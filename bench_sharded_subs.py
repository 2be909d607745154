"""Explicit subscriptions on a sharded engine against a whole-world engine, on the bench_channel_subs.py workload (1 M entities, 100 K
subscribers, r = 50, 15 x 15 cells; one tick subscribes every slot to the cells its sphere touches).
  apply  chd_apply_subscriptions on a whole-world engine and chd_apply_subscriptions_sharded on a one-rank communicator engine, in
         alternating blocks of back-to-back calls: batches of 1 K, 10 K and 100 K ops, a SUB batch and the UNSUB batch of the same
         (slot, channel) pairs in turn, op arrays on the device, out_status NULL (no host synchronisation inside a block).
  tick   the communicator engine with device rings (1024 entries per cell, 4 updates per cell and tick): per tick one 1 K-op batch
         (SUB and UNSUB in turn), chd_rings_append, chd_tick_sharded (TICK_ALL, no summary).  Arm "same": every SUB carries the
         default interval, so no limit rises after the first tick; arm "raised": every SUB carries a longer interval than the last,
         so the next tick exports and imports ring-limit records.  Wall ms per tick of alternating blocks, and, from a separate
         instrumented block, the device ms per tick of CHD_STAGE_IMPORT.
Prints one JSON line with the card and its power limit.  Sets no clocks or power limits, reads nothing outside the repository and
writes nothing.

    python bench_sharded_subs.py [--steps 50] [--warmup 5] [--blocks 3] [--sizes 1000,10000,100000]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_visible_delta import power_limit_w  # noqa: E402

TICK_NS = 33_000_000
UPDATES_PER_CELL = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--sizes", default="1000,10000,100000")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, sharding, synth

    L = capi.lib()

    def ck(st, e):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode())

    wc = synth.CONFIGS["benchmark"]
    ex, ez = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, ex, ez, 50.0)
    S, N, cells = len(conn), wc.n_entities, wc.cols * wc.rows
    halo = sharding.halo_columns(float(np.max(r)), wc.w)
    batch, keep = engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(cx, cz, r))

    whole = engine.Engine(wc.cfg(), N, S, max_pairs=1 << 20)
    whole.set_entities(ex, ez)
    whole.set_subscribers(conn)
    sh = engine.Engine(wc.cfg(), 2 * N + 1024, S, max_pairs=1 << 20)
    sh.comm_init(engine.Engine.comm_unique_id(), 0, 1, halo, N)
    sh.set_subscribers(conn)
    sh.set_entities(ex, ez)
    sh.set_entity_ids(np.arange(N, dtype=np.uint32))
    ck(L.chd_rings_init(sh.h, 1024), sh)
    s1 = whole.tick(batch, TICK_NS, capi.TICK_ALL)
    s2 = sh.tick_sharded(batch, TICK_NS, capi.TICK_ALL)
    assert s1.n_pairs == s2.n_pairs
    rng = np.random.default_rng(1)
    out = {"metric": "sharded_subs", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "pairs": int(s1.n_pairs),
           "apply": {}, "tick": {}}

    def make_ops(n):
        slot = torch.from_numpy(rng.integers(0, S, n).astype(np.uint32).view(np.int32)).cuda()
        ch = torch.from_numpy((engine.SPATIAL_CHANNEL_ID_START + rng.integers(0, cells, n)).astype(np.uint32).view(np.int32)).cuda()
        ops = [torch.full((n,), op, dtype=torch.uint8, device="cuda") for op in (capi.SUBOP_SUB, capi.SUBOP_UNSUB)]
        return slot, ch, ops

    # ---- apply: ms per call, whole-world and sharded blocks in turn
    t_apply = 10 * TICK_NS
    for n in [int(v) for v in a.sizes.split(",")]:
        slot, ch, ops = make_ops(n)
        torch.cuda.synchronize()
        batches = [capi.SubBatch(n=n, slot=slot.data_ptr(), channel_id=ch.data_ptr(), op=o.data_ptr()) for o in ops]
        fns = {"whole": (whole, L.chd_apply_subscriptions), "sharded": (sh, L.chd_apply_subscriptions_sharded)}

        def run(arm, k):
            e, fn = fns[arm]
            for i in range(k):
                ck(fn(e.h, C.byref(batches[i & 1]), t_apply + i, None), e)

        res = {arm: [] for arm in fns}
        for arm in fns:
            run(arm, 2 * a.warmup)
            fns[arm][0].sync()
        for _ in range(a.blocks):
            for arm in fns:
                t0 = time.perf_counter()
                run(arm, 2 * a.steps)
                fns[arm][0].sync()
                res[arm].append(round((time.perf_counter() - t0) * 1e3 / (2 * a.steps), 4))
        out["apply"][str(n)] = res

    # ---- tick: the sharded tick after a 1 K-op batch, with and without raised limits
    n = 1000
    slot, ch, ops = make_ops(n)
    ivs = np.zeros(n, np.uint32)  # (pageable: its upload completes before the call returns, so it may change next tick)
    present = np.full(n, capi.SUBOPT_INTERVAL, np.uint8)
    u_off = torch.from_numpy((np.arange(cells + 1) * UPDATES_PER_CELL).astype(np.int32)).pin_memory()
    u_snd = torch.from_numpy(rng.integers(1, S, cells * UPDATES_PER_CELL).astype(np.int32)).pin_memory()
    u_arr = torch.zeros(cells * UPDATES_PER_CELL, dtype=torch.int64).pin_memory()  # (arrival 0: the rings evict by count)
    state = {"t": 2, "iv": 1000}

    def tick_block(arm, k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(k):
            state["t"] += 1
            t_ns = state["t"] * TICK_NS
            sub = state["t"] % 2 == 0
            b = capi.SubBatch(n=n, slot=slot.data_ptr(), channel_id=ch.data_ptr(), op=ops[0 if sub else 1].data_ptr())
            if sub and arm == "raised":
                state["iv"] += 1
                ivs[:] = state["iv"]
                b.present, b.interval_ms = capi.ptr(present), capi.ptr(ivs)
            ck(L.chd_apply_subscriptions_sharded(sh.h, C.byref(b), t_ns - 1_000_000, None), sh)
            ck(L.chd_rings_append(sh.h, capi.ptr(u_off), cells * UPDATES_PER_CELL, capi.ptr(u_arr), capi.ptr(u_snd)), sh)
            ck(L.chd_tick_sharded(sh.h, C.byref(batch), t_ns, capi.TICK_ALL, None), sh)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / k

    arms = ("same", "raised")
    res = {arm: dict(ms=[]) for arm in arms}
    for arm in arms:
        tick_block(arm, 2 * a.warmup)
    for _ in range(a.blocks):
        for arm in arms:
            res[arm]["ms"].append(round(tick_block(arm, a.steps), 4))
    for arm in arms:  # instrumented (not the timed blocks)
        sh.profile_enable(True)
        tick_block(arm, a.steps)
        ms, k = sh.profile_get(capi.STAGE_IMPORT)
        res[arm]["import_stage_ms"] = round(ms / max(k, 1), 4)
        sh.profile_enable(False)
    out["tick"] = res
    print(json.dumps(out))
    assert L.chd_comm_destroy(sh.h) == capi.OK
    sh.close()
    whole.close()


if __name__ == "__main__":
    main()
