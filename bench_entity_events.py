"""Sparse entity events against position snapshots, at the benchmark configuration (1 M entities, 100 K subscribers, r = 50,
15 x 15 cells), in the pipelined e2e form of bench.py: pinned host inputs, chd_adopt_prefetched + chd_begin_interest + chd_tick,
the next tick's queries / rings (and, for snapshots, positions) prefetched behind it, results read back with
chd_fetch_results_async while the next tick runs (cell CSR, handover list, visible offsets).
    snapshot   every tick uploads all positions as floats (chd_prefetch_entities_f32: 8 bytes per entity)
    f=<frac>   entity-table mode (chd_entity_table_init, 1 M spawned ids): every tick moves that fraction of the entities, in random
               id order, through chd_move_entities_f32 (12 bytes per moved entity, resolved on the device) before chd_tick
The arms run in alternating blocks of ticks (one engine in each mode).  Prints one JSON line: the card and its power limit, wall ms per
tick of each block, the host's enqueue ms per tick, and from a separate instrumented block the device ms per tick of the event stage
(CHD_STAGE_ENTITY_EVENTS) and of the engine stream's tick span (CHD_STAGE_TICK).  Reads nothing outside the repository and writes
nothing.

    python bench_entity_events.py [--steps 30] [--warmup 5] [--blocks 3] [--fractions 0.001,0.01,0.1,1]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--fractions", default="0.001,0.01,0.1,1")
    ap.add_argument("--config", default="benchmark")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()

    def ck(st):
        if st != capi.OK:
            raise capi.ChdError(st, "bench_entity_events")

    def pinned(arr, dtype):
        t = torch.from_numpy(np.ascontiguousarray(arr).view(dtype)).pin_memory()
        return t

    wc = synth.CONFIGS[a.config]
    N, S = wc.n_entities, wc.n_subscribers
    x0, z0 = synth.entities(wc)
    x1, z1 = synth.move_entities(wc, x0, z0, 1, 60.0)
    snaps = [(x0.astype(np.float32), z0.astype(np.float32)), (x1.astype(np.float32), z1.astype(np.float32))]
    snaps_t = [(pinned(x, np.float32), pinned(z, np.float32)) for x, z in snaps]
    ids = (np.arange(N, dtype=np.uint32) * 3 + 1)  # sparse NetGUID-like ids
    idx = (np.arange(S, dtype=np.int64) * (N // S)) % N
    q_cx, q_cz = pinned(x0[idx].astype(np.float64), np.float64), pinned(z0[idx].astype(np.float64), np.float64)
    q_r, q_sub = pinned(np.full(S, wc.radius), np.float64), pinned(np.arange(S, dtype=np.uint32), np.int32)
    batch, batch_keep = engine.make_batch(S, sub=q_sub, sphere=(q_cx, q_cz, q_r))
    _, off, arr, snd, ridx, cmi = synth.update_rings(wc, 0, 0, TICK_NS, 4, S, ring_len=64)
    ring = dict(off=pinned(off.astype(np.uint32), np.int32), arr=pinned(arr.astype(np.int64), np.int64), snd=pinned(snd.astype(np.uint32), np.int32),
                idx=pinned(ridx.astype(np.uint64), np.int64), cmi=pinned(cmi.astype(np.uint64), np.int64), n=int(off[-1]))
    fractions = [float(f) for f in a.fractions.split(",")]
    rng = np.random.default_rng(1)
    moves = {}
    for f in fractions:
        m = max(1, int(round(f * N)))
        sets = []
        for p in range(2):
            sel = rng.permutation(N)[:m]
            sets.append((pinned(ids[sel], np.int32), pinned(snaps[p][0][sel], np.float32), pinned(snaps[p][1][sel], np.float32), m))
        moves[f] = sets

    def result_set(max_ent):
        keep = dict(cs=torch.zeros(wc.cells + 1, dtype=torch.int32).pin_memory(), se=torch.zeros(max_ent, dtype=torch.int32).pin_memory(),
                    ho=[torch.zeros(max_ent, dtype=torch.int32).pin_memory() for _ in range(3)], voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(),
                    hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.cell_start, r.sorted_entity, r.entity_cap = capi.ptr(keep["cs"]), capi.ptr(keep["se"]), max_ent
        r.handover_entity, r.handover_src, r.handover_dst, r.handover_cap = (*[capi.ptr(t) for t in keep["ho"]], max_ent)
        r.vis_off = capi.ptr(keep["voff"])
        return r, keep

    def new_engine(table):
        e = engine.Engine(wc.cfg(), N, S)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        if table:
            e.entity_table_init()
            st = e.spawn_entities_f32(ids, *snaps[0])
            assert (st == capi.EV_OK).all()
        return dict(e=e, table=table, t=0, sets=[result_set(N), result_set(N)])

    eng = {"snapshot": new_engine(False), "table": new_engine(True)}
    arms = ["snapshot"] + ["f=%g" % f for f in fractions]
    res = {arm: dict(ms=[], host_ms=[], wait_ms=[]) for arm in arms}

    def prefetch(rs, arm):
        e = rs["e"]
        ck(L.chd_prefetch_rings(e.h, capi.ptr(ring["off"]), ring["n"], capi.ptr(ring["arr"]), capi.ptr(ring["snd"]), capi.ptr(ring["idx"]),
                                capi.ptr(ring["cmi"])))
        ck(L.chd_prefetch_queries(e.h, C.byref(batch)))
        if arm == "snapshot":
            xs, zs = snaps_t[(rs["t"] + 1) % 2]
            ck(L.chd_prefetch_entities_f32(e.h, capi.ptr(xs), capi.ptr(zs), N))

    def block(arm, n):
        """n pipelined ticks of `arm` -> (wall s, host enqueue s, host wait s)"""
        rs = eng["snapshot" if arm == "snapshot" else "table"]
        e = rs["e"]
        mv = None if arm == "snapshot" else moves[float(arm[2:])]
        summ = capi.TickSummary()
        torch.cuda.synchronize()
        prefetch(rs, arm)
        host = wait = 0.0
        t0 = time.perf_counter()
        for k in range(n):
            h0 = time.perf_counter()
            rs["t"] += 1
            t_ns = rs["t"] * TICK_NS
            ck(L.chd_adopt_prefetched(e.h))
            ck(L.chd_begin_interest(e.h, None, t_ns, 1))
            if mv is not None:
                mi, mx, mz, m = mv[rs["t"] % 2]
                ck(L.chd_move_entities_f32(e.h, capi.ptr(mi), capi.ptr(mx), capi.ptr(mz), m))
            ck(L.chd_tick(e.h, None, t_ns, capi.TICK_ALL, None))
            prefetch(rs, arm)
            r_, k_ = rs["sets"][k % 2]
            ck(L.chd_fetch_results_async(e.h, C.byref(r_), capi.ptr(k_["hdr"])))
            h1 = time.perf_counter()
            host += h1 - h0
            if k:
                ck(L.chd_fetch_wait(e.h, C.byref(summ)))  # the previous tick, while this one runs
                wait += time.perf_counter() - h1
        h1 = time.perf_counter()
        ck(L.chd_fetch_wait(e.h, C.byref(summ)))
        wait += time.perf_counter() - h1
        torch.cuda.synchronize()
        return time.perf_counter() - t0, host, wait

    for arm in arms:
        block(arm, a.warmup)
    for _ in range(a.blocks):
        for arm in arms:
            dt, host, wait = block(arm, a.steps)
            res[arm]["ms"].append(round(dt / a.steps * 1e3, 4))
            res[arm]["host_ms"].append(round(host / a.steps * 1e3, 4))
            res[arm]["wait_ms"].append(round(wait / a.steps * 1e3, 4))
    # instrumented (not the timed blocks): device time of the event stage and of the tick's engine-stream span
    for arm in arms:
        e = eng["snapshot" if arm == "snapshot" else "table"]["e"]
        e.profile_enable(True)
        block(arm, a.steps)
        tick_ms, k = e.profile_get(capi.STAGE_TICK)
        res[arm]["tick_stage_ms"] = round(tick_ms / max(k, 1), 4)
        if arm != "snapshot":
            ev_ms, k = e.profile_get(capi.STAGE_ENTITY_EVENTS)
            res[arm]["event_stage_ms"] = round(ev_ms / max(k, 1), 4)
        e.profile_enable(False)
    for arm in arms:
        res[arm]["h2d_position_bytes_per_tick"] = 8 * N if arm == "snapshot" else 12 * moves[float(arm[2:])][0][3]
    st = eng["table"]["e"].entity_stats()
    out = {"metric": "entity_events", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "config": wc.name,
           "steps": a.steps, "blocks": a.blocks, "arms": res, "table_stats": st}
    print(json.dumps(out))
    for rs in eng.values():
        rs["e"].close()


if __name__ == "__main__":
    main()
