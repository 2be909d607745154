"""Device rings on a sharded engine against host ring snapshots, at world 1 on the benchmark configuration (1 M entities, 100 K
subscribers, 15 x 15 cells).  Two one-rank communicator engines get the same entities and queries and run the same sharded tick
(chd_tick_sharded, TICK_ALL, no summary: nothing synchronises with the host inside a block), in alternating blocks of ticks:
    snapshot  chd_set_rings of a host ring snapshot (64 entries per cell, pinned) before each tick: what a sharded host does
              without device rings
    device    device rings (chd_rings_init, 1024 entries per cell) and chd_rings_append of the tick's updates (4 per cell, pinned):
              the tick exports and imports the ring limits and appends the staged updates before the interest update starts
Prints one JSON line: the card and its power limit; per arm the wall ms per tick of each block and the host's enqueue ms per tick
and, from a separate instrumented block, the device ms per tick of CHD_STAGE_IMPORT and CHD_STAGE_INTEREST and the interest
stage's start in the tick's timeline.  Sets no clocks or power limits, reads nothing outside the repository and writes nothing.

    python bench_sharded_rings.py [--steps 50] [--warmup 10] [--blocks 3]
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
ARMS = ("snapshot", "device")
UPDATES_PER_CELL = 4
CYCLE = 8  # distinct ticks of inputs, reused round robin


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--config", default="benchmark")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, sharding, synth

    L = capi.lib()

    def ck(st, e):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode())

    def pinned(arr, dtype):
        return torch.from_numpy(np.ascontiguousarray(arr).view(dtype)).pin_memory()

    wc = synth.CONFIGS[a.config]
    N, S = wc.n_entities, wc.n_subscribers
    x, z = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, x, z)
    batch, keep = engine.make_batch(S, sub=None, sphere=(cx, cz, r))
    snaps, upds, state = [], [], None
    for k in range(CYCLE):
        t_ns = (k + 1) * TICK_NS
        state, off, arr, snd, idx, cmi = synth.update_rings(wc, k, t_ns, TICK_NS, UPDATES_PER_CELL, S, ring_len=64, state=state)
        snaps.append(dict(off=pinned(off.astype(np.uint32), np.int32), arr=pinned(arr, np.int64), snd=pinned(snd, np.int32),
                          idx=pinned(idx, np.int64), cmi=pinned(cmi, np.int64), n=int(off[-1])))
        # the same tick's updates as an append batch: the last UPDATES_PER_CELL entries of every cell
        last = (np.arange(wc.cells)[:, None] * (len(arr) // wc.cells) + np.arange(len(arr) // wc.cells - UPDATES_PER_CELL, len(arr) // wc.cells)).reshape(-1)
        u_off = (np.arange(wc.cells + 1) * UPDATES_PER_CELL).astype(np.uint32)
        upds.append(dict(off=pinned(u_off, np.int32), arr=pinned(arr[last], np.int64), snd=pinned(snd[last], np.int32), n=len(last)))
    halo = sharding.halo_columns(float(np.max(r)), wc.w)

    def new_engine(arm):
        per_cell = N / wc.cells  # (bench.py's capacities)
        e = engine.Engine(wc.cfg(), 2 * N + 1024, S, max_visible=int(S * 1.3 * per_cell * (1.0 + 4.0 * wc.radius / wc.w) + (1 << 22)),
                          max_due=S * 8 + 4096)
        e.comm_init(engine.Engine.comm_unique_id(), 0, 1, halo, N)
        e.set_subscribers(conn)
        e.set_entities(x, z)
        e.set_entity_ids(np.arange(N, dtype=np.uint32))
        if arm == "device":
            ck(L.chd_rings_init(e.h, 1024), e)
        return dict(e=e, t=0)

    eng = {arm: new_engine(arm) for arm in ARMS}

    def block(arm, n):
        """n sharded ticks -> (wall s, host enqueue s)"""
        rs = eng[arm]
        e = rs["e"]
        torch.cuda.synchronize()
        host = 0.0
        t0 = time.perf_counter()
        for _ in range(n):
            h0 = time.perf_counter()
            rs["t"] += 1
            t_ns = rs["t"] * TICK_NS
            if arm == "device":
                u = upds[rs["t"] % CYCLE]
                ck(L.chd_rings_append(e.h, capi.ptr(u["off"]), u["n"], capi.ptr(u["arr"]), capi.ptr(u["snd"])), e)
            else:
                g = snaps[rs["t"] % CYCLE]
                ck(L.chd_set_rings(e.h, capi.ptr(g["off"]), g["n"], capi.ptr(g["arr"]), capi.ptr(g["snd"]), capi.ptr(g["idx"]), capi.ptr(g["cmi"])), e)
            ck(L.chd_tick_sharded(e.h, C.byref(batch), t_ns, capi.TICK_ALL, None), e)
            host += time.perf_counter() - h0
        torch.cuda.synchronize()
        return time.perf_counter() - t0, host

    out = {arm: dict(ms=[], host_ms=[]) for arm in ARMS}
    for arm in ARMS:
        block(arm, a.warmup)
    for _ in range(a.blocks):
        for arm in ARMS:
            dt, host = block(arm, a.steps)
            out[arm]["ms"].append(round(dt / a.steps * 1e3, 4))
            out[arm]["host_ms"].append(round(host / a.steps * 1e3, 4))
    for arm in ARMS:  # instrumented (not the timed blocks)
        e = eng[arm]["e"]
        e.profile_enable(True)
        block(arm, a.steps)
        for name, sid in (("import", capi.STAGE_IMPORT), ("interest", capi.STAGE_INTEREST)):
            ms, k = e.profile_get(sid)
            out[arm][name + "_stage_ms"] = round(ms / max(k, 1), 4)
        out[arm]["interest_start_ms"] = round(e.profile_timeline(capi.STAGE_INTEREST)[0], 4)
        e.profile_enable(False)
        n0 = e.launch_count()
        block(arm, 1)
        out[arm]["launches_per_tick"] = e.launch_count() - n0
    print(json.dumps({"metric": "sharded_rings", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "config": wc.name,
                      "world": 1, "steps": a.steps, "blocks": a.blocks, "results": out}))
    for rs in eng.values():
        assert L.chd_comm_destroy(rs["e"].h) == capi.OK
        rs["e"].close()


if __name__ == "__main__":
    main()
