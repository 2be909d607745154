"""A mixed world at the benchmark configuration (1 M entities, 100 K subscribers, 15 x 15 cells), entity-table mode: a fraction x of
the subscribers send explicit queries every tick (spheres and boxes anywhere in the world, some with spots; the slots follow nothing),
the rest follow their pawn, and a fraction of the entities moves every tick (chd_move_entities_f32).  Two engines get identical
inputs, in alternating blocks of ticks, in the pipelined loop of bench_follow.py (rings prefetched behind the tick, results read back
with chd_fetch_results_async while the next tick is enqueued):
    two-updates  the explicit batch through chd_update_interest in an update of its own, a synchronous read of its diff and
                 statuses (without it the follow tick's update would overwrite them), then chd_follow_queries(CHD_FOLLOW_MOVED) and the
                 follow tick
    merged       the explicit batch prefetched a tick ahead (chd_prefetch_queries), adopted, merged with
                 chd_follow_queries_with(CHD_FOLLOW_MOVED, NULL), one follow tick
Prints one JSON line: the card and its power limit; per x and arm the wall ms per tick of each block, the host's enqueue ms per tick
and CUDA-graph replays per tick, and, from a separate instrumented block, the device ms per tick of CHD_STAGE_FOLLOW and
CHD_STAGE_INTEREST (both updates for two-updates) and the emit kernel's start in the tick's timeline.  Sets no clocks or power
limits, reads nothing outside the repository and writes nothing.

    python bench_follow_mixed.py [--steps 30] [--warmup 5] [--blocks 3] [--explicit 0.01,0.1,0.5] [--moved 0.01]
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
ARMS = ("two-updates", "merged")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--explicit", default="0.01,0.1,0.5")
    ap.add_argument("--moved", type=float, default=0.01)
    ap.add_argument("--config", default="benchmark")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()

    def ck(st, e=None):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode() if e else "bench_follow_mixed")

    def pinned(arr, dtype):
        return torch.from_numpy(np.ascontiguousarray(arr).view(dtype)).pin_memory()

    wc = synth.CONFIGS[a.config]
    N, S = wc.n_entities, wc.n_subscribers
    x0, z0 = synth.entities(wc)
    x1, z1 = synth.move_entities(wc, x0, z0, 1, 60.0)
    snaps = [(x0.astype(np.float32), z0.astype(np.float32)), (x1.astype(np.float32), z1.astype(np.float32))]
    ids = np.arange(N, dtype=np.uint32) * 3 + 1
    pawn = (np.arange(S, dtype=np.int64) * (N // S)) % N
    rng = np.random.default_rng(1)
    m = max(1, int(round(a.moved * N)))
    moves = []
    for p in range(2):
        sel = rng.permutation(N)[:m]
        moves.append(dict(ids=pinned(ids[sel], np.int32), x=pinned(snaps[p][0][sel], np.float32), z=pinned(snaps[p][1][sel], np.float32), m=m))
    _, off, arr, snd, ridx, cmi = synth.update_rings(wc, 0, 0, TICK_NS, 4, S, ring_len=64)
    ring = dict(off=pinned(off.astype(np.uint32), np.int32), arr=pinned(arr.astype(np.int64), np.int64), snd=pinned(snd.astype(np.uint32), np.int32),
                idx=pinned(ridx.astype(np.uint64), np.int64), cmi=pinned(cmi.astype(np.uint64), np.int64), n=int(off[-1]))
    x0w, x1w = wc.offx, wc.offx + wc.w * wc.cols
    z0w, z1w = wc.offz, wc.offz + wc.h * wc.rows

    def explicit_batches(slots):
        """two variants (alternate ticks) of the explicit queries of `slots`: spheres and boxes, every 10th with two spots"""
        n = len(slots)
        out = []
        for _ in range(2):
            kind = np.where(np.arange(n) % 2 == 0, capi.AOI_SPHERE, capi.AOI_BOX).astype(np.uint8)
            kind[::10] |= capi.AOI_SPOTS
            cx, cz = rng.uniform(x0w, x1w, n), rng.uniform(z0w, z1w, n)
            cnt = np.where(kind & capi.AOI_SPOTS, 2, 0)
            so = np.zeros(n + 1, np.uint32)
            so[1:] = np.cumsum(cnt)
            t = int(so[-1])
            keep = [pinned(slots, np.int32), pinned(kind, np.uint8), pinned(cx, np.float64), pinned(cz, np.float64), pinned(np.full(n, wc.radius), np.float64),
                    pinned(rng.uniform(30, 70, n), np.float64), pinned(rng.uniform(30, 70, n), np.float64), pinned(so, np.int32),
                    pinned(np.zeros(n, np.uint32), np.int32), pinned(rng.uniform(x0w, x1w, max(t, 1)), np.float64),
                    pinned(rng.uniform(z0w, z1w, max(t, 1)), np.float64), pinned(np.zeros(max(t, 1), np.uint32), np.int32)]
            sub, kd, cxp, czp, r, ex, ez, sop, nd, sx, sz, sd = keep
            b, _ = engine.make_batch(n, sub=sub, kind=kd, sphere=(cxp, czp, r), box=(cxp, czp, ex, ez), spots=(sop, nd, sx, sz, sd))
            out.append((b, keep))
        return out

    def result_set():
        keep = dict(cs=torch.zeros(wc.cells + 1, dtype=torch.int32).pin_memory(), se=torch.zeros(N, dtype=torch.int32).pin_memory(),
                    voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(), hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.cell_start, r.sorted_entity, r.entity_cap, r.vis_off = capi.ptr(keep["cs"]), capi.ptr(keep["se"]), N, capi.ptr(keep["voff"])
        return r, keep

    res = {}
    for x in [float(v) for v in a.explicit.split(",")]:
        n_x = max(1, int(round(x * S)))
        perm = rng.permutation(S)
        explicit = np.sort(perm[:n_x]).astype(np.uint32)
        follow = np.sort(perm[n_x:]).astype(np.uint32)
        batches = explicit_batches(explicit)

        def new_engine(arm):
            H = engine.host_part_size(n_x)
            e = engine.Engine(wc.cfg(), N, S, max_queries=H + S, max_spots=max(1024, 2 * n_x))
            e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
            e.entity_table_init()
            assert (e.spawn_entities_f32(ids, *snaps[0]) == capi.EV_OK).all()
            e.follow_bind(follow, ids[pawn[follow]], sph_r=np.full(len(follow), wc.radius))
            rs = dict(e=e, arm=arm, t=0, sets=[result_set(), result_set()])
            if arm == "two-updates":
                P = e.lim.max_pairs
                rs["diff"] = [torch.zeros(P, dtype=torch.int32).pin_memory() for _ in range(4)]
                rs["status"] = torch.zeros(n_x, dtype=torch.int32).pin_memory()
            return rs

        eng = {arm: new_engine(arm) for arm in ARMS}

        def block(arm, n):
            """n pipelined ticks -> (wall s, host enqueue s, graph replays)"""
            rs = eng[arm]
            e = rs["e"]
            summ = capi.TickSummary()
            torch.cuda.synchronize()
            ck(L.chd_prefetch_rings(e.h, capi.ptr(ring["off"]), ring["n"], capi.ptr(ring["arr"]), capi.ptr(ring["snd"]), capi.ptr(ring["idx"]), capi.ptr(ring["cmi"])))
            if arm == "merged":
                ck(L.chd_prefetch_queries(e.h, C.byref(batches[(rs["t"] + 1) % 2][0])), e)
            g0 = e.graph_launch_count()
            host = 0.0
            t0 = time.perf_counter()
            for k in range(n):
                h0 = time.perf_counter()
                rs["t"] += 1
                t_ns = rs["t"] * TICK_NS
                mv = moves[rs["t"] % 2]
                ck(L.chd_move_entities_f32(e.h, capi.ptr(mv["ids"]), capi.ptr(mv["x"]), capi.ptr(mv["z"]), mv["m"]), e)
                ck(L.chd_adopt_prefetched(e.h), e)
                if arm == "merged":
                    ck(L.chd_follow_queries_with(e.h, capi.FOLLOW_MOVED, None), e)
                    if k + 1 < n:  # the next tick's explicit part, behind this tick
                        ck(L.chd_prefetch_queries(e.h, C.byref(batches[(rs["t"] + 1) % 2][0])), e)
                else:
                    ck(L.chd_update_interest(e.h, C.byref(batches[rs["t"] % 2][0]), t_ns), e)
                    ck(L.chd_summary(e.h, C.byref(summ)), e)
                    d = rs["diff"]
                    ck(L.chd_get_diff(e.h, capi.ptr(d[0]), capi.ptr(d[1]), capi.ptr(d[2]), capi.ptr(d[3])), e)
                    ck(L.chd_get_query_status(e.h, capi.ptr(rs["status"]), n_x), e)
                    ck(L.chd_follow_queries(e.h, capi.FOLLOW_MOVED), e)
                ck(L.chd_begin_interest(e.h, None, t_ns, 1), e)
                ck(L.chd_tick(e.h, None, t_ns, capi.TICK_ALL, None), e)
                ck(L.chd_prefetch_rings(e.h, capi.ptr(ring["off"]), ring["n"], capi.ptr(ring["arr"]), capi.ptr(ring["snd"]), capi.ptr(ring["idx"]),
                                        capi.ptr(ring["cmi"])), e)
                r_, k_ = rs["sets"][k % 2]
                ck(L.chd_fetch_results_async(e.h, C.byref(r_), capi.ptr(k_["hdr"])), e)
                host += time.perf_counter() - h0
                if k:
                    ck(L.chd_fetch_wait(e.h, C.byref(summ)), e)
            ck(L.chd_fetch_wait(e.h, C.byref(summ)), e)
            torch.cuda.synchronize()
            return time.perf_counter() - t0, host, e.graph_launch_count() - g0

        out = {arm: dict(ms=[], host_ms=[], graph_replays_per_tick=[]) for arm in ARMS}
        for arm in ARMS:
            block(arm, a.warmup)
        for _ in range(a.blocks):
            for arm in ARMS:
                dt, host, g = block(arm, a.steps)
                out[arm]["ms"].append(round(dt / a.steps * 1e3, 4))
                out[arm]["host_ms"].append(round(host / a.steps * 1e3, 4))
                out[arm]["graph_replays_per_tick"].append(round(g / a.steps, 2))
        for arm in ARMS:  # instrumented (not the timed blocks)
            e = eng[arm]["e"]
            e.profile_enable(True)
            block(arm, a.steps)
            ms, k = e.profile_get(capi.STAGE_INTEREST)
            out[arm]["interest_stage_ms_per_tick"] = round(ms / a.steps, 4)
            out[arm]["interest_stages_per_tick"] = round(k / a.steps, 2)
            ms, k = e.profile_get(capi.STAGE_FOLLOW)
            out[arm]["follow_stage_ms_per_tick"] = round(ms / a.steps, 4)
            out[arm]["emit_kernel_start_ms"] = round(e.profile_timeline(capi.STAGE_EMIT_KERNEL)[0], 4)
            e.profile_enable(False)
        out["explicit_queries"] = n_x
        res["x=%g" % x] = out
        for rs in eng.values():
            rs["e"].close()
    print(json.dumps({"metric": "follow_mixed", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "config": wc.name,
                      "moved": a.moved, "steps": a.steps, "blocks": a.blocks, "results": res}))


if __name__ == "__main__":
    main()
