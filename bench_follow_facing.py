"""Turning followers: re-binding against facings, at the benchmark configuration (1 M entities, 100 K cone followers, 15 x 15 cells),
entity-table mode, in the pipelined loop of bench_follow.py (chd_move_entities_f32 -> chd_follow_queries(CHD_FOLLOW_MOVED) ->
chd_begin_interest -> chd_tick -> chd_fetch_results_async while the next tick is enqueued).  Every tick a fraction f of the pawns
moves and turns (the moved pawns alternate between two position sets and turn to a new facing at every move).  Two engines get
identical moves, in alternating blocks of ticks:
    rebind   today's way: the cone's direction is fixed at bind time, so the host re-binds (chd_follow_bind) the followers whose
             pawn turned, every tick; each bind synchronises with the engine stream
    facing   the moves carry the facing (chd_move_entities_facing_f32) and every follower has a frame (chd_follow_set_frame, identity
             rotation, no offset): the device aims the cones
Prints one JSON line: the card and its power limit; per arm and fraction the wall ms per tick of each block, the host's enqueue ms
per tick and, from a separate instrumented block, the device ms per tick of CHD_STAGE_FOLLOW and the emit kernel's start in the
tick's timeline.  Sets no clocks or power limits, reads nothing outside the repository and writes nothing.

    python bench_follow_facing.py [--steps 30] [--warmup 5] [--blocks 3] [--fractions 0.01,0.1,1]
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
ARMS = ("rebind", "facing")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--fractions", default="0.01,0.1,1")
    ap.add_argument("--config", default="benchmark")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()

    def ck(st, e=None):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode() if e else "bench_follow_facing")

    def pinned(arr, dtype):
        return torch.from_numpy(np.ascontiguousarray(arr).view(dtype)).pin_memory()

    wc = synth.CONFIGS[a.config]
    N, S = wc.n_entities, wc.n_subscribers
    x0, z0 = synth.entities(wc)
    x1, z1 = synth.move_entities(wc, x0, z0, 1, 60.0)
    snaps = [(x0.astype(np.float32), z0.astype(np.float32)), (x1.astype(np.float32), z1.astype(np.float32))]
    ids = np.arange(N, dtype=np.uint32) * 3 + 1
    pawn = (np.arange(S, dtype=np.int64) * (N // S)) % N  # follower j stands on entity pawn[j]
    follower_of = np.full(N, -1, np.int64)
    follower_of[pawn] = np.arange(S)
    fractions = [float(f) for f in a.fractions.split(",")]
    rng = np.random.default_rng(1)
    # tick t moves the pawns of position set t % 2 and turns them to facing set t % 3, so a pawn's facing changes at every move
    moves = {}
    for f in fractions:
        m = max(1, int(round(f * N)))
        sets = []
        for p in range(2):
            sel = rng.permutation(N)[:m]
            fol = follower_of[sel]
            turned = fol >= 0
            m_b = int(turned.sum())
            base = dict(ids=pinned(ids[sel], np.int32), x=pinned(snaps[p][0][sel], np.float32), z=pinned(snaps[p][1][sel], np.float32), m=m,
                        b_slot=np.ascontiguousarray(fol[turned], np.uint32), b_ent=np.ascontiguousarray(ids[sel[turned]]),
                        b_kind=np.full(m_b, capi.AOI_CONE, np.uint8), b_ang=np.full(m_b, 0.8), b_r=np.full(m_b, wc.radius))
            for q in range(3):
                yaw = rng.uniform(0, 2 * np.pi, m)
                fx, fz = np.cos(yaw).astype(np.float32), np.sin(yaw).astype(np.float32)
                # the re-bind batch of the followers whose pawn turned: the same cone along the new facing
                sets.append(dict(base, fx=pinned(fx, np.float32), fz=pinned(fz, np.float32), b_dx=fx[turned].astype(np.float64),
                                 b_dz=fz[turned].astype(np.float64)))
        moves[f] = sets
    _, off, arr, snd, ridx, cmi = synth.update_rings(wc, 0, 0, TICK_NS, 4, S, ring_len=64)
    ring = dict(off=pinned(off.astype(np.uint32), np.int32), arr=pinned(arr.astype(np.int64), np.int64), snd=pinned(snd.astype(np.uint32), np.int32),
                idx=pinned(ridx.astype(np.uint64), np.int64), cmi=pinned(cmi.astype(np.uint64), np.int64), n=int(off[-1]))

    def result_set():
        keep = dict(cs=torch.zeros(wc.cells + 1, dtype=torch.int32).pin_memory(), se=torch.zeros(N, dtype=torch.int32).pin_memory(),
                    voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(), hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.cell_start, r.sorted_entity, r.entity_cap, r.vis_off = capi.ptr(keep["cs"]), capi.ptr(keep["se"]), N, capi.ptr(keep["voff"])
        return r, keep

    def new_engine(arm):
        e = engine.Engine(wc.cfg(), N, S)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.entity_table_init()
        yaw = np.random.default_rng(2).uniform(0, 2 * np.pi, N)
        fx, fz = np.cos(yaw).astype(np.float32), np.sin(yaw).astype(np.float32)
        if arm == "facing":
            assert (e.spawn_entities_facing_f32(ids, *snaps[0], fx, fz) == capi.EV_OK).all()
        else:
            assert (e.spawn_entities_f32(ids, *snaps[0]) == capi.EV_OK).all()
        slots = np.arange(S, dtype=np.uint32)
        e.follow_bind(slots, ids[pawn], kind=np.full(S, capi.AOI_CONE, np.uint8),
                      cone=(fx[pawn].astype(np.float64), fz[pawn].astype(np.float64), np.full(S, 0.8), np.full(S, wc.radius)))
        if arm == "facing":
            e.follow_set_frame(slots, 0.0, 0.0)
        return dict(e=e, arm=arm, t=0, sets=[result_set(), result_set()])

    eng = {arm: new_engine(arm) for arm in ARMS}

    def block(arm, f, n):
        """n pipelined ticks -> (wall s, host enqueue s)"""
        rs = eng[arm]
        e = rs["e"]
        summ = capi.TickSummary()
        torch.cuda.synchronize()
        ck(L.chd_prefetch_rings(e.h, capi.ptr(ring["off"]), ring["n"], capi.ptr(ring["arr"]), capi.ptr(ring["snd"]), capi.ptr(ring["idx"]), capi.ptr(ring["cmi"])))
        host = 0.0
        t0 = time.perf_counter()
        for k in range(n):
            h0 = time.perf_counter()
            rs["t"] += 1
            t_ns = rs["t"] * TICK_NS
            mv = moves[f][3 * (rs["t"] % 2) + rs["t"] % 3]
            if arm == "facing":
                ck(L.chd_move_entities_facing_f32(e.h, capi.ptr(mv["ids"]), capi.ptr(mv["x"]), capi.ptr(mv["z"]), capi.ptr(mv["fx"]), capi.ptr(mv["fz"]),
                                                  mv["m"]), e)
            else:
                ck(L.chd_move_entities_f32(e.h, capi.ptr(mv["ids"]), capi.ptr(mv["x"]), capi.ptr(mv["z"]), mv["m"]), e)
                if len(mv["b_slot"]):
                    b = capi.FollowBatch(n=len(mv["b_slot"]), slot=capi.ptr(mv["b_slot"]), entity=capi.ptr(mv["b_ent"]), kind=capi.ptr(mv["b_kind"]),
                                         cone_dx=capi.ptr(mv["b_dx"]), cone_dz=capi.ptr(mv["b_dz"]), cone_angle=capi.ptr(mv["b_ang"]),
                                         cone_r=capi.ptr(mv["b_r"]))
                    ck(L.chd_follow_bind(e.h, C.byref(b)), e)
            ck(L.chd_follow_queries(e.h, capi.FOLLOW_MOVED), e)
            ck(L.chd_adopt_prefetched(e.h), e)
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
        return time.perf_counter() - t0, host

    res = {}
    for f in fractions:
        out = {arm: dict(ms=[], host_ms=[]) for arm in ARMS}
        for arm in ARMS:
            block(arm, f, a.warmup)
        for _ in range(a.blocks):
            for arm in ARMS:
                dt, host = block(arm, f, a.steps)
                out[arm]["ms"].append(round(dt / a.steps * 1e3, 4))
                out[arm]["host_ms"].append(round(host / a.steps * 1e3, 4))
        for arm in ARMS:  # instrumented (not the timed blocks)
            e = eng[arm]["e"]
            e.profile_enable(True)
            block(arm, f, a.steps)
            ms, k = e.profile_get(capi.STAGE_FOLLOW)
            out[arm]["follow_stage_ms"] = round(ms / max(k, 1), 4)
            out[arm]["emit_kernel_start_ms"] = round(e.profile_timeline(capi.STAGE_EMIT_KERNEL)[0], 4)
            out[arm]["selected_last_tick"] = e.get_follow()["n_selected"]
            e.profile_enable(False)
        res["f=%g" % f] = out
    print(json.dumps({"metric": "follow_facing", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "config": wc.name,
                      "steps": a.steps, "blocks": a.blocks, "results": res}))
    for rs in eng.values():
        rs["e"].close()


if __name__ == "__main__":
    main()
