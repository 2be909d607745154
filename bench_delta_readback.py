"""What it costs a pipelined host to read the visible-set delta back every tick, at the benchmark configuration (1 M entities, 100 K
subscribers, r = 50, 15 x 15 cells), in the e2e loop of bench_entity_events.py: pinned host inputs, chd_adopt_prefetched +
chd_begin_interest + chd_tick(TICK_ALL | TICK_EARLY_RESULTS ...), the next tick's inputs prefetched behind it, tick k's results read
back while tick k+1 runs.  Three arms, one engine each, identical inputs, in alternating blocks of ticks:
    none     TICK_ALL, chd_fetch_results_async (cell CSR, handover list, visible offsets); no delta
    get      TICK_ALL | TICK_VISIBLE_DELTA, the same fetch, and chd_get_visible_delta after each wait (it blocks on the tick in flight)
    fetch    TICK_ALL | TICK_VISIBLE_DELTA, chd_fetch_results_async_delta + chd_fetch_wait_delta (the delta rides in the fetch)
Two workloads: "move60" moves every entity up to 60 per axis per tick (bench_visible_delta.py's), "walk2" up to 2.  The first delta
(everything enters) runs before the timed blocks and is fetched without lists.
Prints one JSON line per run: the card and its power limit; per workload and arm the wall ms per tick of each block and entered + left
per tick; from an instrumented block (per-stage CUDA events on) the CHD_STAGE_READBACK ms per tick and the delta's share of its
PCIe bytes as GB/s, and the next tick's CHD_STAGE_EMIT_KERNEL start (chd_profile_timeline); from a torch.profiler block of the
"fetch" arm the hop-1 copy kernel (HBM -> HBM staging, bulk_copy_kernel on the stream of delta_head_kernel) ms and GB/s (read +
write), next to a write-only fill of the same size.  The profiler trace goes to a temporary directory; nothing is written in the
tree and nothing outside the repository is read.

    python bench_delta_readback.py [--steps 30] [--warmup 5] [--blocks 3] [--workloads move60,walk2]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_visible_delta import power_limit_w  # noqa: E402

TICK_NS = 33_000_000
STEPS = {"move60": 60.0, "walk2": 2.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--workloads", default="move60,walk2")
    ap.add_argument("--config", default="benchmark")
    ap.add_argument("--entity-cap", type=int, default=40_000_000, help="entries per delta list (pinned buffers and the reserve)")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()

    def ck(st, h=None):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(h).decode() if h else "bench_delta_readback")

    def pinned(arr, dtype):
        return torch.from_numpy(np.ascontiguousarray(arr).view(dtype)).pin_memory()

    wc = synth.CONFIGS[a.config]
    N, S = wc.n_entities, wc.n_subscribers
    ECAP = a.entity_cap
    idx = (np.arange(S, dtype=np.int64) * (N // S)) % N
    _, off, arr, snd, ridx, cmi = synth.update_rings(wc, 0, 0, TICK_NS, 4, S, ring_len=64)
    ring = dict(off=pinned(off.astype(np.uint32), np.int32), arr=pinned(arr.astype(np.int64), np.int64), snd=pinned(snd.astype(np.uint32), np.int32),
                idx=pinned(ridx.astype(np.uint64), np.int64), cmi=pinned(cmi.astype(np.uint64), np.int64), n=int(off[-1]))
    q_r, q_sub = pinned(np.full(S, wc.radius), np.float64), pinned(np.arange(S, dtype=np.uint32), np.int32)

    def result_set():
        keep = dict(cs=torch.zeros(wc.cells + 1, dtype=torch.int32).pin_memory(), se=torch.zeros(N, dtype=torch.int32).pin_memory(),
                    ho=[torch.zeros(N, dtype=torch.int32).pin_memory() for _ in range(3)], voff=torch.zeros(S + 1, dtype=torch.int64).pin_memory(),
                    hdr=torch.zeros(64, dtype=torch.int32).pin_memory())
        r = capi.ResultBuffers()
        r.cell_start, r.sorted_entity, r.entity_cap = capi.ptr(keep["cs"]), capi.ptr(keep["se"]), N
        r.handover_entity, r.handover_src, r.handover_dst, r.handover_cap = (*[capi.ptr(t) for t in keep["ho"]], N)
        r.vis_off = capi.ptr(keep["voff"])
        return r, keep

    def delta_set():
        keep = [torch.zeros(S + 1, dtype=torch.int64).pin_memory() for _ in range(2)] + [torch.zeros(ECAP, dtype=torch.int32).pin_memory() for _ in range(2)]
        d = capi.DeltaBuffers()
        d.enter_off, d.leave_off, d.enter_entity, d.leave_entity = (capi.ptr(t) for t in keep)
        d.slot_cap, d.entity_cap = S + 1, ECAP
        return d, keep

    dsets = [delta_set(), delta_set()]  # shared by the arms (one arm runs at a time)
    get_bufs = dsets[0][1]

    def make_positions(step):
        """two alternating position snapshots (the second moved by `step`), pinned f32, and their query centres"""
        x0, z0 = synth.entities(wc)
        x1, z1 = synth.move_entities(wc, x0, z0, 1, step)
        snaps = []
        for x, z in ((x0, z0), (x1, z1)):
            snaps.append(dict(x=pinned(x.astype(np.float32), np.float32), z=pinned(z.astype(np.float32), np.float32),
                              cx=pinned(x[idx].astype(np.float64), np.float64), cz=pinned(z[idx].astype(np.float64), np.float64)))
        return snaps

    arms = {"none": capi.TICK_ALL | capi.TICK_EARLY_RESULTS,
            "get": capi.TICK_ALL | capi.TICK_EARLY_RESULTS | capi.TICK_VISIBLE_DELTA,
            "fetch": capi.TICK_ALL | capi.TICK_EARLY_RESULTS | capi.TICK_VISIBLE_DELTA}
    out = {"metric": "delta_readback", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "config": wc.name,
           "steps": a.steps, "blocks": a.blocks, "entity_cap": ECAP, "workloads": {}}
    for wl in a.workloads.split(","):
        snaps = make_positions(STEPS[wl])
        batches = [engine.make_batch(S, sub=q_sub, sphere=(s_["cx"], s_["cz"], q_r)) for s_ in snaps]
        runs = {}
        for arm, flags in arms.items():
            e = engine.Engine(wc.cfg(), N, S)
            e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
            rs = dict(e=e, flags=flags, t=0, sets=[result_set(), result_set()], ms=[], changes=[])
            if flags & capi.TICK_VISIBLE_DELTA:
                e.reserve_visible_delta(max(ECAP, 600_000_000))  # the first delta enters every visible list (V = 4.9e8)
            runs[arm] = rs

        def prefetch(rs):
            e = rs["e"]
            s_ = snaps[(rs["t"] + 1) % 2]
            ck(L.chd_prefetch_rings(e.h, capi.ptr(ring["off"]), ring["n"], capi.ptr(ring["arr"]), capi.ptr(ring["snd"]), capi.ptr(ring["idx"]),
                                    capi.ptr(ring["cmi"])), e.h)
            ck(L.chd_prefetch_queries(e.h, C.byref(batches[(rs["t"] + 1) % 2][0])), e.h)
            ck(L.chd_prefetch_entities_f32(e.h, capi.ptr(s_["x"]), capi.ptr(s_["z"]), N), e.h)

        def block(arm, n, counts_out=None):
            rs = runs[arm]
            e = rs["e"]
            summ, cnt = capi.TickSummary(), capi.DeltaCounts()
            ne, nl, ns = C.c_uint64(), C.c_uint64(), C.c_uint32()
            torch.cuda.synchronize()
            prefetch(rs)
            t0 = time.perf_counter()

            def after_wait():
                if arm == "get":  # the only read-back before this change: blocks on the tick in flight, returns ITS lists
                    ck(L.chd_get_visible_delta(e.h, capi.ptr(get_bufs[0]), capi.ptr(get_bufs[2]), capi.ptr(get_bufs[1]), capi.ptr(get_bufs[3]), ECAP,
                                               C.byref(ne), C.byref(nl), C.byref(ns)), e.h)
                    if counts_out is not None:
                        counts_out.append(ne.value + nl.value)
                elif arm == "fetch" and counts_out is not None:
                    counts_out.append(cnt.n_entered + cnt.n_left)

            for k in range(n):
                rs["t"] += 1
                t_ns = rs["t"] * TICK_NS
                ck(L.chd_adopt_prefetched(e.h), e.h)
                ck(L.chd_begin_interest(e.h, None, t_ns, 1), e.h)
                ck(L.chd_tick(e.h, None, t_ns, rs["flags"], None), e.h)
                prefetch(rs)
                r_, k_ = rs["sets"][k % 2]
                if arm == "fetch":
                    ck(L.chd_fetch_results_async_delta(e.h, C.byref(r_), C.byref(dsets[k % 2][0]), capi.ptr(k_["hdr"])), e.h)
                else:
                    ck(L.chd_fetch_results_async(e.h, C.byref(r_), capi.ptr(k_["hdr"])), e.h)
                if k:
                    ck(L.chd_fetch_wait_delta(e.h, C.byref(summ), C.byref(cnt)), e.h)
                    after_wait()
            ck(L.chd_fetch_wait_delta(e.h, C.byref(summ), C.byref(cnt)), e.h)
            after_wait()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        for arm, rs in runs.items():  # the first tick (and, with the flag, the delta that enters everything): outside the loop
            e = rs["e"]
            prefetch(rs)
            rs["t"] += 1
            ck(L.chd_adopt_prefetched(e.h), e.h)
            ck(L.chd_begin_interest(e.h, None, rs["t"] * TICK_NS, 1), e.h)
            ck(L.chd_tick(e.h, None, rs["t"] * TICK_NS, rs["flags"], None), e.h)
            ck(L.chd_fetch_results(e.h, C.byref(rs["sets"][0][0]), C.byref(capi.TickSummary())), e.h)
            block(arm, a.warmup)
        for _ in range(a.blocks):
            for arm in arms:
                runs[arm]["ms"].append(round(block(arm, a.steps) / a.steps * 1e3, 4))
        res = {}
        for arm, rs in runs.items():
            e = rs["e"]
            changes = []
            e.profile_enable(True)
            emit_start = []
            for _ in range(3):
                block(arm, a.steps, changes)
                emit_start.append(round(e.profile_timeline(capi.STAGE_EMIT_KERNEL)[0], 4))
            rb_ms, k = e.profile_get(capi.STAGE_READBACK)
            e.profile_enable(False)
            r = dict(wall_ms=rs["ms"], readback_stage_ms=round(rb_ms / max(k, 1), 4), next_emit_kernel_start_ms=emit_start)
            if changes:
                ch = float(np.median(changes))
                r["entered_plus_left_per_tick"] = ch
                if arm == "fetch":
                    dbytes = 4 * ch + 16 * (S + 1)
                    r["delta_readback_bytes_per_tick"] = dbytes
                    r["readback_delta_pcie_gbs"] = round(dbytes / (r["readback_stage_ms"] * 1e-3) / 1e9, 2) if r["readback_stage_ms"] else None
            res[arm] = r
        # hop 1 of the delta fetch under torch.profiler (its own block), and a write-only fill of the same bytes
        from torch.profiler import ProfilerActivity, profile

        with tempfile.TemporaryDirectory() as td:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                block("fetch", 10)
            path = os.path.join(td, "trace.json")
            prof.export_chrome_trace(path)
            ev = [x for x in json.load(open(path))["traceEvents"] if x.get("cat") == "kernel"]
        hop1_streams = {x["args"].get("stream") for x in ev if "delta_head_kernel" in x["name"]}
        hop1 = [x["dur"] for x in ev if "bulk_copy_kernel" in x["name"] and x["args"].get("stream") in hop1_streams]
        hop2 = [x["dur"] for x in ev if "bulk_copy_kernel" in x["name"] and x["args"].get("stream") not in hop1_streams]
        ch = res["fetch"].get("entered_plus_left_per_tick", 0.0)
        hop1_bytes = 4 * ch + 16 * (S + 1)
        fill = torch.empty(max(int(hop1_bytes // 4), 1), dtype=torch.int32, device="cuda")
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            fill.fill_(1)
        t0.record()
        for _ in range(20):
            fill.fill_(1)
        t1.record()
        torch.cuda.synchronize()
        fill_ms = t0.elapsed_time(t1) / 20
        del fill
        h1 = float(np.median(hop1)) / 1e3 if hop1 else None
        res["fetch"]["hop1_copy_ms"] = round(h1, 4) if h1 else None
        res["fetch"]["hop1_copy_gbs_read_plus_write"] = round(2 * hop1_bytes / (h1 * 1e-3) / 1e9, 1) if h1 else None
        res["fetch"]["hop2_copy_ms"] = round(float(np.median(hop2)) / 1e3, 4) if hop2 else None
        res["fetch"]["fill_same_bytes_ms"] = round(fill_ms, 4)
        res["fetch"]["fill_gbs_write"] = round(hop1_bytes / (fill_ms * 1e-3) / 1e9, 1) if fill_ms else None
        out["workloads"][wl] = res
        for rs in runs.values():
            rs["e"].close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
