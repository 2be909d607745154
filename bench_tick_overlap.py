"""How much of each tick's head runs beside the previous tick's visible-list copy, and what a tick costs when the window is closed
only after the last copy kernel.

bench.py closes its timed window with an event on the engine stream.  The two-stream tick leaves its copy kernel running on the
copy stream after chd_tick returns, so that window does not contain the last tick's copy (about 1/steps of it).  This script
times the same loop (one chd_set_rings + chd_set_entities + chd_tick per step, device-resident inputs) with the host clock
around the loop and a final chd_sync, which waits for the last copy.

A second, instrumented pass runs the same steps under torch.profiler and prints for each tick how far into it the copy kernel
starts and how much of the next tick's head overlaps this tick's copy kernels.  A tick starts with its interest update's first
kernel (`stage_begin_kernel`, launched at the fork with the build; the fan-out pass launches the tick's second one), its head
ends where its first copy kernel starts.

    python bench_tick_overlap.py --config benchmark [--tree DIR]

--tree: import channeld_b200 from DIR instead of this script's directory (to compare two checkouts in one session).  Prints one
JSON line.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="benchmark", choices=["benchmark", "10m", "handover"])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-steps", type=int, default=20)
    ap.add_argument("--tree", default=HERE)
    args = ap.parse_args()
    sys.path.insert(0, HERE)
    import bench  # make_snapshots, TICK_NS: the inputs bench.py times

    sys.path.insert(0, os.path.abspath(args.tree))
    import torch

    from channeld_b200 import capi, engine, synth

    assert os.path.dirname(os.path.dirname(os.path.abspath(engine.__file__))) == os.path.abspath(args.tree)
    torch.cuda.init()
    wc = synth.CONFIGS[args.config]
    conn, snaps = bench.make_snapshots(wc)
    N, S = wc.n_entities, wc.n_subscribers
    per_cell = N / wc.cells
    stream = torch.cuda.Stream()
    e = engine.Engine(wc.cfg(), N + 1024, S, max_visible=int(S * 1.3 * max(per_cell, 1.0) * (1.0 + 4.0 * (wc.radius / wc.w)) + (1 << 22)),
                      max_ring_entries=wc.cells * 16 + 1024, max_due=S * 8 + 4096)
    e.set_stream(stream.cuda_stream)
    e.set_subscribers(conn)
    dev = [{k: torch.from_numpy(np.ascontiguousarray(sn[k])).cuda() for k in ("x", "z", "cx", "cz", "r")} for sn in snaps]
    batches, keep = [], []
    for d in dev:
        b, k = engine.make_batch(S, sub=None, sphere=(d["cx"], d["cz"], d["r"]))
        batches.append(b)
        keep.append(k)
    n_rings = args.warmup + args.steps + args.prof_steps + 2
    rings, state = [], None
    for i in range(n_rings):
        state, off, arr, snd, idx, cmi = synth.update_rings(wc, i, (i + 1) * bench.TICK_NS, bench.TICK_NS, 4, S, ring_len=16, state=state)
        rings.append({k_: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k_, v in
                      (("off", off.view(np.int32)), ("arr", arr), ("snd", snd.view(np.int32)), ("idx", idx.view(np.int64)),
                       ("cmi", cmi.view(np.int64)))} | {"n": int(off[-1])})
    L = e.L

    def ck(st):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode())

    def step(i):
        d, rg = dev[i % 2], rings[i]
        ck(L.chd_set_rings(e.h, capi.ptr(rg["off"]), rg["n"], capi.ptr(rg["arr"]), capi.ptr(rg["snd"]), capi.ptr(rg["idx"]), capi.ptr(rg["cmi"])))
        ck(L.chd_set_entities(e.h, capi.ptr(d["x"]), capi.ptr(d["z"]), N))
        ck(L.chd_tick(e.h, C.byref(batches[i % 2]), (i + 1) * bench.TICK_NS, capi.TICK_ALL, None))

    with torch.cuda.stream(stream):
        for i in range(args.warmup):
            step(i)
        e.summary()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(args.steps):
            step(args.warmup + i)
        e.sync()  # waits for the last tick's copy kernel too
        ms = (time.perf_counter() - t0) * 1e3 / args.steps
        s = e.summary()
        assert s.overflow == 0

        base = args.warmup + args.steps
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.prof_steps):
                step(base + i)
            e.sync()
            torch.cuda.synchronize()
    kern = [(ev.time_range.start, ev.time_range.end, ev.name) for ev in prof.events() if ev.device_type.name == "CUDA"]
    kern.sort()
    marks = [k[0] for k in kern if "stage_begin_kernel" in k[2]][::2]
    copies = [k for k in kern if "emit_visible" in k[2]]
    assert len(marks) == args.prof_steps and copies and len(copies) % args.prof_steps == 0, (len(marks), len(copies))
    per = len(copies) // args.prof_steps
    spans = [(copies[i * per][0], max(c[1] for c in copies[i * per:(i + 1) * per])) for i in range(args.prof_steps)]
    start_in_tick = [spans[i][0] - marks[i] for i in range(args.prof_steps)]
    overlap = [max(0.0, min(spans[i][1], spans[i + 1][0]) - max(marks[i + 1], spans[i][0])) for i in range(args.prof_steps - 1)]
    head = [spans[i + 1][0] - marks[i + 1] for i in range(args.prof_steps - 1)]
    props = torch.cuda.get_device_properties(0)
    out = {
        "config": args.config, "tree": os.path.abspath(args.tree), "gpu": props.name, "steps": args.steps,
        "ms_per_step_to_sync": round(ms, 4), "queries_per_s_to_sync": round(S / (ms * 1e-3), 1),
        "copy_start_in_tick_us": {"median": round(float(np.median(start_in_tick)), 1), "min": round(min(start_in_tick), 1),
                                  "max": round(max(start_in_tick), 1)},
        "head_overlapping_previous_copy_us": {"median": round(float(np.median(overlap)), 1), "min": round(min(overlap), 1),
                                              "max": round(max(overlap), 1)},
        "head_us_median": round(float(np.median(head)), 1),
        "copy_us_median": round(float(np.median([b - a for a, b in spans])), 1),
    }
    e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
