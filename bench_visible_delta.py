"""Cost and size of the visible-set delta (chd_visible_delta) at the benchmark configuration (1 M entities, 100 K subscribers,
r = 50, 15 x 15 cells), with every entity moving every tick (synth.move_entities, max step 60) and every subscriber standing on
its entity.  Four tick forms run on four engines with identical inputs, in alternating blocks of ticks:
    all        CHD_TICK_ALL
    all+delta  CHD_TICK_ALL | CHD_TICK_VISIBLE_DELTA
    delta      CHD_TICK_BUILD | CHD_TICK_FANOUT | CHD_TICK_VISIBLE_DELTA  (no expanded lists)
    delta ids  the same in id mode (chd_reserve_visible_delta_ids): the entities carry a fixed permutation as global ids
Prints one JSON line: the card and its power limit, device ms per tick of each form (CHD_STAGE_TICK: the engine stream's span of
the tick, per-stage profiling on), the delta stage's own time (CHD_STAGE_VISIBLE_DELTA) and entered + left entries per tick
against the visible-list size V.  Reads nothing outside the repository and writes nothing.

    python bench_visible_delta.py [--steps 20] [--warmup 5] [--blocks 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--max-step", type=float, default=60.0)
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    wc = synth.CONFIGS["benchmark"]
    N, S = wc.n_entities, wc.n_subscribers
    x0, z0 = synth.entities(wc)
    idx = (np.arange(S, dtype=np.int64) * (N // S)) % N
    r = np.full(S, wc.radius)
    forms = {"all": capi.TICK_ALL, "all+delta": capi.TICK_ALL | capi.TICK_VISIBLE_DELTA,
             "delta": capi.TICK_BUILD | capi.TICK_FANOUT | capi.TICK_VISIBLE_DELTA,
             "delta ids": capi.TICK_BUILD | capi.TICK_FANOUT | capi.TICK_VISIBLE_DELTA}
    _, off, arr, snd, ridx, cmi = synth.update_rings(wc, 0, 0, 33_000_000, 4, S, ring_len=64)
    runs = {}
    for name, flags in forms.items():
        e = engine.Engine(wc.cfg(), N, S)
        e.set_subscribers(np.arange(1, S + 1, dtype=np.uint32))
        e.set_rings(off, arr, snd, ridx, cmi)
        if name == "delta ids":
            e.set_entity_ids(np.random.default_rng(1).permutation(N).astype(np.uint32))
            e.reserve_visible_delta_ids(600_000_000, N)
        elif flags & capi.TICK_VISIBLE_DELTA:
            e.reserve_visible_delta(600_000_000)  # the first delta enters every visible list (V = 4.9e8)
        runs[name] = dict(e=e, flags=flags, x=x0.copy(), z=z0.copy(), t=0, tick_ms=[], delta_ms=[], changes=[], visible=[])

    def run(rs, n, timed):
        e = rs["e"]
        e.profile_enable(timed)
        for _ in range(n):
            rs["t"] += 1
            rs["x"], rs["z"] = synth.move_entities(wc, rs["x"], rs["z"], rs["t"], a.max_step)
            e.set_entities(rs["x"], rs["z"])
            batch, keep = engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(rs["x"][idx].copy(), rs["z"][idx].copy(), r))
            s = e.tick(batch, rs["t"] * 33_000_000, rs["flags"])
            if timed and rs["flags"] & capi.TICK_VISIBLE_DELTA:
                ne, nl, _ = e.visible_delta_counts()
                rs["changes"].append(ne + nl)
                if rs["flags"] & capi.TICK_EMIT:
                    rs["visible"].append(s.n_visible)
        if timed:
            ms, k = e.profile_get(capi.STAGE_TICK)
            rs["tick_ms"].append(ms / max(k, 1))
            if rs["flags"] & capi.TICK_VISIBLE_DELTA:
                ms, k = e.profile_get(capi.STAGE_VISIBLE_DELTA)
                rs["delta_ms"].append(ms / max(k, 1))

    for rs in runs.values():
        run(rs, a.warmup, False)
    for _ in range(a.blocks):
        for rs in runs.values():
            run(rs, a.steps, True)
    V = float(np.median(runs["all+delta"]["visible"]))
    changes = [c for name in ("all+delta", "delta") for c in runs[name]["changes"]]
    out = {
        "metric": "visible_delta", "card": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
        "config": wc.name, "max_step": a.max_step, "steps": a.steps, "blocks": a.blocks,
        "tick_ms": {name: [round(v, 4) for v in rs["tick_ms"]] for name, rs in runs.items()},
        "delta_stage_ms": {name: [round(v, 4) for v in rs["delta_ms"]] for name, rs in runs.items() if rs["delta_ms"]},
        "entered_plus_left_per_tick": float(np.median(changes)), "visible_entries_V": V,
        "delta_fraction_of_V": float(np.median(changes)) / V if V else None,
    }
    print(json.dumps(out))
    for rs in runs.values():
        rs["e"].close()


if __name__ == "__main__":
    main()
