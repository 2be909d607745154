"""Explicit subscriptions (chd_apply_subscriptions) at the benchmark configuration (1 M entities, 100 K subscribers, r = 50, 15 x 15
cells): one tick subscribes every slot to the cells its sphere touches (about 109 K pairs), then batches of 1 K, 10 K and 200 K ops are
applied back to back, alternating a SUB batch and the UNSUB batch of the same (slot, channel) pairs so that the pair count stays put.
The op arrays live on the device and out_status is NULL, so a call adds no host synchronisation: the time per call of a block of
back-to-back calls, taken between two chd_sync, is the stage's device time once it exceeds the host's enqueue time.
Prints one JSON line: the card and its power limit, and per batch size the ms per call of each block.  Sets no clocks or power
limits, reads nothing outside the repository and writes nothing.

    python bench_channel_subs.py [--steps 50] [--warmup 5] [--blocks 3] [--sizes 1000,10000,200000]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--sizes", default="1000,10000,200000")
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()
    wc = synth.CONFIGS["benchmark"]
    ex, ez = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, ex, ez, 50.0)
    S, cells = len(conn), wc.cols * wc.rows
    e = engine.Engine(wc.cfg(), wc.n_entities, S, max_pairs=1 << 20)
    e.set_entities(ex, ez)
    e.set_subscribers(conn)
    batch, keep = engine.make_batch(S, sub=np.arange(S, dtype=np.uint32), sphere=(cx, cz, r))
    s = e.tick(batch, 33_000_000, capi.TICK_ALL)
    rng = np.random.default_rng(1)
    out = {"metric": "chd_apply_subscriptions ms per call", "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(),
           "pairs": int(s.n_pairs), "sizes": {}}
    for n in [int(v) for v in a.sizes.split(",")]:
        slot = rng.integers(0, S, n).astype(np.uint32)
        ch = (engine.SPATIAL_CHANNEL_ID_START + rng.integers(0, cells, n)).astype(np.uint32)
        dev = {k: torch.from_numpy(v).cuda() for k, v in (("slot", slot), ("channel_id", ch))}
        ops = [torch.full((n,), op, dtype=torch.uint8, device="cuda") for op in (capi.SUBOP_SUB, capi.SUBOP_UNSUB)]
        torch.cuda.synchronize()
        batches = [capi.SubBatch(n=n, slot=dev["slot"].data_ptr(), channel_id=dev["channel_id"].data_ptr(), op=o.data_ptr()) for o in ops]

        def run(k):
            for i in range(k):
                e._ck(L.chd_apply_subscriptions(e.h, C.byref(batches[i & 1]), 40_000_000 + i, None))

        run(a.warmup * 2)
        e.sync()
        blocks = []
        for _ in range(a.blocks):
            t0 = time.perf_counter()
            run(a.steps * 2)
            e.sync()
            blocks.append((time.perf_counter() - t0) * 1e3 / (a.steps * 2))
        out["sizes"][str(n)] = {"ms_per_call": [round(b, 4) for b in blocks], "launches_per_call": None}
        l0 = e.launch_count()
        run(2)
        e.sync()
        out["sizes"][str(n)]["launches_per_call"] = (e.launch_count() - l0) / 2
    e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
