"""Wire payloads from host-owned and byte-carrying device rings on the benchmark configuration (1 M entities, 100 K subscribers,
15 x 15 cells), with bench.py's ring generator (synth.update_rings, 4 updates per cell and tick), in alternating blocks of ticks:
    host    host-kept rings (the newest updates, at most 64 per cell: 4 to 64 over the 16-tick input cycle), then chd_set_rings +
            chd_set_payload_bytes of every live entry, then chd_tick(TICK_ALL), chd_assemble_payloads and chd_frame_packets
    device  chd_rings_append_bytes of the tick's new updates only (device rings of 1024 entries, a byte slab of 32 KB per cell),
            then chd_tick(TICK_ALL), chd_assemble_payloads and chd_frame_packets
Every update carries 24 bytes.  The input cycle is replayed with its arrivals and message indices moved forward by whole cycles, so
both arms see one stream that advances with the tick clock.  Prints one JSON line: the card and its power limit; per arm the wall ms
per tick of each block and the bytes it uploads per tick (from the shapes, the mean over the cycle); the device append's time (its copies and rings_append_bytes_kernel, CUDA events
on the engine stream); and a flooded cell: just above 512 live entries in a nearly full byte slab, where a byte slide comes with
almost every update.  Sets no clocks or power limits, reads nothing outside the repository and writes nothing.

    python bench_ring_bytes.py [--steps 30] [--warmup 5] [--blocks 3]
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
ARMS = ("host", "device")
UPDATES_PER_CELL = 4
ENTRY_BYTES = 24
CYCLE = 16         # distinct ticks of inputs, reused round robin (the host rings fill to 64 entries within it)
RING_CAP = 1024
BYTES_PER_CELL = 32 << 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=3)
    a = ap.parse_args()
    import torch

    from channeld_b200 import capi, engine, synth

    L = capi.lib()
    p = capi.ptr

    def ck(st, e):
        if st != capi.OK:
            raise capi.ChdError(st, L.chd_last_error(e.h).decode())

    wc = synth.CONFIGS["benchmark"]
    N, S, Cn = wc.n_entities, wc.n_subscribers, wc.cells
    x, z = synth.entities(wc)
    conn, cx, cz, r = synth.subscribers(wc, x, z)
    batch, keep = engine.make_batch(S, sub=None, sphere=(cx, cz, r))
    compression = (np.arange(S) % 2).astype(np.uint8)
    full_off = (np.arange(Cn + 1) * 200).astype(np.uint64)
    full = np.frombuffer(np.random.default_rng(1).bytes(int(full_off[-1])), np.uint8)
    url = b"type.googleapis.com/chdtest.TestChannelDataMessage"
    pool = np.frombuffer(np.random.default_rng(2).bytes(1 << 20), np.uint8)
    snaps, upds, state = [], [], None
    for k in range(CYCLE):
        state, off, arr, snd, idx, cmi = synth.update_rings(wc, k, (k + 1) * TICK_NS, TICK_NS, UPDATES_PER_CELL, S, ring_len=64, state=state)
        n = int(off[-1])
        eoff = (np.arange(n + 1) * ENTRY_BYTES).astype(np.uint64)
        snaps.append(dict(off=off.astype(np.uint32), arr=arr, snd=snd, idx=idx, cmi=cmi, n=n, eoff=eoff, eb=pool[:n * ENTRY_BYTES].copy()))
        per = n // Cn
        last = (np.arange(Cn)[:, None] * per + np.arange(per - UPDATES_PER_CELL, per)).reshape(-1)
        m = len(last)
        upds.append(dict(off=(np.arange(Cn + 1) * UPDATES_PER_CELL).astype(np.uint32), arr=arr[last].copy(), snd=snd[last].copy(), n=m,
                         boff=(np.arange(m + 1) * ENTRY_BYTES).astype(np.uint64), bytes=pool[:m * ENTRY_BYTES].copy()))

    def new_engine(arm):
        per_cell = N / Cn  # (bench.py's capacities)
        e = engine.Engine(wc.cfg(), N, S, max_visible=int(S * 1.3 * per_cell * (1.0 + 4.0 * wc.radius / wc.w) + (1 << 22)), max_due=S * 8 + 4096,
                          max_ring_entries=Cn * RING_CAP)
        e.set_subscribers(conn)
        e.set_entities(x, z)
        if arm == "device":
            ck(L.chd_rings_init(e.h, RING_CAP), e)
            ck(L.chd_rings_reserve_bytes(e.h, BYTES_PER_CELL), e)
        return dict(e=e, t=0, blob=np.zeros(1 << 26, np.uint8), out=np.zeros(1 << 27, np.uint8))

    eng = {arm: new_engine(arm) for arm in ARMS}

    def payloads(rs):
        e = rs["e"]
        ncls, blen, olen, nd = C.c_uint32(), C.c_uint64(), C.c_uint64(), C.c_uint32()
        ck(L.chd_assemble_payloads(e.h, C.byref(ncls), None, 0, p(rs["blob"]), rs["blob"].size, C.byref(blen)), e)
        ck(L.chd_frame_packets(e.h, p(compression), None, None, None, p(rs["out"]), rs["out"].size, C.byref(olen), C.byref(nd)), e)

    def block(arm, n):
        rs = eng[arm]
        e = rs["e"]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            rs["t"] += 1
            t_ns = rs["t"] * TICK_NS
            k = rs["t"] % CYCLE
            dt, di = (rs["t"] - k - 1) * TICK_NS, (rs["t"] - k) * UPDATES_PER_CELL  # input k was made for the clock (k + 1) * TICK_NS
            if arm == "device":
                u = upds[k]
                arr = u["arr"] + dt
                ck(L.chd_rings_append_bytes(e.h, p(u["off"]), u["n"], p(arr), p(u["snd"]), p(u["boff"]), p(u["bytes"])), e)
                ck(L.chd_set_payload_bytes(e.h, p(np.zeros(1, np.uint64)), 0, None, p(full_off), p(full), url, 8), e)
            else:
                g = snaps[k]
                arr, idx, cmi = g["arr"] + dt, g["idx"] + np.uint64(di), g["cmi"] + np.uint64(di)
                ck(L.chd_set_rings(e.h, p(g["off"]), g["n"], p(arr), p(g["snd"]), p(idx), p(cmi)), e)
                ck(L.chd_set_payload_bytes(e.h, p(g["eoff"]), g["n"], p(g["eb"]), p(full_off), p(full), url, 8), e)
            e.tick(batch, t_ns, capi.TICK_ALL, want_summary=False)
            payloads(rs)
        e.sync()
        return time.perf_counter() - t0

    for arm in ARMS:
        block(arm, a.warmup)
    wall = {arm: [] for arm in ARMS}
    for _ in range(a.blocks):
        for arm in ARMS:
            wall[arm].append(round(1e3 * block(arm, a.steps) / a.steps, 3))
    u = upds[0]
    n_host = np.mean([g["n"] for g in snaps])  # the live entries the host arm uploads, over the cycle
    upload = {"host": round(4 * (Cn + 1) + (8 + 4 + 8) * n_host + 8 * Cn + 8 * (n_host + 1) + n_host * ENTRY_BYTES),
              "device": 4 * (Cn + 1) + (8 + 4) * u["n"] + 8 * (u["n"] + 1) + u["n"] * ENTRY_BYTES}

    def append_ms(e, stream, args, reps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        for k in range(reps):
            ck(L.chd_rings_append_bytes(e.h, *args(k)), e)
        ev[1].record(stream)
        ev[1].synchronize()
        return ev[0].elapsed_time(ev[1]) / reps

    # the append on the benchmark engine's stream
    de = eng["device"]["e"]
    stream = torch.cuda.Stream()
    de.set_stream(stream.cuda_stream)
    app = lambda k: (p(upds[k % CYCLE]["off"]), upds[k % CYCLE]["n"], p(upds[k % CYCLE]["arr"]), p(upds[k % CYCLE]["snd"]),  # noqa: E731
                     p(upds[k % CYCLE]["boff"]), p(upds[k % CYCLE]["bytes"]))
    append_ms(de, stream, app, 5)
    t_append = append_ms(de, stream, app, 50)
    # a flooded cell: 512 live entries of 60 bytes in a slab of 513: each update of 60 bytes finds the tail at the slab end, slides
    # the live bytes by 60, and the 512 rule evicts the oldest entry
    fe = engine.Engine(wc.cfg(), 16, 16, max_ring_entries=Cn * RING_CAP)
    ck(L.chd_rings_init(fe.h, RING_CAP), fe)
    ck(L.chd_rings_reserve_bytes(fe.h, 513 * 60), fe)
    fe.set_stream(stream.cuda_stream)
    F = 64

    def flood(k, n):
        off = np.zeros(Cn + 1, np.uint32)
        off[1:] = n
        arr = (np.arange(n) + k * 1000 + 1).astype(np.int64)  # the same arrivals: maxFanOutIntervalMs 0, the 512 rule evicts past 512
        return off, arr, np.ones(n, np.uint32), (np.arange(n + 1) * 60).astype(np.uint64), pool[:n * 60].copy()

    keep_f = []

    def fl(k):
        args = flood(k + 1, F)
        keep_f.append(args)
        return (p(args[0]), F, p(args[1]), p(args[2]), p(args[3]), p(args[4]))

    first = flood(0, 520)
    ck(L.chd_rings_append_bytes(fe.h, p(first[0]), 520, p(first[1]), p(first[2]), p(first[3]), p(first[4])), fe)
    append_ms(fe, stream, fl, 5)
    t_flood = append_ms(fe, stream, fl, 50)
    s = capi.TickSummary()
    L.chd_summary(fe.h, C.byref(s))
    flood_ok = int(s.overflow) == 0
    fe.close()
    for rs in eng.values():
        rs["e"].close()
    print(json.dumps(dict(bench="ring_bytes", gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit_w(), config="benchmark",
                          steps=a.steps, blocks=a.blocks, wall_ms_per_tick=wall, upload_bytes_per_tick=upload,
                          append_ms=round(t_append, 4), flood_updates_per_append=F, flood_append_ms=round(t_flood, 4),
                          flood_no_overflow=flood_ok)))


if __name__ == "__main__":
    main()
