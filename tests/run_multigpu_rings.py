"""Multi-GPU device rings (one rank per GPU, launched by tests/test_multigpu_rings.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29671 \
        tests/run_multigpu_rings.py

The world of tests/test_gpu_sharded_rings.py (cap 620: the flooded border cells' maximum lives on the right-hand neighbour) on one
communicator engine per GPU, with device rings: every tick every rank stages the same whole-grid updates (chd_rings_append) and runs
chd_tick_sharded, which exchanges the ring limits inside the tick.  Rank 0 also runs a whole-world engine fed the same updates and
queries and checks, every tick and for every rank's served cells: every ring entry and msgIndex, the due list and the pair state of
the rank's subscribers.  Both exchange modes: peer windows (when the ranks can map each other) and chd_comm_use_collective."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding  # noqa: E402
from tests.test_gpu_sharded_rings import COLS, DEFAULT_IV, HALO, ROWS, W, RingWorld, _served  # noqa: E402


def ring_cells(r):
    """get_rings() -> per cell (arrival, sender, index) and the msgIndex"""
    o = r["off"].astype(np.int64)
    return {c: (r["arrival"][o[c]:o[c + 1]].tolist(), r["sender"][o[c]:o[c + 1]].tolist(), r["index"][o[c]:o[c + 1]].tolist(), int(r["msg_index"][c]))
            for c in range(len(o) - 1)}


def due_of(e, n_due, conn):
    d = e.get_due(n_due)
    return {(int(conn[x["sub"]]),) + tuple(int(x[k]) for k in d.dtype.names[1:]) for x in d}


def pairs_of(e, conn):
    p = e.get_pairs()
    slot = np.repeat(np.arange(len(p["off"]) - 1), np.diff(p["off"].astype(np.int64)))
    return {(int(conn[s]), int(p["channel"][k]), int(p["dist"][k]), int(p["interval"][k]), int(p["flags"][k]), int(p["last"][k]),
             int(p["last_index"][k])) for k, s in enumerate(slot)}


def run(rank, world, local, collective):
    split = max(world, 2)  # the world's layout needs two slabs; on one rank, rank 0 hosts both
    rw = RingWorld(split, 620, 77)
    hosted = [p for p in range(split) if p * world // split == rank]
    my_conn = np.concatenate([rw.conn[p] for p in hosted])
    cfg = engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    rng = np.random.default_rng(78)
    n_ent = 4000
    x, z = rng.uniform(0, COLS * W, n_ent), rng.uniform(0, ROWS * W, n_ent)
    lo, hi = sharding.slab_columns(COLS, world, rank)
    mine = np.nonzero(sharding.owner_of_column(sharding.column_of(x, 0.0, W, COLS), COLS, world) == rank)[0]
    e = engine.Engine(cfg, n_ent * (world + 1) + 16, len(my_conn), device=local, default_fanout_interval_ms=DEFAULT_IV)
    uid = [engine.Engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    e.comm_init(uid[0], rank, world, HALO, n_ent)
    if collective:
        e.use_collective(True)
    e.set_subscribers(my_conn)
    e.rings_init(620)
    conn_all = np.concatenate(rw.conn)
    whole = None
    if rank == 0:
        whole = engine.Engine(cfg, n_ent, len(conn_all), device=local, default_fanout_interval_ms=DEFAULT_IV)
        whole.set_subscribers(conn_all)
        whole.set_entities(x, z)
        whole.rings_init(620)
    bad = 0
    for tick, t in enumerate(rw.times()):
        upd = rw.updates(tick, t)  # (same seed on every rank: the same whole-grid batch)
        e.set_entities(x[mine], z[mine])
        e.set_entity_ids(mine.astype(np.uint32))
        e.rings_append(*upd)
        b, keep = engine.make_batch(len(my_conn), sub=np.arange(len(my_conn), dtype=np.uint32),
                                    sphere=tuple(a.copy() for a in rw.queries(hosted, tick)))
        s = e.tick_sharded(b, t, capi.TICK_ALL)
        assert s.overflow == 0
        mine_out = (ring_cells(e.get_rings()), due_of(e, s.n_due, my_conn), pairs_of(e, my_conn))
        got = [None] * world
        dist.all_gather_object(got, mine_out)
        if rank == 0:
            whole.rings_append(*upd)
            wb, wkeep = engine.make_batch(len(conn_all), sub=np.arange(len(conn_all), dtype=np.uint32),
                                          sphere=tuple(a.copy() for a in rw.queries(range(split), tick)))
            sw = whole.tick(wb, t, capi.TICK_ALL)
            W_r, W_d, W_p = ring_cells(whole.get_rings()), due_of(whole, sw.n_due, conn_all), pairs_of(whole, conn_all)
            for r in range(world):
                g_r, g_d, g_p = got[r]
                rl, rh = sharding.slab_columns(COLS, world, r)
                for c in _served(rl, rh):
                    if g_r[c] != W_r[c]:
                        print("tick %d rank %d cell %d: ring differs (%d vs %d entries)" % (tick, r, c, len(g_r[c][2]), len(W_r[c][2])))
                        bad += 1
                conns = set(np.concatenate([rw.conn[p] for p in range(split) if p * world // split == r]).tolist())
                if g_d != {d for d in W_d if d[0] in conns} or g_p != {p for p in W_p if p[0] in conns}:
                    print("tick %d rank %d: due list or pairs differ" % (tick, r))
                    bad += 1
    mode = e.exchange_mode()
    assert e.L.chd_comm_destroy(e.h) == capi.OK
    e.close()
    if whole is not None:
        whole.close()
    return bad, mode


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    failures = 0
    for collective in (False, True):
        bad, mode = run(rank, world, local, collective)
        if rank == 0:
            print("world %d, exchange mode %d: %d mismatches" % (world, mode, bad))
        failures += bad
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0 and failures == 0:
        print("multi-GPU rings OK")
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
