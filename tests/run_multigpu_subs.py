"""Multi-GPU explicit subscriptions (one rank per GPU, launched by tests/test_multigpu_subs.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29681 \
        tests/run_multigpu_subs.py

The world of tests/test_gpu_sharded_subs.py on one communicator engine per GPU, with device rings.  Per tick every rank applies the
ops for the slots it holds (sharding.route_sub_ops: regular connections on their served cells, the server's key per rank on the cells
of that rank's columns) with chd_apply_subscriptions_sharded, stages the same whole-grid updates (chd_rings_append), moves migrants
(chd_migrate_out / chd_migrate_in: querying connections that change rank, with their explicit pairs) and runs chd_tick_sharded,
which exchanges the ring limits inside the tick.  Rank 0 also runs a whole-world engine fed the same ops, updates and queries and
checks, every tick: the statuses, and per connection the pairs and the due list, and every rank's served rings.  Both exchange
modes: peer windows (when the ranks can map each other) and chd_comm_use_collective."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding  # noqa: E402
from tests.run_multigpu_rings import ring_cells  # noqa: E402
from tests.test_gpu_sharded_subs import (COLS, DEFAULT_IV, HALO, MS, N_ENT, RING_CAP, ROWS, SERVER, W, SubWorld, _dues, _pairs,  # noqa: E402
                                         _random_ops, _served_cols)

MIGRATE_AT = 4


class _NS:
    capi, sharding = capi, sharding
    S0 = engine.SPATIAL_CHANNEL_ID_START


def keys_cells(sw, world):
    """the (key, cell) pairs an op may name, for the connections' current ranks"""
    out = []
    for c in sw.regular:
        lo, hi = sharding.slab_columns(COLS, world, sw.table.owner[c])
        out += [(c, int(row * COLS + col)) for col in _served_cols(lo, hi) for row in range(ROWS)]
    col_owner = sharding.owner_of_column(np.arange(COLS), COLS, world)
    return out + [(("server", SERVER, int(col_owner[cell % COLS])), cell) for cell in range(COLS * ROWS)]


def run(rank, world, local, collective):
    sw = SubWorld(_NS, world, 91)  # (same seed on every rank: the same ops and updates)
    cfg = engine.grid_cfg(0.0, 0.0, W, W, COLS, ROWS)
    mig = 4
    e = engine.Engine(cfg, N_ENT * (world + 1) + 16, 7 + 2 * mig, device=local, default_fanout_interval_ms=DEFAULT_IV)
    uid = [engine.Engine.comm_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(uid, src=0)
    e.comm_init(uid[0], rank, world, HALO, N_ENT, migrate_subscribers=mig, migrate_pairs=mig * COLS * ROWS)
    if collective:
        e.use_collective(True)
    e.set_subscribers(sw.conn_of_slot[rank])
    e.rings_init(RING_CAP)
    mine = np.nonzero(sw.ent_owner == rank)[0]
    whole = None
    if rank == 0:
        whole = engine.Engine(cfg, N_ENT, len(sw.whole_conns), device=local, default_fanout_interval_ms=DEFAULT_IV)
        whole.set_subscribers(sw.whole_conns)
        whole.set_entities(sw.x, sw.z)
        whole.rings_init(RING_CAP)
    # the migrants: the first querying connection of each rank moves to the next rank (its centre with it)
    migrants = [next(c for c in sw.regular if sw.table.owner[c] == r and sw.queries[c]) for r in range(world)] if world > 1 else []
    bad = moved = 0
    t = 1000 * MS
    for tick in range(10):
        t += int(sw.rng.integers(90, 131)) * MS
        ops = _random_ops(sw.rng, 40, keys_cells(sw, world))
        keys, cell, op, present, iv, dl, ss, sf = ops
        idx, slots = sharding.route_sub_ops(sw.table, keys)[rank]
        st = e.apply_subscriptions_sharded(slots, _NS.S0 + cell[idx], op[idx], interval=iv[idx], delay=dl[idx], skip_self=ss[idx],
                                           skip_first=sf[idx], now_ns=t - 7 * MS, present=present[idx])
        upd = sw.updates(tick, t)
        e.rings_append(*upd)
        if tick == MIGRATE_AT and migrants:
            new_owner = {}
            for r, c in enumerate(migrants):
                dst = (r + 1) % world
                lo, hi = sharding.slab_columns(COLS, world, dst)
                sw.cx[c] = (lo + 0.5) * W
                new_owner[c] = dst
            arrivals, out_lists, in_calls, vacated = sharding.plan_migrations(sw.table, new_owner)
            e.migrate_out(np.array(vacated[rank], np.uint32))
            for dst, src, first, placed in in_calls:
                if dst == rank:
                    e.migrate_in(src, first, np.array([s for _, s in placed], np.uint32), np.array([c for c, _ in placed], np.uint32))
            moved = len(migrants)
        conn_of_slot = np.zeros(e.n_slots, np.uint32)  # (vacated slots: 0)
        for s_, k in sw.table.at[rank].items():
            conn_of_slot[s_] = k[1] if isinstance(k, tuple) else k
        q = [c for c in sw.regular if sw.queries[c] and sw.table.owner[c] == rank]
        b, keep = engine.make_batch(len(q), sub=np.array([sw.table.slot[c] for c in q], np.uint32),
                                    sphere=(np.array([sw.cx[c] for c in q]), np.array([sw.cz[c] for c in q]), np.full(len(q), 150.0)))
        e.set_entities(sw.x[mine], sw.z[mine])
        e.set_entity_ids(mine.astype(np.uint32))
        s = e.tick_sharded(b, t, capi.TICK_ALL)
        assert s.overflow == 0
        got = [None] * world
        dist.all_gather_object(got, (idx.tolist(), st.tolist(), ring_cells(e.get_rings()), _dues(e, s.n_due, conn_of_slot), _pairs(e, conn_of_slot)))
        if tick == MIGRATE_AT and migrants:
            sw.table.release(rank, vacated[rank])  # (the vacated slots are free from the next tick on)
        if rank != 0:
            continue
        want = whole.apply_subscriptions([sw.whole_slot[k[1] if isinstance(k, tuple) else k] for k in keys], _NS.S0 + cell, op, interval=iv,
                                         delay=dl, skip_self=ss, skip_first=sf, now_ns=t - 7 * MS, present=present)
        whole.rings_append(*upd)
        wq = [c for c in sw.regular if sw.queries[c]]
        wb, wkeep = engine.make_batch(len(wq), sub=np.array([sw.whole_slot[c] for c in wq], np.uint32),
                                      sphere=(np.array([sw.cx[c] for c in wq]), np.array([sw.cz[c] for c in wq]), np.full(len(wq), 150.0)))
        ws = whole.tick(wb, t, capi.TICK_ALL)
        statuses = np.full(len(keys), capi.SUB_ERR_SLOT, np.uint8)
        pairs, dues = [], []
        for r in range(world):
            statuses[np.array(got[r][0], np.int64)] = got[r][1]
            pairs += got[r][4]
            dues += got[r][3]
            W_r = ring_cells(whole.get_rings())
            for c in np.nonzero(np.isin(np.arange(COLS * ROWS) % COLS, _served_cols(*sharding.slab_columns(COLS, world, r))))[0]:
                if got[r][2][c] != W_r[c]:
                    print("tick %d rank %d cell %d: ring differs" % (tick, r, c))
                    bad += 1
        if statuses.tolist() != want.tolist():
            print("tick %d: statuses differ" % tick)
            bad += 1
        if sorted(pairs) != _pairs(whole, sw.whole_conns) or sorted(dues) != _dues(whole, ws.n_due, sw.whole_conns):
            print("tick %d: pairs or due lists differ" % tick)
            bad += 1
    mode = e.exchange_mode()
    assert e.L.chd_comm_destroy(e.h) == capi.OK
    e.close()
    if whole is not None:
        whole.close()
    return bad, mode, moved


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    failures = 0
    for collective in (False, True):
        bad, mode, moved = run(rank, world, local, collective)
        if rank == 0:
            print("world %d, exchange mode %d, %d migrants: %d mismatches" % (world, mode, moved, bad))
        failures += bad
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0 and failures == 0:
        print("multi-GPU subscriptions OK")
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
