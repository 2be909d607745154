"""Multi-GPU followers (one rank per GPU, launched by tests/test_multigpu_follow.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29641 \
        tests/run_multigpu_follow.py

Every rank owns an X-slab and a table engine with subscriber migration.  Every connection follows an entity and lives on the rank
that owns it (sharding.FollowerRegistry, replicated in every process like sharding.EntityRouter).  Per tick, on every rank: the
entity moves are routed; the registry's plan moves followers whose entity changed owner with chd_migrate_out / chd_migrate_in (their
subscriptions and fan-out state travel in the tick's exchange) and binds the arrivals again; chd_follow_queries(CHD_FOLLOW_MOVED);
chd_tick_sharded(NULL, .., CHD_TICK_FOLLOW); chd_handoff_entities, whose lists every rank learns and the destinations adopt.  Each
rank also runs a whole-world table engine with the same bindings on its GPU, and every tick, per connection on the rank: the
visible set, every pair field (cell, dist, interval and the kept fan-out state) and, except on the tick it moves, the follower's
chd_get_follow entry equal the whole world's."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding  # noqa: E402
from tests.test_gpu_sharded_follow import COLS, ROWS, W, Walk, _bind, _shapes  # noqa: E402
from tests.test_gpu_sharded_table import _vis_sets  # noqa: E402

TICK = 33_000_000
FLAGS = capi.TICK_ALL | capi.TICK_FOLLOW
PAIR_FIELDS = ("channel", "dist", "interval", "flags", "last", "last_index")


def per_slot(e):
    """slot -> (visible set, pair fields, follow entry)"""
    vis = _vis_sets(*e.get_visible()) if e.n_slots else []
    p = e.get_pairs()
    f = e.get_follow()
    fol = {int(s): (int(f["entity"][k]), int(f["status"][k]), float(f["cx"][k]), float(f["cz"][k])) for k, s in enumerate(f["slot"])}
    out = {}
    for s in range(e.n_slots):
        a, b = int(p["off"][s]), int(p["off"][s + 1])
        out[s] = (vis[s], tuple(tuple(p[k][a:b].tolist()) for k in PAIR_FIELDS), fol.get(s))
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    failures = 0
    n, F = 6000, 480
    walk = Walk(n, 2025)
    rng = np.random.default_rng(2026)
    fol = rng.choice(walk.ids, F, replace=False)
    kind, shape = _shapes(rng, F)
    halo = sharding.halo_columns(180.0, W) + 1
    cfg = engine.grid_cfg(0, 0, W, W, COLS, ROWS)
    e = engine.Engine(cfg, 2 * n + n * world + 16, F, device=local, max_visible=1 << 24)
    uid = torch.zeros(128, dtype=torch.uint8, device=dev)
    if rank == 0:
        uid.copy_(torch.frombuffer(bytearray(engine.Engine.comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(uid, 0)
    e.comm_init(uid.cpu().numpy().tobytes(), rank, world, halo, n, migrate_subscribers=F)  # the slab first, then the table
    e.entity_table_init()
    whole = engine.Engine(cfg, 2 * n, F, device=local, max_visible=1 << 24)
    whole.entity_table_init()
    whole.set_subscribers(np.arange(1, F + 1, dtype=np.uint32))  # connection c = slot c - 1
    router = sharding.EntityRouter(world, COLS, 0.0, W)
    reg = sharding.FollowerRegistry(world)
    assert (whole.spawn_entities(walk.ids, walk.x, walk.z) == 0).all()
    mine = router.spawn(walk.ids, walk.x, walk.z)[rank]
    assert (e.spawn_entities(*mine) == 0).all()
    _bind(whole, np.arange(F), fol, kind, shape)
    for j in range(F):
        reg.follow(j + 1, int(fol[j]), int(kind[j]), shape[:, j])
    vacated = [[] for _ in range(world)]
    migrated = handed = 0
    for tick in range(8):
        t_ns = (tick + 1) * TICK
        if tick:
            mv = walk.tick()
            whole.move_entities(*mv)
            b = router.move(*mv)[rank]
            if len(b[0]):
                e.move_entities(*b)
        for r in range(world):
            reg.slots.release(r, vacated[r])
        arrivals, out_lists, in_calls, vacated, binds = reg.plan(router)
        e.migrate_out(vacated[rank])  # (unbinds the emigrants)
        moved = set()
        for dst, src, first, pairs in in_calls:
            moved |= {c for c, _ in pairs}
            if dst == rank:
                e.migrate_in(src, first, [s for _, s in pairs], [c for c, _ in pairs])
        if arrivals[rank]:
            e.add_subscribers([s for _, s in arrivals[rank]], [c for c, _ in arrivals[rank]])
        if len(binds[rank]["conn"]):
            _bind(e, binds[rank]["slot"], binds[rank]["entity"], binds[rank]["kind"], binds[rank]["shape"])
        migrated += len(moved)
        e.follow_queries(capi.FOLLOW_MOVED)
        s = e.tick_sharded(None, t_ns, FLAGS)
        whole.follow_queries(capi.FOLLOW_MOVED)
        s1 = whole.tick(None, t_ns, FLAGS)
        bad = int(s.overflow != 0) + int(s1.overflow != 0)
        got, want = per_slot(e), per_slot(whole)
        for c, r in reg.slots.owner.items():
            if r != rank:
                continue
            g, w = got[reg.slots.slot[c]], want[c - 1]
            bad += int(g[0] != w[0]) + int(g[1] != w[1])
            bad += int(g[2] is None or g[2][1] == capi.FOLLOW_OUTSIDE_SLAB)
            if c not in moved:
                bad += int(g[2] != w[2])
        ids, dst, x, z = e.handoff_entities()
        lists = [None] * world
        dist.all_gather_object(lists, (ids.tolist(), dst.tolist(), x.tolist(), z.tolist()))
        adopt = router.handoff(lists)
        handed += sum(len(v[0]) for v in lists)
        if len(adopt[rank][0]):
            bad += int(not (e.spawn_entities(*adopt[rank]) == 0).all())
        failures += bad
        print("rank %d tick %d: followers=%d mismatches=%d migrated=%d handed=%d" % (rank, tick, len(reg.slots.at[rank]), bad, migrated, handed),
              flush=True)
    if handed == 0 or migrated == 0:
        failures += 1
        print("rank %d: no hand-off or no follower migrated (%d, %d)" % (rank, handed, migrated), flush=True)
    e.close()
    whole.close()
    t = torch.tensor([failures], device=dev)
    dist.all_reduce(t)
    dist.destroy_process_group()
    if int(t[0]) != 0:
        raise SystemExit("multi-GPU follow FAILED: %d mismatches" % int(t[0]))
    if rank == 0:
        print("multi-GPU follow OK")


if __name__ == "__main__":
    main()
