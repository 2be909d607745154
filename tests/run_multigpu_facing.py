"""Multi-GPU framed followers (one rank per GPU, launched by tests/test_multigpu_facing.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29661 \
        tests/run_multigpu_facing.py

tests/run_multigpu_follow.py with facings and frames (include/chd_gpu_facing.h).  Every entity has a facing; every tick the walking
entities turn, and their moves carry the facing (chd_move_entities_facing, routed by sharding.EntityRouter).  Every connection
follows an entity with a frame (centre offset and cone rotation, sharding.FollowerRegistry.follow(.., frame=)).  Per tick, on every
rank: the registry's plan moves followers whose entity changed owner with chd_migrate_out (which clears their frames) /
chd_migrate_in, binds the arrivals again and sets their frames from the plan's batch["frame"]; chd_follow_queries(CHD_FOLLOW_MOVED);
chd_tick_sharded(NULL, .., CHD_TICK_FOLLOW); chd_handoff_entities_facing, whose lists (with their facings and the communicator's
destination ranks) every rank learns and the destinations adopt with chd_spawn_entities_facing.  Each rank also runs a whole-world
table engine with the same facings and frames on its GPU, and every tick, per connection on the rank: the follower's status, and
unless its query failed (an offset centre out of the world keeps whatever pairs each engine had) the visible set and every pair
field; except on the tick it moves, its chd_get_follow entry and its chd_get_follow_frame entry (facing, centre, direction, bit for
bit).  The rank's framed slots are exactly its connections' slots: the emigrants' frames are gone."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding  # noqa: E402
from tests.run_multigpu_follow import per_slot  # noqa: E402
from tests.test_gpu_sharded_follow import COLS, ROWS, W, Walk, _bind, _shapes  # noqa: E402

TICK = 33_000_000
FLAGS = capi.TICK_ALL | capi.TICK_FOLLOW
FRAME = ("fx", "fz", "cx", "cz", "dx", "dz")
MAX_OFF = 60.0


def frames_of(e):
    """slot -> the six f64 of chd_get_follow_frame, as bit patterns"""
    g = e.get_follow_frame()
    v = np.stack([np.ascontiguousarray(g[a], np.float64).view(np.uint64) for a in FRAME]) if len(g["slot"]) else np.zeros((6, 0), np.uint64)
    return {int(s): tuple(v[:, k].tolist()) for k, s in enumerate(g["slot"])}


def set_frames(e, b):
    f = b.get("frame")
    if f is not None and len(f["slot"]):
        e.follow_set_frame(f["slot"], f["off_fwd"], f["off_right"], (f["rot_cos"], f["rot_sin"]))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    failures = 0
    n, F = 6000, 480
    walk = Walk(n, 3031)
    rng = np.random.default_rng(3032)
    yaw = rng.uniform(0, 2 * np.pi, n)
    fx, fz = np.cos(yaw), np.sin(yaw)
    fx[::13] = fz[::13] = 0.0  # entities without a facing
    fol = rng.choice(walk.ids, F, replace=False)
    kind, shape = _shapes(rng, F)
    frames = np.stack([rng.uniform(-MAX_OFF, MAX_OFF, F), rng.uniform(-MAX_OFF, MAX_OFF, F), np.ones(F), np.zeros(F)])
    ang = rng.uniform(-np.pi, np.pi, F)
    frames[2, 1::2], frames[3, 1::2] = np.cos(ang[1::2]), np.sin(ang[1::2])
    halo = sharding.halo_columns(180.0 + MAX_OFF * np.sqrt(2), W) + 1  # the reach and the offset, + 1 column crossed per tick
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
    assert (whole.spawn_entities_facing(walk.ids, walk.x, walk.z, fx, fz) == 0).all()
    mine = router.spawn(walk.ids, walk.x, walk.z, fx, fz)[rank]
    if len(mine[0]):
        assert (e.spawn_entities_facing(*mine) == 0).all()
    _bind(whole, np.arange(F), fol, kind, shape)
    whole.follow_set_frame(np.arange(F, dtype=np.uint32), frames[0], frames[1], (frames[2], frames[3]))
    for j in range(F):
        reg.follow(j + 1, int(fol[j]), int(kind[j]), shape[:, j], frame=tuple(frames[:, j]))
    vacated = [[] for _ in range(world)]
    migrated = handed = 0
    for tick in range(8):
        t_ns = (tick + 1) * TICK
        if tick:
            ids, x, z = walk.tick()
            turn = rng.uniform(0, 2 * np.pi, len(ids))
            fx[ids - 1], fz[ids - 1] = np.cos(turn), np.sin(turn)
            mv = (ids, x, z, fx[ids - 1].copy(), fz[ids - 1].copy())
            whole.move_entities_facing(*mv)
            b = router.move(*mv)[rank]
            if len(b[0]):
                e.move_entities_facing(*b)
        for r in range(world):
            reg.slots.release(r, vacated[r])
        arrivals, out_lists, in_calls, vacated, binds = reg.plan(router)
        e.migrate_out(vacated[rank])  # (unbinds the emigrants and clears their frames)
        moved = set()
        for dst, src, first, pairs in in_calls:
            moved |= {c for c, _ in pairs}
            if dst == rank:
                e.migrate_in(src, first, [s for _, s in pairs], [c for c, _ in pairs])
        if arrivals[rank]:
            e.add_subscribers([s for _, s in arrivals[rank]], [c for c, _ in arrivals[rank]])
        if len(binds[rank]["conn"]):
            _bind(e, binds[rank]["slot"], binds[rank]["entity"], binds[rank]["kind"], binds[rank]["shape"])
            set_frames(e, binds[rank])  # (a bind clears the frame: set it again)
        migrated += len(moved)
        e.follow_queries(capi.FOLLOW_MOVED)
        s = e.tick_sharded(None, t_ns, FLAGS)
        whole.follow_queries(capi.FOLLOW_MOVED)
        s1 = whole.tick(None, t_ns, FLAGS)
        bad = int(s.overflow != 0) + int(s1.overflow != 0)
        got, want = per_slot(e), per_slot(whole)
        gf, wf = frames_of(e), frames_of(whole)
        here = {reg.slots.slot[c] for c, r in reg.slots.owner.items() if r == rank}
        bad += int(set(gf) != here)  # every connection of the rank is framed, and no emigrant's frame is left
        for c, r in reg.slots.owner.items():
            if r != rank:
                continue
            sl = reg.slots.slot[c]
            g, w = got[sl], want[c - 1]
            bad += int(g[2] is None or g[2][1] == capi.FOLLOW_OUTSIDE_SLAB or g[2][1] != w[2][1])
            if w[2][1] == capi.Q_OK:
                bad += int(g[0] != w[0]) + int(g[1] != w[1])
            if c not in moved:
                bad += int(g[2] != w[2]) + int(gf.get(sl) != wf[c - 1])
        ids, dst, x, z, hfx, hfz = e.handoff_entities_facing()
        bad += int(bool((dst == rank).any()))
        lists = [None] * world
        dist.all_gather_object(lists, (ids.tolist(), dst.tolist(), x.tolist(), z.tolist(), hfx.tolist(), hfz.tolist()))
        adopt = router.handoff(lists)
        handed += sum(len(v[0]) for v in lists)
        if len(adopt[rank][0]):
            bad += int(not (e.spawn_entities_facing(*adopt[rank]) == 0).all())
        failures += bad
        print("rank %d tick %d: followers=%d mismatches=%d migrated=%d handed=%d" % (rank, tick, len(reg.slots.at[rank]), bad, migrated, handed),
              flush=True)
    if world > 1 and (handed == 0 or migrated == 0):
        failures += 1
        print("rank %d: no hand-off or no follower migrated (%d, %d)" % (rank, handed, migrated), flush=True)
    e.close()
    whole.close()
    t = torch.tensor([failures], device=dev)
    dist.all_reduce(t)
    dist.destroy_process_group()
    if int(t[0]) != 0:
        raise SystemExit("multi-GPU facing FAILED: %d mismatches" % int(t[0]))
    if rank == 0:
        print("multi-GPU facing OK")


if __name__ == "__main__":
    main()
