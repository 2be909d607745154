"""Multi-GPU entity-table mode (one rank per GPU, launched by tests/test_multigpu_table.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29631 \
        tests/run_multigpu_table.py

Every rank owns an X-slab and a table engine, and runs chd_tick_sharded with CHD_TICK_VISIBLE_DELTA (id mode).  Every rank draws the
same seeded event stream and routes it with sharding.EntityRouter; after each tick the ranks exchange their chd_handoff_entities
lists and the receivers adopt the entities with chd_spawn_entities.  Each rank also feeds the whole stream to a whole-world table
engine on its GPU, and every tick: per connection the visible set equals the whole world's, the ranks' handover lists together are
the whole world's (each change once), each rank's delta is the set difference of its visible lists, and after the hand-offs every
live id lives on exactly one rank."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding, synth  # noqa: E402
from tests.test_gpu_sharded_table import ID_SPACE, NO_MOVES, Events, _apply, _live_ids, _vis_sets  # noqa: E402

TICK = 33_000_000
NS = SimpleNamespace(capi=capi)
FLAGS = capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_VISIBLE_DELTA


def keys(off, ent, n):
    off = np.asarray(off, np.uint64)[: n + 1]
    slot = np.repeat(np.arange(len(off) - 1, dtype=np.uint64), np.diff(off).astype(np.int64))
    return set(((slot << np.uint64(32)) | np.asarray(ent[: len(slot)], np.uint64)).tolist())


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    failures = 0
    n_ent, n_sub, radius = 40_000, 2_000, 1000.0
    wc = synth.scaled(synth.CONFIGS["benchmark"], n_ent, n_sub)
    halo = sharding.halo_columns(radius, wc.w)
    ev = Events(wc, 2024)
    router = sharding.EntityRouter(world, wc.cols, wc.offx, wc.w)
    first = ev.spawn(n_ent, n_out=20)
    cx, cz = first[1][20: 20 + 10 * n_sub: 10].copy(), first[2][20: 20 + 10 * n_sub: 10].copy()
    subs = np.nonzero(router.owner_of_x(cx) == rank)[0]
    own_cap, cap = 2 * n_ent, n_ent
    e = engine.Engine(wc.cfg(), own_cap + cap * world + 16, max(len(subs), 1), device=local, max_visible=1 << 26)
    uid = torch.zeros(128, dtype=torch.uint8, device=dev)
    if rank == 0:
        uid.copy_(torch.frombuffer(bytearray(engine.Engine.comm_unique_id()), dtype=torch.uint8))
    dist.broadcast(uid, 0)
    e.comm_init(uid.cpu().numpy().tobytes(), rank, world, halo, cap)  # the slab first, then the table
    e.entity_table_init()
    e.set_subscribers(subs.astype(np.uint32) + 1)
    e.reserve_visible_delta_ids(1 << 24, ID_SPACE)
    whole = engine.Engine(wc.cfg(), own_cap, n_sub, device=local, max_visible=1 << 26)
    whole.entity_table_init()
    whole.set_subscribers(np.arange(1, n_sub + 1, dtype=np.uint32))
    prev = set()
    frozen = set()
    handed = crossing = 0
    for tick in range(7):
        t_ns = (tick + 1) * TICK
        sp, mv, dp = (first, NO_MOVES, np.zeros(0, np.uint32)) if tick == 0 else ev.tick(frozen)
        _apply(whole, sp, mv, dp)
        _apply(e, router.spawn(*sp)[rank], router.move(*mv)[rank], router.despawn(dp)[rank])
        batch, keep = engine.make_batch(len(subs), sub=np.arange(len(subs), dtype=np.uint32), sphere=(cx[subs], cz[subs], np.full(len(subs), radius)))
        s = e.tick_sharded(batch, t_ns, FLAGS)
        b1, k1 = engine.make_batch(n_sub, sphere=(cx, cz, np.full(n_sub, radius)))
        s1 = whole.tick(b1, t_ns, capi.TICK_BUILD | capi.TICK_EMIT)
        bad = int(s.overflow != 0) + int(s1.overflow != 0)
        w_vis = _vis_sets(*whole.get_visible())
        now = e.get_visible()
        bad += sum(1 for k, v in enumerate(_vis_sets(*now)) if v != w_vis[subs[k]])
        # the delta is the set difference of consecutive visible lists, slot by slot
        eo, en, lo, le = e.get_visible_delta()
        n = len(subs)
        now_k = keys(*now, n)
        bad += int(keys(eo, en, n) != now_k - prev) + int(keys(lo, le, n) != prev - now_k)
        prev = now_k
        a, b_, c = e.get_handover(s.n_handover)
        mine_ho = list(zip(a.tolist(), b_.tolist(), c.tolist()))
        all_ho = [None] * world
        dist.all_gather_object(all_ho, mine_ho)
        w_ho = set(zip(*[v.tolist() for v in whole.get_handover(s1.n_handover)]))
        union = set(h for part in all_ho for h in part)
        bad += int(union != w_ho) + int(sum(len(p) for p in all_ho) != len(w_ho))
        crossing += sum(1 for part in all_ho for _, src, dst in part
                        if src and dst and sharding.owner_of_column((src - engine.SPATIAL_CHANNEL_ID_START) % wc.cols, wc.cols, world)
                        != sharding.owner_of_column((dst - engine.SPATIAL_CHANNEL_ID_START) % wc.cols, wc.cols, world))
        # hand-offs: every rank learns every list (the router is replicated), the destinations adopt
        ids, dst, x, z = e.handoff_entities()
        lists = [None] * world
        dist.all_gather_object(lists, (ids.tolist(), dst.tolist(), x.tolist(), z.tolist()))
        adopt = router.handoff(lists)
        handed += sum(len(v[0]) for v in lists)
        if len(adopt[rank][0]):
            bad += int(not (e.spawn_entities(*adopt[rank]) == 0).all())
        frozen = set(i for part in adopt for i in part[0].tolist())
        live = [None] * world
        dist.all_gather_object(live, _live_ids(NS, e))
        w_live = _live_ids(NS, whole)
        bad += int(sum(len(v) for v in live) != len(w_live)) + int(set().union(*live) != w_live)
        bad += int(live[rank] != set(i for i, o in router.owner.items() if o == rank))
        failures += bad
        print("rank %d tick %d: own=%d subs=%d mismatches=%d handed=%d crossing=%d" % (rank, tick, len(live[rank]), n, bad, handed, crossing), flush=True)
    if handed == 0 or crossing == 0:
        failures += 1
        print("rank %d: no hand-off or no handover across slabs (%d, %d)" % (rank, handed, crossing), flush=True)
    e.close()
    whole.close()
    t = torch.tensor([failures], device=dev)
    dist.all_reduce(t)
    dist.destroy_process_group()
    if int(t[0]) != 0:
        raise SystemExit("multi-GPU table FAILED: %d mismatches" % int(t[0]))
    if rank == 0:
        print("multi-GPU table OK")


if __name__ == "__main__":
    main()
