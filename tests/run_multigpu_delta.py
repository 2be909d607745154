"""Multi-GPU id-mode visible-set deltas (one rank per GPU, launched by tests/test_multigpu_delta.py or by hand):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29611 \
        tests/run_multigpu_delta.py

Every rank owns an X-slab and runs chd_tick_sharded with CHD_TICK_VISIBLE_DELTA after chd_reserve_visible_delta_ids.  Entities
drift across slab borders and are re-homed (sender drops, receiver adopts); subscribers follow the owner of their centre's column
through chd_migrate_out / chd_migrate_in, as in tests/run_multigpu_parity.py.  Per connection and tick, the deltas of every rank
(the old slot's on the source rank, the new slot's on the destination) netted with sharding.net_migrant_delta must equal the set
differences of a whole-world single-GPU engine's consecutive visible lists for that connection."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from channeld_b200 import capi, engine, sharding, synth  # noqa: E402

TICK = 33_000_000
FLAGS = capi.TICK_BUILD | capi.TICK_EMIT | capi.TICK_VISIBLE_DELTA


def per_slot(off, ent, slot):
    return ent[int(off[slot]):int(off[slot + 1])] if slot + 1 < len(off) else ent[:0]


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    failures = 0
    n_ticks = int(os.environ.get("CHD_DELTA_TICKS", "6"))
    for name, n_ent, n_sub, radius, max_move in (("benchmark", 60_000, 3_000, 500.0, 900.0), ("2x2", 30_000, 1_500, 500.0, 300.0)):
        wc = synth.scaled(synth.CONFIGS[name], n_ent, n_sub)
        if world > wc.cols:
            continue
        x, z = synth.entities(wc)
        halo = sharding.halo_columns(radius, wc.w)
        ent_owner = sharding.owner_of_column(sharding.column_of(x, wc.offx, wc.w, wc.cols), wc.cols, world)
        mine = np.nonzero(ent_owner == rank)[0]
        cap = n_ent
        stream = torch.cuda.Stream(device=dev)
        e = engine.Engine(wc.cfg(), n_ent + cap * world + 16, n_sub, device=local, max_visible=1 << 26, max_pairs=n_sub * 64 + 1024)
        e.set_stream(stream.cuda_stream)
        uid = torch.zeros(128, dtype=torch.uint8, device=dev)
        if rank == 0:
            uid.copy_(torch.frombuffer(bytearray(engine.Engine.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(uid, 0)
        e.comm_init(uid.cpu().numpy().tobytes(), rank, world, halo, cap, migrate_subscribers=n_sub, migrate_pairs=n_sub * 16)
        e.reserve_visible_delta_ids(1 << 24, n_ent)
        # the whole world on one GPU (slot j = subscriber j, entity index = global id)
        e1 = engine.Engine(wc.cfg(), n_ent, n_sub, device=local, max_visible=1 << 27, max_pairs=n_sub * 64 + 1024)
        e1.set_stream(stream.cuda_stream)
        conn, cx, cz, r = synth.subscribers(wc, x, z, radius)
        e1.set_subscribers(conn)
        table = sharding.SlotTable(world)
        last_owner = np.zeros(n_sub, np.int64)
        prev1 = (np.zeros(n_sub + 1, np.uint64), np.zeros(0, np.uint32))
        n_mig = n_rehome = n_netted = 0
        with torch.cuda.stream(stream):
            for tick in range(n_ticks):
                t_ns = (tick + 1) * TICK
                if tick:
                    x, z = synth.move_entities(wc, x, z, tick, max_move)
                conn, cx, cz, r = synth.subscribers(wc, x, z, radius)
                col = sharding.column_of(cx, wc.offx, wc.w, wc.cols)
                new_owner = np.where(col >= 0, sharding.owner_of_column(col, wc.cols, world), last_owner)
                last_owner = new_owner
                arrivals, out_lists, in_calls, vacated = sharding.plan_migrations(table, new_owner)
                if out_lists[rank]:
                    e.migrate_out(np.array(vacated[rank], np.uint32))
                for (dst, src, first, pairs_) in in_calls:
                    if dst == rank:
                        e.migrate_in(src, first, np.array([s_ for _, s_ in pairs_], np.uint32), conn[[j for j, _ in pairs_]])
                if arrivals[rank]:
                    e.add_subscribers(np.array([s_ for _, s_ in arrivals[rank]], np.uint32), conn[[j for j, _ in arrivals[rank]]])
                n_mig += sum(len(v) for v in out_lists)
                e.set_entities(x[mine], z[mine])
                e.set_entity_ids(mine.astype(np.uint32))
                my_slots = np.array(sorted(table.at[rank]), np.uint32)
                my_subs = np.array([table.at[rank][int(s_)] for s_ in my_slots], np.int64)
                batch, keep = engine.make_batch(len(my_slots), sub=my_slots, sphere=(cx[my_subs], cz[my_subs], r[my_subs]))
                s = e.tick_sharded(batch, t_ns, FLAGS)
                if s.overflow:
                    failures += 1
                    print("rank %d: overflow %#x" % (rank, s.overflow), flush=True)
                for a in range(world):
                    table.release(a, vacated[a])
                e1.set_entities(x, z)
                b1, k1 = engine.make_batch(n_sub, sphere=(cx, cz, r))
                e1.tick(b1, t_ns, capi.TICK_BUILD | capi.TICK_EMIT)
                now1 = e1.get_visible()
                # this rank's part of every connection's delta: its current slots and the slots its emigrants left
                eo, en, lo, le = e.get_visible_delta()
                part = {}
                for s_, j in list(zip(my_slots.tolist(), my_subs.tolist())) + list(zip(vacated[rank], out_lists[rank])):
                    ent_, lea_ = per_slot(eo, en, s_), per_slot(lo, le, s_)
                    if len(ent_) or len(lea_):
                        part[int(j)] = (ent_.tolist(), lea_.tolist())
                parts = [None] * world
                dist.all_gather_object(parts, part)
                bad = 0
                for j in range(n_sub):
                    enters = [g for p in parts if j in p for g in p[j][0]]
                    leaves = [g for p in parts if j in p for g in p[j][1]]
                    enter, leave = sharding.net_migrant_delta(leaves, enters)
                    was, sees = per_slot(*prev1, j), per_slot(*now1, j)
                    if not (np.array_equal(np.sort(enter), np.setdiff1d(sees, was)) and np.array_equal(np.sort(leave), np.setdiff1d(was, sees))):
                        bad += 1
                    if sum(1 for p in parts if j in p) > 1:
                        n_netted += 1
                failures += bad
                prev1 = now1
                # entity re-homing for the next tick: sender drops, receiver adopts
                g_id, g_dst, g_n = e.get_rehome()
                allre = [None] * world
                dist.all_gather_object(allre, (g_id.tolist(), g_dst.tolist()))
                leaving = set(allre[rank][0])
                adopt = [g for (ids, dsts) in allre for g, d_ in zip(ids, dsts) if d_ == rank]
                if leaving or adopt:
                    mine = np.array(sorted((set(mine.tolist()) - leaving) | set(adopt)), np.int64)
                n_rehome += sum(len(v[0]) for v in allre)
                print("rank %d %s tick %d: own=%d slots=%d mismatches=%d migrated=%d netted=%d rehomed=%d" %
                      (rank, name, tick, len(mine), len(my_slots), bad, sum(len(v) for v in out_lists), n_netted, n_rehome), flush=True)
        if name != "2x2" and (n_mig == 0 or n_rehome == 0):
            failures += 1
            print("rank %d %s: nothing migrated or re-homed (%d, %d)" % (rank, name, n_mig, n_rehome), flush=True)
        e.close()
        e1.close()
    t = torch.tensor([failures], device=dev)
    dist.all_reduce(t)
    dist.destroy_process_group()
    if int(t[0]) != 0:
        raise SystemExit("multi-GPU delta FAILED: %d mismatches" % int(t[0]))
    if rank == 0:
        print("multi-GPU delta OK")


if __name__ == "__main__":
    main()
