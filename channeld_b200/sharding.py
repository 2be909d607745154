"""X-slab sharding of the grid across ranks (SURVEY.md §8e): host-side placement logic only.

GPU g of G owns grid columns [floor(g*cols/G), floor((g+1)*cols/G)).  Entities live on the owner of their column,
subscribers on the owner of their centre's column; a query touches at most `halo` columns beyond its slab, so
one all-gather of border-column entity records per tick makes every rank's cell lists complete for its
subscribers.  The per-tick driver (`ShardedTick`) is engine-agnostic so the N>1 control flow is testable on
CPU with the gloo backend.
"""
import math

import numpy as np


def slab_columns(cols: int, world: int, rank: int):
    return (rank * cols) // world, ((rank + 1) * cols) // world


def owner_of_column(col, cols: int, world: int):
    """Inverse of slab_columns for arrays of columns (col < 0 -> rank 0)."""
    col = np.asarray(col, np.int64)
    # the owner is the largest g with floor(g*cols/world) <= col
    g = np.minimum(((col + 1) * world - 1) // cols, world - 1)
    g = np.where(col < 0, 0, g)
    return g.astype(np.int64)


def halo_columns(radius: float, grid_width: float) -> int:
    return max(1, int(math.ceil(radius / grid_width)))


def column_of(x, offx: float, w: float, cols: int):
    """Grid column of each x (placement only; -1 outside the world).  The engine recomputes cells on the GPU."""
    c = np.floor((np.asarray(x, np.float64) - offx) / w)
    return np.where((c >= 0) & (c < cols), c, -1).astype(np.int64)


class SlotTable:
    """Host-managed subscriber slots of every rank (the engine's slots are the host's to assign: chd_add_subscribers /
    chd_migrate_in name them).  Every process of a multi-rank host keeps the tables of ALL ranks (routing decisions are a pure
    function of the subscribers' positions, so they are computed identically everywhere: no host communication)."""

    def __init__(self, world: int):
        self.world = world
        self.owner = {}                              # subscriber -> rank
        self.slot = {}                               # subscriber -> local slot on its rank
        self.at = [dict() for _ in range(world)]     # per rank: slot -> subscriber
        self._free = [list() for _ in range(world)]
        self._used = [0] * world

    def take(self, rank: int) -> int:
        if self._free[rank]:
            return self._free[rank].pop()
        self._used[rank] += 1
        return self._used[rank] - 1

    def release(self, rank: int, slots):
        """Slots vacated by a tick's emigrants are reusable from the NEXT tick on (the engine frees them in that tick's update)."""
        self._free[rank] += list(slots)

    def place(self, j, rank: int) -> int:
        s = self.take(rank)
        self.owner[j], self.slot[j] = rank, s
        self.at[rank][s] = j
        return s

    def remove(self, j):
        rank, s = self.owner.pop(j), self.slot.pop(j)
        del self.at[rank][s]
        return rank, s


def plan_migrations(table: SlotTable, new_owner):
    """One tick's routing changes.  new_owner: dict / sequence subscriber -> rank that owns its centre's column NOW.
    Returns (arrivals, out_lists, in_calls, vacated):
      arrivals[rank]   = [(subscriber, slot)] first placements                      -> chd_add_subscribers
      out_lists[rank]  = [subscriber] emigrants in blob-record order                -> chd_migrate_out(vacated[rank])
      in_calls         = [(dst, src, first_index, [(subscriber, slot)])]            -> chd_migrate_in(dst: src, first_index, slots, conns)
      vacated[rank]    = the emigrants' old slots (release them after the tick)
    and applies the changes to `table`.  Records of one source rank are grouped by destination, so each (src, dst) pair is one
    contiguous run of src's blob."""
    world = table.world
    items = new_owner.items() if hasattr(new_owner, "items") else enumerate(new_owner)
    arrivals = [[] for _ in range(world)]
    moves = {}
    for j, r in items:
        r = int(r)
        if j not in table.owner:
            arrivals[r].append(j)
        elif table.owner[j] != r:
            moves.setdefault((table.owner[j], r), []).append(j)
    out_lists = [[] for _ in range(world)]
    in_calls = []
    for (a, b) in sorted(moves):
        in_calls.append([b, a, len(out_lists[a]), list(moves[(a, b)])])
        out_lists[a] += moves[(a, b)]
    vacated = [[table.slot[j] for j in out_lists[a]] for a in range(world)]
    for a in range(world):
        for j in out_lists[a]:
            table.remove(j)
    for call in in_calls:
        call[3] = [(j, table.place(j, call[0])) for j in call[3]]
    arrivals = [[(j, table.place(j, r)) for j in arrivals[r]] for r in range(world)]
    return arrivals, out_lists, [tuple(c) for c in in_calls], vacated


def route_sub_ops(table: SlotTable, subscribers):
    """Splits a batch of explicit subscription ops (include/chd_gpu_subs_sharded.h) whose ops name subscriber keys into one batch per
    rank: -> [(op indices int64, slots u32)] per rank, the ops of each rank in array order (so several ops on one pair keep theirs).
    Give rank r's batch the op arrays indexed by its op indices and its slots, and put the ranks' statuses back in the batch's order
    with merge_sub_status.  A key the table does not hold is routed nowhere and gets SUB_ERR_SLOT there.

    A slab accepts SUBs of the cells it serves only (columns [col_lo - halo, col_hi + halo)).  A spatial server whose region plus
    border spans more than one rank's served columns is therefore placed once per rank it needs, under one key per (connection,
    rank): SlotTable keys are arbitrary, e.g. ("server", conn, r) placed on rank r.  Each of its ops names the key on the owner of the
    cell's column, owner_of_column((channel - channel_id_start) % cols, cols, world); that rank serves the cell."""
    keys = list(subscribers)
    rank = np.array([table.owner.get(k, -1) for k in keys], np.int64)
    slot = np.array([table.slot.get(k, 0) for k in keys], np.uint32)
    out = []
    for r in range(table.world):
        idx = np.nonzero(rank == r)[0]
        out.append((idx, slot[idx]))
    return out


def merge_sub_status(routes, statuses, n: int):
    """route_sub_ops' inverse for the statuses: statuses[r] = rank r's CHD_SUB_* per op of its batch -> u8[n] in the batch's order,
    SUB_ERR_SLOT for the ops no rank received (unknown keys)."""
    from .capi import SUB_ERR_SLOT

    out = np.full(int(n), SUB_ERR_SLOT, np.uint8)
    for (idx, _), st in zip(routes, statuses):
        out[idx] = np.asarray(st, np.uint8)
    return out


def net_migrant_delta(leave_src, enter_dst):
    """A connection migrated from rank A to rank B (plan_migrations' in_calls), as id-mode visible deltas see it: A's delta
    reports its old slot leaving everything A's snapshot held, B's reports its new slot entering everything it sees now.  The
    connection's own delta is their net:
        enter = enter_B \\ leave_A        leave = leave_A \\ enter_B
    exact when leave_src is A's delta of the tick that ran chd_migrate_out and enter_dst is B's first successful delta for the
    connection.  Global ids in, (enter, leave) out as u32 arrays in the order of the lists they come from."""
    leave_src = np.asarray(leave_src, np.uint32)
    enter_dst = np.asarray(enter_dst, np.uint32)
    return enter_dst[~np.isin(enter_dst, leave_src)], leave_src[~np.isin(leave_src, enter_dst)]


class EntityRouter:
    """Host router of a sharded entity-table host (chd_entity_table_init on X-slabs): every rank's table holds the entities it
    owns, and the router keeps id -> owning rank.  A spawn goes to the owner of its position's column (a spawn outside the world to
    the owner of the clamped column); moves and despawns go to the id's current owner; after each tick the ranks' hand-off lists
    (chd_handoff_entities) become adoption batches (spawns) for their destinations and the map follows.  Ids the router does not
    know are routed nowhere.  Every method returns one batch per rank."""

    def __init__(self, world: int, cols: int, offx: float, w: float):
        self.world, self.cols, self.offx, self.w = int(world), int(cols), float(offx), float(w)
        self.owner = {}  # id -> rank

    def owner_of_x(self, x):
        """Owning rank of the (clamped) column of each x."""
        with np.errstate(invalid="ignore"):
            c = np.floor((np.asarray(x, np.float64) - self.offx) / self.w)
        c = np.where(np.isnan(c), 0, np.clip(c, 0, self.cols - 1)).astype(np.int64)
        return owner_of_column(c, self.cols, self.world)

    def _split(self, rank, *arrays):
        return [tuple(np.asarray(a)[rank == r] for a in arrays) for r in range(self.world)]

    def _rank_of_ids(self, ids):
        return np.array([self.owner.get(int(i), -1) for i in ids], np.int64)

    @staticmethod
    def _facing(fx, fz):
        return () if fx is None else (np.asarray(fx), np.asarray(fz))

    def spawn(self, ids, x, z, fx=None, fz=None):
        """-> per rank (ids u32, x, z), or (ids, x, z, fx, fz) for chd_spawn_entities_facing when facings are given.  An id that is
        already live goes to its owner (which reports it as a duplicate)."""
        ids = np.asarray(ids, np.uint32)
        rank = self.owner_of_x(x)
        known = self._rank_of_ids(ids)
        rank = np.where(known >= 0, known, rank)
        for i, r in zip(ids.tolist(), rank.tolist()):
            self.owner.setdefault(i, r)
        return self._split(rank, ids, np.asarray(x, np.float64), np.asarray(z, np.float64), *self._facing(fx, fz))

    def move(self, ids, x, z, fx=None, fz=None):
        """-> per rank (ids u32, x, z) for chd_move_entities, or (ids, x, z, fx, fz) for chd_move_entities_facing."""
        ids = np.asarray(ids, np.uint32)
        return self._split(self._rank_of_ids(ids), ids, np.asarray(x), np.asarray(z), *self._facing(fx, fz))

    def despawn(self, ids):
        """-> per rank ids u32; the ids leave the map."""
        ids = np.asarray(ids, np.uint32)
        rank = self._rank_of_ids(ids)
        for i in ids.tolist():
            self.owner.pop(i, None)
        return [b[0] for b in self._split(rank, ids)]

    def handoff(self, lists):
        """lists[r] = rank r's chd_handoff_entities result (id, dst_rank, x, z) -> per rank (ids u32, x, z) to adopt with
        chd_spawn_entities; every listed id is owned by its destination from now on.  With chd_handoff_entities_facing results
        (id, dst_rank, x, z, fx, fz) the batches are (ids, x, z, fx, fz) for chd_spawn_entities_facing; when only some lists carry
        facings, the entities of the others get none (0, 0)."""
        facing = any(len(l) == 6 for l in lists)
        out = [tuple([] for _ in range(5 if facing else 3)) for _ in range(self.world)]
        for l in lists:
            if len(l) not in (4, 6):
                raise ValueError("a hand-off list is (id, dst_rank, x, z) or (id, dst_rank, x, z, fx, fz)")
            ids, dst = l[0], l[1]
            cols = [np.asarray(a) for a in l[2:4]]
            if facing:
                cols += [np.asarray(a) for a in l[4:6]] if len(l) == 6 else [np.zeros(len(cols[0]))] * 2
            for k, (i, d) in enumerate(zip(np.asarray(ids).tolist(), np.asarray(dst).tolist())):
                self.owner[i] = d
                out[d][0].append(i)
                for c, a in enumerate(cols):
                    out[d][1 + c].append(a[k])
        return [(np.asarray(o[0], np.uint32),) + tuple(np.asarray(a, np.float64) for a in o[1:]) for o in out]


class FollowerRegistry:
    """Followers on a sharded entity-table host (chd_follow_bind on X-slabs).  A follower lives on the rank that owns its entity, so
    its centre is always an own entity of that rank's table and its exact position is local.  Every process keeps the registry of
    ALL ranks, as it keeps the EntityRouter: connection -> (entity id, kind, shape), and the connections' slots in a SlotTable.

    After each tick's EntityRouter.handoff, plan(router) moves every follower to router.owner[entity] through plan_migrations and
    returns, per destination, the chd_follow_bind batch of its arriving slots (first placements and immigrants).  A follower whose
    entity the router does not know (despawned, not spawned yet) stays where it is; its rank reports CHD_FOLLOW_NO_ENTITY.

    Per tick, on every rank: route the entity events; adopt the hand-offs (spawn); chd_migrate_out / chd_migrate_in (and
    chd_add_subscribers for first placements); bind the arrivals; chd_follow_queries(_with)(CHD_FOLLOW_MOVED);
    chd_tick_sharded(NULL, .., flags | CHD_TICK_FOLLOW); chd_handoff_entities.  chd_migrate_out unbinds the emigrants on the source;
    the binding does not travel in the migration blob, so the destination binds them again."""

    SHAPE = ("sph_r", "box_ex", "box_ez", "cone_dx", "cone_dz", "cone_angle", "cone_r")
    FRAME = ("off_fwd", "off_right", "rot_cos", "rot_sin")

    def __init__(self, world: int):
        self.world = int(world)
        self.slots = SlotTable(world)
        self.bind = {}  # connection -> (entity id, kind, shape: 7 floats in SHAPE order)
        self.frame = {}  # connection -> 4 floats in FRAME order (chd_follow_set_frame), for framed followers only
        self._rebind = set()  # connections bound since the last plan()

    def follow(self, conn, entity, kind, shape, frame=None):
        """Binds (or re-binds) a connection; it is placed or re-bound by the next plan().  frame: (off_fwd, off_right) or
        (off_fwd, off_right, rot_cos, rot_sin) for a follower that turns with its entity (include/chd_gpu_facing.h), None: plain."""
        shape = tuple(float(v) for v in shape)
        if len(shape) != 7:
            raise ValueError("a follower's shape is 7 values: " + ", ".join(self.SHAPE))
        self.bind[conn] = (int(entity), int(kind), shape)
        self.frame.pop(conn, None)
        if frame is not None:
            frame = tuple(float(v) for v in frame)
            if len(frame) == 2:
                frame += (1.0, 0.0)
            if len(frame) != 4:
                raise ValueError("a follower's frame is 2 or 4 values: " + ", ".join(self.FRAME))
            self.frame[conn] = frame
        self._rebind.add(conn)

    def unfollow(self, conn):
        """Forgets a connection -> (rank, slot) it occupied (chd_remove_subscribers there), or None if it was never placed."""
        self.bind.pop(conn, None)
        self.frame.pop(conn, None)
        self._rebind.discard(conn)
        return self.slots.remove(conn) if conn in self.slots.owner else None

    def owner_of(self, conn):
        return self.slots.owner.get(conn)

    def batch(self, conns):
        """The chd_follow_bind arrays of `conns` (placed connections): dict(slot u32, entity u32, kind u8, shape f64 [7][m]), and,
        when some of them have a frame, frame: their chd_follow_set_frame arrays, dict(slot u32, off_fwd, off_right, rot_cos,
        rot_sin), to apply after the bind."""
        conns = list(conns)
        m = len(conns)
        out = dict(slot=np.array([self.slots.slot[c] for c in conns], np.uint32),
                   entity=np.array([self.bind[c][0] for c in conns], np.uint32),
                   kind=np.array([self.bind[c][1] for c in conns], np.uint8),
                   shape=np.array([self.bind[c][2] for c in conns], np.float64).reshape(m, 7).T.copy())
        out["conn"] = conns
        framed = [c for c in conns if c in self.frame]
        if not framed:
            return out
        fr = np.array([self.frame[c] for c in framed], np.float64).reshape(len(framed), 4).T
        out["frame"] = dict(slot=np.array([self.slots.slot[c] for c in framed], np.uint32),
                            **{k: fr[i].copy() for i, k in enumerate(self.FRAME)})
        return out

    def plan(self, router):
        """One tick's placement: -> (arrivals, out_lists, in_calls, vacated, binds) where the first four are plan_migrations' (by
        connection) and binds[rank] is the chd_follow_bind batch (FollowerRegistry.batch) of the connections that arrive on `rank`
        this tick, or were re-bound there with follow(), in connection order, with the frames to set after it when it has framed
        followers (binds[rank]["frame"]: a bind clears a slot's frame, and frames do not travel with migrations either)."""
        conns = sorted(c for c, (e, _, _) in self.bind.items() if e in router.owner)
        new_owner = {c: router.owner[self.bind[c][0]] for c in conns}
        arrivals, out_lists, in_calls, vacated = plan_migrations(self.slots, new_owner)
        fresh = [set() for _ in range(self.world)]
        for r in range(self.world):
            fresh[r] |= {c for c, _ in arrivals[r]}
        for dst, _, _, pairs in in_calls:
            fresh[dst] |= {c for c, _ in pairs}
        for c in self._rebind:
            if c in self.slots.owner:
                fresh[self.slots.owner[c]].add(c)
        self._rebind = {c for c in self._rebind if c not in self.slots.owner}  # (not placed yet: its entity is unknown)
        binds = [self.batch(sorted(fresh[r])) for r in range(self.world)]
        return arrivals, out_lists, in_calls, vacated, binds
