"""Host-side mirror of channeld's SpatialController plugin surface (pkg/channeld/spatial.go:17-35) on top of the
C ABI.  Method names, argument meaning and error behaviour follow the Go interface so the parity tests read
like the reference's own tests (spatial_test.go).  Go returns (value, error); here errors are raised as
SpatialError carrying the same condition.

This class contains NO arithmetic of the hot path: every position -> cell, query and fan-out decision is a
call into libchd_b200.so.  The cgo shim of INTEGRATION.md (go/gpucontroller.go) is the same thing in Go.
"""
import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import capi
from .engine import Engine, grid_cfg, make_batch, SPATIAL_CHANNEL_ID_START


class SpatialError(Exception):
    pass


@dataclass
class ChannelSubscriptionOptions:  # channeld.proto ChannelSubscriptionOptions: the fan-out fields (None = not set in the message)
    FanOutIntervalMs: Optional[int] = None
    FanOutDelayMs: Optional[int] = None
    SkipSelfUpdateFanOut: Optional[bool] = None
    SkipFirstFanOut: Optional[bool] = None


@dataclass
class SpatialInfo:  # pkg/common/common.go:20-24
    X: float = 0.0
    Y: float = 0.0
    Z: float = 0.0


@dataclass
class SpotsAOI:  # channeld.proto:438-443
    Spots: List[SpatialInfo] = field(default_factory=list)
    Dists: List[int] = field(default_factory=list)


@dataclass
class BoxAOI:  # channeld.proto:446-450
    Center: SpatialInfo = None
    Extent: SpatialInfo = None


@dataclass
class SphereAOI:  # channeld.proto:452-456
    Center: SpatialInfo = None
    Radius: float = 0.0


@dataclass
class ConeAOI:  # channeld.proto:458-465
    Center: SpatialInfo = None
    Direction: SpatialInfo = None
    Angle: float = 0.0
    Radius: float = 0.0


@dataclass
class SpatialInterestQuery:  # channeld.proto:436-469
    SpotsAOI: Optional[SpotsAOI] = None
    BoxAOI: Optional[BoxAOI] = None
    SphereAOI: Optional[SphereAOI] = None
    ConeAOI: Optional[ConeAOI] = None


@dataclass
class SpatialRegion:  # channeld.proto:419-424
    Min: SpatialInfo
    Max: SpatialInfo
    ChannelId: int
    ServerIndex: int


MinY = -3.40282347e+38 / 2  # spatial.go:80-83
MaxY = 3.40282347e+38 / 2


def pack_queries(queries: Sequence[SpatialInterestQuery], subs=None):
    """SpatialInterestQuery objects -> chd_query_batch (SoA).  nil Center/Extent/Direction would panic in the
    reference (spatial.go:205,237,272); the shim rejects them up front."""
    n = len(queries)
    kind = np.zeros(n, np.uint8)
    sph = [np.zeros(n) for _ in range(3)]
    box = [np.zeros(n) for _ in range(4)]
    cone = [np.zeros(n) for _ in range(6)]
    spot_off = np.zeros(n + 1, np.uint32)
    spot_ndist = np.zeros(n, np.uint32)
    sx, sz, sd = [], [], []
    for i, q in enumerate(queries):
        if q is None:
            raise SpatialError("query is nil")  # spatial.go:183-185
        if q.SpotsAOI is not None:
            kind[i] |= capi.AOI_SPOTS
            for s in q.SpotsAOI.Spots:
                sx.append(s.X); sz.append(s.Z)
            nd = min(len(q.SpotsAOI.Dists), len(q.SpotsAOI.Spots))
            sd += list(q.SpotsAOI.Dists[:nd]) + [0] * (len(q.SpotsAOI.Spots) - nd)
            spot_ndist[i] = nd
        spot_off[i + 1] = len(sx)
        if q.BoxAOI is not None:
            if q.BoxAOI.Center is None or q.BoxAOI.Extent is None:
                raise SpatialError("BoxAOI with nil Center/Extent")
            kind[i] |= capi.AOI_BOX
            box[0][i], box[1][i], box[2][i], box[3][i] = q.BoxAOI.Center.X, q.BoxAOI.Center.Z, q.BoxAOI.Extent.X, q.BoxAOI.Extent.Z
        if q.SphereAOI is not None:
            if q.SphereAOI.Center is None:
                raise SpatialError("SphereAOI with nil Center")
            kind[i] |= capi.AOI_SPHERE
            sph[0][i], sph[1][i], sph[2][i] = q.SphereAOI.Center.X, q.SphereAOI.Center.Z, q.SphereAOI.Radius
        if q.ConeAOI is not None:
            if q.ConeAOI.Center is None or q.ConeAOI.Direction is None:
                raise SpatialError("ConeAOI with nil Center/Direction")
            kind[i] |= capi.AOI_CONE
            c = q.ConeAOI
            cone[0][i], cone[1][i], cone[2][i], cone[3][i], cone[4][i], cone[5][i] = (
                c.Center.X, c.Center.Z, c.Direction.X, c.Direction.Z, c.Angle, c.Radius)
    spots = None
    if len(sx):
        spots = (spot_off, spot_ndist, np.array(sx, np.float64), np.array(sz, np.float64), np.array(sd, np.uint32))
    return make_batch(n, sub=None if subs is None else np.asarray(subs, np.uint32), kind=kind, sphere=sph, box=box, cone=cone,
                      spots=spots)


class GpuStaticGrid2DSpatialController:
    """Drop-in for StaticGrid2DSpatialController (spatial.go:89-124) backed by the GPU engine."""

    def __init__(self, device=0, max_entities=1 << 16, max_subscribers=1 << 12, **limits):
        self._device, self._ne, self._ns, self._limits = device, max_entities, max_subscribers, limits
        self.engine: Optional[Engine] = None
        self.SpatialChannelIdStart = SPATIAL_CHANNEL_ID_START

    # -- LoadConfig(config []byte) error   (spatial.go:141-159)
    def LoadConfig(self, config) -> None:
        c = json.loads(config) if isinstance(config, (bytes, str)) else dict(config)
        if "Config" in c and "GridWidth" not in c:  # accept the whole -scc file as InitSpatialController reads it (spatial.go:54-68)
            c = c["Config"]
        for k in ("GridWidth", "GridHeight"):
            if not c.get(k, 0) > 0:
                raise SpatialError("GridWidth and GridHeight should be positive")
        for k in ("GridCols", "GridRows"):
            if not c.get(k, 0) > 0:
                raise SpatialError("GridCols and GridRows should be positive")
        for k in ("ServerCols", "ServerRows"):
            if not c.get(k, 0) > 0:
                raise SpatialError("ServerCols and ServerRows should be positive")
        # ServerInterestBorderSize <= 0 is rejected by LoadConfig but InitSpatialController drops the error
        # (spatial.go:68,155-157) and the benchmark configs use 0: tolerated here as well.
        self.GridWidth, self.GridHeight = float(c["GridWidth"]), float(c["GridHeight"])
        self.GridCols, self.GridRows = int(c["GridCols"]), int(c["GridRows"])
        self.WorldOffsetX, self.WorldOffsetZ = float(c.get("WorldOffsetX", 0)), float(c.get("WorldOffsetZ", 0))
        self.ServerCols, self.ServerRows = int(c["ServerCols"]), int(c["ServerRows"])
        self.ServerInterestBorderSize = int(c.get("ServerInterestBorderSize", 0))
        self.cfg = grid_cfg(self.WorldOffsetX, self.WorldOffsetZ, self.GridWidth, self.GridHeight, self.GridCols, self.GridRows,
                            self.ServerCols, self.ServerRows, self.ServerInterestBorderSize, self.SpatialChannelIdStart)
        if self.engine is not None:
            self.engine.close()
        self.engine = Engine(self.cfg, self._ne, self._ns, self._device, **self._limits)

    # -- GetChannelId(info SpatialInfo) (ChannelId, error)   (spatial.go:161-163)
    def GetChannelId(self, info: SpatialInfo) -> int:
        ids, ok = self.engine.cell_of(np.array([info.X]), np.array([info.Z]), with_valid=True)
        cid = int(ids[0])
        if not ok[0]:  # (an explicit flag: with SpatialChannelIdStart == 0 the id 0 is a real cell)
            raise SpatialError("position (%f, %f) is outside the grid" % (info.X, info.Z))
        return cid

    def GetChannelIds(self, x, z) -> np.ndarray:
        """Batched GetChannelId (handleQuerySpatialChannel, message_spatial.go:335-370); 0 marks an error."""
        return self.engine.cell_of(x, z)

    # -- QueryChannelIds(query) (map[ChannelId]uint, error)   (spatial.go:182-317)
    def QueryChannelIds(self, query: SpatialInterestQuery) -> Dict[int, int]:
        if query is None:
            raise SpatialError("query is nil")
        res = self.QueryChannelIdsBatch([query])[0]
        if isinstance(res, SpatialError):
            raise res
        return res

    def QueryChannelIdsBatch(self, queries: Sequence[SpatialInterestQuery]):
        batch, keep = pack_queries(queries)
        status, off, ids, dist = self.engine.query_channel_ids(batch)
        out = []
        for i in range(len(queries)):
            if status[i] != capi.Q_OK:
                out.append(SpatialError({capi.Q_ERR_OUT_OF_WORLD: "center is outside the grid", capi.Q_ERR_BAD_STEP: "invalid radius/extent",
                                         capi.Q_ERR_ITER_BOUND: "step absorbed (reference would not terminate)",
                                         capi.Q_ERR_ANGLE_RANGE: "cone angle out of range"}.get(int(status[i]), "error %d" % status[i])))
            else:
                out.append({int(ids[k]): int(dist[k]) for k in range(off[i], off[i + 1])})
        return out

    # -- GetRegions() ([]*SpatialRegion, error)   (spatial.go:319-356)
    def GetRegions(self) -> List[SpatialRegion]:
        n = self.GridCols * self.GridRows
        a = [np.zeros(n) for _ in range(4)]
        cid, srv = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        import ctypes as C
        st = capi.lib().chd_get_regions(C.byref(self.cfg), *[capi.ptr(v) for v in a], capi.ptr(cid), capi.ptr(srv))
        if st != capi.OK:
            raise SpatialError("GetRegions failed")
        return [SpatialRegion(SpatialInfo(a[0][i], MinY, a[1][i]), SpatialInfo(a[2][i], MaxY, a[3][i]), int(cid[i]), int(srv[i]))
                for i in range(n)]

    # -- GetAdjacentChannels(id) ([]ChannelId, error)   (spatial.go:358-381)
    def GetAdjacentChannels(self, spatialChannelId: int) -> List[int]:
        import ctypes as C
        out = np.zeros(8, np.uint32)
        n = capi.lib().chd_get_adjacent_channels(C.byref(self.cfg), int(spatialChannelId), capi.ptr(out))
        return [int(v) for v in out[:n]]

    # -- Notify(oldInfo, newInfo, provider)   (spatial.go:612-626, the data-parallel prefix), batched:
    # set_entities + build compares every entity's cell with the previous build and returns the crossings
    # (entity, srcChannelId, dstChannelId); the handover orchestration (spatial.go:628-858) stays on the host.
    def NotifyBatch(self, x, z) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        self.engine.set_entities(x, z)
        self.engine.build()
        s = self.engine.summary()
        return self.engine.get_handover(int(s.n_handover))

    # -- entities as the reference delivers them, keyed by NetGUID (entity-table mode, switched on by the first call):
    # SpawnObjects = handleSpawnObject's GetChannelId + addSpatialEntity (pkg/unreal/message.go:20-150), DestroyObjects = the
    # destroy handler (message.go:152-203), MoveEntities = ENTITY-channel updates whose Merge hook calls Notify for that entity only
    # (examples/channeld-ue-tps/tpspb/data.go:227-256, spatial.go:612-626).  Spawns / destroys return a capi.EV_* status per id;
    # results (cells, visible lists, handovers, deltas) name NetGUIDs.
    def _table(self):
        if not getattr(self, "_table_on", False):
            self.engine.entity_table_init()
            self._table_on = True
        return self.engine

    def SpawnObjects(self, net_ids, x, z) -> np.ndarray:
        return self._table().spawn_entities(net_ids, x, z)

    def DestroyObjects(self, net_ids) -> np.ndarray:
        return self._table().despawn_entities(net_ids)

    def MoveEntities(self, net_ids, x, z) -> None:
        self._table().move_entities(net_ids, x, z)

    # -- connections whose interest follows their pawn (a client "stands on its pawn"): bound once, then every Tick(None, ...,
    # follow=...) builds the UPDATE_SPATIAL_INTEREST batch (message_spatial.go:41-129) on the device from the entities' positions.
    # queries[i] gives the AOI SHAPE of connection slot i (SphereAOI / BoxAOI / ConeAOI, any combination); its Center is ignored,
    # the centre is entity net_ids[i] (entity index without SpawnObjects).  SpotsAOI is absolute and cannot follow an entity.
    # On a slab (entity-table mode only) a follower lives on its entity's owner (sharding.FollowerRegistry); a follower whose query
    # would reach columns the slab does not serve reports capi.FOLLOW_OUTSIDE_SLAB.
    def FollowEntities(self, conn_slots, net_ids, queries: Sequence[SpatialInterestQuery]) -> None:
        n = len(queries)
        kind = np.zeros(n, np.uint8)
        sph_r = np.zeros(n)
        box = [np.zeros(n) for _ in range(2)]
        cone = [np.zeros(n) for _ in range(4)]
        for i, q in enumerate(queries):
            if q is None:
                raise SpatialError("query is nil")
            if q.SpotsAOI is not None:
                raise SpatialError("SpotsAOI has absolute positions and cannot follow an entity")
            if q.SphereAOI is not None:
                kind[i] |= capi.AOI_SPHERE
                sph_r[i] = q.SphereAOI.Radius
            if q.BoxAOI is not None:
                if q.BoxAOI.Extent is None:
                    raise SpatialError("BoxAOI with nil Extent")
                kind[i] |= capi.AOI_BOX
                box[0][i], box[1][i] = q.BoxAOI.Extent.X, q.BoxAOI.Extent.Z
            if q.ConeAOI is not None:
                if q.ConeAOI.Direction is None:
                    raise SpatialError("ConeAOI with nil Direction")
                kind[i] |= capi.AOI_CONE
                c = q.ConeAOI
                cone[0][i], cone[1][i], cone[2][i], cone[3][i] = c.Direction.X, c.Direction.Z, c.Angle, c.Radius
            if not kind[i]:
                raise SpatialError("query without an AOI")
        self.engine.follow_bind(conn_slots, net_ids, kind=kind, sph_r=sph_r, box=box, cone=cone)

    def UnfollowEntities(self, conn_slots) -> None:
        self.engine.follow_unbind(conn_slots)

    # -- Tick()   (channel.go:358-387 for all spatial channels at once).  follow = capi.FOLLOW_ALL / FOLLOW_MOVED with batch None:
    # the batch is generated from the FollowEntities bindings.  explicit = the UPDATE_SPATIAL_INTEREST batch of the connections that
    # send their own queries this tick (spectators, SpotsAOI, ...): merged in front of the generated one, and a following
    # connection that sent one uses it for this tick.
    def Tick(self, batch, t_ns, flags=capi.TICK_ALL, follow=None, explicit=None):
        if follow is not None:
            if batch is not None:
                raise SpatialError("a followed tick generates its own batch")
            if explicit is not None:
                self.engine.follow_queries_with(follow, explicit)
            else:
                self.engine.follow_queries(follow)
            flags |= capi.TICK_FOLLOW
        elif explicit is not None:
            raise SpatialError("explicit queries are merged into a followed tick: pass follow=")
        return self.engine.tick(batch, t_ns, flags)

    # -- SubscribeToChannel / UnsubscribeFromChannel for spatial channels (subscription.go:34-125), batched: what handleSubToChannel /
    # handleUnsubFromChannel (message.go:488-605) and a server's subscriptions to its own cells after CreateChannels
    # (message_spatial.go:167-173) do to the fan-out state.  options[i] (None = no options) carries the fields the message set;
    # DataAccess and DataFieldMasks stay with the host.  Applied between ticks, at channel time t_ns; returns capi.SUB_* per op.
    def SubscribeToChannelBatch(self, conn_slots, channel_ids, options: Sequence[Optional["ChannelSubscriptionOptions"]], t_ns) -> np.ndarray:
        n = len(conn_slots)
        present = np.zeros(n, np.uint8)
        iv, dl = np.zeros(n, np.uint32), np.zeros(n, np.int32)
        ss, sf = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        for i, o in enumerate(options):
            if o is None:
                continue
            for v, arr, bit in ((o.FanOutIntervalMs, iv, capi.SUBOPT_INTERVAL), (o.FanOutDelayMs, dl, capi.SUBOPT_DELAY),
                                (o.SkipSelfUpdateFanOut, ss, capi.SUBOPT_SKIP_SELF), (o.SkipFirstFanOut, sf, capi.SUBOPT_SKIP_FIRST)):
                if v is not None:
                    arr[i] = v
                    present[i] |= bit
        return self.engine.apply_subscriptions(conn_slots, channel_ids, np.full(n, capi.SUBOP_SUB, np.uint8), interval=iv, delay=dl, skip_self=ss,
                                               skip_first=sf, now_ns=t_ns, present=present)

    def UnsubscribeFromChannelBatch(self, conn_slots, channel_ids) -> np.ndarray:
        n = len(conn_slots)
        return self.engine.apply_subscriptions(conn_slots, channel_ids, np.full(n, capi.SUBOP_UNSUB, np.uint8))

    # -- per client, the entities to spawn / despawn since the last delta: the net effect of the FULL data a new subscription
    # sends, the despawns of an unsubscription and the handovers between cells (spatial.go:612-858,
    # SpatialChannelData.AddEntity/RemoveEntity).  ReserveVisibleDelta once (and again, larger, after CHD_OVF_DELTA), then
    # Tick with capi.TICK_VISIBLE_DELTA; GetVisibleDelta only reads the last delta back.
    def ReserveVisibleDelta(self, cap_entries):
        self.engine.reserve_visible_delta(cap_entries)

    # The same with entities named by global id in [0, id_space) (engine.set_entity_ids / the halo records): the mode for
    # sharded engines.  Migrated connections are netted on the host (sharding.net_migrant_delta).
    def ReserveVisibleDeltaIds(self, cap_entries, id_space):
        self.engine.reserve_visible_delta_ids(cap_entries, id_space)

    # -> (enter_off, enter, leave_off, leave): CSR by subscriber slot of entity indices (global ids in id mode).
    def GetVisibleDelta(self):
        return self.engine.get_visible_delta()
