// Package channeld (drop this file into pkg/channeld of channeldorg/channeld @ 61fa8add).
//
// GpuStaticGrid2DSpatialController implements the SpatialController interface (spatial.go:17-35) on top of
// libchd_b200.so through cgo.  It embeds the reference StaticGrid2DSpatialController for the control-plane
// methods that stay in Go (CreateChannels, Tick's server-slot bookkeeping, the handover orchestration inside
// Notify) and forwards the data-parallel methods to the GPU engine.
//
// UN-RUN: this image has no Go toolchain; the file is written against include/chd_gpu.h and has not been
// compiled.  INTEGRATION.md lists the three-line change to InitSpatialController that selects it.
package channeld

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../channeld_b200 -lchd_b200 -Wl,-rpath,${SRCDIR}/../../channeld_b200
#include <stdlib.h>
#include "chd_gpu.h"
*/
import "C"

import (
	"encoding/json"
	"errors"
	"fmt"
	"runtime"
	"sync"
	"unsafe"

	"github.com/channeldorg/channeld/pkg/channeldpb"
	"github.com/channeldorg/channeld/pkg/common"
)

type GpuStaticGrid2DSpatialController struct {
	StaticGrid2DSpatialController // LoadConfig fields, GetRegions, CreateChannels, Tick, Notify orchestration

	engine  *C.chd_engine
	mu      sync.Mutex // chd_cell_of / chd_query_channel_ids are internally locked; this guards engine lifetime
	tableOn bool       // entity-table mode (SpawnObjects / DestroyObjects / MoveEntities)
}

// LoadConfig (spatial.go:141-159) + engine creation.  ServerInterestBorderSize == 0 is tolerated like
// InitSpatialController does (it drops LoadConfig's error, spatial.go:68).
func (ctl *GpuStaticGrid2DSpatialController) LoadConfig(config []byte) error {
	if err := json.Unmarshal(config, &ctl.StaticGrid2DSpatialController); err != nil {
		return err
	}
	cfg := C.chd_grid_cfg{
		world_offset_x: C.double(ctl.WorldOffsetX), world_offset_z: C.double(ctl.WorldOffsetZ),
		grid_width: C.double(ctl.GridWidth), grid_height: C.double(ctl.GridHeight),
		grid_cols: C.uint32_t(ctl.GridCols), grid_rows: C.uint32_t(ctl.GridRows),
		server_cols: C.uint32_t(ctl.ServerCols), server_rows: C.uint32_t(ctl.ServerRows),
		server_interest_border_size: C.uint32_t(ctl.ServerInterestBorderSize),
		channel_id_start:            C.uint32_t(GlobalSettings.SpatialChannelIdStart),
	}
	var lim C.chd_limits
	C.chd_default_limits(&cfg, 1<<20, 1<<17, &lim)
	lim.default_fanout_interval_ms = C.uint32_t(GlobalSettings.GetChannelSettings(channeldpb.ChannelType_SPATIAL).DefaultFanOutIntervalMs)
	lim.default_fanout_delay_ms = C.int32_t(GlobalSettings.GetChannelSettings(channeldpb.ChannelType_SPATIAL).DefaultFanOutDelayMs)
	if st := C.chd_create(&cfg, &lim, 0, &ctl.engine); st != C.CHD_OK {
		return fmt.Errorf("chd_create: %s", C.GoString(C.chd_last_error(nil)))
	}
	return nil
}

// GetChannelId (spatial.go:161-163).  One position per cgo call is only for interface compatibility; the
// batched form below (handleQuerySpatialChannel, message_spatial.go:335-370) is the one to use on hot paths.
func (ctl *GpuStaticGrid2DSpatialController) GetChannelId(info common.SpatialInfo) (common.ChannelId, error) {
	x, z := C.double(info.X), C.double(info.Z)
	var id C.uint32_t
	var ok C.uint8_t // explicit validity: with SpatialChannelIdStart == 0 the id 0 is a real cell
	if st := C.chd_cell_of_valid(ctl.engine, &x, &z, 1, &id, &ok); st != C.CHD_OK {
		return 0, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	if ok == 0 {
		return 0, fmt.Errorf("position (%f, %f) is outside the grid", info.X, info.Z)
	}
	return common.ChannelId(id), nil
}

func (ctl *GpuStaticGrid2DSpatialController) GetChannelIds(x, z []float64) ([]uint32, error) {
	n := len(x)
	out := make([]uint32, n)
	if n == 0 {
		return out, nil
	}
	st := C.chd_cell_of(ctl.engine, (*C.double)(unsafe.Pointer(&x[0])), (*C.double)(unsafe.Pointer(&z[0])), C.uint32_t(n),
		(*C.uint32_t)(unsafe.Pointer(&out[0])))
	if st != C.CHD_OK {
		return nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return out, nil
}

// QueryChannelIds (spatial.go:182-317) for one query: a batch of one through chd_query_channel_ids.
func (ctl *GpuStaticGrid2DSpatialController) QueryChannelIds(query *channeldpb.SpatialInterestQuery) (map[common.ChannelId]uint, error) {
	if query == nil {
		return nil, fmt.Errorf("query is nil")
	}
	var b C.chd_query_batch
	b.n = 1
	kind := C.uint8_t(0)
	var sph [3]C.double
	var box [4]C.double
	var cone [6]C.double
	var spotOff [2]C.uint32_t
	var spotN C.uint32_t
	var sx, sz []C.double
	var sd []C.uint32_t
	if q := query.SpotsAOI; q != nil {
		kind |= C.CHD_AOI_SPOTS
		for i, s := range q.Spots {
			sx, sz = append(sx, C.double(s.X)), append(sz, C.double(s.Z))
			if i < len(q.Dists) {
				sd = append(sd, C.uint32_t(q.Dists[i]))
			} else {
				sd = append(sd, 0)
			}
		}
		spotOff[1] = C.uint32_t(len(sx))
		if len(q.Dists) < len(q.Spots) {
			spotN = C.uint32_t(len(q.Dists))
		} else {
			spotN = C.uint32_t(len(q.Spots))
		}
	}
	if q := query.BoxAOI; q != nil {
		if q.Center == nil || q.Extent == nil {
			return nil, errors.New("BoxAOI with nil Center/Extent") // the reference would panic (spatial.go:205)
		}
		kind |= C.CHD_AOI_BOX
		box = [4]C.double{C.double(q.Center.X), C.double(q.Center.Z), C.double(q.Extent.X), C.double(q.Extent.Z)}
	}
	if q := query.SphereAOI; q != nil {
		if q.Center == nil {
			return nil, errors.New("SphereAOI with nil Center")
		}
		kind |= C.CHD_AOI_SPHERE
		sph = [3]C.double{C.double(q.Center.X), C.double(q.Center.Z), C.double(q.Radius)}
	}
	if q := query.ConeAOI; q != nil {
		if q.Center == nil || q.Direction == nil {
			return nil, errors.New("ConeAOI with nil Center/Direction")
		}
		kind |= C.CHD_AOI_CONE
		cone = [6]C.double{C.double(q.Center.X), C.double(q.Center.Z), C.double(q.Direction.X), C.double(q.Direction.Z),
			C.double(q.Angle), C.double(q.Radius)}
	}
	// cgo pointer-passing rule: &b is Go memory that holds Go pointers, which is only legal while those pointers are
	// pinned (runtime.Pinner, Go >= 1.21; go.mod of the reference says 1.25).  The call is synchronous.
	var pin runtime.Pinner
	defer pin.Unpin()
	pin.Pin(&kind)
	pin.Pin(&sph)
	pin.Pin(&box)
	pin.Pin(&cone)
	pin.Pin(&spotOff)
	pin.Pin(&spotN)
	if len(sx) > 0 {
		pin.Pin(&sx[0])
		pin.Pin(&sz[0])
		pin.Pin(&sd[0])
	}
	b.kind = &kind
	b.sph_cx, b.sph_cz, b.sph_r = &sph[0], &sph[1], &sph[2]
	b.box_cx, b.box_cz, b.box_ex, b.box_ez = &box[0], &box[1], &box[2], &box[3]
	b.cone_cx, b.cone_cz, b.cone_dx, b.cone_dz, b.cone_angle, b.cone_r = &cone[0], &cone[1], &cone[2], &cone[3], &cone[4], &cone[5]
	if len(sx) > 0 {
		b.spot_off, b.spot_ndist = &spotOff[0], &spotN
		b.spot_x, b.spot_z, b.spot_dist = &sx[0], &sz[0], &sd[0]
	}
	const capEntries = 1 << 16
	ids := make([]C.uint32_t, capEntries)
	dists := make([]C.uint32_t, capEntries)
	var status C.uint32_t
	var off [2]C.uint32_t
	st := C.chd_query_channel_ids(ctl.engine, &b, &status, &off[0], &ids[0], &dists[0], capEntries)
	if st != C.CHD_OK {
		return nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	if status != C.CHD_Q_OK {
		return nil, fmt.Errorf("spatial query failed with status %d", uint32(status)) // (nil, err) like the reference
	}
	result := make(map[common.ChannelId]uint, int(off[1]))
	for i := 0; i < int(off[1]); i++ {
		result[common.ChannelId(ids[i])] = uint(dists[i])
	}
	return result, nil
}

// GetAdjacentChannels (spatial.go:358-381).
func (ctl *GpuStaticGrid2DSpatialController) GetAdjacentChannels(spatialChannelId common.ChannelId) ([]common.ChannelId, error) {
	var out [8]C.uint32_t
	cfg := ctl.cCfg()
	n := C.chd_get_adjacent_channels(&cfg, C.uint32_t(spatialChannelId), &out[0])
	res := make([]common.ChannelId, int(n))
	for i := range res {
		res[i] = common.ChannelId(out[i])
	}
	return res, nil
}

func (ctl *GpuStaticGrid2DSpatialController) cCfg() C.chd_grid_cfg {
	return C.chd_grid_cfg{
		world_offset_x: C.double(ctl.WorldOffsetX), world_offset_z: C.double(ctl.WorldOffsetZ),
		grid_width: C.double(ctl.GridWidth), grid_height: C.double(ctl.GridHeight),
		grid_cols: C.uint32_t(ctl.GridCols), grid_rows: C.uint32_t(ctl.GridRows),
		server_cols: C.uint32_t(ctl.ServerCols), server_rows: C.uint32_t(ctl.ServerRows),
		server_interest_border_size: C.uint32_t(ctl.ServerInterestBorderSize),
		channel_id_start:            C.uint32_t(GlobalSettings.SpatialChannelIdStart),
	}
}

// ---------------------------------------------------------------------------------------------------------
// Batched tick: replaces the per-channel goroutine loop (channel.go:358-387) for SPATIAL channels.
// The tick driver (one goroutine) gathers, once per tick:
//   - entity positions (SoA, pinned staging from chd_alloc_pinned) from the ENTITY channels' Merge hook
//     (tpspb/data.go:227-256) instead of calling Notify per update,
//   - the UPDATE_SPATIAL_INTEREST messages received since the last tick (message_spatial.go:41) as a
//     chd_query_batch (coalesced to one per connection),
//   - each spatial channel's updateMsgBuffer metadata (data.go:46-51) as the ring CSR,
// then calls chd_tick once and consumes: chd_get_diff -> handleSubToChannel/handleUnsubFromChannel per entry,
// chd_get_due -> fanOutDataUpdate per entry (payload = whole data for kind 0, merge of ring entries selected by
// the returned window for kind 1), chd_get_handover -> the orchestration half of Notify (spatial.go:628-858).
type GpuTickInput struct {
	EntityX, EntityZ []float64 // index = entity slot
	// Alternative to EntityX/EntityZ for hosts whose positions are still the FVector floats of the entity updates
	// (unrealpb.FVector; extension.go:10-24 widens them with float64(*vec.X)): half the PCIe bytes, same results.
	EntityXf, EntityZf []float32
	ConnSlot         []uint32  // per query: subscriber slot
	SphX, SphZ, SphR []float64
	RingOff          []uint32 // [cells+1]
	RingArrival      []int64
	RingSender       []uint32
	RingIndex        []uint64
	ChannelMsgIndex  []uint64
}

func (ctl *GpuStaticGrid2DSpatialController) TickBatch(in *GpuTickInput, now ChannelTime) (C.chd_tick_summary, error) {
	var sum C.chd_tick_summary
	e := ctl.engine
	// The query batch struct below holds pointers into in.*: legal for Go-heap slices only while pinned (see
	// QueryChannelIds); slices carved out of chd_alloc_pinned memory (PinnedFloat64s & co.) are C memory and need no pin.
	// chd_tick is called with a summary, i.e. synchronously: every async copy has completed when it returns.
	var pin runtime.Pinner
	defer pin.Unpin()
	if len(in.ConnSlot) > 0 {
		pin.Pin(&in.ConnSlot[0])
		pin.Pin(&in.SphX[0])
		pin.Pin(&in.SphZ[0])
		pin.Pin(&in.SphR[0])
	}
	if n := len(in.EntityXf); n > 0 {
		pin.Pin(&in.EntityXf[0])
		pin.Pin(&in.EntityZf[0])
		if st := C.chd_set_entities_f32(e, (*C.float)(unsafe.Pointer(&in.EntityXf[0])), (*C.float)(unsafe.Pointer(&in.EntityZf[0])), C.uint32_t(n)); st != C.CHD_OK {
			return sum, errors.New(C.GoString(C.chd_last_error(e)))
		}
	} else if n := len(in.EntityX); n > 0 {
		if st := C.chd_set_entities(e, (*C.double)(unsafe.Pointer(&in.EntityX[0])), (*C.double)(unsafe.Pointer(&in.EntityZ[0])), C.uint32_t(n)); st != C.CHD_OK {
			return sum, errors.New(C.GoString(C.chd_last_error(e)))
		}
	}
	if len(in.RingOff) > 0 {
		total := in.RingOff[len(in.RingOff)-1]
		var a *C.int64_t
		var s *C.uint32_t
		var i *C.uint64_t
		if total > 0 {
			a, s, i = (*C.int64_t)(unsafe.Pointer(&in.RingArrival[0])), (*C.uint32_t)(unsafe.Pointer(&in.RingSender[0])), (*C.uint64_t)(unsafe.Pointer(&in.RingIndex[0]))
		}
		if st := C.chd_set_rings(e, (*C.uint32_t)(unsafe.Pointer(&in.RingOff[0])), C.uint32_t(total), a, s, i,
			(*C.uint64_t)(unsafe.Pointer(&in.ChannelMsgIndex[0]))); st != C.CHD_OK {
			return sum, errors.New(C.GoString(C.chd_last_error(e)))
		}
	}
	var b C.chd_query_batch
	var bp *C.chd_query_batch
	if nq := len(in.ConnSlot); nq > 0 {
		b.n = C.uint32_t(nq)
		b.sub = (*C.uint32_t)(unsafe.Pointer(&in.ConnSlot[0]))
		b.sph_cx, b.sph_cz, b.sph_r = (*C.double)(unsafe.Pointer(&in.SphX[0])), (*C.double)(unsafe.Pointer(&in.SphZ[0])), (*C.double)(unsafe.Pointer(&in.SphR[0]))
		bp = &b
	}
	if st := C.chd_tick(e, bp, C.int64_t(now), C.CHD_TICK_ALL, &sum); st != C.CHD_OK {
		return sum, errors.New(C.GoString(C.chd_last_error(e)))
	}
	return sum, nil
}

// PrefetchTick / TickPrefetched are the pipelined form of TickBatch (INTEGRATION.md §2): while tick k is in flight the
// driver hands the inputs of tick k+1 — collected into a SECOND set of pinned staging slices — to PrefetchTick, which
// only starts asynchronous uploads on the engine's upload stream; tick k+1 is then started with TickPrefetched, which
// adopts them, starts the interest / fan-out chain, runs build + emit with CHD_TICK_EARLY_RESULTS and leaves the read-back
// to FetchResults (chd_fetch_results copies each list as soon as it is final, while the expanded-list kernel still runs).
// The uploads are ASYNCHRONOUS: the slices passed to PrefetchTick must be carved out of chd_alloc_pinned memory
// (PinnedFloat64s / PinnedUint32s / ...: C memory, so no Go pointer is retained by C after the call returns — the cgo
// rule) and must stay untouched until the tick that consumes them has been fetched.
func (ctl *GpuStaticGrid2DSpatialController) PrefetchTick(in *GpuTickInput) error {
	e := ctl.engine
	fail := func() error { return errors.New(C.GoString(C.chd_last_error(e))) }
	if len(in.RingOff) > 0 {
		total := in.RingOff[len(in.RingOff)-1]
		var a *C.int64_t
		var s *C.uint32_t
		var i *C.uint64_t
		if total > 0 {
			a, s, i = (*C.int64_t)(unsafe.Pointer(&in.RingArrival[0])), (*C.uint32_t)(unsafe.Pointer(&in.RingSender[0])), (*C.uint64_t)(unsafe.Pointer(&in.RingIndex[0]))
		}
		if st := C.chd_prefetch_rings(e, (*C.uint32_t)(unsafe.Pointer(&in.RingOff[0])), C.uint32_t(total), a, s, i,
			(*C.uint64_t)(unsafe.Pointer(&in.ChannelMsgIndex[0]))); st != C.CHD_OK {
			return fail()
		}
	}
	if nq := len(in.ConnSlot); nq > 0 {
		var b C.chd_query_batch
		b.n = C.uint32_t(nq)
		b.sub = (*C.uint32_t)(unsafe.Pointer(&in.ConnSlot[0]))
		b.sph_cx, b.sph_cz, b.sph_r = (*C.double)(unsafe.Pointer(&in.SphX[0])), (*C.double)(unsafe.Pointer(&in.SphZ[0])), (*C.double)(unsafe.Pointer(&in.SphR[0]))
		if st := C.chd_prefetch_queries(e, &b); st != C.CHD_OK {
			return fail()
		}
	}
	if n := len(in.EntityXf); n > 0 {
		if st := C.chd_prefetch_entities_f32(e, (*C.float)(unsafe.Pointer(&in.EntityXf[0])), (*C.float)(unsafe.Pointer(&in.EntityZf[0])), C.uint32_t(n)); st != C.CHD_OK {
			return fail()
		}
	} else if n := len(in.EntityX); n > 0 {
		if st := C.chd_prefetch_entities(e, (*C.double)(unsafe.Pointer(&in.EntityX[0])), (*C.double)(unsafe.Pointer(&in.EntityZ[0])), C.uint32_t(n)); st != C.CHD_OK {
			return fail()
		}
	}
	return nil
}

// TickPrefetched starts the tick whose inputs PrefetchTick uploaded.  hadQueries = that input carried a query batch.
func (ctl *GpuStaticGrid2DSpatialController) TickPrefetched(now ChannelTime, hadQueries bool) error {
	e := ctl.engine
	fail := func() error { return errors.New(C.GoString(C.chd_last_error(e))) }
	if st := C.chd_adopt_prefetched(e); st != C.CHD_OK {
		return fail()
	}
	if hadQueries {
		if st := C.chd_begin_interest(e, nil, C.int64_t(now), 1); st != C.CHD_OK {
			return fail()
		}
	}
	if st := C.chd_tick(e, nil, C.int64_t(now), C.CHD_TICK_ALL|C.CHD_TICK_EARLY_RESULTS, nil); st != C.CHD_OK {
		return fail()
	}
	return nil
}

// FetchResults copies every host-facing result of the tick into caller-owned (pinned) buffers.
func (ctl *GpuStaticGrid2DSpatialController) FetchResults(buffers *C.chd_result_buffers) (C.chd_tick_summary, error) {
	var sum C.chd_tick_summary
	if st := C.chd_fetch_results(ctl.engine, buffers, &sum); st != C.CHD_OK {
		return sum, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return sum, nil
}

// AdjacentBroadcast replaces the per-message map merge of message.go:188-239 for a batch of
// BroadcastType_ADJACENT_CHANNELS messages: recipients of message m are slots[off[m]:off[m+1]] (subscriber slots).
// Connection types for the ALL_BUT_CLIENT / ALL_BUT_SERVER filters are registered once with chd_set_subscriber_types.
func (ctl *GpuStaticGrid2DSpatialController) AdjacentBroadcast(channelIds []common.ChannelId, broadcast, senderConnId, clientConnId []uint32, capSlots int) (status, off, slots []uint32, err error) {
	n := len(channelIds)
	status, off, slots = make([]uint32, n), make([]uint32, n+1), make([]uint32, capSlots)
	if n == 0 {
		return status, off, slots[:0], nil
	}
	var pin runtime.Pinner // the batch struct holds pointers to Go slices: pinned for this synchronous call
	defer pin.Unpin()
	pin.Pin(&channelIds[0])
	pin.Pin(&broadcast[0])
	b := C.chd_broadcast_batch{n: C.uint32_t(n), channel_id: (*C.uint32_t)(unsafe.Pointer(&channelIds[0])), broadcast: (*C.uint32_t)(unsafe.Pointer(&broadcast[0]))}
	if len(senderConnId) == n {
		pin.Pin(&senderConnId[0])
		b.sender_conn_id = (*C.uint32_t)(unsafe.Pointer(&senderConnId[0]))
	}
	if len(clientConnId) == n {
		pin.Pin(&clientConnId[0])
		b.client_conn_id = (*C.uint32_t)(unsafe.Pointer(&clientConnId[0]))
	}
	var slotPtr *C.uint32_t
	if capSlots > 0 {
		slotPtr = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
	}
	if st := C.chd_adjacent_broadcast(ctl.engine, &b, (*C.uint32_t)(unsafe.Pointer(&status[0])), (*C.uint32_t)(unsafe.Pointer(&off[0])), slotPtr, C.uint64_t(capSlots)); st != C.CHD_OK {
		return nil, nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return status, off, slots[:off[n]], nil
}

// DueClasses groups the due list of the last tick by payload identity (data.go:248-252 merges afresh per subscriber):
// the host merges / marshals the window of due record rep[k] once and sends it to every record i with classOf[i] == k.
// A CHD_DUE_VOID hole of an overflowed list has classOf[i] == CHD_DUE_VOID (0xFFFFFFFF) and belongs to no class.
func (ctl *GpuStaticGrid2DSpatialController) DueClasses(nDue int) (classOf, rep, count []uint32, err error) {
	if nDue == 0 {
		return nil, nil, nil, nil
	}
	classOf, rep, count = make([]uint32, nDue), make([]uint32, nDue), make([]uint32, nDue)
	var n C.uint32_t
	if st := C.chd_due_classes(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&classOf[0])), (*C.uint32_t)(unsafe.Pointer(&rep[0])),
		(*C.uint32_t)(unsafe.Pointer(&count[0])), C.uint32_t(nDue), &n); st != C.CHD_OK {
		return nil, nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return classOf, rep[:n], count[:n], nil
}

// VisibleDelta returns, per subscriber slot, the entity indices to spawn (enter) and despawn (leave) since the last visible
// delta: the net effect of the FULL data a new subscription sends, the despawns of an unsubscription and the handovers between
// cells (spatial.go:612-858).  Call ReserveVisibleDelta once, then tick with CHD_TICK_VISIBLE_DELTA.  VisibleDelta makes two
// blocking calls on the engine stream: in the pipelined loop it waits for the tick in flight and returns ITS lists.  A pipelined
// host reads the lists with the tick's other results instead: FetchResultsAsyncDelta / FetchWaitDelta.  UN-RUN like the rest
// of this file.
func (ctl *GpuStaticGrid2DSpatialController) ReserveVisibleDelta(capEntries uint64) error {
	if st := C.chd_reserve_visible_delta(ctl.engine, C.uint64_t(capEntries)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// ReserveVisibleDeltaIds picks id mode instead: the deltas name global ids in [0, idSpace) (SetEntityIds, the halo records),
// which also works on sharded engines.  A connection migrated from rank A to rank B is netted by the host: enter = enter_B \
// leave_A, leave = leave_A \ enter_B.
func (ctl *GpuStaticGrid2DSpatialController) ReserveVisibleDeltaIds(capEntries uint64, idSpace uint32) error {
	if st := C.chd_reserve_visible_delta_ids(ctl.engine, C.uint64_t(capEntries), C.uint32_t(idSpace)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) VisibleDelta() (enterOff []uint64, enter []uint32, leaveOff []uint64, leave []uint32, err error) {
	var ne, nl C.uint64_t
	var slots C.uint32_t
	if st := C.chd_get_visible_delta(ctl.engine, nil, nil, nil, nil, 0, &ne, &nl, &slots); st != C.CHD_OK {
		return nil, nil, nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	enterOff, leaveOff = make([]uint64, int(slots)+1), make([]uint64, int(slots)+1)
	enter, leave = make([]uint32, int(ne)+1), make([]uint32, int(nl)+1)
	capEntries := ne
	if nl > capEntries {
		capEntries = nl
	}
	if st := C.chd_get_visible_delta(ctl.engine, (*C.uint64_t)(unsafe.Pointer(&enterOff[0])), (*C.uint32_t)(unsafe.Pointer(&enter[0])),
		(*C.uint64_t)(unsafe.Pointer(&leaveOff[0])), (*C.uint32_t)(unsafe.Pointer(&leave[0])), capEntries+1, nil, nil, nil); st != C.CHD_OK {
		return nil, nil, nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return enterOff, enter[:ne], leaveOff, leave[:nl], nil
}

// SpawnObjects / DestroyObjects / MoveEntities deliver entities the way channeld does, keyed by NetGUID (entity-table mode,
// chd_entity_table_init, switched on by the first call): SpawnObjects = handleSpawnObject's GetChannelId + addSpatialEntity
// (pkg/unreal/message.go:20-150), DestroyObjects = the destroy handler (message.go:152-203), MoveEntities = ENTITY-channel updates
// whose Merge hook calls Notify for that entity alone (spatial.go:612-626).  Every result then names NetGUIDs (cells, visible
// lists, handovers, deltas).  Spawn / destroy statuses (CHD_EV_*) come back before the call returns, so Go slices are fine there;
// MoveEntities is stream-ordered and its arrays must be C memory (PinnedUint32s / PinnedFloat32s).  UN-RUN like the rest of this file.
func (ctl *GpuStaticGrid2DSpatialController) entityTable() error {
	if ctl.tableOn {
		return nil
	}
	if st := C.chd_entity_table_init(ctl.engine); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	ctl.tableOn = true
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) SpawnObjects(netIds []uint32, x, z []float64) ([]uint8, error) {
	if len(x) != len(netIds) || len(z) != len(netIds) {
		return nil, errors.New("SpawnObjects: array sizes differ")
	}
	if err := ctl.entityTable(); err != nil || len(netIds) == 0 {
		return nil, err
	}
	status := make([]uint8, len(netIds))
	if st := C.chd_spawn_entities(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&netIds[0])), (*C.double)(unsafe.Pointer(&x[0])),
		(*C.double)(unsafe.Pointer(&z[0])), C.uint32_t(len(netIds)), (*C.uint8_t)(unsafe.Pointer(&status[0]))); st != C.CHD_OK {
		return nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return status, nil
}

func (ctl *GpuStaticGrid2DSpatialController) DestroyObjects(netIds []uint32) ([]uint8, error) {
	if err := ctl.entityTable(); err != nil || len(netIds) == 0 {
		return nil, err
	}
	status := make([]uint8, len(netIds))
	if st := C.chd_despawn_entities(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&netIds[0])), C.uint32_t(len(netIds)),
		(*C.uint8_t)(unsafe.Pointer(&status[0]))); st != C.CHD_OK {
		return nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return status, nil
}

// FollowOutsideSlab: the follower status (chd_get_follow) of a generated query that would reach columns the slab does not serve.
const FollowOutsideSlab = uint32(C.CHD_FOLLOW_OUTSIDE_SLAB)

// FollowEntities binds connection slots to the entities they stand on (chd_follow_bind); kind[i] is a CHD_AOI_SPHERE | BOX | CONE
// mask (nil: all sphere) and shape the per-binding parameters in the order sph_r, box_ex, box_ez, cone_dx, cone_dz, cone_angle,
// cone_r (a nil entry: no binding uses that kind).  The arrays are copied before the call returns, so Go slices are fine.
// FollowQueries then generates each tick's interest batch on the device (mode CHD_FOLLOW_ALL / CHD_FOLLOW_MOVED); BeginInterest(nil)
// or a Tick with CHD_TICK_FOLLOW consumes it.  Clients with a pawn are bound; server connections keep sending explicit queries.
// On N GPUs (entity-table mode on slabs) a follower lives on the rank that owns its entity: TickSharded with CHD_TICK_FOLLOW consumes
// the batch, MigrateOut unbinds the emigrants and the destination binds them again after MigrateIn; a follower whose query would reach
// columns the slab does not serve gets FollowOutsideSlab.
// UN-RUN like the rest of this file.
func (ctl *GpuStaticGrid2DSpatialController) FollowEntities(slots, netIds []uint32, kind []uint8, shape [7][]float64) error {
	if len(netIds) != len(slots) || len(slots) == 0 {
		return errors.New("FollowEntities: array sizes differ or are empty")
	}
	var b C.chd_follow_batch
	b.n = C.uint32_t(len(slots))
	b.slot = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
	b.entity = (*C.uint32_t)(unsafe.Pointer(&netIds[0]))
	if kind != nil {
		b.kind = (*C.uint8_t)(unsafe.Pointer(&kind[0]))
	}
	dst := [7]**C.double{&b.sph_r, &b.box_ex, &b.box_ez, &b.cone_dx, &b.cone_dz, &b.cone_angle, &b.cone_r}
	for i, a := range shape {
		if a != nil {
			*dst[i] = (*C.double)(unsafe.Pointer(&a[0]))
		}
	}
	if st := C.chd_follow_bind(ctl.engine, &b); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) UnfollowEntities(slots []uint32) error {
	if len(slots) == 0 {
		return nil
	}
	if st := C.chd_follow_unbind(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&slots[0])), C.uint32_t(len(slots))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) FollowQueries(mode uint32) error {
	if st := C.chd_follow_queries(ctl.engine, C.uint32_t(mode)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// FollowQueriesWith merges the tick's explicit queries (connections that follow nothing, such as spectators and SpotsAOI users, or a
// follower's own query for this tick) in front of the generated ones, so one interest update covers both.  explicit == nil: the batch
// PrefetchQueries uploaded and AdoptPrefetched handed over (the pipelined form); otherwise a batch as UpdateInterest takes it, with
// sub set.  Consumed like FollowQueries' batch; chd_gpu.h gives the layout of the statuses.  UN-RUN like the rest of this file.
func (ctl *GpuStaticGrid2DSpatialController) FollowQueriesWith(mode uint32, explicit *C.chd_query_batch) error {
	if st := C.chd_follow_queries_with(ctl.engine, C.uint32_t(mode), explicit); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// MoveEntities: netIds / x / z in C memory, valid until the next Summary / FetchResults.  The last move of an id in one call wins;
// moves of ids that are not live are ignored (counted in EntityStats).
func (ctl *GpuStaticGrid2DSpatialController) MoveEntities(netIds []uint32, x, z []float32) error {
	if len(x) != len(netIds) || len(z) != len(netIds) {
		return errors.New("MoveEntities: array sizes differ")
	}
	if err := ctl.entityTable(); err != nil || len(netIds) == 0 {
		return err
	}
	if st := C.chd_move_entities_f32(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&netIds[0])), (*C.float)(unsafe.Pointer(&x[0])),
		(*C.float)(unsafe.Pointer(&z[0])), C.uint32_t(len(netIds))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) EntityStats() (C.chd_entity_stats, error) {
	var s C.chd_entity_stats
	if st := C.chd_get_entity_stats(ctl.engine, &s); st != C.CHD_OK {
		return s, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return s, nil
}

// PinnedFloat64s / PinnedUint32s / PinnedInt64s / PinnedUint64s carve staging slices out of page-locked C memory
// (chd_alloc_pinned): uploads from them are truly asynchronous and, being C memory, they may be referenced by the
// engine after a cgo call has returned (PrefetchTick).  Release with FreePinned(unsafe.Pointer(&s[0])).
func PinnedFloat64s(n int) []float64 {
	return unsafe.Slice((*float64)(C.chd_alloc_pinned(C.uint64_t(8*n))), n)
}
func PinnedFloat32s(n int) []float32 {
	return unsafe.Slice((*float32)(C.chd_alloc_pinned(C.uint64_t(4*n))), n)
}
func PinnedUint32s(n int) []uint32 {
	return unsafe.Slice((*uint32)(C.chd_alloc_pinned(C.uint64_t(4*n))), n)
}
func PinnedInt64s(n int) []int64 {
	return unsafe.Slice((*int64)(C.chd_alloc_pinned(C.uint64_t(8*n))), n)
}
func PinnedUint64s(n int) []uint64 {
	return unsafe.Slice((*uint64)(C.chd_alloc_pinned(C.uint64_t(8*n))), n)
}
func FreePinned(p unsafe.Pointer) { C.chd_free_pinned(p) }

// ---- round 2 additions: the entry points a sharded / long-running channeld host needs ----

// FetchResultsAsync / FetchWait: the non-blocking read-back.  buffers and header must live in C (pinned) memory
// (chd_alloc_pinned); up to two fetches may be outstanding, FetchWait returns the OLDEST one's summary.
func (ctl *GpuStaticGrid2DSpatialController) FetchResultsAsync(buffers *C.chd_result_buffers, pinnedHeader unsafe.Pointer) error {
	if st := C.chd_fetch_results_async(ctl.engine, buffers, pinnedHeader); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) FetchWait() (C.chd_tick_summary, error) {
	var s C.chd_tick_summary
	if st := C.chd_fetch_wait(ctl.engine, &s); st != C.CHD_OK {
		return s, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return s, nil
}

// FetchResultsAsyncDelta / FetchWaitDelta: the same read-back carrying the visible-set delta of the tick (delta buffers in C
// pinned memory as well).  counts.deltas: 0 = the tick ran no delta, 1 = these are its lists, > 1 = earlier deltas were never
// fetched.  After CHD_OVF_DELTA the wait returns an error and counts holds the required sizes (grow with ReserveVisibleDelta).
func (ctl *GpuStaticGrid2DSpatialController) FetchResultsAsyncDelta(buffers *C.chd_result_buffers, delta *C.chd_delta_buffers, pinnedHeader unsafe.Pointer) error {
	if st := C.chd_fetch_results_async_delta(ctl.engine, buffers, delta, pinnedHeader); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) FetchWaitDelta() (C.chd_tick_summary, C.chd_delta_counts, error) {
	var s C.chd_tick_summary
	var c C.chd_delta_counts
	if st := C.chd_fetch_wait_delta(ctl.engine, &s, &c); st != C.CHD_OK {
		return s, c, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return s, c, nil
}

// AddSubscribers / RemoveSubscribers: connection lifecycle (subscription.go:104-125, channel.go:414-475).  The host owns the
// slot table; the slices are copied before the call returns (plain Go memory is fine).
func (ctl *GpuStaticGrid2DSpatialController) AddSubscribers(slots, connIds []uint32) error {
	if len(slots) == 0 {
		return nil
	}
	if st := C.chd_add_subscribers(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&slots[0])), (*C.uint32_t)(unsafe.Pointer(&connIds[0])), C.uint32_t(len(slots))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) RemoveSubscribers(slots []uint32) error {
	if len(slots) == 0 {
		return nil
	}
	if st := C.chd_remove_subscribers(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&slots[0])), C.uint32_t(len(slots))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// CommUniqueId / CommInit / TickSharded: multi-GPU, one channeld process per GPU.  Rank 0 creates the id and ships the 128 bytes to
// the other processes over any channel it likes (channeld already has TCP connections between its own processes); the NCCL
// all-gather itself is issued inside libchd_b200.so.
func CommUniqueId() ([C.CHD_COMM_ID_BYTES]byte, error) {
	var id [C.CHD_COMM_ID_BYTES]byte
	if st := C.chd_comm_unique_id(unsafe.Pointer(&id[0])); st != C.CHD_OK {
		return id, errors.New("chd_comm_unique_id failed (libnccl.so.2 not loadable?)")
	}
	return id, nil
}

func (ctl *GpuStaticGrid2DSpatialController) CommInit(id [C.CHD_COMM_ID_BYTES]byte, rank, world int, haloCols, borderCapacity, migrateSubscribers, migratePairs uint32) error {
	if st := C.chd_comm_init(ctl.engine, unsafe.Pointer(&id[0]), C.int(rank), C.int(world), C.uint32_t(haloCols), C.uint32_t(borderCapacity),
		C.uint32_t(migrateSubscribers), C.uint32_t(migratePairs)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// TickSharded replaces TickPrefetched on a sharded host (inputs prefetched + adopted, or set with the chd_set_* calls).
func (ctl *GpuStaticGrid2DSpatialController) TickSharded(now ChannelTime, flags uint32) error {
	if st := C.chd_tick_sharded(ctl.engine, nil, C.int64_t(now), C.uint32_t(flags), nil); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// MigrateOut / MigrateIn: a subscriber whose centre crossed into another rank's slab moves with its subscriptions and fan-out
// state inside the same all-gather (no FULL resend).  Both sides call before the same TickSharded.
func (ctl *GpuStaticGrid2DSpatialController) MigrateOut(slots []uint32) error {
	var p *C.uint32_t
	if len(slots) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&slots[0]))
	}
	if st := C.chd_migrate_out(ctl.engine, p, C.uint32_t(len(slots))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) MigrateIn(srcRank, firstIndex uint32, slots, connIds []uint32) error {
	if len(slots) == 0 {
		return nil
	}
	if st := C.chd_migrate_in(ctl.engine, C.uint32_t(srcRank), C.uint32_t(firstIndex), (*C.uint32_t)(unsafe.Pointer(&slots[0])),
		(*C.uint32_t)(unsafe.Pointer(&connIds[0])), C.uint32_t(len(slots))); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// Rehome: own entities whose column now belongs to another rank (global id, destination rank): the host re-routes their feed.
func (ctl *GpuStaticGrid2DSpatialController) Rehome(capEntities int) (gid, dstRank []uint32, err error) {
	gid, dstRank = make([]uint32, capEntities), make([]uint32, capEntities)
	var n C.uint32_t
	var pg, pd *C.uint32_t
	if capEntities > 0 {
		pg, pd = (*C.uint32_t)(unsafe.Pointer(&gid[0])), (*C.uint32_t)(unsafe.Pointer(&dstRank[0]))
	}
	if st := C.chd_get_rehome(ctl.engine, pg, pd, C.uint32_t(capEntities), &n); st != C.CHD_OK {
		return nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	k := int(n)
	if k > capEntities {
		k = capEntities
	}
	return gid[:k], dstRank[:k], nil
}

// HandoffEntities (entity-table mode on slabs, after the tick): the own entities whose column another rank owns, removed from
// this rank's table with their exact positions; the destination rank adopts each one with SpawnObjects.  A list longer than
// capEntities is asked for again with room for it (nothing is removed by the refused call).
func (ctl *GpuStaticGrid2DSpatialController) HandoffEntities(capEntities int) (netIds, dstRank []uint32, x, z []float64, err error) {
	for {
		netIds, dstRank = make([]uint32, capEntities+1), make([]uint32, capEntities+1)
		x, z = make([]float64, capEntities+1), make([]float64, capEntities+1)
		var n C.uint32_t
		st := C.chd_handoff_entities(ctl.engine, (*C.uint32_t)(unsafe.Pointer(&netIds[0])), (*C.uint32_t)(unsafe.Pointer(&dstRank[0])),
			(*C.double)(unsafe.Pointer(&x[0])), (*C.double)(unsafe.Pointer(&z[0])), C.uint32_t(capEntities), &n)
		if st == C.CHD_ERR_CAPACITY && int(n) > capEntities {
			capEntities = int(n)
			continue
		}
		if st != C.CHD_OK {
			return nil, nil, nil, nil, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
		}
		k := int(n)
		return netIds[:k], dstRank[:k], x[:k], z[:k], nil
	}
}

// RingsInit / RingsAppend: ChannelData.OnUpdate's buffer on the GPU (data.go:149-173); updOff is the CSR by cell of this tick's
// updates (arrival order per cell), arrival / sender in C memory when the call is used on the tick path.
func (ctl *GpuStaticGrid2DSpatialController) RingsInit(capacityPerCell uint32) error {
	if st := C.chd_rings_init(ctl.engine, C.uint32_t(capacityPerCell)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) RingsAppend(updOff *C.uint32_t, n uint32, arrival *C.int64_t, sender *C.uint32_t) error {
	if st := C.chd_rings_append(ctl.engine, updOff, C.uint32_t(n), arrival, sender); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

// AssemblePayloads / FramePackets: the byte half of the fan-out.  The host hands over the serialized updateMsg of every ring
// entry and gets back, per connection, bytes it can pass to conn.Write unchanged (tag + marshalled Packet, snappy if asked).
func (ctl *GpuStaticGrid2DSpatialController) SetPayloadBytes(entryOff []uint64, entryBytes []byte, fullOff []uint64, fullBytes []byte, typeUrl string) error {
	curl := C.CString(typeUrl)
	defer C.free(unsafe.Pointer(curl))
	var pe, pf *C.uint8_t
	if len(entryBytes) > 0 {
		pe = (*C.uint8_t)(unsafe.Pointer(&entryBytes[0]))
	}
	if len(fullBytes) > 0 {
		pf = (*C.uint8_t)(unsafe.Pointer(&fullBytes[0]))
	}
	if st := C.chd_set_payload_bytes(ctl.engine, (*C.uint64_t)(unsafe.Pointer(&entryOff[0])), C.uint32_t(len(entryOff)-1), pe,
		(*C.uint64_t)(unsafe.Pointer(&fullOff[0])), pf, curl, C.uint32_t(channeldpb.MessageType_CHANNEL_DATA_UPDATE)); st != C.CHD_OK {
		return errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return nil
}

func (ctl *GpuStaticGrid2DSpatialController) FramePackets(compression []uint8, connOff []uint64, connLen []uint32, out []byte) (uint64, uint32, error) {
	var nClasses C.uint32_t
	if st := C.chd_assemble_payloads(ctl.engine, &nClasses, nil, 0, nil, 0, nil); st != C.CHD_OK {
		return 0, 0, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	var total C.uint64_t
	var dropped C.uint32_t
	var pc *C.uint8_t
	if len(compression) > 0 {
		pc = (*C.uint8_t)(unsafe.Pointer(&compression[0]))
	}
	if st := C.chd_frame_packets(ctl.engine, pc, (*C.uint64_t)(unsafe.Pointer(&connOff[0])), (*C.uint32_t)(unsafe.Pointer(&connLen[0])), nil,
		(*C.uint8_t)(unsafe.Pointer(&out[0])), C.uint64_t(len(out)), &total, &dropped); st != C.CHD_OK {
		return 0, 0, errors.New(C.GoString(C.chd_last_error(ctl.engine)))
	}
	return uint64(total), uint32(dropped), nil
}
