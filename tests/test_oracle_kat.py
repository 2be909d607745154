"""Pins the CPU oracle against every known-answer test the reference holds for the spatial hot path.

Transcribed (inputs + expected results only) from the reference's pkg/channeld/spatial_test.go:
  TestGetChannelId1 :803-848, TestGetChannelId2 :762-801, TestSphereAOI :244-360, TestBoxAOI :362-491,
  TestConeAOI :21-242, TestGetAdjacentChannels :493-526
and the reference's pkg/channeld/data_test.go TestFanOutChannelData :98-166 (doc/design.md:94-109).
SpatialChannelIdStart = 65536 (settings.go:94).
"""
import math

import numpy as np

from tests._oracle import ERR_BAD_STEP, ERR_OUT_OF_WORLD, OK, make_grid

S = 65536
MS = 1_000_000


def test_get_channel_id1(oracle):  # spatial_test.go:803-848
    g = make_grid(-450, -200, 100, 50, 9, 8, 3, 4, 2)
    assert oracle.get_channel_id(g, -450, -200) == (S + 0, OK)
    assert oracle.get_channel_id(g, -350, -200) == (S + 1, OK)
    assert oracle.get_channel_id(g, -450, -150) == (S + 9, OK)
    assert oracle.get_channel_id(g, 0, 0) == (S + 9 * 4 + 4, OK)
    assert oracle.get_channel_id(g, 449.99, 199.99) == (S + 9 * 8 - 1, OK)
    for x, z in [(-500, 0), (500, 0), (0, -300), (0, 300), (450, 200)]:
        assert oracle.get_channel_id(g, x, z)[1] == ERR_OUT_OF_WORLD


def test_get_channel_id2(oracle):  # spatial_test.go:762-801
    g = make_grid(0, 0, 100, 50, 9, 8, 3, 4, 2)
    assert oracle.get_channel_id(g, 0, 0) == (S + 0, OK)
    assert oracle.get_channel_id(g, 100, 0) == (S + 1, OK)
    assert oracle.get_channel_id(g, 0, 50) == (S + 9, OK)
    assert oracle.get_channel_id(g, 899.99, 399.99) == (S + 9 * 8 - 1, OK)
    for x, z in [(-1, 0), (1.7976931348623157e308, 0), (0, -1), (900, 400)]:
        assert oracle.get_channel_id(g, x, z)[1] == ERR_OUT_OF_WORLD
    # beyond the reference's KATs: non-finite inputs take the same error path (Go int(NaN) = MinInt64 on amd64)
    for x in [float("nan"), float("inf"), float("-inf")]:
        assert oracle.get_channel_id(g, x, 0)[1] == ERR_OUT_OF_WORLD
        assert oracle.get_channel_id(g, 0, x)[1] == ERR_OUT_OF_WORLD


def test_sphere_aoi(oracle):  # spatial_test.go:244-360
    g1 = make_grid(0, 0, 10, 10, 1, 1)
    res, st = oracle.query(g1, sphere=(5, 5, 1))
    assert st == OK and S in res
    res, st = oracle.query(g1, sphere=(5, 5, 100))
    assert st == OK and S in res

    g2 = make_grid(-5, -5, 5, 5, 2, 2)
    res, st = oracle.query(g2, sphere=(0, 0, 1))
    assert st == OK and len(res) == 4
    res, st = oracle.query(g2, sphere=(4.9, 4.9, 1))
    assert st == OK and set(res) == {65539}
    res, st = oracle.query(g2, sphere=(4.9, 4.9, 4.9))
    assert st == OK and len(res) == 1
    res, st = oracle.query(g2, sphere=(4.9, 4.9, 10))
    assert st == OK and len(res) == 4

    g3 = make_grid(-150, -150, 100, 100, 3, 3)
    res, st = oracle.query(g3, sphere=(0, 0, 150))
    assert st == OK and len(res) == 9
    res, st = oracle.query(g3, sphere=(0, 0, 99))
    assert st == OK and len(res) == 5
    # "Radious = 100 would count the top-right corner channel in the result" (spatial_test.go:354)
    res100, _ = oracle.query(g3, sphere=(0, 0, 100))
    assert S + 8 in res100


def test_box_aoi(oracle):  # spatial_test.go:362-491
    g1 = make_grid(0, 0, 10, 10, 1, 1)
    res, st = oracle.query(g1, box=(5, 5, 1, 1))
    assert st == OK and S in res
    res, st = oracle.query(g1, box=(5, 5, 100, 100))
    assert st == OK and S in res

    g2 = make_grid(-5, -5, 5, 5, 2, 2)
    res, st = oracle.query(g2, box=(0, 0, 1, 1))
    assert st == OK and len(res) == 4
    res, st = oracle.query(g2, box=(4.9, 4.9, 1, 1))
    assert st == OK and set(res) == {65539}
    res, st = oracle.query(g2, box=(4.9, 4.9, 4.9, 4.9))
    assert st == OK and len(res) == 1
    res, st = oracle.query(g2, box=(4.9, 4.9, 4.9, 10))
    assert st == OK and len(res) == 2  # "Should contain 65539, 65537"
    assert set(res) == {65539, 65537}

    g3 = make_grid(-150, -150, 100, 100, 3, 3)
    res, st = oracle.query(g3, box=(0, 0, 150, 150))
    assert st == OK and len(res) == 9
    res, st = oracle.query(g3, box=(0, 0, 100, 100))
    assert st == OK and len(res) == 9


def test_cone_aoi(oracle):  # spatial_test.go:21-242
    g1 = make_grid(0, 0, 10, 10, 1, 1)
    res, st = oracle.query(g1, cone=(5, 5, 1, 0, math.pi / 4, 1))
    assert st == OK and S in res

    g2 = make_grid(0, 0, 10, 10, 4, 1)
    res, st = oracle.query(g2, cone=(0, 5, 1, 0, math.pi / 4, 1))
    assert st == OK and S in res
    res, st = oracle.query(g2, cone=(0, 5, 1, 0, math.pi / 4, 25))
    assert st == OK and len(res) == 3
    res, st = oracle.query(g2, cone=(0, 5, 1, 0, math.pi / 4, 100))
    assert st == OK and len(res) == 4
    res, st = oracle.query(g2, cone=(0, 5, 0, 1, math.pi / 4, 100))
    assert st == OK and len(res) == 1

    g3 = make_grid(0, 0, 10, 10, 3, 3)
    res, st = oracle.query(g3, cone=(5, 5, 1, 0, 0.1, 100))
    assert st == OK and len(res) == 3
    assert set(res) == {65536, 65537, 65538}  # drawn at spatial_test.go:141-149
    res, st = oracle.query(g3, cone=(5, 5, 1, 0, math.pi / 4, 100))
    assert st == OK and len(res) == 6
    assert set(res) == {65536, 65537, 65538, 65540, 65541, 65544}  # :155-163
    res, st = oracle.query(g3, cone=(15, 15, -1, 0, math.pi / 4, 100))
    assert st == OK and len(res) == 4
    assert set(res) == {65536, 65539, 65540, 65542}  # :169-177
    res, st = oracle.query(g3, cone=(5, 15, 0, -1, math.pi / 4, 100))
    assert st == OK and len(res) == 3
    assert set(res) == {65536, 65537, 65539}  # :191-199

    g4 = make_grid(-2000, -500, 1000, 1000, 4, 1, 2, 1, 1)
    res, st = oracle.query(g4, cone=(1250, 0, -0.087, 0.996, 0.5236, 30000))
    assert st == OK and len(res) == 1


def test_get_adjacent_channels(oracle):  # spatial_test.go:493-526
    assert oracle.adjacent(make_grid(0, 0, 10, 10, 1, 1, 1, 1, 1), S) == []
    assert len(oracle.adjacent(make_grid(-5, -5, 5, 5, 2, 2), S)) == 3
    # reference order is row-major over the 3x3 neighbourhood (spatial.go:363-378)
    g = make_grid(0, 0, 10, 10, 3, 3)
    assert oracle.adjacent(g, S + 4) == [S + 0, S + 1, S + 2, S + 3, S + 5, S + 6, S + 7, S + 8]
    assert oracle.adjacent(g, S + 8) == [S + 4, S + 5, S + 7]


def test_regions_server_layout(oracle):
    # server<->cell layout of TestCreateSpatialChannels1 (spatial_test.go:613-683): 4x3 grid, 2x3 servers
    g = make_grid(-40, -60, 20, 40, 4, 3, 2, 3, 1)
    minx, minz, maxx, maxz, cid, srv = oracle.regions(g)
    assert list(cid) == [S + i for i in range(12)]
    assert list(srv) == [0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5]
    assert minx[0] == -40 and minz[0] == -60 and maxx[0] == -20 and maxz[0] == -20
    assert minx[11] == 20 and minz[11] == 20 and maxx[11] == 40 and maxz[11] == 60


def test_query_error_paths(oracle):  # spatial.go:208-215,240-247,228-231,263-266
    g = make_grid(-5, -5, 5, 5, 2, 2)
    assert oracle.query(g, sphere=(0, 0, 0))[1] == ERR_BAD_STEP
    assert oracle.query(g, sphere=(0, 0, -1))[1] == ERR_BAD_STEP
    assert oracle.query(g, box=(0, 0, 0, 1))[1] == ERR_BAD_STEP
    assert oracle.query(g, box=(0, 0, 1, -2))[1] == ERR_BAD_STEP
    # centre out of the world: the whole query fails even though in-world samples exist
    assert oracle.query(g, sphere=(5.5, 0, 2))[1] == ERR_OUT_OF_WORLD
    assert oracle.query(g, box=(-6, 0, 3, 3))[1] == ERR_OUT_OF_WORLD
    assert oracle.query(g, cone=(0, 7, 1, 0, 1.0, 4))[1] == ERR_OUT_OF_WORLD


def test_dist_and_last_write_wins(oracle):
    # dist = ceil(Dist2D(centre, sample)/gridSize), last sample in z-outer/x-inner order wins, centre cell = 0
    g = make_grid(-150, -150, 100, 100, 3, 3)
    res, st = oracle.query(g, sphere=(0, 0, 150))
    assert st == OK
    assert res[S + 4] == 0
    gs = oracle.grid_size(g)
    assert gs == math.sqrt(100.0 * 100.0 + 100.0 * 100.0)
    # cell 8 (top-right) samples with x,z in {50,100}: last kept in order is (100,100) -> r=141.4 <= 150
    assert res[S + 8] == math.ceil(math.sqrt(100.0 * 100.0 + 100.0 * 100.0) / gs) == 1
    assert set(res.values()) <= {0, 1, 2}


def test_spots_and_combined_kinds(oracle):  # spatial.go:189-202 + the independent `if`s
    g = make_grid(0, 0, 10, 10, 3, 3)
    res, st = oracle.query(g, spots=[(5, 5), (25, 25), (-1, 5), (25, 26)], spot_dists=[3, 2])
    assert st == OK and res == {S + 0: 3, S + 8: 0}  # 2nd spot dist 2 overwritten by 4th spot (no dist -> 0)
    res, st = oracle.query(g, spots=[(5, 5), (25, 25)], spot_dists=[3, 2], sphere=(5, 5, 1))
    assert st == OK and res == {S + 0: 0, S + 8: 2}
    # an error in a later kind voids the whole result (reference returns nil, err)
    res, st = oracle.query(g, spots=[(5, 5)], sphere=(-5, 5, 1))
    assert res is None and st == ERR_OUT_OF_WORLD


def test_damping_and_diff(oracle):  # message_spatial.go:16-38, util.go:105-113
    assert [oracle.damping(d, 77) for d in range(5)] == [20, 50, 100, 77, 77]
    un, sn, kp = oracle.interest_diff([S + 1, S + 2, S + 3], [S + 3, S + 4])
    assert list(un) == [S + 1, S + 2] and list(sn) == [S + 4] and list(kp) == [S + 3]
    un, sn, kp = oracle.interest_diff([], [S + 9, S + 1])
    assert list(un) == [] and list(sn) == [S + 1, S + 9] and list(kp) == []


def test_go_cos_matches_libm_closely(oracle):
    xs = np.concatenate([np.linspace(-10, 10, 4001), [math.pi / 4, 0.1, 0.5236, 0.0, 1e-9, 100.0, 12345.678]])
    for x in xs:
        assert abs(oracle.go_cos(x) - math.cos(x)) <= 4 * np.spacing(1.0)
    assert oracle.go_cos(0.0) == 1.0
    assert math.isnan(oracle.go_cos(float("inf")))


def test_fan_out_channel_data(oracle):  # data_test.go:98-166; timeline of doc/design.md:94-109
    C0, C1, C2 = 1, 2, 3
    ch = oracle.channel()
    t0 = 100 * MS  # channelStartTime
    # c0 subscribes with defaults (GLOBAL settings: interval 20, delay 0; settings.go:97-103), c1 with 50 ms;
    # ch.GetTime() at subscribe time is ~0 in the reference test (real clock, microseconds after creation).
    ch.subscribe(C0, 0, 20)
    ch.subscribe(C1, 0, 50)
    sends = ch.tick_data(t0)  # F0 = the whole data
    c1 = [s for s in sends if s["conn"] == C1]
    assert len(c1) == 1 and c1[0]["kind"] == 0
    assert [s for s in sends if s["conn"] == C2] == []
    n1, n2 = 1, 0

    ch.subscribe(C2, 0, 100)
    sends = ch.tick_data(t0 + 50 * MS)  # F1 = no data, F7 = whole data
    n1 += len([s for s in sends if s["conn"] == C1])
    c2 = [s for s in sends if s["conn"] == C2]
    n2 += len(c2)
    assert (n1, n2) == (1, 1) and c2[0]["kind"] == 0

    ch.on_update(t0 + 60 * MS, C0)  # U1, message index 1
    sends = ch.tick_data(t0 + 100 * MS)  # F2 = U1
    c1 = [s for s in sends if s["conn"] == C1]
    n1 += len(c1)
    n2 += len([s for s in sends if s["conn"] == C2])
    assert (n1, n2) == (2, 1)
    assert c1[0]["kind"] == 1 and c1[0]["n"] == 1 and c1[0]["hash"] == 1

    ch.on_update(t0 + 120 * MS, C0)  # U2, message index 2
    sends = ch.tick_data(t0 + 150 * MS)  # F8 = U1+U2 ; F3 = U2
    c1 = [s for s in sends if s["conn"] == C1]
    c2 = [s for s in sends if s["conn"] == C2]
    n1 += len(c1)
    n2 += len(c2)
    assert (n1, n2) == (3, 2)
    assert c1[0]["n"] == 1 and c1[0]["hash"] == 2 and c1[0]["last_index"] == 2
    assert c2[0]["n"] == 2 and c2[0]["hash"] == 3 and c2[0]["first"] == 0 and c2[0]["last"] == 1


def test_fan_out_catch_up_and_skip_self(oracle):
    # lagging subscriber advances one interval per step, several steps per tick (data.go:208,224,271)
    ch = oracle.channel()
    ch.subscribe(7, 0, 20)
    assert [s["kind"] for s in ch.tick_data(20 * MS)] == [0]
    for k in range(5):
        ch.on_update((25 + 10 * k) * MS, 9)  # 25,35,45,55,65
    ch.on_update(50 * MS, 7)  # own update: skipped (SkipSelfUpdateFanOut default true)
    sends = ch.tick_data(100 * MS)
    # windows [20,40],[40,60],[60,80],[80,100]: {25,35},{45,55},{65},{} -> 3 sends
    assert [(s["n"], s["hash"]) for s in sends] == [(2, 1 + 2), (2, 3 + 4), (1, 5)]
    last, had, idx = ch.state(7)
    assert last == 100 * MS and had and idx == 5
