"""orc_query_batch (the batched, threaded QueryChannelIds the GPU scale tests compare against) equals orc_query_channel_ids called
query by query: statuses, and every query's (channel id, dist) list in the same order.  No GPU needed."""
import numpy as np
import pytest

from tests import _queries as Q
from tests._oracle import make_grid
from tests.golden import golden_io as gio

# the grids of tests/test_gpu_parity.py's random query parity
GRIDS = [
    (-150, -150, 100, 100, 3, 3), (-5, -5, 5, 5, 2, 2), (0, 0, 10, 10, 4, 1), (-2000, -2000, 2000, 2000, 2, 2),
    (-15000, -15000, 2000, 2000, 15, 15), (-450, -200, 100, 50, 9, 8), (-12.5, 3.25, 7.3, 11.9, 13, 7), (0, 0, 33, 77, 2, 2),
]


def _one(q, i):
    """query i of a batch as Oracle.query keyword arguments"""
    k, kw = int(q["kind"][i]), {}
    if k & Q.AOI_SPOTS:
        off, nd, sx, sz, sd = q["spots"]
        a, b = int(off[i]), int(off[i + 1])
        kw["spots"] = list(zip(sx[a:b], sz[a:b]))
        kw["spot_dists"] = sd[a:a + min(int(nd[i]), b - a)].tolist()
    if k & Q.AOI_BOX:
        kw["box"] = tuple(a[i] for a in q["box"])
    if k & Q.AOI_SPHERE:
        kw["sphere"] = tuple(a[i] for a in q["sphere"])
    if k & Q.AOI_CONE:
        kw["cone"] = tuple(a[i] for a in q["cone"])
    return kw


def _check(oracle, og, q, n_threads):
    st, off, ids, dist = oracle.query_batch(og, q["n"], n_threads=n_threads, **Q.batch_kwargs(q))
    assert off.dtype == np.uint64 and len(off) == q["n"] + 1
    for i in range(q["n"]):
        want, wst = oracle.query(og, **_one(q, i))
        assert st[i] == wst, (i, st[i], wst)
        a, b = int(off[i]), int(off[i + 1])
        if wst != 0:
            assert a == b
        else:
            assert list(zip(ids[a:b].tolist(), dist[a:b].tolist())) == list(want.items()), i
    return st, off


@pytest.mark.parametrize("gi", range(len(GRIDS)))
def test_batch_equals_single_queries(oracle, gi):
    g = GRIDS[gi]
    rng = np.random.default_rng(700 + gi)
    q = Q.make_queries(rng, g, 2500, p_err=0.1, long_cells=6.0, max_spots=80)
    st, off = _check(oracle, make_grid(*g), q, n_threads=1 + gi % 4)
    kinds = q["kind"]
    assert set(kinds.tolist()) == set(range(16))
    assert {0, 1, 2, 5, 6} <= set(st.tolist())  # OK and every error path the generator aims at
    assert (st[kinds == 0] == 0).all() and (off[1:][kinds == 0] == off[:-1][kinds == 0]).all()  # no AOI: an empty answer
    # the batch does not depend on how it is split over threads
    st1, off1, ids1, d1 = oracle.query_batch(make_grid(*g), q["n"], n_threads=1, **Q.batch_kwargs(q))
    st8, off8, ids8, d8 = oracle.query_batch(make_grid(*g), q["n"], n_threads=8, **Q.batch_kwargs(q))
    for a, b in ((st1, st8), (off1, off8), (ids1, ids8), (d1, d8)):
        np.testing.assert_array_equal(a, b)


def test_batch_replays_golden_queries(oracle):
    for grid in gio.load_queries():
        g, cases = grid["grid"], grid["cases"]
        n = len(cases)
        kind = np.zeros(n, np.uint8)
        arr = {k: np.zeros(n) for k in ("sph_cx", "sph_cz", "sph_r", "box_cx", "box_cz", "box_ex", "box_ez", "cone_cx", "cone_cz",
                                        "cone_dx", "cone_dz", "cone_angle", "cone_r")}
        off, nd, sx, sz, sd = [0], [], [], [], []
        for i, c in enumerate(cases):
            qd = c["query"]
            if "sphere" in qd:
                kind[i] |= Q.AOI_SPHERE
                arr["sph_cx"][i], arr["sph_cz"][i], arr["sph_r"][i] = qd["sphere"]
            if "box" in qd:
                kind[i] |= Q.AOI_BOX
                arr["box_cx"][i], arr["box_cz"][i], arr["box_ex"][i], arr["box_ez"][i] = qd["box"]
            if "cone" in qd:
                kind[i] |= Q.AOI_CONE
                for k, v in zip(("cone_cx", "cone_cz", "cone_dx", "cone_dz", "cone_angle", "cone_r"), qd["cone"]):
                    arr[k][i] = v
            spots, dists = qd.get("spots"), qd.get("spot_dists") or []
            if spots is not None:
                kind[i] |= Q.AOI_SPOTS
                sx += [s[0] for s in spots]
                sz += [s[1] for s in spots]
                # spot_dist is indexed like the spots: dists past the last spot are never read
                sd += (list(dists) + [0] * len(spots))[:len(spots)]
            nd.append(len(dists))
            off.append(len(sx))
        st, o, ids, dist = oracle.query_batch(
            make_grid(*g), n, kind=kind, sphere=(arr["sph_cx"], arr["sph_cz"], arr["sph_r"]),
            box=(arr["box_cx"], arr["box_cz"], arr["box_ex"], arr["box_ez"]),
            cone=tuple(arr[k] for k in ("cone_cx", "cone_cz", "cone_dx", "cone_dz", "cone_angle", "cone_r")),
            spots=(np.array(off), np.array(nd), np.array(sx), np.array(sz), np.array(sd)))
        for i, c in enumerate(cases):
            assert st[i] == c["status"], (g, i)
            got = list(map(list, zip(ids[o[i]:o[i + 1]].tolist(), dist[o[i]:o[i + 1]].tolist())))
            assert got == (c["result"] or []), (g, i)


def test_batch_capacity_and_missing_arrays(oracle):
    g = GRIDS[5]
    og = make_grid(*g)
    q = Q.make_queries(np.random.default_rng(3), g, 300)
    st, off, ids, dist = oracle.query_batch(og, q["n"], **Q.batch_kwargs(q))
    assert int(off[-1]) > 100
    import ctypes as C

    from tests._oracle import ERR_CAPACITY, ERR_NIL, QuerySoA, u32p, u64p
    # too small a capacity: offsets written, nothing else
    b = QuerySoA()
    b.n = 3
    centre, r = np.zeros(3), np.array([50.0, 120.0, 10.0])
    b.sph_cx, b.sph_cz, b.sph_r = (a.ctypes.data_as(C.POINTER(C.c_double)) for a in (centre, centre, r))
    s3, o3, i3, d3 = np.zeros(3, np.uint32), np.zeros(4, np.uint64), np.full(2, 7, np.uint32), np.full(2, 7, np.uint32)
    rc = oracle.lib.orc_query_batch(C.byref(og), C.byref(b), s3.ctypes.data_as(u32p), o3.ctypes.data_as(u64p), i3.ctypes.data_as(u32p),
                                    d3.ctypes.data_as(u32p), 2, 2)
    assert rc == ERR_CAPACITY and o3[-1] > 2 and (i3 == 7).all()
    # a kind bit without its arrays
    k = np.array([4, 2, 4], np.uint8)
    b.kind = k.ctypes.data
    rc = oracle.lib.orc_query_batch(C.byref(og), C.byref(b), s3.ctypes.data_as(u32p), o3.ctypes.data_as(u64p), None, None, 0, 1)
    assert rc == ERR_NIL
