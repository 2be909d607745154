// chd_query.cuh — QueryChannelIds (spatial.go:182-317) for a batch of SpatialInterestQuery, one thread per
// query, reproducing the reference's sequential `v += step` lattice walk operation-for-operation in FP64.
//
// Data structure: instead of a Go map per query, each query owns a dense "window" over the bounding box of
// cells its samples can reach (columns/rows of the first and last lattice coordinate — exact, because
// floor((v-off)/W) is monotone in v and every sample lies between the loop bounds).  A window slot holds the
// dist of the LAST sample written (z-outer / x-inner order = Go's map overwrite order) or CHD_ABSENT.
// Row-major windows enumerate cells in ascending channel id: the canonical output order.  SpotsAOI cells
// outside the window go to a small per-query side list (last-write-wins, then sorted).
#pragma once
#include "chd_types.cuh"

namespace chd {

// Guards against the reference's non-terminating lattice walks (SURVEY.md §8c'): an absorbed step (v + step == v) is
// detected directly; a walk of more than 2^24 samples is cut off as well (a documented deviation: the reference would
// answer such a query after minutes of CPU time; the oracle applies the same bound).
constexpr uint32_t QUERY_ITER_BOUND = 1u << 24;

struct BboxAcc {
    uint32_t gx0, gx1, gy0, gy1;
    bool any;
    __device__ void init() {
        any = false;
        gx0 = gy0 = 0;
        gx1 = gy1 = 0;
    }
    __device__ void add_cells(uint32_t a0, uint32_t a1, uint32_t b0, uint32_t b1) {
        if (!any) {
            gx0 = a0; gx1 = a1; gy0 = b0; gy1 = b1;
            any = true;
        } else {
            gx0 = min(gx0, a0); gx1 = max(gx1, a1); gy0 = min(gy0, b0); gy1 = max(gy1, b1);
        }
    }
    // lattice coordinates run over [xlo, xhi] x [zlo, zhi]
    __device__ void add_range(const GridDev& g, double xlo, double xhi, double zlo, double zhi) {
        if (!(xlo <= xhi) || !(zlo <= zhi)) return;  // the reference's loops never execute (also NaN)
        const double fl = floor(f64div(f64sub(xlo, g.off_x), g.w)), fh = floor(f64div(f64sub(xhi, g.off_x), g.w));
        const double rl = floor(f64div(f64sub(zlo, g.off_z), g.h)), rh = floor(f64div(f64sub(zhi, g.off_z), g.h));
        if (!(fh >= 0.0) || !(fl < g.fcols) || !(rh >= 0.0) || !(rl < g.frows)) return;
        const uint32_t a0 = fl < 0.0 ? 0u : (uint32_t)fl, a1 = fh >= g.fcols ? g.cols - 1 : (uint32_t)fh;
        const uint32_t b0 = rl < 0.0 ? 0u : (uint32_t)rl, b1 = rh >= g.frows ? g.rows - 1 : (uint32_t)rh;
        add_cells(a0, a1, b0, b1);
    }
    __device__ void add_point(const GridDev& g, double x, double z) {
        uint32_t gx, gy;
        if (grid_coord(g, x, z, gx, gy)) add_cells(gx, gx, gy, gy);
    }
};

// Q1: bounding box of the cells a query's lattice samples can reach.
__device__ __forceinline__ Bbox query_bbox(const GridDev& g, const QueryDev& q, uint32_t i, uint32_t kind) {
    BboxAcc acc;
    acc.init();
    if (kind & CHD_AOI_BOX) {
        const double cx = q.box_cx[i], cz = q.box_cz[i], ex = q.box_ex[i], ez = q.box_ez[i];
        acc.add_range(g, f64sub(cx, ex), f64add(cx, ex), f64sub(cz, ez), f64add(cz, ez));
        acc.add_point(g, cx, cz);
    }
    if (kind & CHD_AOI_SPHERE) {
        const double cx = q.sph_cx[i], cz = q.sph_cz[i], r = q.sph_r[i];
        acc.add_range(g, f64sub(cx, r), f64add(cx, r), f64sub(cz, r), f64add(cz, r));
        acc.add_point(g, cx, cz);
    }
    if (kind & CHD_AOI_CONE) {
        const double cx = q.cone_cx[i], cz = q.cone_cz[i], r = q.cone_r[i];
        acc.add_range(g, go_max(g.off_x, f64sub(cx, r)), go_min(g.world_x_hi, f64add(cx, r)), go_max(g.off_z, f64sub(cz, r)),
                      go_min(g.world_z_hi, f64add(cz, r)));
        acc.add_point(g, cx, cz);
    }
    Bbox b;
    if (acc.any) {
        b.gx0 = acc.gx0; b.gy0 = acc.gy0; b.bw = acc.gx1 - acc.gx0 + 1; b.bh = acc.gy1 - acc.gy0 + 1;
    } else {
        b.gx0 = b.gy0 = 0; b.bw = b.bh = 0;
    }
    return b;
}

struct WinRef {
    uint32_t* w;
    Bbox b;
    __device__ __forceinline__ bool put(uint32_t gx, uint32_t gy, uint32_t dist) const {
        const uint32_t ix = gx - b.gx0, iy = gy - b.gy0;  // unsigned wrap => out of window
        if (ix >= b.bw || iy >= b.bh) return false;
        w[iy * b.bw + ix] = dist;
        return true;
    }
};

// The whole query in ONE launch: bounding box -> window scratch -> lattice walk.  A query's window is private scratch, so
// its location does not matter: the block's windows are carved out of `window` with one atomicAdd per block on a bump
// cursor (zeroed by the stage's first kernel) instead of a device-wide prefix sum (two launches less per tick).
// A query whose window does not fit the scratch gets CHD_Q_ERR_CAPACITY: like any failed query it leaves the subscriber's
// subscriptions untouched; CHD_OVF_WINDOW is raised and the cursor's final value is the required capacity.
// A query that sets a kind bit without supplying that kind's arrays gets CHD_Q_ERR_MISSING_ARRAY; in a merged batch the host
// part's entries are judged by the arrays the host part supplied (q.missing, written by follow_merge_kernel).
__global__ void __launch_bounds__(128)
    query_kernel(GridDev g, QueryDev q, Bbox* __restrict__ bbox, uint64_t* __restrict__ win_off, uint64_t win_cap,
                 unsigned long long* __restrict__ win_cursor, uint32_t* __restrict__ window, uint32_t* __restrict__ side_cell,
                 uint32_t* __restrict__ side_dist, uint32_t* __restrict__ side_cnt, uint32_t* __restrict__ status, uint32_t* __restrict__ count,
                 uint32_t* __restrict__ overflow) {
    __shared__ unsigned long long s_warp[4], s_base;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
    uint32_t kind = 0;
    bool missing = false;
    WinRef win;
    win.b.gx0 = win.b.gy0 = win.b.bw = win.b.bh = 0;
    if (i < q.n) {
        kind = query_kind(q, i);
        missing = query_arrays_missing(q, kind) || (q.missing && q.missing[i]);
        if (!missing) win.b = query_bbox(g, q, i, kind);
    }
    const uint32_t wn = win.b.bw * win.b.bh;
    // block-aggregated reservation of the window scratch
    unsigned long long incl = wn;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long a = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += a;
    }
    if (lane == 31) s_warp[wp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long tot = s_warp[0] + s_warp[1] + s_warp[2] + s_warp[3];
        s_base = tot ? atomicAdd(win_cursor, tot) : 0ull;
    }
    __syncthreads();
    unsigned long long off = s_base + incl - wn;
    for (int k = 0; k < wp; k++) off += s_warp[k];
    if (i >= q.n) return;
    bbox[i] = win.b;
    win_off[i] = off;
    if (missing || off + wn > win_cap) {
        if (!missing) atomicOr(overflow, (uint32_t)CHD_OVF_WINDOW);
        status[i] = missing ? CHD_Q_ERR_MISSING_ARRAY : CHD_Q_ERR_CAPACITY;
        count[i] = 0;
        if (side_cnt) side_cnt[i] = 0;
        return;
    }
    win.w = window + off;
    for (uint32_t k = 0; k < wn; k++) win.w[k] = CHD_ABSENT;
    uint32_t st = CHD_Q_OK;
    uint32_t n_side = 0;
    uint32_t gx, gy;

    if ((kind & CHD_AOI_SPOTS) && q.spot_off) {  // spatial.go:189-202
        const uint32_t s0 = q.spot_off[i], s1 = q.spot_off[i + 1];
        const uint32_t nd = q.spot_ndist ? q.spot_ndist[i] : 0u;
        for (uint32_t k = s0; k < s1; k++) {
            if (!grid_coord(g, q.spot_x[k], q.spot_z[k], gx, gy)) continue;
            const uint32_t d = (k - s0) < nd ? q.spot_dist[k] : 0u;
            if (win.put(gx, gy, d)) continue;
            const uint32_t c = gx + gy * g.cols;
            uint32_t j = 0;
            for (; j < n_side; j++)
                if (side_cell[s0 + j] == c) break;
            side_cell[s0 + j] = c;
            side_dist[s0 + j] = d;
            if (j == n_side) n_side++;
        }
    }

    if (kind & CHD_AOI_BOX) {  // spatial.go:204-233
        const double cx = q.box_cx[i], cz = q.box_cz[i], ex = q.box_ex[i], ez = q.box_ez[i];
        const double stepZ = f64mul(go_min(ez, g.h), 0.5);
        if (stepZ <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double stepX = f64mul(go_min(ex, g.w), 0.5);
        if (stepX <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double zhi = f64add(cz, ez), xhi = f64add(cx, ex), xlo = f64sub(cx, ex);
        uint32_t iters = 0;
        for (double z = f64sub(cz, ez), zn; z <= zhi; z = zn) {
            zn = f64add(z, stepZ);
            if (zn == z) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
            for (double x = xlo, xn; x <= xhi; x = xn) {
                xn = f64add(x, stepX);
                if (xn == x || ++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }  // absorbed step: the reference never terminates
                if (!grid_coord(g, x, z, gx, gy)) continue;
                win.put(gx, gy, cell_dist(g, cx, cz, x, z));
            }
            if (++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
        }
        if (!grid_coord(g, cx, cz, gx, gy)) { st = CHD_Q_ERR_OUT_OF_WORLD; goto done; }
        win.put(gx, gy, 0u);
    }

    if (kind & CHD_AOI_SPHERE) {  // spatial.go:235-268
        const double cx = q.sph_cx[i], cz = q.sph_cz[i], r = q.sph_r[i];
        const double stepZ = f64mul(go_min(r, g.h), 0.5);
        if (stepZ <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double stepX = f64mul(go_min(r, g.w), 0.5);
        if (stepX <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double zhi = f64add(cz, r), xhi = f64add(cx, r), xlo = f64sub(cx, r), rr = f64mul(r, r);
        uint32_t iters = 0;
        for (double z = f64sub(cz, r), zn; z <= zhi; z = zn) {
            zn = f64add(z, stepZ);
            if (zn == z) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
            const double dz = f64sub(z, cz);
            const double dz2 = f64mul(dz, dz);
            for (double x = xlo, xn; x <= xhi; x = xn) {
                xn = f64add(x, stepX);
                if (xn == x || ++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }  // absorbed step: the reference never terminates
                const double dx = f64sub(x, cx);
                if (f64add(f64mul(dx, dx), dz2) > rr) continue;
                if (!grid_coord(g, x, z, gx, gy)) continue;
                win.put(gx, gy, cell_dist(g, cx, cz, x, z));
            }
            if (++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
        }
        if (!grid_coord(g, cx, cz, gx, gy)) { st = CHD_Q_ERR_OUT_OF_WORLD; goto done; }
        win.put(gx, gy, 0u);
    }

    if (kind & CHD_AOI_CONE) {  // spatial.go:270-314
        const double cx = q.cone_cx[i], cz = q.cone_cz[i], r = q.cone_r[i];
        double ddx = q.cone_dx[i], ddz = q.cone_dz[i];
        {  // common.go:56-60 Normalize2D
            const double mag = f64sqrt(f64add(f64mul(ddx, ddx), f64mul(ddz, ddz)));
            ddx = f64div(ddx, mag);
            ddz = f64div(ddz, mag);
        }
        const double stepZ = f64mul(go_min(r, g.h), 0.5);
        if (stepZ <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double stepX = f64mul(go_min(r, g.w), 0.5);
        if (stepX <= 0) { st = CHD_Q_ERR_BAD_STEP; goto done; }
        const double zhi = go_min(g.world_z_hi, f64add(cz, r)), xhi = go_min(g.world_x_hi, f64add(cx, r));
        const double xlo = go_max(g.off_x, f64sub(cx, r)), rr = f64mul(r, r);
        bool cos_ok;
        const double cosv = go_cos(q.cone_angle[i], cos_ok);  // spatial.go:295 (loop invariant)
        if (!cos_ok) { st = CHD_Q_ERR_ANGLE_RANGE; goto done; }
        uint32_t iters = 0;
        for (double z = go_max(g.off_z, f64sub(cz, r)), zn; z <= zhi; z = zn) {
            zn = f64add(z, stepZ);
            if (zn == z) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
            const double dz = f64sub(z, cz);
            const double dz2 = f64mul(dz, dz);
            for (double x = xlo, xn; x <= xhi; x = xn) {
                xn = f64add(x, stepX);
                if (xn == x || ++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }  // absorbed step: the reference never terminates
                const double dx = f64sub(x, cx);
                if (f64add(f64mul(dx, dx), dz2) > rr) continue;
                const double mag = f64sqrt(f64add(f64mul(dx, dx), dz2));
                const double ux = f64div(dx, mag), uz = f64div(dz, mag);  // 0/0 = NaN at the centre sample
                const double dot = f64add(f64mul(ux, ddx), f64mul(uz, ddz));
                if (dot < cosv) continue;  // NaN < cos is false: the centre sample passes (spatial.go:297)
                if (!grid_coord(g, x, z, gx, gy)) continue;
                win.put(gx, gy, cell_dist(g, cx, cz, x, z));
            }
            if (++iters > QUERY_ITER_BOUND) { st = CHD_Q_ERR_ITER_BOUND; goto done; }
        }
        if (!grid_coord(g, cx, cz, gx, gy)) { st = CHD_Q_ERR_OUT_OF_WORLD; goto done; }
        win.put(gx, gy, 0u);
    }

done:
    uint32_t cnt = 0;
    if (st == CHD_Q_OK) {
        for (uint32_t k = 0; k < wn; k++) cnt += win.w[k] != CHD_ABSENT;
        cnt += n_side;
        if (n_side > 1) {  // insertion sort of the side list by cell
            const uint32_t s0 = q.spot_off[i];
            for (uint32_t a = 1; a < n_side; a++) {
                const uint32_t c = side_cell[s0 + a], d = side_dist[s0 + a];
                uint32_t b = a;
                while (b > 0 && side_cell[s0 + b - 1] > c) {
                    side_cell[s0 + b] = side_cell[s0 + b - 1];
                    side_dist[s0 + b] = side_dist[s0 + b - 1];
                    b--;
                }
                side_cell[s0 + b] = c;
                side_dist[s0 + b] = d;
            }
        }
    } else {
        n_side = 0;
    }
    status[i] = st;
    count[i] = cnt;
    if (side_cnt) side_cnt[i] = n_side;
}

// Iterates a query's result entries (window U side list) in ascending cell order.
struct ResultIter {
    const uint32_t* w;
    Bbox b;
    uint32_t wn, k;  // window cursor
    const uint32_t *sc, *sd;
    uint32_t ns, j;  // side cursor
    uint32_t cols;
    __device__ void init(const uint32_t* window, const uint64_t* win_off, const Bbox* bbox, const uint32_t* side_cell,
                         const uint32_t* side_dist, const uint32_t* side_cnt, const uint32_t* spot_off, uint32_t q, uint32_t cols_) {
        b = bbox[q];
        w = window + win_off[q];
        wn = b.bw * b.bh;
        k = 0;
        cols = cols_;
        ns = side_cnt ? side_cnt[q] : 0u;
        j = 0;
        if (ns) {
            sc = side_cell + spot_off[q];
            sd = side_dist + spot_off[q];
        } else {
            sc = sd = nullptr;
        }
        while (k < wn && w[k] == CHD_ABSENT) k++;
    }
    __device__ bool next(uint32_t& cell, uint32_t& dist) {
        const bool hw = k < wn, hs = j < ns;
        if (!hw && !hs) return false;
        uint32_t wc = 0;
        if (hw) wc = (b.gx0 + k % b.bw) + (b.gy0 + k / b.bw) * cols;
        if (hw && (!hs || wc < sc[j])) {
            cell = wc;
            dist = w[k];
            k++;
            while (k < wn && w[k] == CHD_ABSENT) k++;
        } else {
            cell = sc[j];
            dist = sd[j];
            j++;
        }
        return true;
    }
};

// Q3 (stateless path): write the CSR result of chd_query_channel_ids.
__global__ void __launch_bounds__(128)
    query_write_kernel(GridDev g, uint32_t n, const uint32_t* __restrict__ status, const Bbox* __restrict__ bbox,
                       const uint64_t* __restrict__ win_off, const uint32_t* __restrict__ window,
                       const uint32_t* __restrict__ side_cell, const uint32_t* __restrict__ side_dist,
                       const uint32_t* __restrict__ side_cnt, const uint32_t* __restrict__ spot_off,
                       const uint64_t* __restrict__ out_off, uint64_t cap, uint32_t* __restrict__ out_id, uint32_t* __restrict__ out_dist) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || status[i] != CHD_Q_OK) return;
    if (out_off[n] > cap) return;
    ResultIter it;
    it.init(window, win_off, bbox, side_cell, side_dist, side_cnt, spot_off, i, g.cols);
    uint64_t o = out_off[i];
    uint32_t c, d;
    while (it.next(c, d)) {
        out_id[o] = c + g.id_start;
        out_dist[o] = d;
        o++;
    }
}

}  // namespace chd
