// chd_device.cuh — device-side arithmetic shared by all kernels.
//
// Bit-exactness contract (SURVEY.md §8c): every FP64 operation below is a single correctly-rounded IEEE
// binary64 op in the order the Go source performs it — explicit __dadd_rn/__dsub_rn/__dmul_rn/__ddiv_rn/
// __dsqrt_rn so that nvcc can never contract a*b+c into an FMA (Go on amd64 does not fuse), independent of
// -fmad.  floor/ceil are exact.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/chd_gpu.h"

// look-back scan epochs (chd_scan.cuh) are 22 bits and skip 0, the value of a never-written descriptor
__host__ __device__ __forceinline__ unsigned long long chd_next_epoch(unsigned long long e) {
    e = (e + 1) & ((1ull << 22) - 1);
    return e ? e : 1ull;
}

#define CHD_INVALID_CELL 0xFFFFFFFFu
#define CHD_ABSENT 0xFFFFFFFFu

struct GridDev {
    double off_x, off_z, w, h;
    double grid_size;          // sqrt(w*w+h*h), spatial.go:134-139
    double world_x_hi, world_z_hi;  // off + w*cols, off + h*rows (spatial.go:126-132,286-287)
    double fcols, frows;
    uint32_t cols, rows, cells, id_start;
    // slab served by this engine (multi-GPU): queries may touch columns [col_lo_halo, col_hi_halo)
    uint32_t col_lo, col_hi, halo;
    uint32_t default_interval_ms;
    int32_t default_delay_ms;
    // a column this slab serves: [col_lo - halo, col_hi + halo), clipped to the grid (col < cols); the halo import keeps the
    // records of these columns, the ring limits are exchanged for them, and explicit subscriptions may name them
    __device__ __forceinline__ bool serves_column(uint32_t col) const { return col + halo >= col_lo && col < col_hi + halo; }
};

// The rank owning grid column `col` when `world` ranks split the columns into X-slabs (chd_comm_init): the largest rank r with
// floor(r * cols / world) <= col.
__device__ __forceinline__ uint32_t slab_owner(uint32_t col, uint32_t cols, uint32_t world) {
    return min((uint32_t)((((uint64_t)col + 1) * world - 1) / cols), world - 1);
}

__device__ __forceinline__ double f64sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double f64add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double f64mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double f64div(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double f64sqrt(double a) { return __dsqrt_rn(a); }

// Go math.Min / math.Max (NaN-propagating; -0 < +0).  Call sites spatial.go:207,212,239,244,276,281,286,287.
__device__ __forceinline__ double go_min(double x, double y) {
    if (isinf(x) && x < 0) return x;
    if (isinf(y) && y < 0) return y;
    if (isnan(x) || isnan(y)) return __longlong_as_double(0x7FF8000000000001ll);
    if (x == 0 && x == y) return signbit(x) ? x : y;
    return x < y ? x : y;
}
__device__ __forceinline__ double go_max(double x, double y) {
    if (isinf(x) && x > 0) return x;
    if (isinf(y) && y > 0) return y;
    if (isnan(x) || isnan(y)) return __longlong_as_double(0x7FF8000000000001ll);
    if (x == 0 && x == y) return signbit(x) ? y : x;
    return x > y ? x : y;
}

// GetChannelIdWithOffset (spatial.go:169-180): grid coordinates, or false where the reference errors.
// Go's int(math.Floor(v)) is MinInt64 for NaN/out-of-range v on amd64 and then fails `< 0`
// (pinned by spatial_test.go:793-794); testing the double before converting is equivalent.
__device__ __forceinline__ bool grid_coord(const GridDev& g, double x, double z, uint32_t& gx, uint32_t& gy) {
    const double fx = floor(f64div(f64sub(x, g.off_x), g.w));
    if (!(fx >= 0.0) || !(fx < g.fcols)) return false;
    const double fz = floor(f64div(f64sub(z, g.off_z), g.h));
    if (!(fz >= 0.0) || !(fz < g.frows)) return false;
    gx = (uint32_t)fx;
    gy = (uint32_t)fz;
    return true;
}
__device__ __forceinline__ uint32_t cell_index(const GridDev& g, double x, double z) {
    uint32_t gx, gy;
    if (!grid_coord(g, x, z, gx, gy)) return CHD_INVALID_CELL;
    return gx + gy * g.cols;
}

// uint(math.Ceil(center.Dist2D(&spot) / ctl.GridSize()))  (spatial.go:224,259,305; common.go:44-46)
__device__ __forceinline__ uint32_t cell_dist(const GridDev& g, double cx, double cz, double x, double z) {
    const double dx = f64sub(cx, x), dz = f64sub(cz, z);
    const double d = f64sqrt(f64add(f64mul(dx, dx), f64mul(dz, dz)));
    return (uint32_t)ceil(f64div(d, g.grid_size));
}

// message_spatial.go:16-38 + :65-80
__device__ __host__ __forceinline__ uint32_t damping_interval_ms(uint32_t dist, uint32_t default_ms) {
    return dist == 0 ? 20u : dist == 1 ? 50u : dist == 2 ? 100u : default_ms;
}

// Go math.Cos (src/math/sin.go; Cephes polynomials + 3-part pi/4 reduction), call site spatial.go:295.
// Restated from the published algorithm (the Go stdlib source is not in the reference tree: parity of the
// cone AOI is pinned only by TestConeAOI).  ok=false for |x| >= 2^29 (Payne-Hanek branch not reproduced).
__device__ __forceinline__ double go_cos(double x, bool& ok) {
    ok = true;
    if (isnan(x) || isinf(x)) return __longlong_as_double(0x7FF8000000000001ll);
    const double PI4A = 7.85398125648498535156e-1, PI4B = 3.77489470793079817668e-8, PI4C = 2.69515142907905952645e-15;
    bool sign = false;
    x = fabs(x);
    if (x >= 536870912.0) {
        ok = false;
        return 0.0;
    }
    // 4/Pi is a compile-time constant in Go: float64(4/Pi) = 0x3FF45F306DC9C883
    unsigned long long j = (unsigned long long)f64mul(x, __longlong_as_double(0x3FF45F306DC9C883ll));
    double y = (double)j;
    if (j & 1) {
        j++;
        y = f64add(y, 1.0);
    }
    j &= 7;
    const double z = f64sub(f64sub(f64sub(x, f64mul(y, PI4A)), f64mul(y, PI4B)), f64mul(y, PI4C));
    if (j > 3) {
        j -= 4;
        sign = !sign;
    }
    if (j > 1) sign = !sign;
    const double zz = f64mul(z, z);
    double r;
    if (j == 1 || j == 2) {
        double p = f64mul(1.58962301576546568060e-10, zz);
        p = f64mul(f64add(p, -2.50507477628578072866e-8), zz);
        p = f64mul(f64add(p, 2.75573136213857245213e-6), zz);
        p = f64mul(f64add(p, -1.98412698295895385996e-4), zz);
        p = f64mul(f64add(p, 8.33333333332211858878e-3), zz);
        p = f64add(p, -1.66666666666666307295e-1);
        r = f64add(z, f64mul(f64mul(z, zz), p));
    } else {
        double p = f64mul(-1.13585365213876817300e-11, zz);
        p = f64mul(f64add(p, 2.08757008419747316778e-9), zz);
        p = f64mul(f64add(p, -2.75573141792967388112e-7), zz);
        p = f64mul(f64add(p, 2.48015872888517045348e-5), zz);
        p = f64mul(f64add(p, -1.38888888888730564116e-3), zz);
        p = f64add(p, 4.16666666666665929218e-2);
        r = f64add(f64sub(1.0, f64mul(0.5, zz)), f64mul(f64mul(zz, zz), p));
    }
    return sign ? -r : r;
}
