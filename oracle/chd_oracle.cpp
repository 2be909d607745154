// chd_oracle.cpp — CPU ORACLE (test infrastructure only; see chd_oracle.h for the pin status).
// C++17 restatement of channeld's Go spatial hot path.  Build: g++ -O2 -ffp-contract=off (Makefile).
// No code here is reachable from the product path (channeld_b200/).
#include "chd_oracle.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <mutex>
#include <list>
#include <map>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

// Go math.Min / math.Max (NaN-propagating, signed-zero aware); call sites spatial.go:207,212,239,244,276,281,286,287.
inline double go_min(double x, double y) {
    if (std::isinf(x) && x < 0) return x;
    if (std::isinf(y) && y < 0) return y;
    if (std::isnan(x) || std::isnan(y)) return std::nan("");
    if (x == 0 && x == y) return std::signbit(x) ? x : y;
    return x < y ? x : y;
}
inline double go_max(double x, double y) {
    if (std::isinf(x) && x > 0) return x;
    if (std::isinf(y) && y > 0) return y;
    if (std::isnan(x) || std::isnan(y)) return std::nan("");
    if (x == 0 && x == y) return std::signbit(x) ? y : x;
    return x > y ? x : y;
}

// common.go:44-46  Dist2D (receiver = centre, argument = spot)
inline double dist2d(double x1, double z1, double x2, double z2) {
    return std::sqrt((x1 - x2) * (x1 - x2) + (z1 - z2) * (z1 - z2));
}

// spatial.go:126-132
inline double world_width(const orc_grid* g) { return g->grid_width * double(g->grid_cols); }
inline double world_height(const orc_grid* g) { return g->grid_height * double(g->grid_rows); }

// spatial.go:169-180 with offsets; returns false on the error path.
// Go's int(math.Floor(v)) on amd64 yields MinInt64 for NaN / out-of-range v, which then fails `gridX < 0`
// (pinned by spatial_test.go:793-794, X = MaxFloat64 must error).  Testing the double before converting is
// equivalent and avoids C++ UB.
inline bool cell_index(const orc_grid* g, double x, double z, uint32_t* idx) {
    double fx = std::floor((x - g->world_offset_x) / g->grid_width);
    if (!(fx >= 0.0) || !(fx < double(g->grid_cols))) return false;
    double fz = std::floor((z - g->world_offset_z) / g->grid_height);
    if (!(fz >= 0.0) || !(fz < double(g->grid_rows))) return false;
    *idx = uint32_t(fx) + uint32_t(fz) * g->grid_cols;
    return true;
}

// Guard against the reference's non-terminating walks (SURVEY §8c'): an absorbed step (v + step == v) loops forever in Go;
// walks of more than 2^24 samples are cut off too.  The CUDA path applies the same two rules (chd_query.cuh).
const uint64_t kIterBound = 1ull << 24;

// spatial.go:182-317 into any map-like container M (operator[] overwrite = Go map assignment).
template <class M>
int query_into(const orc_grid* g, const orc_query* q, M& result) {
    if (!q) return ORC_ERR_NIL;
    const double grid_size = orc_grid_size(g);
    const uint32_t base = g->channel_id_start;
    uint32_t idx;

    if (q->kind_mask & ORC_AOI_SPOTS) {  // spatial.go:189-202
        for (uint32_t i = 0; i < q->n_spots; i++) {
            if (!cell_index(g, q->spot_x[i], q->spot_z[i], &idx)) continue;
            result[idx + base] = (i < q->n_spot_dists) ? q->spot_dist[i] : 0u;
        }
    }

    if (q->kind_mask & ORC_AOI_BOX) {  // spatial.go:204-233
        const double cx = q->box_cx, cz = q->box_cz;
        const double stepZ = go_min(q->box_ez, g->grid_height) * 0.5;
        if (stepZ <= 0) return ORC_ERR_BAD_STEP;
        const double stepX = go_min(q->box_ex, g->grid_width) * 0.5;
        if (stepX <= 0) return ORC_ERR_BAD_STEP;
        uint64_t iters = 0;
        for (double z = cz - q->box_ez; z <= cz + q->box_ez; z += stepZ) {
            for (double x = cx - q->box_ex; x <= cx + q->box_ex; x += stepX) {
                if (x + stepX == x || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
                if (!cell_index(g, x, z, &idx)) continue;
                result[idx + base] = uint32_t(std::ceil(dist2d(cx, cz, x, z) / grid_size));
            }
            if (z + stepZ == z || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
        }
        if (!cell_index(g, cx, cz, &idx)) return ORC_ERR_OUT_OF_WORLD;
        result[idx + base] = 0;
    }

    if (q->kind_mask & ORC_AOI_SPHERE) {  // spatial.go:235-268
        const double r = q->sph_r, cx = q->sph_cx, cz = q->sph_cz;
        const double stepZ = go_min(r, g->grid_height) * 0.5;
        if (stepZ <= 0) return ORC_ERR_BAD_STEP;
        const double stepX = go_min(r, g->grid_width) * 0.5;
        if (stepX <= 0) return ORC_ERR_BAD_STEP;
        uint64_t iters = 0;
        for (double z = cz - r; z <= cz + r; z += stepZ) {
            for (double x = cx - r; x <= cx + r; x += stepX) {
                if (x + stepX == x || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
                if ((x - cx) * (x - cx) + (z - cz) * (z - cz) > r * r) continue;
                if (!cell_index(g, x, z, &idx)) continue;
                result[idx + base] = uint32_t(std::ceil(dist2d(cx, cz, x, z) / grid_size));
            }
            if (z + stepZ == z || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
        }
        if (!cell_index(g, cx, cz, &idx)) return ORC_ERR_OUT_OF_WORLD;
        result[idx + base] = 0;
    }

    if (q->kind_mask & ORC_AOI_CONE) {  // spatial.go:270-314
        const double r = q->cone_r, cx = q->cone_cx, cz = q->cone_cz;
        double ddx = q->cone_dx, ddz = q->cone_dz;
        {  // common.go:56-60 Normalize2D
            const double mag = std::sqrt(ddx * ddx + ddz * ddz);
            ddx /= mag;
            ddz /= mag;
        }
        const double stepZ = go_min(r, g->grid_height) * 0.5;
        if (stepZ <= 0) return ORC_ERR_BAD_STEP;
        const double stepX = go_min(r, g->grid_width) * 0.5;
        if (stepX <= 0) return ORC_ERR_BAD_STEP;
        const double z_hi = go_min(g->world_offset_z + world_height(g), cz + r);
        const double x_hi = go_min(g->world_offset_x + world_width(g), cx + r);
        // |angle| >= 2^29: Go's math.Cos switches to Payne-Hanek reduction, which is not restated; both this oracle and the CUDA
        // path reject such a query (documented deviation, DESIGN.md) instead of answering with a different cosine
        if (std::fabs(q->cone_angle) >= double(1 << 29)) return ORC_ERR_ANGLE_RANGE;
        const double cosv = orc_go_cos(q->cone_angle);  // spatial.go:295 (loop-invariant)
        uint64_t iters = 0;
        for (double z = go_max(g->world_offset_z, cz - r); z <= z_hi; z += stepZ) {
            for (double x = go_max(g->world_offset_x, cx - r); x <= x_hi; x += stepX) {
                if (x + stepX == x || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
                if ((x - cx) * (x - cx) + (z - cz) * (z - cz) > r * r) continue;
                double vx = x - cx, vz = z - cz;
                const double mag = std::sqrt(vx * vx + vz * vz);
                vx /= mag;  // 0/0 = NaN at the centre sample; NaN < cos is false so it passes (spatial.go:297)
                vz /= mag;
                const double dot = vx * ddx + vz * ddz;  // common.go:48-50
                if (dot < cosv) continue;
                if (!cell_index(g, x, z, &idx)) continue;
                result[idx + base] = uint32_t(std::ceil(dist2d(cx, cz, x, z) / grid_size));
            }
            if (z + stepZ == z || ++iters > kIterBound) return ORC_ERR_ITER_BOUND;
        }
        if (!cell_index(g, cx, cz, &idx)) return ORC_ERR_OUT_OF_WORLD;
        result[idx + base] = 0;
    }
    return ORC_OK;
}

}  // namespace

extern "C" {

double orc_grid_size(const orc_grid* g) {  // spatial.go:134-139
    if (g->grid_width > 0 && g->grid_height > 0)
        return std::sqrt(g->grid_width * g->grid_width + g->grid_height * g->grid_height);
    return 0.0;
}

// Go math.Cos (src/math/sin.go; Cephes cosf/sinf polynomials, 3-part pi/4 reduction).  The Go source is not
// in the reference tree; this restates the published algorithm.  |x| >= 2^29 uses Payne-Hanek in Go; that branch
// is not restated: QueryChannelIds rejects such cone angles (ORC_ERR_ANGLE_RANGE); this function alone falls back to libm.
double orc_go_cos(double x) {
    static const double kSin[6] = {1.58962301576546568060e-10, -2.50507477628578072866e-8, 2.75573136213857245213e-6,
                                   -1.98412698295895385996e-4, 8.33333333332211858878e-3,  -1.66666666666666307295e-1};
    static const double kCos[6] = {-1.13585365213876817300e-11, 2.08757008419747316778e-9, -2.75573141792967388112e-7,
                                   2.48015872888517045348e-5,   -1.38888888888730564116e-3, 4.16666666666665929218e-2};
    const double PI4A = 7.85398125648498535156e-1, PI4B = 3.77489470793079817668e-8, PI4C = 2.69515142907905952645e-15;
    if (std::isnan(x) || std::isinf(x)) return std::nan("");
    bool sign = false;
    x = std::fabs(x);
    if (x >= double(1 << 29)) return std::cos(x);
    uint64_t j = uint64_t(x * (4.0 / M_PI));
    double y = double(j);
    if (j & 1) {
        j++;
        y++;
    }
    j &= 7;
    const double z = ((x - y * PI4A) - y * PI4B) - y * PI4C;
    if (j > 3) {
        j -= 4;
        sign = !sign;
    }
    if (j > 1) sign = !sign;
    const double zz = z * z;
    if (j == 1 || j == 2)
        y = z + z * zz * ((((((kSin[0] * zz) + kSin[1]) * zz + kSin[2]) * zz + kSin[3]) * zz + kSin[4]) * zz + kSin[5]);
    else
        y = 1.0 - 0.5 * zz +
            zz * zz * ((((((kCos[0] * zz) + kCos[1]) * zz + kCos[2]) * zz + kCos[3]) * zz + kCos[4]) * zz + kCos[5]);
    return sign ? -y : y;
}

int orc_get_channel_id(const orc_grid* g, double x, double z, uint32_t* out_id) {
    uint32_t idx;
    if (!cell_index(g, x, z, &idx)) {
        *out_id = 0;
        return ORC_ERR_OUT_OF_WORLD;
    }
    *out_id = idx + g->channel_id_start;
    return ORC_OK;
}

void orc_cell_of(const orc_grid* g, const double* x, const double* z, uint32_t n, uint32_t* out) {
    for (uint32_t i = 0; i < n; i++) orc_get_channel_id(g, x[i], z[i], &out[i]);
}

int orc_query_channel_ids(const orc_grid* g, const orc_query* q, uint32_t* out_ids, uint32_t* out_dists, uint32_t cap,
                          uint32_t* out_n) {
    std::map<uint32_t, uint32_t> result;  // ordered => canonical output order
    *out_n = 0;
    int st = query_into(g, q, result);
    if (st != ORC_OK) return st;  // reference returns (nil, err): no partial result
    if (result.size() > cap) {
        *out_n = uint32_t(result.size());
        return ORC_ERR_CAPACITY;
    }
    uint32_t n = 0;
    for (auto& kv : result) {
        out_ids[n] = kv.first;
        out_dists[n] = kv.second;
        n++;
    }
    *out_n = n;
    return ORC_OK;
}

uint32_t orc_get_adjacent_channels(const orc_grid* g, uint32_t channel_id, uint32_t* out8) {  // spatial.go:358-381
    const uint32_t index = channel_id - g->channel_id_start;
    const int32_t gx = int32_t(index % g->grid_cols), gy = int32_t(index / g->grid_cols);
    uint32_t n = 0;
    for (int32_t y = gy - 1; y <= gy + 1; y++) {
        if (y < 0 || y > int32_t(g->grid_rows - 1)) continue;
        for (int32_t x = gx - 1; x <= gx + 1; x++) {
            if (x < 0 || x > int32_t(g->grid_cols - 1)) continue;
            if (x == gx && y == gy) continue;
            out8[n++] = uint32_t(x) + uint32_t(y) * g->grid_cols + g->channel_id_start;
        }
    }
    return n;
}

uint32_t orc_adjacent_broadcast(const orc_grid* g, uint32_t channel_id, uint32_t broadcast, uint32_t sender_conn_id,
                                uint32_t client_conn_id, const uint32_t* cell_off, const uint32_t* conn_id,
                                const uint8_t* conn_type, uint32_t* out_conn, uint32_t cap) {  // message.go:188-239
    enum : uint32_t { ALL_BUT_SENDER = 4, ALL_BUT_OWNER = 8, ALL_BUT_CLIENT = 16, ALL_BUT_SERVER = 32 };  // channeld.proto BroadcastType
    const auto check = [&](uint32_t bit) { return (broadcast & bit) > 0; };  // channeldpb/extension.go:5-7
    uint32_t ids[9];
    uint32_t n = orc_get_adjacent_channels(g, channel_id, ids);  // message.go:197
    if (!check(ALL_BUT_OWNER)) ids[n++] = channel_id;            // :203-205
    std::map<uint32_t, uint8_t> adjacent_conns;                  // :208-219 (connection -> its type)
    const uint32_t cells = g->grid_cols * g->grid_rows;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t cell = ids[i] - g->channel_id_start;
        if (cell >= cells) continue;  // GetChannel(id) == nil
        for (uint32_t k = cell_off[cell]; k < cell_off[cell + 1]; k++) adjacent_conns[conn_id[k]] = conn_type ? conn_type[k] : uint8_t(0);
    }
    uint32_t out = 0;
    for (const auto& kv : adjacent_conns) {  // :220-238
        if (check(ALL_BUT_SENDER) && kv.first == sender_conn_id) continue;
        if (check(ALL_BUT_CLIENT) && kv.second == 2) continue;
        if (check(ALL_BUT_SERVER) && kv.second == 1) continue;
        if (kv.first == client_conn_id) continue;
        if (out < cap) out_conn[out] = kv.first;
        out++;
    }
    return out;
}

void orc_get_regions(const orc_grid* g, double* min_x, double* min_z, double* max_x, double* max_z, uint32_t* channel_id,
                     uint32_t* server_index) {  // spatial.go:319-356
    uint32_t sgc = g->grid_cols / g->server_cols;
    if (g->grid_cols % g->server_cols > 0) sgc++;
    uint32_t sgr = g->grid_rows / g->server_rows;
    if (g->grid_rows % g->server_rows > 0) sgr++;
    for (uint32_t y = 0; y < g->grid_rows; y++)
        for (uint32_t x = 0; x < g->grid_cols; x++) {
            const uint32_t index = x + y * g->grid_cols;
            min_x[index] = g->world_offset_x + g->grid_width * double(x);
            min_z[index] = g->world_offset_z + g->grid_height * double(y);
            max_x[index] = g->world_offset_x + g->grid_width * double(x + 1);
            max_z[index] = g->world_offset_z + g->grid_height * double(y + 1);
            channel_id[index] = g->channel_id_start + index;
            server_index[index] = (x / sgc) + (y / sgr) * g->server_cols;
        }
}

uint32_t orc_damping_interval_ms(uint32_t dist, uint32_t default_ms) {  // message_spatial.go:16-38,65-80
    static const uint32_t max_dist[3] = {0, 1, 2};
    static const uint32_t interval[3] = {20, 50, 100};
    for (int i = 0; i < 3; i++)
        if (dist <= max_dist[i]) return interval[i];
    return default_ms;
}

void orc_interest_diff(const uint32_t* existing, uint32_t n_existing, const uint32_t* wanted, uint32_t n_wanted,
                       uint32_t* unsub, uint32_t* n_unsub, uint32_t* sub_new, uint32_t* n_sub_new, uint32_t* kept,
                       uint32_t* n_kept) {
    std::map<uint32_t, int> ex, wa;
    for (uint32_t i = 0; i < n_existing; i++) ex[existing[i]] = 1;
    for (uint32_t i = 0; i < n_wanted; i++) wa[wanted[i]] = 1;
    uint32_t nu = 0, ns = 0, nk = 0;
    for (auto& kv : ex)  // util.go:105-113 Difference(existing, wanted)
        if (!wa.count(kv.first)) unsub[nu++] = kv.first;
    for (auto& kv : wa) {  // message_spatial.go:110-128 -> handleSubToChannel -> subscription.go:43-58 / :60-102
        if (ex.count(kv.first))
            kept[nk++] = kv.first;
        else
            sub_new[ns++] = kv.first;
    }
    *n_unsub = nu;
    *n_sub_new = ns;
    *n_kept = nk;
}

/* ------------------------------------------------------------------ fan-out ------ */
struct RingEl {  // data.go:46-51
    int64_t arrival;
    uint32_t sender;
    uint64_t index;
};
struct Foc {  // data.go:39-44 + the ChannelSubscription options it is looked up with (subscription.go:13-31)
    uint32_t conn;
    bool had_first;
    int64_t last;
    uint64_t last_index;
    uint32_t interval_ms;
    bool skip_self;
};
struct orc_channel {
    std::list<Foc> queue;  // ch.fanOutQueue (container/list)
    std::unordered_map<uint32_t, std::list<Foc>::iterator> subs;
    std::list<RingEl> ring;  // d.updateMsgBuffer
    uint32_t max_interval_ms = 0;
    uint64_t msg_index = 0;
};

static inline int64_t add_ms(int64_t t, int64_t ms) { return t + ms * 1000000ll; }  // channel.go:28-37

orc_channel* orc_channel_new(void) { return new orc_channel(); }
void orc_channel_free(orc_channel* c) { delete c; }

int orc_channel_subscribe(orc_channel* ch, uint32_t conn_id, int64_t now_ns, uint32_t interval_ms, int32_t delay_ms,
                          int skip_self, int skip_first) {
    auto it = ch->subs.find(conn_id);
    if (it != ch->subs.end()) {  // subscription.go:43-58: options merged, fan-out state untouched
        it->second->interval_ms = interval_ms;
        it->second->skip_self = skip_self != 0;
        return 1;
    }
    Foc f;
    f.conn = conn_id;
    f.had_first = skip_first != 0;          // subscription.go:72
    f.last = add_ms(now_ns, delay_ms);      // subscription.go:74
    f.last_index = 0;
    f.interval_ms = interval_ms;
    f.skip_self = skip_self != 0;
    ch->queue.push_front(f);                // subscription.go:70
    ch->subs[conn_id] = ch->queue.begin();
    if (ch->max_interval_ms < interval_ms) ch->max_interval_ms = interval_ms;  // subscription.go:84-86
    return 0;
}

int orc_channel_unsubscribe(orc_channel* ch, uint32_t conn_id) {  // subscription.go:104-125
    auto it = ch->subs.find(conn_id);
    if (it == ch->subs.end()) return 1;
    ch->queue.erase(it->second);
    ch->subs.erase(it);
    return 0;
}

void orc_channel_on_update(orc_channel* ch, int64_t arrival_ns, uint32_t sender) {  // data.go:149-173
    ch->msg_index++;
    ch->ring.push_back(RingEl{arrival_ns, sender, ch->msg_index});
    if (ch->ring.size() > 512) {  // MaxUpdateMsgBufferSize, data.go:53-55,166-172
        if (add_ms(ch->ring.front().arrival, ch->max_interval_ms) < arrival_ns) ch->ring.pop_front();
    }
}

uint32_t orc_channel_ring_len(const orc_channel* ch) { return uint32_t(ch->ring.size()); }

uint32_t orc_channel_tick_data(orc_channel* ch, int64_t t, orc_send* out, uint32_t cap) {
    return orc_channel_tick_data_ex(ch, t, out, cap, nullptr, nullptr, nullptr, nullptr, 0);
}

uint32_t orc_channel_tick_data_ex(orc_channel* ch, int64_t t, orc_send* out, uint32_t cap, int64_t* window_lo, uint32_t* self_skipped,
                                  uint32_t* sel_off, uint32_t* sel_pos, uint32_t sel_cap) {  // data.go:175-291
    uint32_t n_out = 0;
    uint32_t n_sel = 0;
    if (sel_off) sel_off[0] = 0;
    uint64_t guard = 0;
    auto focp = ch->queue.begin();
    while (focp != ch->queue.end()) {
        if (++guard > (1ull << 22)) return uint32_t(-1);
        Foc& foc = *focp;
        const int64_t next = add_ms(foc.last, foc.interval_ms);  // data.go:205
        if (t >= next) {
            int64_t latest = next;
            int64_t last_update_time = 0;
            bool merged = false;
            if (!foc.had_first) {  // data.go:218-224
                if (n_out >= cap) return uint32_t(-1);
                foc.had_first = true;
                foc.last_index = ch->msg_index;
                latest = t;
                if (window_lo) window_lo[n_out] = foc.last;
                if (self_skipped) self_skipped[n_out] = 0;
                out[n_out++] = orc_send{foc.conn, 0u, 0u, 0u, 0u, 0ull, foc.last_index, next};
                if (sel_off) sel_off[n_out] = n_sel;
            } else if (!ch->ring.empty()) {  // data.go:225-265
                if (foc.last >= last_update_time) last_update_time = foc.last;
                orc_send s{foc.conn, 1u, 0u, 0u, 0u, 0ull, 0ull, next};
                uint32_t pos = 0, skipped = 0;
                const uint32_t sel_begin = n_sel;
                for (auto& be : ch->ring) {
                    const uint32_t p = pos++;
                    if (be.sender == foc.conn && foc.skip_self) {
                        if (be.arrival >= last_update_time && be.arrival <= next) skipped++;  // would have been merged
                        continue;
                    }
                    if (be.arrival >= last_update_time && be.arrival <= next) {
                        if (sel_pos) {
                            if (n_sel >= sel_cap) return uint32_t(-1);
                            sel_pos[n_sel] = p;
                        }
                        n_sel++;
                        if (!merged) s.first_sel = p;
                        merged = true;
                        s.last_sel = p;
                        s.n_selected++;
                        s.sel_hash += be.index;
                        last_update_time = be.arrival;
                        foc.last_index = be.index;
                    }
                }
                if (merged) {
                    if (n_out >= cap) return uint32_t(-1);
                    s.last_message_index = foc.last_index;
                    if (window_lo) window_lo[n_out] = foc.last;
                    if (self_skipped) self_skipped[n_out] = skipped;
                    out[n_out++] = s;
                    if (sel_off) sel_off[n_out] = n_sel;
                } else {
                    n_sel = sel_begin;  // nothing merged: nothing sent
                }
            }
            foc.last = latest;  // data.go:268
            // data.go:270-286: walk from the back, MoveAfter the first element whose time is <= ours
            const bool had_prev = focp != ch->queue.begin();
            auto temp = had_prev ? std::prev(focp) : ch->queue.end();
            for (auto be = ch->queue.end(); be != ch->queue.begin();) {
                --be;
                if (be->last <= foc.last) {
                    if (be != focp) {  // list.MoveAfter(e, mark): no-op when e == mark
                        auto after = std::next(be);
                        ch->queue.splice(after, ch->queue, focp);  // iterators (and `subs`) stay valid
                    }
                    focp = had_prev ? std::next(temp) : ch->queue.begin();
                    break;
                }
            }
        } else {
            ++focp;
        }
    }
    return n_out;
}

int orc_channel_get_state(const orc_channel* ch, uint32_t conn_id, int64_t* last_fanout, int* had_first,
                          uint64_t* last_msg_index) {
    auto it = ch->subs.find(conn_id);
    if (it == ch->subs.end()) return 1;
    *last_fanout = it->second->last;
    *had_first = it->second->had_first ? 1 : 0;
    *last_msg_index = it->second->last_index;
    return 0;
}

void orc_channels_subscribe(orc_channel* const* ch, const uint32_t* chan, const uint32_t* conn_id, const uint32_t* interval_ms,
                            uint64_t n, int64_t now_ns, int32_t delay_ms, int skip_self, int skip_first) {
    for (uint64_t i = 0; i < n; i++) orc_channel_subscribe(ch[chan[i]], conn_id[i], now_ns, interval_ms[i], delay_ms, skip_self, skip_first);
}

void orc_channels_unsubscribe(orc_channel* const* ch, const uint32_t* chan, const uint32_t* conn_id, uint64_t n) {
    for (uint64_t i = 0; i < n; i++) orc_channel_unsubscribe(ch[chan[i]], conn_id[i]);
}

void orc_channels_on_update(orc_channel* const* ch, const uint32_t* chan, const int64_t* arrival_ns, const uint32_t* sender_conn_id,
                            uint64_t n) {
    for (uint64_t i = 0; i < n; i++) orc_channel_on_update(ch[chan[i]], arrival_ns[i], sender_conn_id[i]);
}

uint64_t orc_channels_tick_data(orc_channel* const* ch, uint32_t n_ch, int64_t t_ns, orc_send* out, uint64_t cap, uint64_t* out_off) {
    uint64_t total = 0;
    out_off[0] = 0;
    for (uint32_t c = 0; c < n_ch; c++) {
        const uint64_t room = cap - total;
        const uint32_t k = orc_channel_tick_data(ch[c], t_ns, out + total, room > 0xFFFFFFFEull ? 0xFFFFFFFEu : uint32_t(room));
        if (k == uint32_t(-1)) return uint64_t(-1);
        total += k;
        out_off[c + 1] = total;
    }
    return total;
}

uint64_t orc_channels_tick_data_ex(orc_channel* const* ch, uint32_t n_ch, int64_t t_ns, orc_send* out, uint64_t cap, uint64_t* out_off,
                                   int64_t* window_lo, uint32_t* self_skipped, uint64_t* sel_off, uint32_t* sel_pos, uint64_t sel_cap) {
    uint64_t total = 0, n_sel = 0;
    out_off[0] = 0;
    sel_off[0] = 0;
    std::vector<uint32_t> off1;  // one channel's selection offsets, relative to its first selected position
    for (uint32_t c = 0; c < n_ch; c++) {
        const uint64_t room = cap - total, sel_room = sel_cap - n_sel;
        const uint32_t r = room > 0xFFFFFFFEull ? 0xFFFFFFFEu : uint32_t(room);
        off1.resize(uint64_t(r) + 1);
        const uint32_t k = orc_channel_tick_data_ex(ch[c], t_ns, out + total, r, window_lo + total, self_skipped + total, off1.data(),
                                                    sel_pos + n_sel, sel_room > 0xFFFFFFFEull ? 0xFFFFFFFEu : uint32_t(sel_room));
        if (k == uint32_t(-1)) return uint64_t(-1);
        for (uint32_t j = 1; j <= k; j++) sel_off[total + j] = n_sel + off1[j];
        n_sel += off1[k];
        total += k;
        out_off[c + 1] = total;
    }
    return total;
}

uint64_t orc_channels_get_rings(orc_channel* const* ch, uint32_t n_ch, uint64_t* ring_off, int64_t* arrival_ns, uint32_t* sender_conn_id,
                                uint64_t* message_index, uint64_t cap, uint64_t* msg_index, uint32_t* max_interval_ms) {
    uint64_t total = 0;
    ring_off[0] = 0;
    for (uint32_t c = 0; c < n_ch; c++) {
        total += ch[c]->ring.size();
        ring_off[c + 1] = total;
        if (msg_index) msg_index[c] = ch[c]->msg_index;
        if (max_interval_ms) max_interval_ms[c] = ch[c]->max_interval_ms;
    }
    if (total > cap) return total;
    for (uint32_t c = 0; c < n_ch; c++) {
        uint64_t k = ring_off[c];
        for (const RingEl& r : ch[c]->ring) {
            if (arrival_ns) arrival_ns[k] = r.arrival;
            if (sender_conn_id) sender_conn_id[k] = r.sender;
            if (message_index) message_index[k] = r.index;
            k++;
        }
    }
    return total;
}

void orc_channels_get_state(orc_channel* const* ch, const uint32_t* chan, const uint32_t* conn_id, uint64_t n, int64_t* last_fanout,
                            uint8_t* had_first, uint64_t* last_msg_index, uint8_t* found) {
    for (uint64_t i = 0; i < n; i++) {
        int had = 0;
        found[i] = orc_channel_get_state(ch[chan[i]], conn_id[i], &last_fanout[i], &had, &last_msg_index[i]) == 0;
        had_first[i] = uint8_t(had);
    }
}

/* ------------------------------------------------------------------ visible sets ------ */
namespace {
struct CellLists {
    std::vector<uint32_t> start;   // [C+1]
    std::vector<uint32_t> sorted;  // entity indices, (cell asc, entity asc)
};
void build_cell_lists(const orc_grid* g, const double* ex, const double* ez, uint32_t n, CellLists& cl) {
    const uint32_t C = g->grid_cols * g->grid_rows;
    std::vector<uint32_t> cell(n);
    cl.start.assign(C + 1, 0);
    for (uint32_t i = 0; i < n; i++) {
        uint32_t idx;
        if (cell_index(g, ex[i], ez[i], &idx)) {
            cell[i] = idx;
            cl.start[idx + 1]++;
        } else
            cell[i] = 0xFFFFFFFFu;
    }
    for (uint32_t c = 0; c < C; c++) cl.start[c + 1] += cl.start[c];
    cl.sorted.resize(cl.start[C]);
    std::vector<uint32_t> cur(cl.start.begin(), cl.start.end() - 1);
    for (uint32_t i = 0; i < n; i++)
        if (cell[i] != 0xFFFFFFFFu) cl.sorted[cur[cell[i]]++] = i;
}
}  // namespace

int orc_sphere_tick(const orc_grid* g, const double* ex, const double* ez, uint32_t n_ent, const double* cx,
                    const double* cz, const double* r, uint32_t nq, uint32_t* status, uint64_t* pair_off,
                    uint32_t* pair_cell, uint32_t* pair_dist, uint64_t pair_cap, uint64_t* vis_off, uint32_t* vis_entity,
                    uint64_t vis_cap, int n_threads) {
    (void)n_threads;
    CellLists cl;
    build_cell_lists(g, ex, ez, n_ent, cl);
    uint64_t np = 0, nv = 0;
    int rc = ORC_OK;
    for (uint32_t s = 0; s < nq; s++) {
        pair_off[s] = np;
        vis_off[s] = nv;
        orc_query q;
        std::memset(&q, 0, sizeof(q));
        q.kind_mask = ORC_AOI_SPHERE;
        q.sph_cx = cx[s];
        q.sph_cz = cz[s];
        q.sph_r = r[s];
        std::map<uint32_t, uint32_t> res;
        const int st = query_into(g, &q, res);
        status[s] = uint32_t(st);
        if (st != ORC_OK) continue;
        for (auto& kv : res) {
            const uint32_t c = kv.first - g->channel_id_start;
            if (pair_cell) {
                if (np >= pair_cap) rc = ORC_ERR_CAPACITY;
                else {
                    pair_cell[np] = kv.first;
                    pair_dist[np] = kv.second;
                }
            }
            np++;
            const uint32_t b = cl.start[c], e = cl.start[c + 1];
            if (vis_entity) {
                if (nv + (e - b) > vis_cap) rc = ORC_ERR_CAPACITY;
                else std::memcpy(vis_entity + nv, cl.sorted.data() + b, size_t(e - b) * 4);
            }
            nv += e - b;
        }
    }
    pair_off[nq] = np;
    vis_off[nq] = nv;
    return rc;
}

// ---- CPU baseline (bench.py cpu_baseline / --impl reference): the reference's per-query algorithm over all host threads.
// A persistent pool (workers park on a condition variable between calls) replaces the thread-per-call spawning of round 1,
// and the per-cell entity lists are built in parallel (per-thread histograms over contiguous slices + prefix + stable scatter:
// same (cell asc, entity asc) order as the serial build).  Round 1's serial build made the 128-thread figure Amdahl-bound.
namespace {
class Pool {
public:
    static Pool& get() {
        static Pool* p = new Pool();  // leaked on purpose: parked workers must never see the pool destroyed at exit
        return *p;
    }
    // runs fn(tid) for tid in [0, n) on n threads (the caller is tid 0) and waits
    void run(int n, const std::function<void(int)>& fn) {
        std::unique_lock<std::mutex> call_lock(call_mu_);  // one parallel region at a time
        grow(n - 1);
        {
            std::lock_guard<std::mutex> lk(mu_);
            fn_ = &fn;
            active_ = n - 1;
            pending_ = n - 1;
            gen_++;
        }
        cv_.notify_all();
        fn(0);
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [&] { return pending_ == 0; });
        fn_ = nullptr;
    }

private:
    void grow(int workers) {
        while ((int)th_.size() < workers) {
            const int id = (int)th_.size() + 1;
            th_.emplace_back([this, id] { loop(id); });
            th_.back().detach();
        }
    }
    void loop(int id) {
        uint64_t seen = 0;
        for (;;) {
            const std::function<void(int)>* fn = nullptr;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
                if (id <= active_) fn = fn_;
            }
            if (!fn) continue;
            (*fn)(id);
            {
                std::lock_guard<std::mutex> lk(mu_);
                if (--pending_ == 0) done_cv_.notify_one();
            }
        }
    }
    std::mutex mu_, call_mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> th_;
    const std::function<void(int)>* fn_ = nullptr;
    int active_ = 0, pending_ = 0;
    uint64_t gen_ = 0;
};

void build_cell_lists_mt(const orc_grid* g, const double* ex, const double* ez, uint32_t n, CellLists& cl, int n_threads) {
    if (n_threads <= 1 || n < 65536) {
        build_cell_lists(g, ex, ez, n, cl);
        return;
    }
    const uint32_t C = g->grid_cols * g->grid_rows;
    static std::vector<uint32_t> cell;       // reused between ticks
    static std::vector<uint32_t> hist;       // [thread][C]
    cell.resize(n);
    hist.assign(size_t(n_threads) * C, 0);
    auto slice = [&](int t, uint32_t& lo, uint32_t& hi) {
        lo = uint32_t(uint64_t(n) * uint64_t(t) / uint64_t(n_threads));
        hi = uint32_t(uint64_t(n) * uint64_t(t + 1) / uint64_t(n_threads));
    };
    Pool::get().run(n_threads, [&](int t) {
        uint32_t lo, hi;
        slice(t, lo, hi);
        uint32_t* h = hist.data() + size_t(t) * C;
        for (uint32_t i = lo; i < hi; i++) {
            uint32_t idx;
            if (cell_index(g, ex[i], ez[i], &idx)) {
                cell[i] = idx;
                h[idx]++;
            } else
                cell[i] = 0xFFFFFFFFu;
        }
    });
    cl.start.assign(C + 1, 0);
    uint32_t run = 0;
    for (uint32_t c = 0; c < C; c++) {  // exclusive offsets in (cell, thread) order = stable
        cl.start[c] = run;
        for (int t = 0; t < n_threads; t++) {
            const uint32_t v = hist[size_t(t) * C + c];
            hist[size_t(t) * C + c] = run;
            run += v;
        }
    }
    cl.start[C] = run;
    cl.sorted.resize(run);
    Pool::get().run(n_threads, [&](int t) {
        uint32_t lo, hi;
        slice(t, lo, hi);
        uint32_t* h = hist.data() + size_t(t) * C;
        for (uint32_t i = lo; i < hi; i++)
            if (cell[i] != 0xFFFFFFFFu) cl.sorted[h[cell[i]]++] = i;
    });
}
}  // namespace

uint64_t orc_baseline_run(const orc_grid* g, const double* ex, const double* ez, uint32_t n_ent, const double* cx,
                          const double* cz, const double* r, uint32_t q_begin, uint32_t q_end, int n_threads, int build) {
    static CellLists cached;
    static uint32_t cached_n = 0;
    if (n_threads < 1) n_threads = 1;
    if (build || cached_n != n_ent) {
        if (build == 2) build_cell_lists(g, ex, ez, n_ent, cached);  // round-1 behaviour (serial build), kept for comparison
        else build_cell_lists_mt(g, ex, ez, n_ent, cached, n_threads);
        cached_n = n_ent;
    }
    const CellLists& cl = cached;
    std::vector<uint64_t> sums(size_t(n_threads), 0);
    auto work = [&](int tid) {
        std::vector<uint32_t> scratch;
        uint64_t acc = 0;
        const uint64_t total = q_end - q_begin;
        const uint32_t lo = q_begin + uint32_t(total * uint64_t(tid) / uint64_t(n_threads));
        const uint32_t hi = q_begin + uint32_t(total * uint64_t(tid + 1) / uint64_t(n_threads));
        for (uint32_t s = lo; s < hi; s++) {
            orc_query q;
            std::memset(&q, 0, sizeof(q));
            q.kind_mask = ORC_AOI_SPHERE;
            q.sph_cx = cx[s];
            q.sph_cz = cz[s];
            q.sph_r = r[s];
            std::unordered_map<uint32_t, uint32_t> res;  // per-call map allocation kept, as in Go (spatial.go:187)
            if (query_into(g, &q, res) != ORC_OK) continue;
            scratch.clear();
            for (auto& kv : res) {
                const uint32_t c = kv.first - g->channel_id_start;
                scratch.insert(scratch.end(), cl.sorted.begin() + cl.start[c], cl.sorted.begin() + cl.start[c + 1]);
                acc += kv.second;
            }
            acc += scratch.size() + res.size();
            if (!scratch.empty()) acc += scratch[scratch.size() / 2] & 1u;
        }
        sums[size_t(tid)] = acc;
    };
    Pool::get().run(n_threads, work);
    uint64_t total = 0;
    for (auto v : sums) total += v;
    return total;
}

/* ------------------------------------------------------------------ visible-set deltas ------ */
namespace {
struct DeltaState {
    const uint32_t* cell;
    uint32_t n;
    const uint64_t* pair_off;
    const uint32_t* pair_cell;
    uint32_t slots;
    std::vector<uint32_t> start, members;  // the state's entities by cell (cell asc, entity asc)

    uint32_t cell_of(uint32_t e, uint32_t cells) const { return e < n && cell[e] < cells ? cell[e] : cells; }
    void build(uint32_t cells) {
        start.assign(size_t(cells) + 1, 0);
        for (uint32_t e = 0; e < n; e++)
            if (cell[e] < cells) start[cell[e] + 1]++;
        for (uint32_t c = 0; c < cells; c++) start[c + 1] += start[c];
        members.resize(start[cells]);
        std::vector<uint32_t> cur(start.begin(), start.end() - 1);
        for (uint32_t e = 0; e < n; e++)
            if (cell[e] < cells) members[cur[cell[e]]++] = e;
    }
    // slot s's cells, ascending (a slot at or above the state's slot count has none)
    void slot_cells(uint32_t s, uint32_t cells, std::vector<uint32_t>& out) const {
        out.clear();
        if (s < slots)
            for (uint64_t k = pair_off[s]; k < pair_off[s + 1]; k++)
                if (pair_cell[k] < cells) out.push_back(pair_cell[k]);
        std::sort(out.begin(), out.end());
        out.erase(std::unique(out.begin(), out.end()), out.end());
    }
};

// the members of the cells `from` in state a whose cell in state b is not marked; counts them, and stores them from out on
uint64_t delta_side(const DeltaState& a, const std::vector<uint32_t>& from, const DeltaState& b, const std::vector<uint8_t>& mark_b,
                    uint32_t cells, uint32_t* out) {
    uint64_t k = 0;
    for (uint32_t c : from)
        for (uint32_t j = a.start[c]; j < a.start[c + 1]; j++) {
            const uint32_t e = a.members[j];
            const uint32_t cb = b.cell_of(e, cells);
            if (cb < cells && mark_b[cb]) continue;
            if (out) out[k] = e;
            k++;
        }
    return k;
}
}  // namespace

int orc_visible_delta(uint32_t cells, const uint32_t* prev_cell, uint32_t prev_n, const uint64_t* prev_pair_off, const uint32_t* prev_pair_cell,
                      uint32_t prev_slots, const uint32_t* now_cell, uint32_t now_n, const uint64_t* now_pair_off, const uint32_t* now_pair_cell,
                      uint32_t now_slots, uint64_t* enter_off, uint32_t* enter, uint64_t enter_cap, uint64_t* leave_off, uint32_t* leave,
                      uint64_t leave_cap, int n_threads) {
    if (n_threads < 1) n_threads = 1;
    DeltaState prev{prev_cell, prev_n, prev_pair_off, prev_pair_cell, prev_slots, {}, {}};
    DeltaState now{now_cell, now_n, now_pair_off, now_pair_cell, now_slots, {}, {}};
    prev.build(cells);
    now.build(cells);
    const uint32_t n_out = std::max(prev_slots, now_slots);
    // pass 1 counts (into the offsets, shifted by one); pass 2 writes at the scanned offsets
    auto pass = [&](bool write) {
        Pool::get().run(n_threads, [&](int t) {
            const uint32_t lo = uint32_t(uint64_t(n_out) * uint64_t(t) / uint64_t(n_threads));
            const uint32_t hi = uint32_t(uint64_t(n_out) * uint64_t(t + 1) / uint64_t(n_threads));
            std::vector<uint8_t> mark_p(cells, 0), mark_q(cells, 0);
            std::vector<uint32_t> P, Q;
            for (uint32_t s = lo; s < hi; s++) {
                prev.slot_cells(s, cells, P);
                now.slot_cells(s, cells, Q);
                for (uint32_t c : P) mark_p[c] = 1;
                for (uint32_t c : Q) mark_q[c] = 1;
                const uint64_t ne = delta_side(now, Q, prev, mark_p, cells, write && enter ? enter + enter_off[s] : nullptr);
                const uint64_t nl = delta_side(prev, P, now, mark_q, cells, write && leave ? leave + leave_off[s] : nullptr);
                if (!write) {
                    enter_off[s + 1] = ne;
                    leave_off[s + 1] = nl;
                }
                for (uint32_t c : P) mark_p[c] = 0;
                for (uint32_t c : Q) mark_q[c] = 0;
            }
        });
    };
    pass(false);
    enter_off[0] = leave_off[0] = 0;
    for (uint32_t s = 0; s < n_out; s++) {
        enter_off[s + 1] += enter_off[s];
        leave_off[s + 1] += leave_off[s];
    }
    if ((enter && enter_off[n_out] > enter_cap) || (leave && leave_off[n_out] > leave_cap)) return ORC_ERR_CAPACITY;
    if (enter || leave) pass(true);
    return ORC_OK;
}

/* ------------------------------------------------------------------ batched QueryChannelIds ------ */
int orc_query_batch(const orc_grid* g, const orc_query_soa* b, uint32_t* status, uint64_t* out_off, uint32_t* out_ids,
                    uint32_t* out_dists, uint64_t cap, int n_threads) {
    const uint32_t n = b->n;
    const auto has = [](std::initializer_list<const void*> ps) {
        for (const void* p : ps)
            if (!p) return false;
        return true;
    };
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t k = b->kind ? b->kind[i] : uint32_t(ORC_AOI_SPHERE);
        if (((k & ORC_AOI_SPOTS) && !has({b->spot_off, b->spot_x, b->spot_z})) ||
            ((k & ORC_AOI_BOX) && !has({b->box_cx, b->box_cz, b->box_ex, b->box_ez})) ||
            ((k & ORC_AOI_SPHERE) && !has({b->sph_cx, b->sph_cz, b->sph_r})) ||
            ((k & ORC_AOI_CONE) && !has({b->cone_cx, b->cone_cz, b->cone_dx, b->cone_dz, b->cone_angle, b->cone_r})))
            return ORC_ERR_NIL;
    }
    if (n_threads < 1) n_threads = 1;
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> res(n);
    std::atomic<uint32_t> next{0};
    const uint32_t chunk = 64;
    Pool::get().run(n_threads, [&](int) {
        std::map<uint32_t, uint32_t> m;
        for (uint32_t lo; (lo = next.fetch_add(chunk)) < n;) {
            for (uint32_t i = lo; i < std::min(n, lo + chunk); i++) {
                orc_query q;
                std::memset(&q, 0, sizeof(q));
                q.kind_mask = b->kind ? b->kind[i] : uint32_t(ORC_AOI_SPHERE);
                if (q.kind_mask & ORC_AOI_SPOTS) {
                    const uint32_t s0 = b->spot_off[i];
                    q.n_spots = b->spot_off[i + 1] - s0;
                    q.n_spot_dists = b->spot_ndist ? b->spot_ndist[i] : 0u;
                    if (!b->spot_dist) q.n_spot_dists = 0;  // no dists given: every spot has dist 0
                    q.spot_x = b->spot_x + s0;
                    q.spot_z = b->spot_z + s0;
                    q.spot_dist = b->spot_dist ? b->spot_dist + s0 : nullptr;
                }
                if (q.kind_mask & ORC_AOI_BOX) {
                    q.box_cx = b->box_cx[i]; q.box_cz = b->box_cz[i]; q.box_ex = b->box_ex[i]; q.box_ez = b->box_ez[i];
                }
                if (q.kind_mask & ORC_AOI_SPHERE) {
                    q.sph_cx = b->sph_cx[i]; q.sph_cz = b->sph_cz[i]; q.sph_r = b->sph_r[i];
                }
                if (q.kind_mask & ORC_AOI_CONE) {
                    q.cone_cx = b->cone_cx[i]; q.cone_cz = b->cone_cz[i]; q.cone_dx = b->cone_dx[i]; q.cone_dz = b->cone_dz[i];
                    q.cone_angle = b->cone_angle[i]; q.cone_r = b->cone_r[i];
                }
                m.clear();
                status[i] = uint32_t(query_into(g, &q, m));
                if (status[i] == ORC_OK) res[i].assign(m.begin(), m.end());
            }
        }
    });
    out_off[0] = 0;
    for (uint32_t i = 0; i < n; i++) out_off[i + 1] = out_off[i] + res[i].size();
    if (!out_ids) return ORC_OK;
    if (out_off[n] > cap) return ORC_ERR_CAPACITY;
    for (uint32_t i = 0; i < n; i++)
        for (size_t k = 0; k < res[i].size(); k++) {
            out_ids[out_off[i] + k] = res[i][k].first;
            out_dists[out_off[i] + k] = res[i][k].second;
        }
    return ORC_OK;
}

}  // extern "C"
