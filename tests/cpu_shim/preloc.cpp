/*
 * tests/cpu_shim/preloc.cpp — TEST-ONLY host build of lv_prelocalize (csrc/lv_preloc.h) and lv_prelocalize_global
 * (csrc/lv_preloc_bound.h).
 *
 * The occupancy comes from a block table this file fills itself with the map's block_mark (lv_voxel_map.h) over the map points
 * the map would store (finite, below 1e9 m), so a device score that equals this one also says that the device map's occupancy
 * bits are those of its points.
 *
 * lv_prelocalize: every candidate is scored serially with the header's functions in the kernel's order: frames per heading,
 * offsets per position, preloc_rows then preloc_hit per point, preloc_key for the winner.
 *
 * lv_prelocalize_global: the extent and the bitmap pyramid are built from the same block table serially with the header's
 * functions (occ_block_range, occ_layout, occ_bit), as the device's occ_extent and occ_bits kernels do.  The search is the
 * header's PrelocSearch with a serial evaluator in place of the device launches, so its winner and every count of its stats
 * are what the device call must report.
 *
 * Not part of the product.
 */
#include <string.h>

#include <vector>

#include "../../limo-velo_b200/csrc/lv_preloc_bound.h"

using namespace lv;

namespace {

struct HostBlocks {
    std::vector<uint4> btable;
    uint32_t counters[kMapCounters] = {};
    VoxelMapView view;
};

void build_blocks(HostBlocks& b, const float* map_xyz, int64_t m, float ds, float voxel_size) {
    MapGrid g;
    g.ds = ds;
    int k = (int)floor((double)voxel_size / (double)ds + 0.5);   /* map_alloc */
    g.k = k < 1 ? 1 : (k > kMaxCellsPerVoxel ? kMaxCellsPerVoxel : k);
    g.cell0 = (float)g.k * ds;
    uint32_t slots = 1024;
    while ((int64_t)slots < 4 * m) slots <<= 1;
    b.btable.assign(slots, uint4{0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u});
    VoxelMapRW rw;
    memset(&rw, 0, sizeof(rw));
    rw.btable = b.btable.data();
    rw.bmask = slots - 1;
    rw.counters = b.counters;
    rw.grid = g;
    for (int64_t p = 0; p < m; ++p) {
        const float x = map_xyz[3 * p], y = map_xyz[3 * p + 1], z = map_xyz[3 * p + 2];
        if (!(fabsf(x) < 1e9f && fabsf(y) < 1e9f && fabsf(z) < 1e9f)) continue;   /* map_point_key */
        block_mark(rw, voxel_coord(g, x), voxel_coord(g, y), voxel_coord(g, z));
    }
    memset(&b.view, 0, sizeof(b.view));
    b.view.btable = b.btable.data();
    b.view.bmask = slots - 1;
    b.view.grid = g;
}

/* the block table with the occupancy summary of lv_prelocalize_global */
struct HostOcc : HostBlocks {
    std::vector<uint32_t> bits;
    PrelocOcc occ;
    bool empty = true;
};

void build_occ(HostOcc& b, const float* map_xyz, int64_t m, float ds, float voxel_size) {
    build_blocks(b, map_xyz, m, ds, voxel_size);
    PrelocOcc& o = b.occ;
    memset(&o, 0, sizeof(o));
    o.map = b.view;
    for (int a = 0; a < 3; ++a) { o.lo[a] = 0xFFFFFFFFu; o.hi[a] = 0u; }
    for (const uint4& e : b.btable) {                                 /* occ_extent_kernel */
        const uint64_t mask = (uint64_t)e.z | ((uint64_t)e.w << 32);
        if ((e.x & e.y) == 0xFFFFFFFFu || !mask) continue;
        uint32_t lo[3], hi[3];
        occ_block_range((uint64_t)e.x | ((uint64_t)e.y << 32), mask, lo, hi);
        for (int a = 0; a < 3; ++a) {
            o.lo[a] = lo[a] < o.lo[a] ? lo[a] : o.lo[a];
            o.hi[a] = hi[a] > o.hi[a] ? hi[a] : o.hi[a];
        }
    }
    b.empty = o.lo[0] > o.hi[0];
    if (b.empty) return;
    b.bits.assign(occ_layout(o), 0u);
    for (const uint4& e : b.btable) {                                 /* occ_bits_kernel */
        if ((e.x & e.y) == 0xFFFFFFFFu) continue;
        const uint64_t key = (uint64_t)e.x | ((uint64_t)e.y << 32), mask = (uint64_t)e.z | ((uint64_t)e.w << 32);
        for (int v = 0; v < 64; ++v) {
            if (!((mask >> v) & 1ull)) continue;
            const uint32_t x = 4 * ((uint32_t)key & 0x1FFFFFu) + (v & 3), y = 4 * ((uint32_t)(key >> 21) & 0x1FFFFFu) + ((v >> 2) & 3),
                           z = 4 * ((uint32_t)(key >> 42) & 0x1FFFFFu) + (v >> 4);
            for (int l = o.m0; l <= o.M; ++l) {
                const uint64_t bit = occ_bit(o, l, x, y, z);
                b.bits[o.off[l] + (bit >> 5)] |= 1u << (bit & 31);
            }
        }
    }
    o.bits = b.bits.data();
}

/* the evaluator of PrelocSearch: the device kernels' work, serially */
struct HostEval {
    const PrelocOcc* occ;
    const float* xyz;
    int64_t n, S, I, K;
    float step;
    PrelocAxes ax;
    std::vector<Rt32> frames;
    std::vector<float> rows;
    void rotate(int64_t h) {
        rows.resize((size_t)S * 3);
        for (int64_t s = 0; s < S; ++s) {
            const int64_t p = preloc_point_index(s, n, S);
            preloc_rows(frames[(size_t)h], xyz[3 * p], xyz[3 * p + 1], xyz[3 * p + 2], &rows[(size_t)(3 * s)]);
        }
    }
    int32_t bound(const PrelocCell& c) {
        const Rt32& F = frames[(size_t)c.h];
        int64_t i0, i1, j0, j1;
        preloc_cell_range(c, I, &i0, &i1, &j0, &j1);
        float tlo[3], thi[3];
        preloc_cell_t(ax, F.t, step, i0, i1, j0, j1, tlo, thi);
        rotate(c.h);
        int32_t b = 0;
        for (int64_t s = 0; s < S; ++s) b += preloc_bound_point(*occ, &rows[(size_t)(3 * s)], tlo, thi);
        return b;
    }
    void bounds(const PrelocCell* c, int64_t cnt, int32_t* out) {
        for (int64_t t = 0; t < cnt; ++t) out[t] = bound(c[t]);
    }
    void exact(const PrelocCell* c, int64_t cnt, PrelocBest* out) {
        for (int64_t t = 0; t < cnt; ++t) {
            const Rt32& F = frames[(size_t)c[t].h];
            rotate(c[t].h);
            int64_t i0, i1, j0, j1;
            preloc_cell_range(c[t], I, &i0, &i1, &j0, &j1);
            PrelocBest best;
            best.score = -1; best.pad_ = 0; best.tie = 0; best.idx = 0;
            for (int64_t i = i0; i <= i1; ++i)
                for (int64_t j = j0; j <= j1; ++j) {
                    float o[3];
                    preloc_offset(ax, dmul((double)i, (double)step), dmul((double)j, (double)step), o);
                    const float tt[3] = {fadd(F.t[0], o[0]), fadd(F.t[1], o[1]), fadd(F.t[2], o[2])};
                    int32_t score = 0;
                    for (int64_t s = 0; s < S; ++s) score += preloc_hit(occ->map, rows[3 * s], rows[3 * s + 1], rows[3 * s + 2], tt);
                    const PrelocBest b = preloc_best_of(score, c[t].h - K, i, j, I, K);
                    if (preloc_better(b, best)) best = b;
                }
            out[t] = best;
        }
    }
};

void setup(HostEval& ev, const PrelocOcc& occ, const double* x, const float* xyz, int64_t n, int64_t S, int64_t I, int64_t K, float step,
           float yaw_step) {
    ev.occ = &occ;
    ev.xyz = xyz;
    ev.n = n;
    ev.S = S;
    ev.I = I;
    ev.K = K;
    ev.step = step;
    ev.ax = preloc_axes(x);
    ev.frames.resize((size_t)(2 * K + 1));
    for (int64_t k = -K; k <= K; ++k) ev.frames[(size_t)(k + K)] = preloc_heading_frame(x, ev.ax, (double)k * (double)yaw_step);
}

}  // namespace

extern "C" {

/* ---- lv_prelocalize ---------------------------------------------------------------------------------------------------------- */

/* every candidate's score into scores ((2K+1)(2I+1)^2, linear index order); returns the winner's linear index (-1 for a
 * window of more than 2^24 candidates); frames (2K+1 x 12) and offsets ((2I+1)^2 x 3) may be NULL */
int64_t shim_preloc_scores(const double* x, const float* xyz, int64_t n, const float* map_xyz, int64_t m, float ds, float voxel_size,
                           float radius, float step, float yaw_range, float yaw_step, int32_t max_points, int32_t* scores, float* frames,
                           float* offsets) {
    HostBlocks blk;
    build_blocks(blk, map_xyz, m, ds, voxel_size);
    const int64_t I = (int64_t)preloc_half(radius, step), K = (int64_t)preloc_half(yaw_range, yaw_step);
    const int64_t W = 2 * I + 1, P = W * W, H = 2 * K + 1;
    if (H * P > LV_PRELOC_MAX_CANDIDATES) return -1;
    const int64_t S = n < max_points ? n : max_points;
    const PrelocAxes ax = preloc_axes(x);
    std::vector<float> off((size_t)P * 3);
    for (int64_t i = -I; i <= I; ++i)
        for (int64_t j = -I; j <= I; ++j) preloc_offset(ax, (double)i * (double)step, (double)j * (double)step, &off[(size_t)(((i + I) * W + (j + I)) * 3)]);
    if (offsets) memcpy(offsets, off.data(), sizeof(float) * off.size());
    std::vector<float> rows((size_t)S * 3);
    uint64_t best = 0;
    for (int64_t h = 0; h < H; ++h) {
        const Rt32 F = preloc_heading_frame(x, ax, (double)(h - K) * (double)yaw_step);
        if (frames) {
            memcpy(frames + 12 * h, F.R, sizeof(float) * 9);
            memcpy(frames + 12 * h + 9, F.t, sizeof(float) * 3);
        }
        for (int64_t s = 0; s < S; ++s) {
            const int64_t p = preloc_point_index(s, n, S);
            preloc_rows(F, xyz[3 * p], xyz[3 * p + 1], xyz[3 * p + 2], &rows[(size_t)(3 * s)]);
        }
        for (int64_t q = 0; q < P; ++q) {
            const float* o = &off[(size_t)(3 * q)];
            const float t[3] = {fadd(F.t[0], o[0]), fadd(F.t[1], o[1]), fadd(F.t[2], o[2])};
            int32_t score = 0;
            for (int64_t s = 0; s < S; ++s) score += preloc_hit(blk.view, rows[3 * s], rows[3 * s + 1], rows[3 * s + 2], t);
            const int64_t idx = h * P + q;
            if (scores) scores[idx] = score;
            const uint64_t key = preloc_key(score, h - K, q / W - I, q % W - I, I, idx);
            if (key > best) best = key;
        }
    }
    return preloc_key_index(best);
}

/* the state of candidate (k, i, j) (preloc_candidate) */
void shim_preloc_candidate(const double* x, float step, float yaw_step, int32_t k, int32_t i, int32_t j, double* out) {
    const PrelocAxes ax = preloc_axes(x);
    preloc_candidate(x, ax, (double)k * (double)yaw_step, (double)i * (double)step, (double)j * (double)step, out);
}

/* the rotation axis and the position axes (g, u, v: 9 doubles) */
void shim_preloc_axes(const double* x, double* out) {
    const PrelocAxes ax = preloc_axes(x);
    for (int c = 0; c < 3; ++c) { out[c] = ax.g[c]; out[3 + c] = ax.u[c]; out[6 + c] = ax.v[c]; }
}

/* ---- lv_prelocalize_global --------------------------------------------------------------------------------------------------- */

/* the bound of each cell (cells: nc x (h, l, ci, cj)); returns -1 for an empty map */
int shim_pg_bounds(const double* x, const float* xyz, int64_t n, const float* map_xyz, int64_t m, float ds, float voxel_size, float step,
                   float yaw_step, int64_t I, int64_t K, int64_t S, const int32_t* cells, int64_t nc, int32_t* out) {
    HostOcc occ;
    build_occ(occ, map_xyz, m, ds, voxel_size);
    if (occ.empty) return -1;
    HostEval ev;
    setup(ev, occ.occ, x, xyz, n, S, I, K, step, yaw_step);
    ev.bounds(reinterpret_cast<const PrelocCell*>(cells), nc, out);
    return 0;
}

/* the search: winner (score, tie, index) into best[3], stats (candidates, cells_bounded, candidates_scored, probes, launches)
 * into stats[5] (launches: those of the search, as the device call reports them); returns -1 for an empty map */
int shim_pg_search(const double* x, const float* xyz, int64_t n, const float* map_xyz, int64_t m, float ds, float voxel_size,
                   float radius, float step, float yaw_range, float yaw_step, int32_t max_points, int prune, int64_t* best,
                   int64_t* stats) {
    HostOcc occ;
    build_occ(occ, map_xyz, m, ds, voxel_size);
    if (occ.empty) return -1;
    const int64_t I = (int64_t)preloc_half(radius, step), K = (int64_t)preloc_half(yaw_range, yaw_step);
    const int64_t S = n < max_points ? n : max_points;
    HostEval ev;
    setup(ev, occ.occ, x, xyz, n, S, I, K, step, yaw_step);
    PrelocSearch<HostEval> search(ev, I, K, S, prune != 0);
    search.run();
    best[0] = search.best.score;
    best[1] = search.best.tie;
    best[2] = search.best.idx;
    stats[0] = search.st.candidates;
    stats[1] = search.st.cells_bounded;
    stats[2] = search.st.candidates_scored;
    stats[3] = search.st.probes;
    stats[4] = search.st.launches;
    return 0;
}

/* the occupied voxels' extent (biased voxel coordinates lo[3], hi[3]) and the bitmap levels (m0, M) */
int shim_pg_extent(const float* map_xyz, int64_t m, float ds, float voxel_size, uint32_t* ext, int32_t* levels) {
    HostOcc occ;
    build_occ(occ, map_xyz, m, ds, voxel_size);
    if (occ.empty) return -1;
    for (int a = 0; a < 3; ++a) { ext[a] = occ.occ.lo[a]; ext[3 + a] = occ.occ.hi[a]; }
    levels[0] = occ.occ.m0;
    levels[1] = occ.occ.M;
    return 0;
}

/* the top level of a window's cells (preloc_top_level) */
int shim_pg_top_level(int64_t I, int64_t K) { return preloc_top_level(I, K); }

}  // extern "C"
