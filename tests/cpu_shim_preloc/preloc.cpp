/*
 * tests/cpu_shim_preloc/preloc.cpp — TEST-ONLY host build of lv_prelocalize's arithmetic (csrc/lv_preloc.h).
 *
 * The occupancy comes from a block table this file fills itself with the map's block_mark (lv_voxel_map.h) over the map points
 * the map would store (finite, below 1e9 m), so a device score that equals this one also says that the device map's occupancy
 * bits are those of its points.  Every candidate is scored serially with the header's functions in the kernel's order: frames
 * per heading, offsets per position, preloc_rows then preloc_hit per point, preloc_key for the winner.  Not part of the product.
 */
#include <string.h>

#include <vector>

#include "../../limo-velo_b200/csrc/lv_preloc.h"

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

}  // namespace

extern "C" {

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

}  // extern "C"
