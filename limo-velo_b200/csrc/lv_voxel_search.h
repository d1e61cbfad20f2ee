/*
 * lv_voxel_search.h — exact 5-NN on the device map, host+device.
 *
 * Replaces KD_TREE<Point>::Nearest_Search / Search (include/ikd-Tree/ikd_Tree/ikd_Tree.cpp:
 * 426-461, 1062-1243) as LIMO-Velo uses it: k = 5, max_dist = infinity, result ascending,
 * followed by Plane's gate "5th squared distance < MAX_DIST_PLANE^2" (src/Objects/Plane.cpp:
 * 36-43).  Because every query whose 5th neighbour is not inside that radius is rejected by the
 * gate, the device search is an EXACT 5-NN restricted to the open ball of radius MAX_DIST_PLANE:
 * identical neighbour sets for every point the reference can accept, "fewer than 5" otherwise.
 *
 * Map layout: lv_voxel_map.h (hashed voxels with halo buckets, maintained incrementally).
 *
 * Search, two tiers:
 *   level 0     ONE probe finds the query's home voxel and ONE contiguous scan of its halo bucket sees every map
 *               point within Chebyshev ring 1, i.e. within the certified radius (edge + distance to the nearest
 *               face) of the query.  If the 5th best lies inside that radius the answer is exact and final (the
 *               bulk of a sweep).  lv_measure.cu runs this tier with 4 or 8 lanes per query.
 *   knn5_rings  the rest — sparse spot, or a query more than a voxel away from the map — one warp per query:
 *               every voxel whose box lies closer than the bound level 0 established (or the search radius) is
 *               visited through the 4x4x4 block occupancy masks; exact by construction.
 * No tree descent: the pointer chasing of the kd-tree becomes streaming reads, paid for with ~27x the map in HBM for
 * the halo buckets.
 */
#ifndef LV_VOXEL_SEARCH_H_
#define LV_VOXEL_SEARCH_H_

#include "lv_voxel_map.h"

#if defined(__CUDACC__)
#define LV_UNROLL_N(n) _Pragma("unroll")
#else
#define LV_UNROLL_N(n)
#endif

#ifndef LV_PROBE_COUNT
#define LV_PROBE_COUNT()      /* tuning build: counts hash probes */
#endif

namespace lv {

/* ascending top-5 kept in registers.  id = position in the scanned array (-1 = none). */
struct Top5 {
    float d0, d1, d2, d3, d4;
    int i0, i1, i2, i3, i4;
    float d5;   /* smallest squared distance seen that is NOT in the list (the 6th neighbour so far): feeds the
                 * reuse test of later evaluations (query_reusable) */
};
LV_HD void top5_init(Top5& t, float bound) {
    t.d0 = t.d1 = t.d2 = t.d3 = t.d4 = bound;
    t.i0 = t.i1 = t.i2 = t.i3 = t.i4 = -1;
    t.d5 = INFINITY;
}
/* insert if strictly better than the current 5th (ikd_Tree.cpp:1087: dist < q.top().dist);
 * equal distances keep the earlier candidate in front.                                      */
LV_HD void top5_insert(Top5& t, float d, int id) {
    if (!(d < t.d4)) { t.d5 = d < t.d5 ? d : t.d5; return; }
    t.d5 = t.d4 < t.d5 ? t.d4 : t.d5;   /* the old 5th drops out (a `bound` placeholder is >= every real candidate kept) */
    /* branch-free bubble through the sorted list: every lane of a warp executes the same selects */
    bool s;
    float td; int ti;
    s = d < t.d0; td = s ? t.d0 : d; ti = s ? t.i0 : id; t.d0 = s ? d : t.d0; t.i0 = s ? id : t.i0; d = td; id = ti;
    s = d < t.d1; td = s ? t.d1 : d; ti = s ? t.i1 : id; t.d1 = s ? d : t.d1; t.i1 = s ? id : t.i1; d = td; id = ti;
    s = d < t.d2; td = s ? t.d2 : d; ti = s ? t.i2 : id; t.d2 = s ? d : t.d2; t.i2 = s ? id : t.i2; d = td; id = ti;
    s = d < t.d3; td = s ? t.d3 : d; ti = s ? t.i3 : id; t.d3 = s ? d : t.d3; t.i3 = s ? id : t.i3; d = td; id = ti;
    t.d4 = d; t.i4 = id;   /* d < old d4 is known: whatever falls out of slot 3 (or the new value) is the new 5th */
}

/* scan `n` consecutive points starting at p; ids are base + j */
LV_HD void scan_run(const float4* p, uint32_t n, int base, float gx, float gy, float gz, Top5& t) {
    uint32_t j = 0;
    for (; j + 4 <= n; j += 4) {   /* four independent 16-byte loads in flight, then the insertions */
        const float4 q0 = load_point(p + j), q1 = load_point(p + j + 1), q2 = load_point(p + j + 2), q3 = load_point(p + j + 3);
        top5_insert(t, sq_dist(gx, gy, gz, q0.x, q0.y, q0.z), base + (int)j);
        top5_insert(t, sq_dist(gx, gy, gz, q1.x, q1.y, q1.z), base + (int)j + 1);
        top5_insert(t, sq_dist(gx, gy, gz, q2.x, q2.y, q2.z), base + (int)j + 2);
        top5_insert(t, sq_dist(gx, gy, gz, q3.x, q3.y, q3.z), base + (int)j + 3);
    }
    for (; j < n; ++j) {
        const float4 q = load_point(p + j);
        top5_insert(t, sq_dist(gx, gy, gz, q.x, q.y, q.z), base + (int)j);
    }
}

LV_HD void top5_pop(Top5& t, float bound) {
    t.d0 = t.d1; t.i0 = t.i1;
    t.d1 = t.d2; t.i1 = t.i2;
    t.d2 = t.d3; t.i2 = t.i3;
    t.d3 = t.d4; t.i3 = t.i4;
    t.d4 = bound; t.i4 = -1;
}
/* smallest distance this list still holds or has seen dropped: what a merge leaves behind */
LV_HD float top5_rest(const Top5& t) { return t.d0 < t.d5 ? t.d0 : t.d5; }

/* ---- lane groups: the rare queries level 0 cannot settle are finished by a whole warp ---------- */
struct GroupSerial {   /* host / single lane */
    enum { size = 1 };
    LV_HD static int lane() { return 0; }
    LV_HD static uint32_t bcast(uint32_t v, int src) { (void)src; return v; }
    LV_HD static void merge(Top5& loc, float bound, Top5& out) { out = loc; (void)bound; }
    LV_HD static float min_all(float v) { return v; }
};
#if defined(__CUDACC__)
template <int G>
struct GroupLanes {    /* G consecutive lanes of a warp (G = 4 or 8 per level-0 query, 32 = GroupWarp for the ring search); every lane of the WARP must call merge() */
    enum { size = G };
    __device__ __forceinline__ static int lane() { return (int)(threadIdx.x & (G - 1)); }
    __device__ __forceinline__ static uint32_t bcast(uint32_t v, int src) {
        return __shfl_sync(0xffffffffu, v, (int)((threadIdx.x & 31u) & ~(unsigned)(G - 1)) + src);
    }
    /* group-wide ascending top-5 of the union of the lanes' lists -> out (identical in all lanes) */
    __device__ __forceinline__ static void merge(Top5& loc, float bound, Top5& out) {
        const int l = lane();
        const unsigned gbase = (threadIdx.x & 31u) & ~(unsigned)(G - 1);
        float od[5];
        int oi[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) {
            float m = loc.d0;
#pragma unroll
            for (int s = 1; s < G; s <<= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, s));
            const unsigned b = (__ballot_sync(0xffffffffu, loc.d0 == m) >> gbase) & (0xffffffffu >> (32 - G));
            const int winner = __ffs(b) - 1;                       /* lowest lane on ties */
            od[k] = m;
            oi[k] = __shfl_sync(0xffffffffu, loc.i0, (int)gbase + winner);
            if (l == winner) top5_pop(loc, bound);
        }
        out.d0 = od[0]; out.d1 = od[1]; out.d2 = od[2]; out.d3 = od[3]; out.d4 = od[4];
        out.i0 = oi[0]; out.i1 = oi[1]; out.i2 = oi[2]; out.i3 = oi[3]; out.i4 = oi[4];
        out.d5 = min_all(top5_rest(loc));   /* heads left after five extractions, and what the lanes dropped earlier */
    }
    __device__ __forceinline__ static float min_all(float v) {
#pragma unroll
        for (int s = 1; s < G; s <<= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, s));
        return v;
    }
};
typedef GroupLanes<32> GroupWarp;
#endif

/* the query inside its home voxel: distances to the six faces, minus `slack` (a few ulp of the largest
 * coordinate: fp32 rounding of the voxel assignment floor(fl(v / ds)) / k can never make a bound optimistic) */
struct HomeGeom {
    float lo[3], hi[3];     /* distance to the low / high face per axis, >= 0 */
    float edge;
    float slack;
};
LV_HD HomeGeom home_geom(const MapGrid& grid, uint32_t bx0, uint32_t by0, uint32_t bz0, float gx, float gy, float gz) {
    HomeGeom h;
    const float c = grid.cell0;
    const uint32_t b[3] = {bx0, by0, bz0};
    const float g[3] = {gx, gy, gz};
    for (int a = 0; a < 3; ++a) {
        float v = g[a] - voxel_low(grid, b[a]);
        v = v < 0.f ? 0.f : (v > c ? c : v);
        h.lo[a] = v;
        h.hi[a] = c - v;
    }
    float amax = fabsf(gx) > fabsf(gy) ? fabsf(gx) : fabsf(gy);
    amax = amax > fabsf(gz) ? amax : fabsf(gz);
    h.edge = c;
    h.slack = 2e-6f * (amax + 4.0f);
    return h;
}
/* squared radius certified once ring 1 of the home voxel has been searched: every other map point
 * is at least edge + (distance to the nearest face) away */
LV_HD float certified_d2(const HomeGeom& h) {
    float gap = h.lo[0] < h.hi[0] ? h.lo[0] : h.hi[0];
    gap = gap < h.lo[1] ? gap : h.lo[1]; gap = gap < h.hi[1] ? gap : h.hi[1];
    gap = gap < h.lo[2] ? gap : h.lo[2]; gap = gap < h.hi[2] ? gap : h.hi[2];
    float cert = h.edge + gap - h.slack;
    cert = cert > 0.f ? cert : 0.f;
    return cert * cert;
}
/* squared distance from the query to the voxel at offset (dx, dy, dz) from its home voxel, rounded down */
LV_HD float voxel_box_d2(const HomeGeom& h, int dx, int dy, int dz) {
    const int d[3] = {dx, dy, dz};
    float s = 0.f;
    for (int a = 0; a < 3; ++a) {
        float v = d[a] < 0 ? h.lo[a] + (float)(-d[a] - 1) * h.edge : (d[a] > 0 ? h.hi[a] + (float)(d[a] - 1) * h.edge : 0.f);
        v = d[a] == 0 ? 0.f : v - h.slack * (float)(d[a] < 0 ? -d[a] : d[a]);
        v = v > 0.f ? v : 0.f;
        s += v * v;
    }
    return s;
}

/*
 * Level 0 in two steps so that a thread block can put ALL its probes and bucket fetches in flight
 * before anything waits on them.
 *   level0_probe   ONE hash probe -> the halo bucket (start, count) of the query's home voxel.
 *                  Slots exist for every occupied voxel AND for every empty voxel adjacent to one, so a query only
 *                  misses here when it is farther than one voxel from all map points (returns -1).
 *   level0_scan    one GROUP of lanes per query: ONE contiguous scan + one merge.  Returns true when `out`
 *                  (identical in all lanes of the group) is final, i.e. certified exact.  `active` = the group has a
 *                  query with a bucket; inactive groups only take part in the collectives.
 * Ids are positions in the arena.
 */
LV_HD int level0_probe(const VoxelMapView& m, float gx, float gy, float gz, uint32_t* bstart, uint32_t* bcount, uint32_t* vox = nullptr) {
    const uint32_t bx0 = voxel_coord(m.grid, gx), by0 = voxel_coord(m.grid, gy), bz0 = voxel_coord(m.grid, gz);
    if (vox) { vox[0] = bx0; vox[1] = by0; vox[2] = bz0; }    /* three IEEE divisions: callers hand them on to level0_scan */
    const int slot = voxel_find(m, voxel_key(bx0, by0, bz0));
    *bstart = 0;
    *bcount = 0;
    if (slot < 0) return -1;
    const uint4 b = load_slot(m.table + 2 * (size_t)slot + 1);
    *bstart = b.x;
    *bcount = b.y;
    return slot;
}
LV_HD float level0_certified(const VoxelMapView& m, float gx, float gy, float gz) {
    const uint32_t bx0 = voxel_coord(m.grid, gx), by0 = voxel_coord(m.grid, gy), bz0 = voxel_coord(m.grid, gz);
    return certified_d2(home_geom(m.grid, bx0, by0, bz0, gx, gy, gz));
}

template <class Grp>
LV_HD bool level0_scan(const VoxelMapView& m, float gx, float gy, float gz, float max_d2, uint32_t bstart, uint32_t bcount,
                       bool active, Top5& out, float* region_d2 = nullptr, const uint32_t* vox = nullptr) {
    Top5 loc;
    top5_init(loc, max_d2);
    if (active) {
        const float4* p = m.arena + bstart;
        const uint32_t n = bcount, step = (uint32_t)Grp::size;
        uint32_t j = (uint32_t)Grp::lane();
        if (Grp::size <= 4) {                        /* few lanes per query: eight loads in flight per lane, or a 36-point bucket is three round trips */
            for (; j + 7 * step < n; j += 8 * step) {
                float4 q[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) q[u] = load_point(p + j + (uint32_t)u * step);
#pragma unroll
                for (int u = 0; u < 8; ++u) top5_insert(loc, sq_dist(gx, gy, gz, q[u].x, q[u].y, q[u].z), (int)(bstart + j + (uint32_t)u * step));
            }
        }
        for (; j + 3 * step < n; j += 4 * step) {   /* four independent 16-byte loads in flight per lane */
            const float4 q0 = load_point(p + j), q1 = load_point(p + j + step), q2 = load_point(p + j + 2 * step),
                         q3 = load_point(p + j + 3 * step);
            top5_insert(loc, sq_dist(gx, gy, gz, q0.x, q0.y, q0.z), (int)(bstart + j));
            top5_insert(loc, sq_dist(gx, gy, gz, q1.x, q1.y, q1.z), (int)(bstart + j + step));
            top5_insert(loc, sq_dist(gx, gy, gz, q2.x, q2.y, q2.z), (int)(bstart + j + 2 * step));
            top5_insert(loc, sq_dist(gx, gy, gz, q3.x, q3.y, q3.z), (int)(bstart + j + 3 * step));
        }
        for (; j < n; j += step) {
            const float4 q = load_point(p + j);
            top5_insert(loc, sq_dist(gx, gy, gz, q.x, q.y, q.z), (int)(bstart + j));
        }
    }
    Grp::merge(loc, max_d2, out);
    if (!active) return false;
    const float cert = vox ? certified_d2(home_geom(m.grid, vox[0], vox[1], vox[2], gx, gy, gz)) : level0_certified(m, gx, gy, gz);
    if (region_d2) *region_d2 = cert;     /* every map point outside the bucket is at least this far (squared) */
    return out.d4 <= cert;                /* out.d4 <= max_d2 always */
}

/*
 * The queries level 0 could not settle, executed by a whole warp on the device (one lane on the host).
 *   bound0  squared 5th distance level 0 found among real points (an upper bound of the answer), or max_d2 if it
 *           found fewer than 5.  Every map point that can still matter lies closer than that, so it is enough to
 *           visit the voxels whose box does: voxel offsets within r = ceil(sqrt(bound) / edge) of the home voxel,
 *           pruned by their exact box distance.  The occupied ones are found through the 4x4x4 block masks (a
 *           surface-like map occupies ~10 % of the voxels of such a region): lanes fetch the masks of up to 32 blocks
 *           at a time; then, block by block, lane c looks at child voxel c (and c + 32), probes it if it is
 *           occupied and in range, a warp scan of the counts flattens the voxels' own points into one index
 *           range that the lanes stride over with independent loads.  One merge at the end.
 */
template <class Grp>
LV_HD void knn5_rings(const VoxelMapView& m, float gx, float gy, float gz, float max_d2, float bound0, Top5& out,
                      float* region_d2 = nullptr) {
    const uint32_t bx0 = voxel_coord(m.grid, gx), by0 = voxel_coord(m.grid, gy), bz0 = voxel_coord(m.grid, gz);
    const HomeGeom h = home_geom(m.grid, bx0, by0, bz0, gx, gy, gz);
    /* strictly above bound0 so that the points level 0 saw are found again; 10 % farther than needed so that the
     * answer comes with a margin to the nearest point NOT in it: later evaluations of the same sweep reuse it while
     * the iterate moves less than that margin (query_reusable) */
    float bound = nextafterf(bound0, INFINITY);
    {
        const float wide = bound0 * 1.21f;
        bound = bound > wide ? bound : wide;
    }
    bound = bound < max_d2 ? bound : max_d2;
    if (region_d2) *region_d2 = bound;
    int r = (int)ceilf(fsqrt(bound) / h.edge * 1.0001f);
    r = r < 1 ? 1 : (r > 64 ? 64 : r);
    const int hx = (int)bx0, hy = (int)by0, hz = (int)bz0;
    Top5 loc;
    top5_init(loc, bound);
    for (int dz = -r; dz <= r; ++dz)          /* single-lane form (host shim); the device runs knn5_rings_warp below */
        for (int dy = -r; dy <= r; ++dy)
            for (int dx = -r; dx <= r; ++dx) {
                const int cx = hx + dx, cy = hy + dy, cz = hz + dz;
                if (cx < 0 || cy < 0 || cz < 0 || cx > 0x1FFFFF || cy > 0x1FFFFF || cz > 0x1FFFFF) continue;
                if (!(voxel_box_d2(h, dx, dy, dz) < bound)) continue;
                if (!((block_find(m, voxel_key((uint32_t)cx >> 2, (uint32_t)cy >> 2, (uint32_t)cz >> 2)) >> block_bit((uint32_t)cx, (uint32_t)cy, (uint32_t)cz)) & 1ull)) continue;
                const int slot = voxel_find(m, voxel_key((uint32_t)cx, (uint32_t)cy, (uint32_t)cz));
                if (slot < 0) continue;
                const uint4 e = load_slot(m.table + 2 * (size_t)slot);
                scan_run(m.arena + e.z, e.w, (int)e.z, gx, gy, gz, loc);
            }
    Grp::merge(loc, bound, out);
}

/* The bits of a 4x4x4 block (bit = x + 4 y + 16 z) whose voxel offsets (cbx + x, cby + y, cbz + z) lie in [-r, r]^3. */
LV_HD unsigned long long block_cube_mask(int cbx, int cby, int cbz, int r) {
    const int xl = -r - cbx > 0 ? -r - cbx : 0, xh = r - cbx < 3 ? r - cbx : 3;
    const int yl = -r - cby > 0 ? -r - cby : 0, yh = r - cby < 3 ? r - cby : 3;
    const int zl = -r - cbz > 0 ? -r - cbz : 0, zh = r - cbz < 3 ? r - cbz : 3;
    if (xl > xh || yl > yh || zl > zh) return 0ull;
    const uint32_t nibble = (0xFu >> (3 - xh)) & (0xFu << xl) & 0xFu;                       /* x in [xl, xh]        */
    const uint32_t rows = (0xFFFFu >> (4 * (3 - yh))) & (0xFFFFu << (4 * yl)) & 0xFFFFu;   /* y in [yl, yh], all x */
    const unsigned long long slices = (~0ull >> (16 * (3 - zh))) & (~0ull << (16 * zl));   /* z in [zl, zh]        */
    return (0x1111111111111111ull * nibble) & (0x0001000100010001ull * rows) & slices;
}

#if defined(__CUDACC__)
/*
 * knn5_rings for one WARP (same voxel set, same result as the single-lane form above), arranged so that a query costs a
 * handful of dependent memory round trips:
 *   1. the occupancy masks of all blocks overlapping the voxel range (<= 128: four per lane, kept in registers)
 *   2. every lane clips its masks to the cube of the wanted rings (block_cube_mask: no walk), walks the SET bits that remain
 *      (work proportional to the occupied voxels of the cube, not to its volume), keeps the voxels whose box lies inside the
 *      bound, and the warp compacts them into a candidate list in shared memory (count, scan, write: deterministic order)
 *   3. the candidates, 32 at a time: one slot probe per lane, a warp scan of the counts flattens their own points into
 *      one index range, the lanes stride over it with four independent loads in flight
 * A query that knows nothing yet (no bucket at level 0: bound0 = the search radius) first derives a bound from the list
 * itself (the five nearest occupied voxels hold five points), so it too visits a few dozen voxels, not the whole ball.
 */
enum { kRingBlocksPerLane = 4, kRingBlocks = 32 * kRingBlocksPerLane, kRingCands = 1024, kRingMaxR = 15 };
struct RingScratch {
    uint32_t seg_pk[kRingCands];          /* every occupied voxel of the cube: (dx + 64) | (dy + 64) << 8 | (dz + 64) << 16; then, compacted
                                             in place, the candidates of the pass                                          */
    float seg_d2[kRingCands];             /* their box distances                                                             */
    unsigned long long blk_mask[kRingBlocks];   /* occupancy of the blocks over the cube, clipped to it                      */
    uint32_t blk_incl[kRingBlocks];       /* inclusive prefix of their popcounts: voxel ranks [incl - popc, incl)             */
    uint32_t blk_pk[kRingBlocks];         /* packed offset of the block's first voxel (same packing as seg_pk)                */
    float axis_d2[3][2 * kRingMaxR + 1];  /* squared per-axis part of the box distance for offsets -r .. r                    */
};
__device__ __forceinline__ void rings_process_candidates(const VoxelMapView& m, const uint32_t* cand, uint32_t n_cand, int hx, int hy, int hz,
                                                         float gx, float gy, float gz, Top5& loc) {
    const int lane = (int)(threadIdx.x & 31u);
    for (uint32_t c0 = 0; c0 < n_cand; c0 += 32) {
        uint32_t s = 0, cnt = 0;
        if (c0 + (uint32_t)lane < n_cand) {
            const uint32_t pk = cand[c0 + lane];
            const int vx = hx + (int)(pk & 0xFFu) - 64, vy = hy + (int)((pk >> 8) & 0xFFu) - 64, vz = hz + (int)((pk >> 16) & 0xFFu) - 64;
            const int slot = voxel_find(m, voxel_key((uint32_t)vx, (uint32_t)vy, (uint32_t)vz));
            if (slot >= 0) { const uint4 e = load_slot(m.table + 2 * (size_t)slot); s = e.z; cnt = e.w; }
        }
        uint32_t incl = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        const uint32_t excl = incl - cnt;
        for (uint32_t j0 = 0; j0 < total; j0 += 128) {           /* four independent loads in flight per lane */
            uint32_t idx[4];
            bool ok[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t j = j0 + 32u * (uint32_t)u + (uint32_t)lane;
                ok[u] = j < total;
                int lo = 0;                                      /* first voxel whose inclusive prefix exceeds j */
#pragma unroll
                for (int step = 16; step > 0; step >>= 1) {
                    const uint32_t v = __shfl_sync(0xffffffffu, incl, lo + step - 1);
                    if (v <= j) lo += step;
                }
                lo = lo > 31 ? 31 : lo;
                const uint32_t sv = __shfl_sync(0xffffffffu, s, lo), ev = __shfl_sync(0xffffffffu, excl, lo);
                idx[u] = sv + (j - ev);
            }
            float4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) q[u] = ok[u] ? load_point(m.arena + idx[u]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (ok[u]) top5_insert(loc, sq_dist(gx, gy, gz, q[u].x, q[u].y, q[u].z), (int)idx[u]);
        }
    }
}
__device__ __forceinline__ void broadcast_top5(Top5& t, int src) {
    t.d0 = __shfl_sync(0xffffffffu, t.d0, src); t.d1 = __shfl_sync(0xffffffffu, t.d1, src); t.d2 = __shfl_sync(0xffffffffu, t.d2, src);
    t.d3 = __shfl_sync(0xffffffffu, t.d3, src); t.d4 = __shfl_sync(0xffffffffu, t.d4, src); t.d5 = __shfl_sync(0xffffffffu, t.d5, src);
    t.i0 = __shfl_sync(0xffffffffu, t.i0, src); t.i1 = __shfl_sync(0xffffffffu, t.i1, src); t.i2 = __shfl_sync(0xffffffffu, t.i2, src);
    t.i3 = __shfl_sync(0xffffffffu, t.i3, src); t.i4 = __shfl_sync(0xffffffffu, t.i4, src);
}
__device__ __forceinline__ void knn5_rings_warp(const VoxelMapView& m, float gx, float gy, float gz, float max_d2, float bound0, Top5& out,
                                                float* region_d2, RingScratch* sm) {
    const uint32_t bx0 = voxel_coord(m.grid, gx), by0 = voxel_coord(m.grid, gy), bz0 = voxel_coord(m.grid, gz);
    const HomeGeom h = home_geom(m.grid, bx0, by0, bz0, gx, gy, gz);
    float bound = nextafterf(bound0, INFINITY);
    {
        const float wide = bound0 * 1.21f;
        bound = bound > wide ? bound : wide;
    }
    bound = bound < max_d2 ? bound : max_d2;
    int r = (int)ceilf(fsqrt(bound) / h.edge * 1.0001f);
    r = r < 1 ? 1 : (r > 63 ? 63 : r);
    const int hx = (int)bx0, hy = (int)by0, hz = (int)bz0;
    const int lane = (int)(threadIdx.x & 31u);
    const int vx0 = hx - r < 0 ? 0 : hx - r, vx1 = hx + r > 0x1FFFFF ? 0x1FFFFF : hx + r;
    const int vy0 = hy - r < 0 ? 0 : hy - r, vy1 = hy + r > 0x1FFFFF ? 0x1FFFFF : hy + r;
    const int vz0 = hz - r < 0 ? 0 : hz - r, vz1 = hz + r > 0x1FFFFF ? 0x1FFFFF : hz + r;
    const int x0 = vx0 >> 2, y0 = vy0 >> 2, z0 = vz0 >> 2;
    const int nx = (vx1 >> 2) - x0 + 1, ny = (vy1 >> 2) - y0 + 1, nz = (vz1 >> 2) - z0 + 1;
    const int nb = nx * ny * nz;
    if (nb > 32 * kRingBlocksPerLane || r > kRingMaxR) {   /* a range no 2 m search produces: the single-lane form, on lane 0 */
        Top5 t1;
        top5_init(t1, bound);
        float reg = bound;
        if (lane == 0) knn5_rings<GroupSerial>(m, gx, gy, gz, max_d2, bound0, t1, &reg);
        broadcast_top5(t1, 0);
        out = t1;
        if (region_d2) *region_d2 = __shfl_sync(0xffffffffu, reg, 0);
        return;
    }
    /* 1. block masks */
    unsigned long long mk[kRingBlocksPerLane];
    int cb[kRingBlocksPerLane][3];       /* voxel offset of each block's first voxel from the home voxel */
    {
        /* block index -> (ix, iy, iz) with two reciprocal multiplies (exact for indices < 2^16 / n; the index is < 128):
         * runtime integer divisions were a third of this kernel's instructions */
        const uint32_t inv_nx = (65536u + (uint32_t)nx - 1u) / (uint32_t)nx, inv_ny = (65536u + (uint32_t)ny - 1u) / (uint32_t)ny;
        /* the first probe of all four lookups in flight together (a probe is a dependent round trip; the table is sparse,
         * so the first slot nearly always decides); block_find() finishes the rare collision */
        uint64_t key[kRingBlocksPerLane];
        uint4 e[kRingBlocksPerLane];
#pragma unroll
        for (int u = 0; u < kRingBlocksPerLane; ++u) {
            const uint32_t bi = (uint32_t)(lane + 32 * u);
            const uint32_t t = (bi * inv_nx) >> 16, ix = bi - t * (uint32_t)nx;
            const uint32_t iz = (t * inv_ny) >> 16, iy = t - iz * (uint32_t)ny;
            cb[u][0] = (x0 + (int)ix) * 4 - hx; cb[u][1] = (y0 + (int)iy) * 4 - hy; cb[u][2] = (z0 + (int)iz) * 4 - hz;
            key[u] = voxel_key((uint32_t)(x0 + (int)ix), (uint32_t)(y0 + (int)iy), (uint32_t)(z0 + (int)iz));
            e[u] = (int)bi < nb ? load_slot(m.btable + (size_t)((voxel_hash(key[u]) * 0x9E3779B1u) & m.bmask)) : make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
        }
#pragma unroll
        for (int u = 0; u < kRingBlocksPerLane; ++u) {
            if (e[u].x == (uint32_t)key[u] && e[u].y == (uint32_t)(key[u] >> 32)) mk[u] = (uint64_t)e[u].z | ((uint64_t)e[u].w << 32);
            else if ((e[u].x & e[u].y) == 0xFFFFFFFFu) mk[u] = 0ull;
            else mk[u] = block_find(m, key[u]);
        }
    }
    /* per-axis parts of the box distance (voxel_box_d2, one table entry per offset) */
    if (lane <= 2 * r) {                  /* 2 r + 1 <= 31 offsets per axis: one lane each */
        const int d = lane - r;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            float v = d < 0 ? h.lo[a] + (float)(-d - 1) * h.edge : (d > 0 ? h.hi[a] + (float)(d - 1) * h.edge : 0.f);
            v = d == 0 ? 0.f : v - h.slack * (float)(d < 0 ? -d : d);
            v = v > 0.f ? v : 0.f;
            sm->axis_d2[a][lane] = v * v;
        }
    }
    __syncwarp();
    /* 2. the occupied voxels of the cube with their box distances, as ONE dense list in block order.  The masks are clipped
     * to the cube (no walk), their popcounts scanned, and the voxel RANKS are dealt out evenly: lane j lists ranks
     * [j * per, (j + 1) * per) whichever blocks they fall in — a dense block no longer makes one lane walk 64 bits while the
     * others wait.  The list order (block, bit) is fixed, so the result does not depend on the dealing. */
    uint32_t n_list = 0;
    {
        uint32_t mine = 0, pc[kRingBlocksPerLane];
#pragma unroll
        for (int u = 0; u < kRingBlocksPerLane; ++u) {
            const int cbx = cb[u][0], cby = cb[u][1], cbz = cb[u][2];
            mk[u] &= block_cube_mask(cbx, cby, cbz, r);
            pc[u] = (uint32_t)__popcll(mk[u]);
            mine += pc[u];
            sm->blk_mask[kRingBlocksPerLane * lane + u] = mk[u];
            /* offsets of a clipped-away block may fall outside the 8-bit fields; its mask is 0 and it is never decoded */
            sm->blk_pk[kRingBlocksPerLane * lane + u] = (uint32_t)(cbx + 64) | ((uint32_t)(cby + 64) << 8) | ((uint32_t)(cbz + 64) << 16);
        }
        uint32_t incl = mine;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += v;
        }
        n_list = __shfl_sync(0xffffffffu, incl, 31);
        uint32_t run = incl - mine;
#pragma unroll
        for (int u = 0; u < kRingBlocksPerLane; ++u) {
            run += pc[u];
            sm->blk_incl[kRingBlocksPerLane * lane + u] = run;
        }
        __syncwarp();
        if (n_list <= (uint32_t)kRingCands && n_list > 0) {
            const uint32_t per = (n_list + 31u) >> 5;
            uint32_t rank = per * (uint32_t)lane;
            const uint32_t stop = rank + per < n_list ? rank + per : n_list;
            if (rank < stop) {
                int b = 0;                                      /* first block whose inclusive prefix exceeds rank */
#pragma unroll
                for (int step = kRingBlocks / 2; step > 0; step >>= 1)
                    if (sm->blk_incl[b + step - 1] <= rank) b += step;
                unsigned long long mm = sm->blk_mask[b];
                uint32_t skip = rank - (sm->blk_incl[b] - (uint32_t)__popcll(mm));
                /* drop the `skip` lowest set bits: whole 16-bit slices first */
#pragma unroll
                for (int z = 0; z < 3; ++z) {
                    const uint32_t in_slice = (uint32_t)__popc((uint32_t)(mm >> (16 * z)) & 0xFFFFu);
                    if (skip >= in_slice) { skip -= in_slice; mm &= ~(0xFFFFull << (16 * z)); }   /* skip < popc(mm): bits remain above */
                    else break;
                }
                for (; skip > 0; --skip) mm &= mm - 1ull;
                uint32_t base = sm->blk_pk[b];
                while (rank < stop) {
                    while (mm == 0ull) { ++b; mm = sm->blk_mask[b]; base = sm->blk_pk[b]; }
                    const int c = __ffsll((long long)mm) - 1;
                    mm &= mm - 1ull;
                    const uint32_t pk = base + (uint32_t)(c & 3) + ((uint32_t)((c >> 2) & 3) << 8) + ((uint32_t)(c >> 4) << 16);
                    const int ox = (int)(pk & 0xFFu) - 64 + r, oy = (int)((pk >> 8) & 0xFFu) - 64 + r, oz = (int)((pk >> 16) & 0xFFu) - 64 + r;
                    sm->seg_pk[rank] = pk;
                    sm->seg_d2[rank] = (sm->axis_d2[0][ox] + sm->axis_d2[1][oy]) + sm->axis_d2[2][oz];   /* == voxel_box_d2(h, dx, dy, dz) */
                    ++rank;
                }
            }
        }
    }
    __syncwarp();
    if (n_list > (uint32_t)kRingCands) {              /* more occupied voxels in range than the list holds (volumetric map, tiny voxels) */
        Top5 t1;
        top5_init(t1, bound);
        float reg = bound;
        if (lane == 0) knn5_rings<GroupSerial>(m, gx, gy, gz, max_d2, bound0, t1, &reg);
        broadcast_top5(t1, 0);
        out = t1;
        if (region_d2) *region_d2 = __shfl_sync(0xffffffffu, reg, 0);
        return;
    }
    /* A query that knows nothing (no bucket at level 0: bound0 = the search radius) would have to visit every occupied voxel
     * within 2 m.  The list tells it better: every listed voxel holds at least one point, so the five voxels with the smallest
     * box distances hold five points no farther than (5th smallest box distance + the voxel diagonal) — an upper bound of the
     * 5th neighbour distance, and the only voxels that can matter are those whose box lies inside it. */
    Top5 loc;
    float first_d2 = -1.f;                /* voxels with a box distance <= first_d2 are searched first (blind queries only) */
    if (!(bound0 < max_d2)) {
        Top5 sel;
        top5_init(sel, bound);
        for (uint32_t i = (uint32_t)lane; i < n_list; i += 32) top5_insert(sel, sm->seg_d2[i], (int)i);
        Top5 s5;
        GroupWarp::merge(sel, bound, s5);
        if (s5.i4 >= 0) {
            const float reach = (fsqrt(s5.d4) + h.slack * (float)(r + 1) + 1.7320509f * h.edge) * 1.0001f;
            const float b1 = reach * reach;
            bound = b1 < bound ? b1 : bound;
            /* ... and the points of those nearest voxels give the real thing: search them first, take the 5th distance found
             * as the bound for the rest (their list lives in blk_pk, free since the walk) */
            uint32_t n_first = 0;
            for (uint32_t i0 = 0; i0 < n_list && n_first <= (uint32_t)kRingBlocks; i0 += 32) {
                const uint32_t i = i0 + (uint32_t)lane;
                const bool pick = i < n_list && sm->seg_d2[i] <= s5.d4;
                const unsigned bal = __ballot_sync(0xffffffffu, pick);
                const uint32_t at = n_first + (uint32_t)__popc(bal & ((1u << lane) - 1u));
                if (pick && at < (uint32_t)kRingBlocks) sm->blk_pk[at] = sm->seg_pk[i];
                n_first += (uint32_t)__popc(bal);
            }
            __syncwarp();
            if (n_first <= (uint32_t)kRingBlocks) {
                Top5 part, t5;
                top5_init(part, bound);
                rings_process_candidates(m, sm->blk_pk, n_first, hx, hy, hz, gx, gy, gz, part);
                GroupWarp::merge(part, bound, t5);
                if (t5.i4 >= 0) {
                    const float b2 = nextafterf(t5.d4, INFINITY);
                    bound = b2 < bound ? b2 : bound;
                }
                first_d2 = s5.d4;
                top5_init(loc, bound);
                if (lane == 0) loc = t5;                    /* the rest joins what the first voxels gave */
            }
        }
    }
    if (first_d2 < 0.f) top5_init(loc, bound);
    /* the candidates: the listed voxels inside the bound (and not searched yet), in list order */
    uint32_t total = 0;
    for (uint32_t i0 = 0; i0 < n_list; i0 += 32) {
        const uint32_t i = i0 + (uint32_t)lane;
        const float d2 = i < n_list ? sm->seg_d2[i] : INFINITY;
        const bool sel = d2 < bound && d2 > first_d2;
        const unsigned bal = __ballot_sync(0xffffffffu, sel);
        const uint32_t pk = sel ? sm->seg_pk[i] : 0u;
        __syncwarp();                                   /* in place: the slots written (<= i0 + lane) have been read */
        if (sel) sm->seg_pk[total + (uint32_t)__popc(bal & ((1u << lane) - 1u))] = pk;
        total += (uint32_t)__popc(bal);
    }
    __syncwarp();
    /* 3. probe + scan, one merge */
    rings_process_candidates(m, sm->seg_pk, total, hx, hy, hz, gx, gy, gz, loc);
    if (region_d2) *region_d2 = bound;     /* every voxel whose box lies inside the bound has been visited */
    GroupWarp::merge(loc, bound, out);
}
#endif

/*
 * The reference orders neighbours of (nearly) equal distance by x: PointType_CMP (ikd_Tree.h:109-115) compares x when
 * |dist - dist'| < 1e-10, so Nearest_Search's list is ascending in (distance, x).  Which of two equidistant points a
 * search meets first depends on how it walks the map (lanes, buckets, rings); that must not leak into the plane fit,
 * whose rounding depends on the order of its five points.  Called on the five neighbours (ascending distances) before
 * the fit.  (Seen on the bench data: one query of 65 536 in sweep 1 has its 3rd and 4th neighbour at equal distance.)
 * Points the comparator leaves unordered (equal x: mirror images about the query, duplicates) are put in (y, z, map point id)
 * order: the reference pops them in whatever order its tree walk left, so any fixed order is as faithful, and without one
 * the lane count of the search (4 or 8 per query, 32 in the ring search) would decide the plane's last bits.  `id` is the
 * map point id (insertion order), not a position in the arena.
 */
LV_HD bool neighbour_before(const float* a, int ia, const float* b, int ib) {
    if (a[0] != b[0]) return a[0] < b[0];
    if (a[1] != b[1]) return a[1] < b[1];
    if (a[2] != b[2]) return a[2] < b[2];
    return ia < ib;
}
LV_HD void canonical_neighbour_order(float (*q)[3], float* d, int* id) {
    /* ascending distances: a tie anywhere shows in one of the four adjacent gaps (a float test first: the fp64 compare of the
     * reference's comparator costs more than the rest of the function and one query in 10^5 has a tie at all) */
    const float gap = fminf(fminf(d[1] - d[0], d[2] - d[1]), fminf(d[3] - d[2], d[4] - d[3]));
    if (!(gap < 2e-10f)) return;
    /* exactly equal distances first: the search hands them over in lane order, so put them in key order before the 1e-10
     * relation (not transitive: a chain of near-ties can exceed 1e-10) is applied, and the result depends only on the set */
    for (int pass = 0; pass < 4; ++pass)
        for (int k = 0; k < 4; ++k)
            if (d[k + 1] == d[k] && neighbour_before(q[k + 1], id[k + 1], q[k], id[k])) {
                for (int a = 0; a < 3; ++a) { const float t = q[k][a]; q[k][a] = q[k + 1][a]; q[k + 1][a] = t; }
                const int ti = id[k]; id[k] = id[k + 1]; id[k + 1] = ti;
            }
    for (int pass = 0; pass < 4; ++pass)
        for (int k = 0; k < 4; ++k)
            if (fabs((double)(d[k + 1] - d[k])) < 1e-10 && neighbour_before(q[k + 1], id[k + 1], q[k], id[k])) {
                for (int a = 0; a < 3; ++a) { const float t = q[k][a]; q[k][a] = q[k + 1][a]; q[k + 1][a] = t; }
                const float td = d[k]; d[k] = d[k + 1]; d[k + 1] = td;
                const int ti = id[k]; id[k] = id[k + 1]; id[k + 1] = ti;
            }
}

/*
 * Reuse of a query's neighbours by a later evaluation of the SAME sweep (the iterate moved, the map did not).
 *   ref    (gx, gy, gz, lb): the world position the neighbours were searched from and lb, a lower bound (metres,
 *          rounded down) of the distance from there to every map point that is not one of the five
 *          (outsider_bound()).
 *   g      the query's world position now; q[k], id[k] the five stored neighbours.
 * A map point outside the five is now at least lb - |g - ref| away, so if the farthest of the five is closer
 * than that (with room for the fp32 rounding of every computed distance) the exact search would return the
 * same five: they only need their distances recomputed and their order restored.  Returns false (search
 * again) on any doubt: fewer than five, a tie among the new distances, the 5th beyond the search radius.
 */
LV_HD float outsider_bound(float d5_sq, float region_sq) {
    const float m = d5_sq < region_sq ? d5_sq : region_sq;
    const float r = fsqrt(m > 0.f ? m : 0.f);
    return r * (1.0f - 1e-6f);
}
LV_HD bool query_reusable(const float ref[4], const float g[3], const float (*q)[3], const int* id, float max_d2,
                          Top5& out) {
    if (!(ref[3] > 0.f)) return false;
    float d[5];
    int o[5];
    for (int k = 0; k < 5; ++k) {
        if (id[k] == -1) return false;
        d[k] = sq_dist(g[0], g[1], g[2], q[k][0], q[k][1], q[k][2]);
        o[k] = id[k];
    }
    /* 9-comparator sorting network for 5 keys */
#define LV_CE(a, b) { if (d[b] < d[a]) { const float td = d[a]; d[a] = d[b]; d[b] = td; const int ti = o[a]; o[a] = o[b]; o[b] = ti; } }
    LV_CE(0, 1) LV_CE(3, 4) LV_CE(2, 4) LV_CE(2, 3) LV_CE(0, 3) LV_CE(0, 2) LV_CE(1, 4) LV_CE(1, 3) LV_CE(1, 2)
#undef LV_CE
    if (d[0] == d[1] || d[1] == d[2] || d[2] == d[3] || d[3] == d[4]) return false;
    if (!(d[4] < max_d2)) return false;
    const float dx = g[0] - ref[0], dy = g[1] - ref[1], dz = g[2] - ref[2];
    const float moved = fsqrt(dx * dx + dy * dy + dz * dz);
    const float far5 = fsqrt(d[4]);
    const float need = far5 + moved + 1e-5f * (far5 + moved + ref[3]) + 1e-5f;
    if (!(need < ref[3])) return false;
    out.d0 = d[0]; out.d1 = d[1]; out.d2 = d[2]; out.d3 = d[3]; out.d4 = d[4];
    out.i0 = o[0]; out.i1 = o[1]; out.i2 = o[2]; out.i3 = o[3]; out.i4 = o[4];
    out.d5 = INFINITY;
    return true;
}

}  // namespace lv
#endif
