/*
 * lv_preloc_bound.h — lv_prelocalize_global: an exact branch-and-bound form of lv_prelocalize's search, host+device.
 *
 * The search maximises the same score as lv_prelocalize (lv_preloc.h): the number of the S scored sweep points whose world
 * point lands in an occupied map voxel.  Instead of scoring every candidate it bounds the score over blocks of candidates and
 * scores exactly only the blocks whose bound can still reach the best score found.
 *
 * Cell.  One heading k together with an aligned block of positions: (i + I) in [ci 2^l, (ci + 1) 2^l), (j + I) in
 * [cj 2^l, (cj + 1) 2^l), clipped at the window's edge (2I + 1 positions per axis).  Level l = 0 is one candidate.
 *
 * Why the bound is exact.  Every step from (i, j) to a point's voxel is monotone per axis:
 *   - (double)i * step is exact; dmul by u_c is monotone (non-decreasing for u_c >= 0, non-increasing below), and dadd is
 *     monotone in each argument, so each component of the fp64 offset a_i u + b_j v is monotone in i and in j separately;
 *   - the rounding to float in preloc_offset is monotone;
 *   - fadd(F.t, o), then fadd(r, t): monotone in o, then in t;
 *   - floorf(fdiv(w, ds)), floor_div and the clamp of voxel_of_cell: monotone in w.
 * A function monotone in i and in j separately takes its extremes over a rectangle at its corners.  So over a cell, each
 * voxel coordinate of a scored point lies between its values at the cell's four corners: that per-axis range is the point's
 * VOXEL BOX, computed from the corner offsets with the same preloc_offset / fadd / voxel_coord arithmetic as preloc_hit.
 * The cell's BOUND is the number of scored points whose voxel box holds at least one occupied voxel (or a superset of that
 * test: the box test below is exact for small boxes and conservative for large ones; a conservative answer only loosens the
 * bound).  Then:
 *   - the bound is at least every candidate's exact score in the cell: a point that scores at a candidate lands in an
 *     occupied voxel inside its box;
 *   - for a single-candidate cell the box is one voxel, so the bound equals preloc_hit's score;
 *   - preloc_hit never scores a coordinate not below 1e9 in magnitude; the box is cut to that range first (a point whose
 *     range is empty there is not counted).  A point whose floor(w / ds) reaches 2^30 in magnitude (2e8 m at 0.2 m cells) is
 *     counted without a test (the integer voxel arithmetic is not monotone that far out): the bound may count it, the exact
 *     score never does.
 * The search prunes a cell only when its bound is STRICTLY below a score some candidate is known to reach, so every candidate
 * that could win, or tie the winner, is scored exactly with lv_prelocalize's own arithmetic (preloc_rows + preloc_hit) and
 * the tie rule picks the same winner.
 *
 * Box test (PrelocOcc, built per call from the block table):
 *   - a box that touches at most 2 blocks (4 x 4 x 4 voxels) per axis: the box's bits AND-ed with the 64-bit occupancy masks
 *     of those blocks (block_find): exact;
 *   - a larger box: a pyramid of dense bitmaps over the occupied voxels' extent, level m keyed (x >> m, y >> m, z) (x and y
 *     coarsened, z at voxel resolution: the position offsets lie in the plane normal to gravity, so for the usual world frame
 *     the box is wide in x and y and one or two voxels tall).  The box is cut to the extent, then tested against the at most
 *     2 x 2 coarse columns that cover it at the finest level where it fits: conservative.
 *
 * The schedule (PrelocSearch, host code shared by lv_capi.cu and tests/cpu_shim/preloc.cpp): bound every top-level cell
 * and order the cells by bound (descending, ties by cell index); find a first score by diving from the first cell through
 * the child of highest bound at each level; then take the cells in batches and descend level by level, each level's
 * survivors highest bound first, scoring the surviving level-1 cells exactly; stop when the next top cell's bound is below
 * the best score.  Every decision is taken on
 * the host between launches from values that do not depend on timing, so the counts (PrelocStats) are deterministic.
 */
#ifndef LV_PRELOC_BOUND_H_
#define LV_PRELOC_BOUND_H_

#include "lv_preloc.h"

#include <algorithm>
#include <vector>

namespace lv {

#define LV_PRELOC_GLOBAL_MAX_CANDIDATES ((int64_t)1 << 40)

enum {
    kOccLevels = 22,           /* bitmap levels m = 0 .. 21 (biased voxel coordinates have 21 bits)          */
    kPrelocTopLevel = 5,       /* top-level cells are 32 x 32 positions ...                                   */
    kPrelocMaxTopCells = 1 << 20,  /* ... or larger, so that there are at most this many                      */
    kPrelocChunk = 1 << 16,    /* cells per launch                                                            */
    kPrelocBatch = 4096        /* top-level cells per batch                                                   */
};
#define LV_OCC_MAX_BITS ((uint64_t)1 << 30)   /* the finest bitmap level holds at most this many bits (128 MB) */

/* the occupancy summary of one call */
struct PrelocOcc {
    uint32_t lo[3], hi[3];         /* biased voxel coordinates of the occupied voxels' extent (inclusive)        */
    int32_t m0, M;                 /* bitmap levels m0 .. M (m0 >= 3); at M the extent spans <= 2 columns per axis */
    uint64_t off[kOccLevels];      /* word offset of level m's bitmap                                           */
    uint32_t nx[kOccLevels], ny[kOccLevels];
    const uint32_t* bits;
    VoxelMapView map;
};

/* the voxel range of the occupied voxels of one block (key, mask != 0) */
LV_HD void occ_block_range(uint64_t key, uint64_t mask, uint32_t* lo, uint32_t* hi) {
    uint32_t xm = 0, ym = 0, zm = 0;
    for (int z = 0; z < 4; ++z) {
        const uint32_t slab = (uint32_t)(mask >> (16 * z)) & 0xFFFFu;
        if (!slab) continue;
        zm |= 1u << z;
        for (int y = 0; y < 4; ++y) {
            const uint32_t row = (slab >> (4 * y)) & 0xFu;
            if (row) { ym |= 1u << y; xm |= row; }
        }
    }
    const uint32_t b[3] = {(uint32_t)key & 0x1FFFFFu, (uint32_t)(key >> 21) & 0x1FFFFFu, (uint32_t)(key >> 42) & 0x1FFFFFu};
    const uint32_t m[3] = {xm, ym, zm};
    for (int a = 0; a < 3; ++a) {
        int l = 0, h = 3;
        while (!((m[a] >> l) & 1u)) ++l;
        while (!((m[a] >> h) & 1u)) --h;
        lo[a] = 4u * b[a] + (uint32_t)l;
        hi[a] = 4u * b[a] + (uint32_t)h;
    }
}

/* bit of voxel (x, y, z) (inside the extent) in level m's bitmap */
LV_HD uint64_t occ_bit(const PrelocOcc& o, int m, uint32_t x, uint32_t y, uint32_t z) {
    return ((uint64_t)(z - o.lo[2]) * o.ny[m] + ((y >> m) - (o.lo[1] >> m))) * o.nx[m] + ((x >> m) - (o.lo[0] >> m));
}

/* the layout of the bitmaps from the extent: levels, dimensions, word offsets; returns the words needed */
inline uint64_t occ_layout(PrelocOcc& o) {
    const uint64_t nz = o.hi[2] - o.lo[2] + 1;
    o.m0 = 3;
    for (;;) {
        const uint64_t nx = (o.hi[0] >> o.m0) - (o.lo[0] >> o.m0) + 1, ny = (o.hi[1] >> o.m0) - (o.lo[1] >> o.m0) + 1;
        if (nx * ny * nz <= LV_OCC_MAX_BITS || o.m0 == kOccLevels - 1) break;
        ++o.m0;
    }
    o.M = o.m0;
    while (o.M < kOccLevels - 1 && ((o.hi[0] >> o.M) - (o.lo[0] >> o.M) > 1 || (o.hi[1] >> o.M) - (o.lo[1] >> o.M) > 1)) ++o.M;
    uint64_t words = 0;
    for (int m = 0; m < kOccLevels; ++m) {
        o.off[m] = words;
        o.nx[m] = o.ny[m] = 0;
        if (m < o.m0 || m > o.M) continue;
        o.nx[m] = (o.hi[0] >> m) - (o.lo[0] >> m) + 1;
        o.ny[m] = (o.hi[1] >> m) - (o.lo[1] >> m) + 1;
        words += ((uint64_t)o.nx[m] * o.ny[m] * nz + 31) / 32;
    }
    return words;
}

/* the 64-bit mask of the voxels x in [xl, xh], y in [yl, yh], z in [zl, zh] of a block (local coordinates 0..3) */
LV_HD uint64_t occ_box_mask(uint32_t xl, uint32_t xh, uint32_t yl, uint32_t yh, uint32_t zl, uint32_t zh) {
    const uint64_t row = (uint64_t)((1u << (xh + 1)) - (1u << xl));
    uint64_t slab = 0, m = 0;
    for (uint32_t y = yl; y <= yh; ++y) slab |= row << (4 * y);
    for (uint32_t z = zl; z <= zh; ++z) m |= slab << (16 * z);
    return m;
}

/* 1 when the voxel box [lo, hi] (inclusive, biased coordinates) may hold an occupied voxel; 0 only when it holds none */
LV_HD int occ_box_hits(const PrelocOcc& o, const uint32_t* lo_in, const uint32_t* hi_in) {
    uint32_t lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        lo[a] = lo_in[a] > o.lo[a] ? lo_in[a] : o.lo[a];
        hi[a] = hi_in[a] < o.hi[a] ? hi_in[a] : o.hi[a];
        if (lo[a] > hi[a]) return 0;
    }
    if ((hi[0] >> 2) - (lo[0] >> 2) <= 1 && (hi[1] >> 2) - (lo[1] >> 2) <= 1 && (hi[2] >> 2) - (lo[2] >> 2) <= 1) {
        for (uint32_t bz = lo[2] >> 2; bz <= hi[2] >> 2; ++bz)
            for (uint32_t by = lo[1] >> 2; by <= hi[1] >> 2; ++by)
                for (uint32_t bx = lo[0] >> 2; bx <= hi[0] >> 2; ++bx) {
                    const uint64_t mask = block_find(o.map, voxel_key(bx, by, bz));
                    if (!mask) continue;
                    const uint32_t x0 = 4 * bx, y0 = 4 * by, z0 = 4 * bz;
                    const uint64_t box = occ_box_mask((lo[0] > x0 ? lo[0] : x0) - x0, (hi[0] < x0 + 3 ? hi[0] : x0 + 3) - x0,
                                                      (lo[1] > y0 ? lo[1] : y0) - y0, (hi[1] < y0 + 3 ? hi[1] : y0 + 3) - y0,
                                                      (lo[2] > z0 ? lo[2] : z0) - z0, (hi[2] < z0 + 3 ? hi[2] : z0 + 3) - z0);
                    if (mask & box) return 1;
                }
        return 0;
    }
    int m = o.m0;
    while (m < o.M && ((hi[0] >> m) - (lo[0] >> m) > 1 || (hi[1] >> m) - (lo[1] >> m) > 1)) ++m;
    for (uint32_t z = lo[2]; z <= hi[2]; ++z)
        for (uint32_t y = lo[1] >> m; y <= hi[1] >> m; ++y)
            for (uint32_t x = lo[0] >> m; x <= hi[0] >> m; ++x) {
                const uint64_t b = occ_bit(o, m, x << m, y << m, z);
                if ((o.bits[o.off[m] + (b >> 5)] >> (b & 31)) & 1u) return 1;
            }
    return 0;
}

/* the fp32 translation range of a cell: tlo / thi = fadd(F.t, min / max over the four corner offsets) */
LV_HD void preloc_cell_t(const PrelocAxes& ax, const float* Ft, float step, int64_t i0, int64_t i1, int64_t j0, int64_t j1,
                         float* tlo, float* thi) {
    float olo[3], ohi[3];
    for (int c = 0; c < 4; ++c) {
        float o[3];
        preloc_offset(ax, dmul((double)(c & 1 ? i1 : i0), (double)step), dmul((double)(c & 2 ? j1 : j0), (double)step), o);
        for (int a = 0; a < 3; ++a) {
            olo[a] = c == 0 || o[a] < olo[a] ? o[a] : olo[a];
            ohi[a] = c == 0 || o[a] > ohi[a] ? o[a] : ohi[a];
        }
    }
    for (int a = 0; a < 3; ++a) { tlo[a] = fadd(Ft[a], olo[a]); thi[a] = fadd(Ft[a], ohi[a]); }
}

/* 1 when the point with rows r may score at some candidate of the cell (its voxel box may hold an occupied voxel) */
LV_HD int preloc_bound_point(const PrelocOcc& o, const float* r, const float* tlo, const float* thi) {
    const float kMax = 999999936.f;                 /* the largest float below 1e9 */
    uint32_t lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        float wl = fadd(r[a], tlo[a]), wh = fadd(r[a], thi[a]);
        wl = wl < -kMax ? -kMax : wl;
        wh = wh > kMax ? kMax : wh;
        if (!(wl <= wh)) return 0;                  /* no candidate of the cell can score it (also NaN) */
        const float ql = floorf(fdiv(wl, o.map.grid.ds)), qh = floorf(fdiv(wh, o.map.grid.ds));
        if (!(ql > -1073741824.f && qh < 1073741824.f)) return 1;
        lo[a] = voxel_of_cell((int)ql, o.map.grid.k);
        hi[a] = voxel_of_cell((int)qh, o.map.grid.k);
    }
    return occ_box_hits(o, lo, hi);
}

/* ---- cells ----------------------------------------------------------------------------------------------------------------- */
struct PrelocCell {
    int32_t h, l, ci, cj;      /* heading index k + K, level, cell coordinates at that level */
};
/* the positions of a cell as i, j ranges ([-I, I]) */
LV_HD void preloc_cell_range(const PrelocCell& c, int64_t I, int64_t* i0, int64_t* i1, int64_t* j0, int64_t* j1) {
    const int64_t W = 2 * I + 1, s = (int64_t)1 << c.l;
    const int64_t pi1 = ((int64_t)c.ci + 1) * s < W ? ((int64_t)c.ci + 1) * s : W;
    const int64_t pj1 = ((int64_t)c.cj + 1) * s < W ? ((int64_t)c.cj + 1) * s : W;
    *i0 = (int64_t)c.ci * s - I;
    *i1 = pi1 - 1 - I;
    *j0 = (int64_t)c.cj * s - I;
    *j1 = pj1 - 1 - I;
}

/* the best candidate seen: highest score, then smaller tie = |k| (2 I^2 + 1) + i^2 + j^2, then smaller linear index */
struct PrelocBest {
    int32_t score, pad_;
    int64_t tie, idx;
};
LV_HD bool preloc_better(const PrelocBest& a, const PrelocBest& b) {
    if (a.score != b.score) return a.score > b.score;
    if (a.tie != b.tie) return a.tie < b.tie;
    return a.idx < b.idx;
}
LV_HD PrelocBest preloc_best_of(int32_t score, int64_t k, int64_t i, int64_t j, int64_t I, int64_t K) {
    PrelocBest b;
    const int64_t W = 2 * I + 1;
    b.score = score;
    b.pad_ = 0;
    b.tie = (k < 0 ? -k : k) * (2 * I * I + 1) + i * i + j * j;
    b.idx = ((k + K) * W + (i + I)) * W + (j + I);
    return b;
}

/* ---- the schedule (host) --------------------------------------------------------------------------------------------------- */
struct PrelocSearchStats {
    int64_t candidates, cells_bounded, candidates_scored, probes;
    int32_t launches;
};

/* top level: 32 x 32 positions, less for a narrow window (at least 1), more when there would be over kPrelocMaxTopCells cells.
 * Cells split positions only, so the count never drops below the 2K + 1 headings: the level stops growing once one cell covers
 * every position (lv_prelocalize_global refuses more than kPrelocMaxTopCells headings). */
inline int preloc_top_level(int64_t I, int64_t K) {
    const int64_t W = 2 * I + 1, H = 2 * K + 1;
    int L = 1;
    while (L < kPrelocTopLevel && ((int64_t)1 << L) < W) ++L;
    for (;;) {
        const int64_t C = (W + ((int64_t)1 << L) - 1) >> L;
        if (H * C * C <= kPrelocMaxTopCells || C == 1) return L;
        ++L;
    }
}

/*
 * The search.  Ev provides
 *   void bounds(const PrelocCell* c, int64_t n, int32_t* out)     the bound of each cell (one launch)
 *   void exact(const PrelocCell* c, int64_t n, PrelocBest* out)   the best candidate of each cell, every candidate scored
 *                                                                 exactly (one launch)
 * prune == false scores every candidate (top-level cells exactly, in index order, nothing bounded).
 */
template <class Ev>
struct PrelocSearch {
    Ev& ev;
    int64_t I, K, S;
    bool prune;
    PrelocBest best;
    PrelocSearchStats st;
    std::vector<int32_t> bnd;
    std::vector<PrelocBest> res;
    PrelocCell dived;              /* the level-1 cell dive() scored: its candidates are in best already */
    bool has_dived = false;

    PrelocSearch(Ev& e, int64_t I_, int64_t K_, int64_t S_, bool prune_) : ev(e), I(I_), K(K_), S(S_), prune(prune_) {
        best.score = -1; best.pad_ = 0; best.tie = 0; best.idx = 0;
        st.candidates = (2 * K + 1) * (2 * I + 1) * (2 * I + 1);
        st.cells_bounded = st.candidates_scored = st.probes = 0;
        st.launches = 0;
    }
    int64_t cell_size(const PrelocCell& c) const {
        int64_t i0, i1, j0, j1;
        preloc_cell_range(c, I, &i0, &i1, &j0, &j1);
        return (i1 - i0 + 1) * (j1 - j0 + 1);
    }
    void bound(const std::vector<PrelocCell>& c, size_t at, size_t n) {
        bnd.resize(n);
        ev.bounds(c.data() + at, (int64_t)n, bnd.data());
        st.launches += 1;
        st.cells_bounded += (int64_t)n;
    }
    void exact(const std::vector<PrelocCell>& c) {
        for (size_t at = 0; at < c.size(); at += kPrelocChunk) {
            const size_t n = std::min(c.size() - at, (size_t)kPrelocChunk);
            res.resize(n);
            ev.exact(c.data() + at, (int64_t)n, res.data());
            st.launches += 1;
            for (size_t t = 0; t < n; ++t) {
                st.candidates_scored += cell_size(c[at + t]);
                if (preloc_better(res[t], best)) best = res[t];
            }
        }
    }
    /* the children of cell c (level l >= 1) that hold positions */
    void children(const PrelocCell& c, std::vector<PrelocCell>& out) const {
        const int64_t W = 2 * I + 1, s = (int64_t)1 << (c.l - 1);
        for (int q = 0; q < 4; ++q) {
            const PrelocCell k = {c.h, c.l - 1, 2 * c.ci + (q >> 1), 2 * c.cj + (q & 1)};
            if ((int64_t)k.ci * s < W && (int64_t)k.cj * s < W) out.push_back(k);
        }
    }
    /* a first score to prune against: from cell c down through the child of highest bound (the first of equal ones) at each
     * level, then the level-1 cell scored exactly */
    void dive(PrelocCell c) {
        std::vector<PrelocCell> kids;
        while (c.l > 1) {
            kids.clear();
            children(c, kids);
            bound(kids, 0, kids.size());
            size_t b = 0;
            for (size_t t = 1; t < kids.size(); ++t)
                if (bnd[t] > bnd[b]) b = t;
            c = kids[b];
        }
        exact(std::vector<PrelocCell>(1, c));
        dived = c;
        has_dived = true;
    }
    bool is_dived(const PrelocCell& c) const {
        return has_dived && c.h == dived.h && c.l == dived.l && c.ci == dived.ci && c.cj == dived.cj;
    }
    /* cells of level l, each with a bound; those still at or above the best score descend, highest bound first */
    void descend(int l, const std::vector<PrelocCell>& cells, const std::vector<int32_t>& bounds) {
        std::vector<size_t> live;
        for (size_t t = 0; t < cells.size(); ++t)
            if (bounds[t] >= best.score) live.push_back(t);
        if (live.empty()) return;
        std::stable_sort(live.begin(), live.end(), [&](size_t a, size_t b) { return bounds[a] > bounds[b]; });
        std::vector<PrelocCell> kids;
        if (l == 1) {                  /* scored exactly, each candidate once: the dived cell is not scored again */
            for (size_t t : live)
                if (!is_dived(cells[t])) kids.push_back(cells[t]);
            if (!kids.empty()) exact(kids);
            return;
        }
        for (size_t t : live) children(cells[t], kids);
        for (size_t at = 0; at < kids.size(); at += kPrelocChunk) {
            const size_t n = std::min(kids.size() - at, (size_t)kPrelocChunk);
            bound(kids, at, n);
            std::vector<PrelocCell> part(kids.begin() + at, kids.begin() + at + n);
            std::vector<int32_t> pb(bnd.begin(), bnd.begin() + n);
            descend(l - 1, part, pb);
        }
    }
    void run() {
        const int L = preloc_top_level(I, K);
        const int64_t W = 2 * I + 1, C = (W + ((int64_t)1 << L) - 1) >> L, T = (2 * K + 1) * C * C;
        std::vector<PrelocCell> top((size_t)T);
        for (int64_t t = 0; t < T; ++t) top[(size_t)t] = {(int32_t)(t / (C * C)), L, (int32_t)(t % (C * C) / C), (int32_t)(t % C)};
        if (!prune) {
            exact(top);
        } else {
            std::vector<int32_t> tb((size_t)T);
            for (size_t at = 0; at < top.size(); at += kPrelocChunk) {
                const size_t n = std::min(top.size() - at, (size_t)kPrelocChunk);
                bound(top, at, n);
                std::copy(bnd.begin(), bnd.begin() + n, tb.begin() + at);
            }
            std::vector<int64_t> order((size_t)T);
            for (int64_t t = 0; t < T; ++t) order[(size_t)t] = t;
            std::sort(order.begin(), order.end(), [&](int64_t a, int64_t b) {
                return tb[(size_t)a] != tb[(size_t)b] ? tb[(size_t)a] > tb[(size_t)b] : a < b;
            });
            dive(top[(size_t)order[0]]);
            for (size_t at = 0; at < order.size(); at += kPrelocBatch) {
                if (tb[(size_t)order[at]] < best.score) break;      /* every later cell is bounded lower still */
                const size_t n = std::min(order.size() - at, (size_t)kPrelocBatch);
                std::vector<PrelocCell> cells(n);
                std::vector<int32_t> b(n);
                for (size_t t = 0; t < n; ++t) { cells[t] = top[(size_t)order[at + t]]; b[t] = tb[(size_t)order[at + t]]; }
                descend(L, cells, b);
            }
        }
        st.probes = S * (st.cells_bounded + st.candidates_scored);
    }
};

}  // namespace lv
#endif
