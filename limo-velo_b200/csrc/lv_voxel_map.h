/*
 * lv_voxel_map.h — the device map: an INCREMENTAL hashed voxel grid with halo buckets, host+device.
 *
 * Replaces the ikd-Tree of the reference as a container (include/ikd-Tree/ikd_Tree/ikd_Tree.cpp): Build (:409-423),
 * Add_Points with the voxel-downsample rule (:478-573) and what Nearest_Search needs to run (lv_voxel_search.h).
 * Round 1 rebuilt a Morton-sorted pyramid from scratch after every sweep (sort of the whole map + ~0.5 GB of halo
 * copies per 1 M points).  Here a sweep only touches what it changes:
 *
 *   cell      the reference's downsample voxel, edge ds = map_downsample_size (0.2 m, Mapper.cpp:64-66), coordinate
 *             floor(x / ds) in fp32 exactly as ikd_Tree.cpp:493 computes it
 *   voxel     k x k x k cells (edge k * ds, 0.4 m by default); one 32-byte hash slot (= one DRAM / L2 sector):
 *               { key_lo, key_hi, own_start, own_count | halo_start, halo_count, caps, flags }
 *             own   = the voxel's points, one contiguous extent of the arena (capacity own_cap)
 *             halo  = "halo bucket": own points followed by those of the 26 neighbours, one contiguous extent
 *                     (capacity halo_cap): a query sees everything within Chebyshev ring 1 of its voxel with ONE
 *                     probe and ONE contiguous read (or one bulk copy into shared memory)
 *             every occupied voxel keeps slots (count 0) for its 26 neighbours ("dilation"), so a query landing in
 *             an empty voxel next to the map still finds a bucket
 *   block     4 x 4 x 4 voxels; one 16-byte slot { key, 64-bit occupancy mask }: the sparse-spot search
 *             (knn5_rings) walks blocks instead of probing up to 13^3 voxels
 *   arena     one float4 array (x, y, z, bits(point id)) for all extents, bump-allocated; an extent that outgrows
 *             its capacity moves to a fresh one (the old one is abandoned: the arena is sized for it, and
 *             lv_map_build / a rebuild compacts)
 *
 * Adding n points (Mapper::add): key + find-or-insert slot per point -> radix sort of n 32-bit (slot, cell) keys ->
 * one thread per touched voxel merges its run into the own extent under the reference's rule -> touched voxels mark
 * their 27 neighbourhoods dirty -> one warp per dirty voxel regenerates its halo bucket.  Work is proportional to
 * the sweep, not to the map; no host round trip (all counts live on the device), so the whole sequence can sit in a
 * CUDA graph or overlap the next sweep's transfer.  Build is the same path on an empty table without the rule.
 *
 * All per-item functions are LV_HD: tests/cpu_shim runs them serially on the host.
 */
#ifndef LV_VOXEL_MAP_H_
#define LV_VOXEL_MAP_H_

#include "lv_point_math.h"

#if !defined(__CUDACC__)
struct float4 { float x, y, z, w; };
struct uint4 { unsigned int x, y, z, w; };
#endif

namespace lv {

#define LV_KEY_BIAS (1 << 20)
#define LV_EMPTY_KEY 0xFFFFFFFFFFFFFFFFull

enum {
    kMaxProbes = 128,           /* an insertion that needs more probes fails (table full): lookups never need more */
    kBlockEdge = 4,             /* voxels per block edge                                                              */
    kCellBits = 5,              /* cell index inside a voxel: k <= 3 -> k^3 <= 27                                     */
    kMaxCellsPerVoxel = 3
};
/* device counters of the map (MapCounters index) */
/* kCtrIds: ids handed out so far; kCtrIdBase: the first id of the add in flight; kCtrAddN: points of the add in flight;
 * kCtrBuild: 1 when the add in flight builds the map (no downsampling) */
enum { kCtrArenaTop = 0, kCtrPoints, kCtrTouched, kCtrDirty, kCtrError, kCtrSlotsUsed, kCtrGather, kCtrBlocksUsed,
       kCtrIds, kCtrIdBase, kCtrAddN, kCtrBuild, kMapCounters = 16 };
/* bits of kCtrError */
enum { kErrTableFull = 1, kErrArenaFull = 2, kErrExtentTooLarge = 4, kErrListFull = 8, kErrBlockTableFull = 16 };

/* ---- host/device atomics (the host build is single-threaded) ---------------------------------------- */
LV_HD unsigned long long atomic_cas_u64(unsigned long long* p, unsigned long long cmp, unsigned long long val) {
#if defined(__CUDA_ARCH__)
    return atomicCAS(p, cmp, val);
#else
    const unsigned long long old = *p;
    if (old == cmp) *p = val;
    return old;
#endif
}
LV_HD unsigned long long atomic_or_u64(unsigned long long* p, unsigned long long v) {
#if defined(__CUDA_ARCH__)
    return atomicOr(p, v);
#else
    const unsigned long long old = *p;
    *p = old | v;
    return old;
#endif
}
LV_HD uint32_t atomic_add_u32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, v);
#else
    const uint32_t old = *p;
    *p = old + v;
    return old;
#endif
}
LV_HD uint32_t atomic_or_u32(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    return atomicOr(p, v);
#else
    const uint32_t old = *p;
    *p = old | v;
    return old;
#endif
}

/* ---- geometry of the grid ----------------------------------------------------------------------------- */
struct MapGrid {
    float ds;        /* cell edge = map_downsample_size                          */
    int32_t k;       /* cells per voxel edge (1..3)                              */
    float cell0;     /* voxel edge k * ds                                        */
};

LV_HD int cell_coord(float v, float ds) { return (int)floorf(fdiv(v, ds)); }   /* ikd_Tree.cpp:493 */
/* floor(a / k).  k is 1, 2 or 3 on every map this library builds (MapGrid::k): those cases cost a shift or a
 * multiply-high instead of a runtime integer division (three of them per query in every search kernel). */
LV_HD int floor_div(int a, int k) {
    if (k == 1) return a;
    if (k == 2) return a >> 1;                                   /* arithmetic shift: floor for negative a too */
    return a >= 0 ? a / 3 : -((-a + 2) / 3);                     /* k == 3 (map_alloc clamps k to 1..3) */
}
/* biased (non-negative, 21-bit) voxel coordinate of cell coordinate c */
LV_HD uint32_t voxel_of_cell(int c, int k) {
    int v = floor_div(c, k) + LV_KEY_BIAS;
    v = v < 0 ? 0 : (v > 0x1FFFFF ? 0x1FFFFF : v);
    return (uint32_t)v;
}
LV_HD uint32_t voxel_coord(const MapGrid& g, float v) { return voxel_of_cell(cell_coord(v, g.ds), g.k); }
/* low corner of voxel b along one axis (biased coordinate b) */
LV_HD float voxel_low(const MapGrid& g, uint32_t b) { return fmul((float)(((int)b - LV_KEY_BIAS) * g.k), g.ds); }

/* table key of a voxel / block given its biased coordinates: any injective packing will do */
LV_HD uint64_t voxel_key(uint32_t bx, uint32_t by, uint32_t bz) { return (uint64_t)bx | ((uint64_t)by << 21) | ((uint64_t)bz << 42); }
LV_HD uint32_t voxel_hash(uint64_t k) {   /* classic spatial hash of the three coordinates + a finaliser */
    uint32_t h = ((uint32_t)k & 0x1FFFFFu) * 73856093u ^ ((uint32_t)(k >> 21) & 0x1FFFFFu) * 19349663u ^
                 ((uint32_t)(k >> 42) & 0x1FFFFFu) * 83492791u;
    h ^= h >> 15;
    h *= 0x2c1b3c6du;
    h ^= h >> 12;
    return h;
}

LV_HD uint4 load_slot(const uint4* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
LV_HD float4 load_point(const float4* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

/* caps word of a voxel slot: own capacity / 4 in the low half, halo capacity / 8 in the high half */
LV_HD uint32_t caps_own(uint32_t caps) { return (caps & 0xFFFFu) * 4u; }
LV_HD uint32_t caps_halo(uint32_t caps) { return (caps >> 16) * 8u; }
LV_HD uint32_t caps_pack(uint32_t own_cap, uint32_t halo_cap) { return (own_cap / 4u) | ((halo_cap / 8u) << 16); }
enum { kMaxOwnCap = 0xFFFFu * 4u, kMaxHaloCap = 0xFFFFu * 8u };

/* read-only view: what the search kernels take as a kernel argument */
struct VoxelMapView {
    const uint4* table;      /* voxel slots, 2 x uint4 each           */
    uint32_t mask;           /* slots - 1                             */
    const uint4* btable;     /* block slots, 1 x uint4 each           */
    uint32_t bmask;
    const float4* arena;
    MapGrid grid;
};

/* slot of voxel `key`, or -1.  READ-ONLY lookups of kernels that do not modify the table (nc loads). */
LV_HD int voxel_find(const VoxelMapView& m, uint64_t key) {
    const uint32_t klo = (uint32_t)key, khi = (uint32_t)(key >> 32);
    uint32_t slot = voxel_hash(key) & m.mask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        const uint4 e = load_slot(m.table + 2 * (size_t)slot);
        if (e.x == klo && e.y == khi) return (int)slot;
        if ((e.x & e.y) == 0xFFFFFFFFu) break;
        slot = (slot + 1) & m.mask;
    }
    return -1;
}
/* occupancy mask of block `key` (0 when the block does not exist) */
LV_HD uint64_t block_find(const VoxelMapView& m, uint64_t key) {
    const uint32_t klo = (uint32_t)key, khi = (uint32_t)(key >> 32);
    uint32_t slot = (voxel_hash(key) * 0x9E3779B1u) & m.bmask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        const uint4 e = load_slot(m.btable + (size_t)slot);
        if (e.x == klo && e.y == khi) return (uint64_t)e.z | ((uint64_t)e.w << 32);
        if ((e.x & e.y) == 0xFFFFFFFFu) break;
        slot = (slot + 1) & m.bmask;
    }
    return 0ull;
}
LV_HD int block_bit(uint32_t bx, uint32_t by, uint32_t bz) {
    return (int)((bx & 3u) | ((by & 3u) << 2) | ((bz & 3u) << 4));
}

/* ---- the mutable side: map update kernels (lv_map.cu) and the host shim --------------------------------- */
struct VoxelMapRW {
    uint4* table;
    uint32_t mask;
    uint4* btable;
    uint32_t bmask;
    float4* arena;
    uint32_t arena_cap;      /* float4 elements                      */
    uint32_t* counters;      /* kMapCounters words                   */
    uint32_t* touched;       /* slots changed by the current add     */
    uint32_t* dirty;         /* slots whose halo bucket is stale     */
    uint32_t list_cap;       /* capacity of either list              */
    MapGrid grid;
};
LV_HD VoxelMapView map_view_of(const VoxelMapRW& m) {
    VoxelMapView v;
    v.table = m.table; v.mask = m.mask; v.btable = m.btable; v.bmask = m.bmask; v.arena = m.arena; v.grid = m.grid;
    return v;
}

/* plain (coherent) loads for kernels that write the table they read */
LV_HD int voxel_find_rw(const VoxelMapRW& m, uint64_t key) {
    const unsigned long long* tab64 = reinterpret_cast<const unsigned long long*>(m.table);
    uint32_t slot = voxel_hash(key) & m.mask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        const unsigned long long e = tab64[4 * (size_t)slot];
        if (e == (unsigned long long)key) return (int)slot;
        if (e == LV_EMPTY_KEY) break;
        slot = (slot + 1) & m.mask;
    }
    return -1;
}
/* find or insert; -1 when the table is full (sets kErrTableFull).  Most calls find the key: plain loads first, the
 * CAS only on an empty slot.  Once the table has been declared full nothing more is inserted (fail fast: a scattered map
 * would otherwise spend kMaxProbes probes on each of millions of points). */
LV_HD int voxel_insert(const VoxelMapRW& m, uint64_t key) {
    unsigned long long* tab64 = reinterpret_cast<unsigned long long*>(m.table);
    uint32_t slot = voxel_hash(key) & m.mask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(tab64 + 4 * (size_t)slot);
        if (cur == LV_EMPTY_KEY) {
            if (*reinterpret_cast<volatile uint32_t*>(m.counters + kCtrError) & (uint32_t)kErrTableFull) return -1;
            cur = atomic_cas_u64(tab64 + 4 * (size_t)slot, LV_EMPTY_KEY, (unsigned long long)key);
            if (cur == LV_EMPTY_KEY) {
                const uint32_t used = atomic_add_u32(m.counters + kCtrSlotsUsed, 1u);
                if (used > m.mask - (m.mask >> 3)) atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrTableFull);   /* load 0.875 */
                return (int)slot;
            }
        }
        if (cur == (unsigned long long)key) return (int)slot;
        slot = (slot + 1) & m.mask;
    }
    atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrTableFull);
    return -1;
}
/* set the occupancy bit of voxel (bx, by, bz) in its block */
LV_HD void block_mark(const VoxelMapRW& m, uint32_t bx, uint32_t by, uint32_t bz) {
    const uint64_t key = voxel_key(bx >> 2, by >> 2, bz >> 2);
    unsigned long long* tab64 = reinterpret_cast<unsigned long long*>(m.btable);
    uint32_t slot = (voxel_hash(key) * 0x9E3779B1u) & m.bmask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        const unsigned long long prev = atomic_cas_u64(tab64 + 2 * (size_t)slot, LV_EMPTY_KEY, (unsigned long long)key);
        if (prev == LV_EMPTY_KEY || prev == (unsigned long long)key) {
            if (prev == LV_EMPTY_KEY) atomic_add_u32(m.counters + kCtrBlocksUsed, 1u);
            atomic_or_u64(tab64 + 2 * (size_t)slot + 1, 1ull << block_bit(bx, by, bz));
            return;
        }
        slot = (slot + 1) & m.bmask;
    }
    atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrBlockTableFull);
}
/* ---- growth: the tables re-hashed into larger ones (lv_map.cu map_grow, lv_map_reserve / lv_map_set_growth) ------------
 * The arena keeps its indices (its used prefix is copied as it is), so a slot's 32 bytes stay valid word for word: key,
 * own and halo extents, caps and flags.  Only where a key lives changes.  The new table starts empty and holds at most
 * half as many keys per slot as the old one; a key that finds no free slot within kMaxProbes (as voxel_insert) sets the
 * table-full flag, so a lookup never has to probe further than it does today. */
/* old voxel slot `slot` -> m (same hash and linear probing as voxel_insert); counts kCtrSlotsUsed */
LV_HD void voxel_rehash_item(const VoxelMapRW& m, const uint4* old_table, uint32_t slot) {
    const uint4 e0 = old_table[2 * (size_t)slot], e1 = old_table[2 * (size_t)slot + 1];
    if ((e0.x & e0.y) == 0xFFFFFFFFu) return;
    const uint64_t key = (uint64_t)e0.x | ((uint64_t)e0.y << 32);
    unsigned long long* tab64 = reinterpret_cast<unsigned long long*>(m.table);
    uint32_t s = voxel_hash(key) & m.mask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        if (atomic_cas_u64(tab64 + 4 * (size_t)s, LV_EMPTY_KEY, (unsigned long long)key) == LV_EMPTY_KEY) {
            uint32_t* d32 = reinterpret_cast<uint32_t*>(m.table + 2 * (size_t)s);
            d32[2] = e0.z; d32[3] = e0.w;
            m.table[2 * (size_t)s + 1] = e1;
            atomic_add_u32(m.counters + kCtrSlotsUsed, 1u);
            return;
        }
        s = (s + 1) & m.mask;
    }
    atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrTableFull);
}
/* old block slot `slot` -> m (block_mark's hash and probing, occupancy mask OR-ed in); counts kCtrBlocksUsed */
LV_HD void block_rehash_item(const VoxelMapRW& m, const uint4* old_btable, uint32_t slot) {
    const uint4 e = old_btable[slot];
    if ((e.x & e.y) == 0xFFFFFFFFu) return;
    const uint64_t key = (uint64_t)e.x | ((uint64_t)e.y << 32);
    unsigned long long* tab64 = reinterpret_cast<unsigned long long*>(m.btable);
    uint32_t s = (voxel_hash(key) * 0x9E3779B1u) & m.bmask;
    for (int probes = 0; probes < kMaxProbes; ++probes) {
        const unsigned long long prev = atomic_cas_u64(tab64 + 2 * (size_t)s, LV_EMPTY_KEY, (unsigned long long)key);
        if (prev == LV_EMPTY_KEY || prev == (unsigned long long)key) {
            if (prev == LV_EMPTY_KEY) atomic_add_u32(m.counters + kCtrBlocksUsed, 1u);
            atomic_or_u64(tab64 + 2 * (size_t)s + 1, (unsigned long long)e.z | ((unsigned long long)e.w << 32));
            return;
        }
        s = (s + 1) & m.bmask;
    }
    atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrBlockTableFull);
}

/* bump allocation of `cap` float4 from the arena; 0xFFFFFFFF when exhausted (sets kErrArenaFull) */
LV_HD uint32_t arena_alloc(const VoxelMapRW& m, uint32_t cap) {
    const uint32_t at = atomic_add_u32(m.counters + kCtrArenaTop, cap);
    if (at > m.arena_cap || cap > m.arena_cap - at) {
        atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrArenaFull);
        return 0xFFFFFFFFu;
    }
    return at;
}

/* ---- step 1: the sort key of a new point --------------------------------------------------------------- */
/* (slot << kCellBits) | cell index inside the voxel; 0xFFFFFFFF for a point that cannot be stored */
LV_HD uint32_t map_point_key(const VoxelMapRW& m, float x, float y, float z) {
    const bool finite = (fabsf(x) < 1e9f) && (fabsf(y) < 1e9f) && (fabsf(z) < 1e9f);
    if (!finite) return 0xFFFFFFFFu;
    const int k = m.grid.k;
    const int cx = cell_coord(x, m.grid.ds), cy = cell_coord(y, m.grid.ds), cz = cell_coord(z, m.grid.ds);
    const uint32_t bx = voxel_of_cell(cx, k), by = voxel_of_cell(cy, k), bz = voxel_of_cell(cz, k);
    const int slot = voxel_insert(m, voxel_key(bx, by, bz));
    if (slot < 0) return 0xFFFFFFFFu;
    const int lx = cx - ((int)bx - LV_KEY_BIAS) * k, ly = cy - ((int)by - LV_KEY_BIAS) * k, lz = cz - ((int)bz - LV_KEY_BIAS) * k;
    const uint32_t cell = (uint32_t)((lx < 0 ? 0 : (lx >= k ? k - 1 : lx)) + k * ((ly < 0 ? 0 : (ly >= k ? k - 1 : ly)) +
                                     k * (lz < 0 ? 0 : (lz >= k ? k - 1 : lz))));
    return ((uint32_t)slot << kCellBits) | cell;
}

/* ---- step 2: merge one voxel's run of new points into its own extent ----------------------------------- */
/* Cell of an OLD map point as Search_by_range sees it (ikd_Tree.cpp:1262): the box of cell c is
 * [fl(c * ds), fl(c * ds) + ds) in fp32, so a point within an ulp of a face can belong to the cell next to
 * floor(q / ds). */
LV_HD int cell_coord_old(float v, float ds) {
    int c = cell_coord(v, ds);
    const float lo = fmul((float)c, ds);
    if (v < lo) --c;
    else if (!(v < fadd(lo, ds))) ++c;
    return c;
}
/* squared distance of p to the centre of cell (cx, cy, cz), evaluated like ikd_Tree.cpp:493-503 */
LV_HD float cell_centre_dist(float x, float y, float z, int cx, int cy, int cz, float ds) {
    float c[3];
    const int cc[3] = {cx, cy, cz};
    for (int a = 0; a < 3; ++a) {
        const float bmin = fmul((float)cc[a], ds);
        const float bmax = fadd(bmin, ds);
        c[a] = (float)((double)bmin + (double)fsub(bmax, bmin) / 2.0);
    }
    return sq_dist(x, y, z, c[0], c[1], c[2]);
}

LV_HD float4 make_point(float x, float y, float z, uint32_t id) {
    float4 p;
    p.x = x; p.y = y; p.z = z;
#if defined(__CUDA_ARCH__)
    p.w = __int_as_float((int)id);
#else
    memcpy(&p.w, &id, 4);
#endif
    return p;
}

/*
 * One thread per voxel: skeys[j .. e) is the voxel's run of new points (sorted by cell, input order inside a cell).
 *   downsample == 0   KD_TREE::Build / Add_Points(..., false): append everything (ikd_Tree.cpp:409-423, 549-571)
 *   downsample != 0   Add_Points' rule per cell (:487-522): with E = the map points already in the cell and N the
 *                     new ones, the cell ends up holding the single point of E u N closest to its centre — unless
 *                     E is one point and it wins, in which case nothing changes.  Tie rule (measure zero on float
 *                     data, kept for determinism): a new point beats an old one at equal distance (strict '<' at
 *                     :507), the later of two equal new points wins.
 * Ids: a new point gets id_base + its index in the batch.
 */
LV_HD_NOINLINE void map_merge_run(const VoxelMapRW& m, const uint32_t* skeys, const uint32_t* svals, uint32_t j, uint32_t n,
                                  const float* xyz, uint32_t id_base, int downsample) {
    const uint32_t slot = skeys[j] >> kCellBits;
    uint32_t e = j + 1, groups = 1;
    while (e < n && (skeys[e] >> kCellBits) == slot) { groups += skeys[e] != skeys[e - 1] ? 1u : 0u; ++e; }
    uint32_t* s32 = reinterpret_cast<uint32_t*>(m.table + 2 * (size_t)slot);
    const uint64_t key = (uint64_t)s32[0] | ((uint64_t)s32[1] << 32);
    uint32_t own_start = s32[2], cnt = s32[3];
    const uint32_t cnt0 = cnt;
    uint32_t caps = s32[6];
    uint32_t cap = caps_own(caps);
    const uint32_t need = downsample ? cnt + groups : cnt + (e - j);
    if (need > cap) {                                    /* move to a larger extent */
        uint32_t ncap = need + need / 2u + 4u;
        ncap = (ncap + 3u) & ~3u;
        if (ncap > (uint32_t)kMaxOwnCap) ncap = (uint32_t)kMaxOwnCap;
        if (need > ncap) { atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrExtentTooLarge); return; }
        const uint32_t at = arena_alloc(m, ncap);
        if (at == 0xFFFFFFFFu) return;
        for (uint32_t t = 0; t < cnt; ++t) m.arena[at + t] = m.arena[own_start + t];
        own_start = at;
        cap = ncap;
    }
    float4* own = m.arena + own_start;
    bool changed = false;
    if (!downsample) {
        for (uint32_t t = j; t < e; ++t) {
            const uint32_t src = svals[t];
            own[cnt++] = make_point(xyz[3 * (size_t)src], xyz[3 * (size_t)src + 1], xyz[3 * (size_t)src + 2], id_base + src);
        }
        changed = true;
    } else {
        const float ds = m.grid.ds;
        /* the cell of every own point, once (cell_coord_old costs three IEEE divisions per point): 5 bits per point, packed;
         * own extents beyond kCellCache points (dense first-sweep voxels) fall back to recomputing */
        enum { kCellCache = 48 };
        const int k = m.grid.k;
        const int vx0 = ((int)((uint32_t)key & 0x1FFFFFu) - LV_KEY_BIAS) * k, vy0 = ((int)((uint32_t)(key >> 21) & 0x1FFFFFu) - LV_KEY_BIAS) * k,
                  vz0 = ((int)((uint32_t)(key >> 42) & 0x1FFFFFu) - LV_KEY_BIAS) * k;
        uint8_t ocell[kCellCache];
        const bool cached = cnt + groups <= (uint32_t)kCellCache;   /* every group appends at most one point */
        if (cached)
            for (uint32_t t = 0; t < cnt; ++t) {
                const float4 q = own[t];
                const int lx = cell_coord_old(q.x, ds) - vx0, ly = cell_coord_old(q.y, ds) - vy0, lz = cell_coord_old(q.z, ds) - vz0;
                ocell[t] = (lx < 0 || ly < 0 || lz < 0 || lx >= k || ly >= k || lz >= k) ? (uint8_t)255 : (uint8_t)(lx + k * (ly + k * lz));   /* 255: an ulp outside */
            }
        uint32_t g0 = j;
        while (g0 < e) {
            uint32_t g1 = g0 + 1;
            while (g1 < e && skeys[g1] == skeys[g0]) ++g1;
            /* the cell of this group, from its first point (all points of a group share it) */
            const uint32_t s0 = svals[g0];
            const int cx = cell_coord(xyz[3 * (size_t)s0], ds), cy = cell_coord(xyz[3 * (size_t)s0 + 1], ds),
                      cz = cell_coord(xyz[3 * (size_t)s0 + 2], ds);
            const int lcx = cx - vx0, lcy = cy - vy0, lcz = cz - vz0;
            const uint8_t gcell = (lcx < 0 || lcy < 0 || lcz < 0 || lcx >= k || lcy >= k || lcz >= k) ? (uint8_t)254 : (uint8_t)(lcx + k * (lcy + k * lcz));
            int best_old = -1;
            uint32_t n_old = 0;
            float best_d = INFINITY;
            for (uint32_t t = 0; t < cnt; ++t) {
                const float4 q = own[t];
                const bool in_cell = cached ? ocell[t] == gcell
                                            : (cell_coord_old(q.x, ds) == cx && cell_coord_old(q.y, ds) == cy && cell_coord_old(q.z, ds) == cz);
                if (!in_cell) continue;
                ++n_old;
                const float d = cell_centre_dist(q.x, q.y, q.z, cx, cy, cz, ds);
                if (best_old < 0 || d < best_d) { best_old = (int)t; best_d = d; }   /* among old points: first strict minimum */
            }
            int best_new = -1;
            for (uint32_t t = g0; t < g1; ++t) {
                const uint32_t src = svals[t];
                const float d = cell_centre_dist(xyz[3 * (size_t)src], xyz[3 * (size_t)src + 1], xyz[3 * (size_t)src + 2], cx, cy, cz, ds);
                const bool take = (best_old < 0 && best_new < 0) ? true : !(best_d < d);   /* a new point replaces unless the kept one is strictly closer */
                if (take) { best_new = (int)src; best_d = d; }
            }
            bool same = false;                        /* the winner is the point the cell already holds (a re-observed static scene): nothing changes */
            if (best_new >= 0 && n_old == 1) {
                const float4 q = own[best_old];
                same = q.x == xyz[3 * (size_t)best_new] && q.y == xyz[3 * (size_t)best_new + 1] && q.z == xyz[3 * (size_t)best_new + 2];
            }
            if ((best_new >= 0 || n_old > 1) && !same) {
                const float4 w = best_new >= 0 ? make_point(xyz[3 * (size_t)best_new], xyz[3 * (size_t)best_new + 1],
                                                            xyz[3 * (size_t)best_new + 2], id_base + (uint32_t)best_new)
                                               : own[best_old];
                uint32_t wr = 0;
                for (uint32_t t = 0; t < cnt; ++t) {
                    const float4 q = own[t];
                    const bool in_cell = cached ? ocell[t] == gcell
                                                : (cell_coord_old(q.x, ds) == cx && cell_coord_old(q.y, ds) == cy && cell_coord_old(q.z, ds) == cz);
                    if (in_cell) continue;
                    if (cached) ocell[wr] = ocell[t];
                    own[wr++] = q;
                }
                if (cached) {
                    /* the winner is an old point for the later groups: filed under its box cell like every other own point
                     * (a new point on a face inside the voxel can lie in the box of the next cell, a later group) */
                    if (best_new >= 0) {
                        const int lx = cell_coord_old(w.x, ds) - vx0, ly = cell_coord_old(w.y, ds) - vy0, lz = cell_coord_old(w.z, ds) - vz0;
                        ocell[wr] = (lx < 0 || ly < 0 || lz < 0 || lx >= k || ly >= k || lz >= k) ? (uint8_t)255 : (uint8_t)(lx + k * (ly + k * lz));
                    } else {
                        ocell[wr] = gcell;                        /* an old winner was filed under this group's cell */
                    }
                }
                own[wr++] = w;
                cnt = wr;
                changed = true;
            }
            g0 = g1;
        }
    }
    s32[2] = own_start;
    s32[3] = cnt;
    s32[6] = caps_pack(cap, caps_halo(caps));
    if (!changed) return;
    if (cnt != cnt0) atomic_add_u32(m.counters + kCtrPoints, cnt - cnt0);   /* wraps for a net removal: the counter is a signed sum */
    if (cnt0 == 0 && cnt > 0) block_mark(m, (uint32_t)key & 0x1FFFFFu, (uint32_t)(key >> 21) & 0x1FFFFFu, (uint32_t)(key >> 42) & 0x1FFFFFu);
    const uint32_t at = atomic_add_u32(m.counters + kCtrTouched, 1u);
    if (at < m.list_cap) m.touched[at] = slot;
    else atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrListFull);
}

/* ---- step 3: a touched voxel marks its 27 neighbourhoods dirty (and makes sure the neighbour slots exist) ---- */
LV_HD void map_dilate_item(const VoxelMapRW& m, uint32_t slot, int nb) {
    const uint32_t* s32 = reinterpret_cast<const uint32_t*>(m.table + 2 * (size_t)slot);
    const uint64_t key = (uint64_t)s32[0] | ((uint64_t)s32[1] << 32);
    const int cx = (int)((uint32_t)key & 0x1FFFFFu) + nb % 3 - 1, cy = (int)((uint32_t)(key >> 21) & 0x1FFFFFu) + (nb / 3) % 3 - 1,
              cz = (int)((uint32_t)(key >> 42) & 0x1FFFFFu) + nb / 9 - 1;
    if (cx < 0 || cy < 0 || cz < 0 || cx > 0x1FFFFF || cy > 0x1FFFFF || cz > 0x1FFFFF) return;
    const int ns = nb == 13 ? (int)slot : voxel_insert(m, voxel_key((uint32_t)cx, (uint32_t)cy, (uint32_t)cz));
    if (ns < 0) return;
    uint32_t* flags = reinterpret_cast<uint32_t*>(m.table + 2 * (size_t)ns) + 7;
    if (atomic_or_u32(flags, 1u) & 1u) return;                /* already on the dirty list */
    const uint32_t at = atomic_add_u32(m.counters + kCtrDirty, 1u);
    if (at < m.list_cap) m.dirty[at] = (uint32_t)ns;
    else atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrListFull);
}

/* ---- step 4: regenerate the halo bucket of one dirty voxel ----------------------------------------------- */
/* lane l < 27 looks at neighbour nb(l); lane 0 = the voxel itself, so its points come first in the bucket */
LV_HD int halo_lane_to_nb(int lane) { return lane == 0 ? 13 : (lane <= 13 ? lane - 1 : lane); }

/* Capacity of a bucket that must hold `total` points: 25 % slack the first time, 50 % when it has outgrown an earlier
 * extent.  Growth is geometric, so the extents a voxel abandons over its life sum to at most twice its last one: the
 * arena (96 float4 per map point of capacity) never needs a free list. */
LV_HD uint32_t halo_new_cap(uint32_t total, uint32_t old_cap) {
    uint32_t ncap = total + (old_cap ? total / 2u : total / 4u) + 8u;
    ncap = (ncap + 7u) & ~7u;
    return ncap > (uint32_t)kMaxHaloCap ? (uint32_t)kMaxHaloCap : ncap;
}
/* serial form (host shim; the device kernel in lv_map.cu does the same with one warp) */
LV_HD_NOINLINE void map_halo_voxel_serial(const VoxelMapRW& m, uint32_t slot) {
    uint32_t* s32 = reinterpret_cast<uint32_t*>(m.table + 2 * (size_t)slot);
    const uint64_t key = (uint64_t)s32[0] | ((uint64_t)s32[1] << 32);
    const int bx = (int)((uint32_t)key & 0x1FFFFFu), by = (int)((uint32_t)(key >> 21) & 0x1FFFFFu), bz = (int)((uint32_t)(key >> 42) & 0x1FFFFFu);
    uint32_t st[27], ct[27], total = 0;
    for (int l = 0; l < 27; ++l) {
        const int nb = halo_lane_to_nb(l);
        const int cx = bx + nb % 3 - 1, cy = by + (nb / 3) % 3 - 1, cz = bz + nb / 9 - 1;
        st[l] = ct[l] = 0;
        if (cx < 0 || cy < 0 || cz < 0 || cx > 0x1FFFFF || cy > 0x1FFFFF || cz > 0x1FFFFF) continue;
        const int ns = l == 0 ? (int)slot : voxel_find_rw(m, voxel_key((uint32_t)cx, (uint32_t)cy, (uint32_t)cz));
        if (ns < 0) continue;
        const uint32_t* n32 = reinterpret_cast<const uint32_t*>(m.table + 2 * (size_t)ns);
        st[l] = n32[2];
        ct[l] = n32[3];
        total += ct[l];
    }
    uint32_t hstart = s32[4], caps = s32[6];
    uint32_t hcap = caps_halo(caps);
    if (total > hcap) {
        uint32_t ncap = halo_new_cap(total, hcap);
        if (total > ncap) { atomic_or_u32(m.counters + kCtrError, (uint32_t)kErrExtentTooLarge); s32[7] = 0u; return; }
        const uint32_t at = arena_alloc(m, ncap);
        if (at == 0xFFFFFFFFu) { s32[7] = 0u; return; }
        hstart = at;
        hcap = ncap;
    }
    uint32_t w = hstart;
    for (int l = 0; l < 27; ++l)
        for (uint32_t t = 0; t < ct[l]; ++t) m.arena[w++] = m.arena[st[l] + t];
    s32[4] = hstart;
    s32[5] = total;
    s32[6] = caps_pack(caps_own(caps), hcap);
    s32[7] = 0u;
}

}  // namespace lv
#endif
