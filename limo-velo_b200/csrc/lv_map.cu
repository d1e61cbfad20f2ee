/*
 * lv_map.cu — Mapper::add / KD_TREE::Build / Add_Points on the device map (layout and per-item logic: lv_voxel_map.h).
 *
 * Replaces KD_TREE::Build (include/ikd-Tree/ikd_Tree/ikd_Tree.cpp:409-423) and Add_Points with the voxel-downsample
 * rule (:478-573) as called from Mapper::add (src/Modules/Mapper.cpp:22-30,64-76).  One add is six kernels plus a
 * radix sort of the NEW points only, all on the handle's stream, with every count on the device:
 *
 *   begin    reset the touched / dirty lists
 *   keys     per new point: cell (floor(x / ds), ikd_Tree.cpp:493), voxel, find-or-insert the voxel's slot,
 *            32-bit sort key (slot, cell inside the voxel)
 *   sort     cub::DeviceRadixSort over the n new (key, index) pairs            [library: CCCL ships with the toolkit]
 *   merge    one thread per touched voxel: the reference's rule per cell (map_merge_run)
 *   dilate   touched voxels create their neighbours' slots and mark the 27 neighbourhoods dirty
 *   halo     one warp per dirty voxel: 27 probes, warp scan, coalesced copy of the neighbours' points into the
 *            voxel's halo bucket (in place when it fits its capacity, else a fresh extent)
 *
 * HBM traffic is proportional to the sweep: ~20 B per new point for keys and sort, ~0.6 KB per dirty voxel for its
 * bucket (27 x 32 B probes + the copy); the 1 M points already in the map are not touched.  Nothing synchronises the
 * stream: errors (table / arena exhausted) are flagged on the device and read with the next result that is read
 * anyway (lv_map_size, lv_correct, lv_synchronize).
 */
#include <cub/device/device_radix_sort.cuh>

#include "lv_internal.h"

namespace lv {

__global__ void __launch_bounds__(256) lv_map_clear_kernel(uint4* table, uint32_t slots, uint4* btable, uint32_t bslots,
                                                            uint32_t* counters) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = i0; i < 2 * (size_t)slots; i += stride)
        table[i] = (i & 1u) ? make_uint4(0u, 0u, 0u, 0u) : make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
    for (size_t i = i0; i < (size_t)bslots; i += stride) btable[i] = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
    if (i0 < (size_t)kMapCounters) counters[i0] = i0 == (size_t)kCtrArenaTop ? 16u : 0u;   /* position 0 is never handed out */
}

/* the add's point count (n, or the device count of MapAddCount), its first id and whether it builds the map */
__global__ void lv_map_begin_kernel(uint32_t* counters, int64_t n, const int64_t* d_n, int64_t min_points, int build_if_empty,
                                    uint32_t* err) {
    if (threadIdx.x == 0) {
        counters[kCtrTouched] = 0u;
        counters[kCtrDirty] = 0u;
        int64_t k = device_count(d_n, n, err);
        if (d_n && k < (min_points > 1 ? min_points : 1)) k = 0;              /* main.cpp:81: the tick breaks before map.add */
        counters[kCtrAddN] = (uint32_t)k;
        counters[kCtrIdBase] = counters[kCtrIds];                            /* a new point gets id_base + its index in the batch */
        counters[kCtrIds] += (uint32_t)k;
        counters[kCtrBuild] = (build_if_empty && counters[kCtrPoints] == 0u) ? 1u : 0u;
    }
}

/* slots past the add's count get the key of a point that cannot be stored: the merge skips them */
__global__ void __launch_bounds__(256) lv_map_keys_kernel(const VoxelMapRW m, const float* __restrict__ xyz, uint32_t n,
                                                           uint32_t* __restrict__ skeys, uint32_t* __restrict__ svals) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    skeys[i] = i < m.counters[kCtrAddN] ? map_point_key(m, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]) : 0xFFFFFFFFu;
    svals[i] = i;
}

__global__ void __launch_bounds__(128) lv_map_merge_kernel(const VoxelMapRW m, const uint32_t* __restrict__ skeys,
                                                            const uint32_t* __restrict__ svals, uint32_t n,
                                                            const float* __restrict__ xyz, int downsample) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t key = skeys[j];
    if (key == 0xFFFFFFFFu) return;                                          /* not storable (non-finite / table full) */
    if (j > 0 && (skeys[j - 1] >> kCellBits) == (key >> kCellBits)) return;  /* not the head of its voxel's run */
    map_merge_run(m, skeys, svals, j, n, xyz, m.counters[kCtrIdBase], m.counters[kCtrBuild] ? 0 : downsample);
}

__global__ void __launch_bounds__(256) lv_map_dilate_kernel(const VoxelMapRW m) {
    const uint32_t n = min(m.counters[kCtrTouched], m.list_cap) * 27u;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) map_dilate_item(m, m.touched[t / 27u], (int)(t % 27u));
}

/* one warp per dirty voxel (the warp form of map_halo_voxel_serial) */
__global__ void __launch_bounds__(256) lv_map_halo_kernel(const VoxelMapRW m) {
    const uint32_t n = min(m.counters[kCtrDirty], m.list_cap);
    const int lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t d = warp; d < n; d += n_warps) {
        const uint32_t slot = m.dirty[d];
        uint32_t* s32 = reinterpret_cast<uint32_t*>(m.table + 2 * (size_t)slot);
        const uint64_t key = (uint64_t)s32[0] | ((uint64_t)s32[1] << 32);
        const int bx = (int)((uint32_t)key & 0x1FFFFFu), by = (int)((uint32_t)(key >> 21) & 0x1FFFFFu), bz = (int)((uint32_t)(key >> 42) & 0x1FFFFFu);
        uint32_t s = 0, cnt = 0;
        if (lane < 27) {
            const int nb = halo_lane_to_nb(lane);
            const int cx = bx + nb % 3 - 1, cy = by + (nb / 3) % 3 - 1, cz = bz + nb / 9 - 1;
            if (cx >= 0 && cy >= 0 && cz >= 0 && cx <= 0x1FFFFF && cy <= 0x1FFFFF && cz <= 0x1FFFFF) {
                const int ns = lane == 0 ? (int)slot : voxel_find_rw(m, voxel_key((uint32_t)cx, (uint32_t)cy, (uint32_t)cz));
                if (ns >= 0) {
                    const uint32_t* n32 = reinterpret_cast<const uint32_t*>(m.table + 2 * (size_t)ns);
                    s = n32[2];
                    cnt = n32[3];
                }
            }
        }
        uint32_t incl = cnt;   /* inclusive warp scan of the counts */
#pragma unroll
        for (int k = 1; k < 32; k <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl, k);
            if (lane >= k) incl += v;
        }
        const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
        const uint32_t excl = incl - cnt;
        uint32_t hstart = 0, caps = 0, hcap = 0;
        int ok = 1;
        if (lane == 0) {
            hstart = s32[4];
            caps = s32[6];
            hcap = caps_halo(caps);
            if (total > hcap) {
                const uint32_t ncap = halo_new_cap(total, hcap);
                if (total > ncap) { atomicOr(m.counters + kCtrError, (uint32_t)kErrExtentTooLarge); ok = 0; }
                else {
                    const uint32_t at = arena_alloc(m, ncap);
                    if (at == 0xFFFFFFFFu) ok = 0;
                    else { hstart = at; hcap = ncap; }
                }
            }
        }
        ok = __shfl_sync(0xffffffffu, ok, 0);
        hstart = __shfl_sync(0xffffffffu, hstart, 0);
        if (ok) {
            for (uint32_t j0 = 0; j0 < total; j0 += 32) {                     /* coalesced 16-byte stores, gathers from <= 27 runs */
                const uint32_t j = j0 + (uint32_t)lane;
                int lo = 0;                                                  /* first neighbour whose inclusive prefix exceeds j */
#pragma unroll
                for (int step = 16; step > 0; step >>= 1) {
                    const uint32_t v = __shfl_sync(0xffffffffu, incl, lo + step - 1);
                    if (v <= j) lo += step;
                }
                lo = lo > 31 ? 31 : lo;
                const uint32_t sv = __shfl_sync(0xffffffffu, s, lo), ev = __shfl_sync(0xffffffffu, excl, lo);
                if (j < total) m.arena[hstart + j] = m.arena[sv + (j - ev)];
            }
        }
        if (lane == 0) {
            if (ok) {
                s32[4] = hstart;
                s32[5] = total;
                s32[6] = caps_pack(caps_own(caps), hcap);
            }
            s32[7] = 0u;
        }
        __syncwarp();
    }
}

/* lv_map_points: all own points -> out[], unordered; cursor = counters[kCtrGather] */
__global__ void __launch_bounds__(256) lv_map_gather_kernel(const VoxelMapRW m, float4* __restrict__ out, uint32_t out_cap) {
    const uint32_t slots = m.mask + 1u;
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < slots; slot += stride) {
        const uint4 e = m.table[2 * (size_t)slot];
        if ((e.x & e.y) == 0xFFFFFFFFu || e.w == 0u) continue;
        const uint32_t at = atomicAdd(m.counters + kCtrGather, e.w);
        for (uint32_t t = 0; t < e.w && at + t < out_cap; ++t) out[at + t] = m.arena[e.z + t];
    }
}
__global__ void __launch_bounds__(256) lv_map_ids_kernel(const float4* __restrict__ pts, uint32_t n, uint32_t* __restrict__ ids,
                                                          uint32_t* __restrict__ idx) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    ids[i] = (uint32_t)__float_as_int(pts[i].w);
    idx[i] = i;
}
__global__ void __launch_bounds__(256) lv_map_unpack_kernel(const float4* __restrict__ pts, const uint32_t* __restrict__ idx, uint32_t n,
                                                             float* __restrict__ xyz) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 p = pts[idx[i]];
    xyz[3 * (size_t)i] = p.x; xyz[3 * (size_t)i + 1] = p.y; xyz[3 * (size_t)i + 2] = p.z;
}

/* main.cpp:91-93,99-105 on the device: a cloud (LiDAR frame) in world coordinates with the state the update just produced,
 * Xt2 * Xt2.I_Rt_L() * p in fp32 (State.cpp:79-89, RotTransl.cpp:36-48) — the very transform Mapper::match applies.
 * *count points: the map add's (kCtrAddN) or lv_sweep_to_world_device_async's (lv_world_count_kernel).  xyz may equal out. */
__global__ void __launch_bounds__(256) lv_sweep_to_world_kernel(const UpdateCtrl* __restrict__ c, const float* xyz,
                                                                 const uint32_t* __restrict__ count, float* out) {
    __shared__ Frame s_frame;
    if (threadIdx.x == 0) make_frame(c->x, &s_frame);
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *count) return;
    float g[3];
    rt_apply(s_frame.lidar_to_world, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], g);
    out[3 * (size_t)i] = g[0]; out[3 * (size_t)i + 1] = g[1]; out[3 * (size_t)i + 2] = g[2];
}

/* ---- growth (map_grow) ------------------------------------------------------------------------------------ */
/* the new tables start empty; the re-hash recounts the slots and blocks it re-inserts */
__global__ void __launch_bounds__(256) lv_map_grow_init_kernel(uint4* table, uint32_t slots, uint4* btable, uint32_t bslots,
                                                                uint32_t* counters) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = i0; i < 2 * (size_t)slots; i += stride)
        table[i] = (i & 1u) ? make_uint4(0u, 0u, 0u, 0u) : make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
    for (size_t i = i0; i < (size_t)bslots; i += stride) btable[i] = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u);
    if (i0 == 0) { counters[kCtrSlotsUsed] = 0u; counters[kCtrBlocksUsed] = 0u; }
}
/* one thread per old slot: voxel slots first, then block slots (the two tables are independent) */
__global__ void __launch_bounds__(256) lv_map_rehash_kernel(const VoxelMapRW m, const uint4* __restrict__ old_table, uint32_t old_slots,
                                                             const uint4* __restrict__ old_btable, uint32_t old_bslots) {
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < old_slots + old_bslots; t += stride) {
        if (t < old_slots) voxel_rehash_item(m, old_table, t);
        else block_rehash_item(m, old_btable, t - old_slots);
    }
}
/* the used prefix [0, counters[kCtrArenaTop]) of the arena, read on the device: the host never needs the count */
__global__ void __launch_bounds__(256) lv_map_arena_copy_kernel(const float4* __restrict__ src, float4* __restrict__ dst, uint32_t old_cap,
                                                                 const uint32_t* __restrict__ counters) {
    const uint32_t top = min(counters[kCtrArenaTop], old_cap);
    const uint32_t stride = gridDim.x * blockDim.x;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < top; i += stride) dst[i] = src[i];
}

/* ---- host side ------------------------------------------------------------------------------------------- */
static VoxelMapRW map_rw(const MapBuffers& b) {
    VoxelMapRW m;
    m.table = b.table; m.mask = b.slots - 1u; m.btable = b.btable; m.bmask = b.bslots - 1u;
    m.arena = b.arena; m.arena_cap = b.arena_cap; m.counters = b.counters; m.touched = b.touched; m.dirty = b.dirty;
    m.list_cap = b.list_cap; m.grid = b.grid;
    return m;
}

static uint32_t pow2_at_least(uint64_t v, uint32_t lo, uint32_t hi) {
    uint64_t p = lo;
    while (p < v && p < hi) p <<= 1;
    return (uint32_t)p;
}

MapSizes map_sizes(int64_t cap, int64_t max_points, bool scratch) {
    MapSizes z;
    /* occupied + dilated voxels of a surface-like map: ~1 slot per map point; 4x keeps the load below 0.3, scattered
     * maps (27 slots per isolated point) run out and report LV_ERR_CAPACITY instead of hanging */
    z.slots = pow2_at_least(4ull * (uint64_t)cap, 1u << 16, (uint32_t)kMaxSlots);
    z.bslots = pow2_at_least((uint64_t)z.slots / 4u, 1u << 14, 1u << 27);
    /* own extents (~1.5x the map) + halo buckets (27 copies of every point, up to 50 % slack) + the extents that
     * buckets outgrow (geometric growth: at most twice the live ones): 1.5 KB per map point of capacity */
    uint64_t arena = 96ull * (uint64_t)cap + (4ull << 20);
    if (arena > kMaxArena) arena = kMaxArena;                                /* ids are int32 */
    z.arena_cap = (uint32_t)arena;
    z.add_cap = cap > max_points ? cap : max_points;
    z.sort_tmp_bytes = 0;
    if (scratch)
        cub::DeviceRadixSort::SortPairs(nullptr, z.sort_tmp_bytes, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                        (uint32_t*)nullptr, (int)z.add_cap, 0, 32);
    return z;
}
const char* map_ceiling(int64_t cap) {
    if (4ull * (uint64_t)cap > (uint64_t)kMaxSlots) return "voxel table ceiling (2^26 slots, 4 per point)";
    if (96ull * (uint64_t)cap + (4ull << 20) > (uint64_t)kMaxArena) return "arena ceiling (0x7FFFFFF0 entries: point ids are int32)";
    return nullptr;
}
int64_t map_bytes(const MapBuffers& b) {
    return (int64_t)(sizeof(uint4) * (2 * (size_t)b.slots + (size_t)b.bslots) + sizeof(float4) * (size_t)b.arena_cap +
                     sizeof(uint32_t) * (2 * (size_t)b.list_cap + 4 * (size_t)b.add_cap + kMapCounters) + sizeof(float) * 3 * (size_t)b.add_cap +
                     b.sort_tmp_bytes);
}

/* every device buffer of the map comes from the stream-ordered allocator: a growth frees the old ones with cudaFreeAsync
 * behind the kernels that read them, without synchronising the device */
struct MapStore {
    uint4 *table, *btable;
    float4* arena;
    uint32_t *touched, *dirty;
    float* stage_xyz;
    uint32_t *skeys, *skeys_alt, *svals, *svals_alt;
    void* sort_tmp;
};
static void store_free(MapStore& s, cudaStream_t st) {
    void* p[] = {s.table, s.btable, s.arena, s.touched, s.dirty, s.stage_xyz, s.skeys, s.skeys_alt, s.svals, s.svals_alt, s.sort_tmp};
    for (void* q : p) if (q) cudaFreeAsync(q, st);
    memset(&s, 0, sizeof(s));
}
static cudaError_t store_alloc(MapStore& s, const MapSizes& z, cudaStream_t st) {
    memset(&s, 0, sizeof(s));
    cudaError_t e;
    if ((e = cudaMallocAsync((void**)&s.table, sizeof(uint4) * 2 * (size_t)z.slots, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.btable, sizeof(uint4) * (size_t)z.bslots, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.arena, sizeof(float4) * (size_t)z.arena_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.touched, sizeof(uint32_t) * (size_t)z.slots, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.dirty, sizeof(uint32_t) * (size_t)z.slots, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.stage_xyz, sizeof(float) * 3 * (size_t)z.add_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.skeys, sizeof(uint32_t) * (size_t)z.add_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.skeys_alt, sizeof(uint32_t) * (size_t)z.add_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.svals, sizeof(uint32_t) * (size_t)z.add_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync((void**)&s.svals_alt, sizeof(uint32_t) * (size_t)z.add_cap, st)) == cudaSuccess &&
        (e = cudaMallocAsync(&s.sort_tmp, z.sort_tmp_bytes, st)) == cudaSuccess)
        return cudaSuccess;
    store_free(s, st);
    cudaGetLastError();                       /* an allocation failure is not sticky: the old map stays usable */
    return e;
}
static MapStore store_of(const MapBuffers& b) {
    MapStore s = {b.table, b.btable, b.arena, b.touched, b.dirty, b.stage_xyz, b.skeys, b.skeys_alt, b.svals, b.svals_alt, b.sort_tmp};
    return s;
}
static void store_adopt(MapBuffers& b, const MapStore& s, const MapSizes& z, int64_t cap) {
    b.table = s.table; b.btable = s.btable; b.arena = s.arena; b.touched = s.touched; b.dirty = s.dirty; b.stage_xyz = s.stage_xyz;
    b.skeys = s.skeys; b.skeys_alt = s.skeys_alt; b.svals = s.svals; b.svals_alt = s.svals_alt; b.sort_tmp = s.sort_tmp;
    b.cap = cap;
    b.slots = z.slots; b.bslots = z.bslots; b.arena_cap = z.arena_cap; b.list_cap = z.slots;
    b.add_cap = z.add_cap; b.sort_tmp_bytes = z.sort_tmp_bytes;
    b.sort_bits = kCellBits;
    for (uint32_t s2 = b.slots; s2 > 1; s2 >>= 1) b.sort_bits++;
}

cudaError_t map_alloc(MapBuffers& b, int64_t max_map_points, int64_t max_points, float voxel_size, float ds, cudaStream_t st) {
    memset(&b, 0, sizeof(b));
    b.grid.ds = ds;
    int k = (int)floor((double)voxel_size / (double)ds + 0.5);
    k = k < 1 ? 1 : (k > kMaxCellsPerVoxel ? kMaxCellsPerVoxel : k);
    b.grid.k = k;
    b.grid.cell0 = (float)k * ds;
    b.max_points = max_points;
    b.stream = st;
    const MapSizes z = map_sizes(max_map_points, max_points);
    MapStore s;
    cudaError_t e;
    if ((e = store_alloc(s, z, st)) != cudaSuccess) return e;
    store_adopt(b, s, z, max_map_points);
    if ((e = cudaMalloc(&b.counters, sizeof(uint32_t) * kMapCounters)) != cudaSuccess) return e;
    if ((e = cudaMallocHost(&b.h_counters, sizeof(uint32_t) * kMapCounters)) != cudaSuccess) return e;
    b.empty = true;
    return cudaSuccess;
}

void map_free(MapBuffers& b) {
    MapStore s = store_of(b);
    store_free(s, b.stream);
    if (b.stream) cudaStreamSynchronize(b.stream);
    cudaFree(b.counters); cudaFreeHost(b.h_counters);
    memset(&b, 0, sizeof(b));
}

/* re-hash both tables into tables sized for `cap` points, copy the arena's used prefix into a larger arena, grow the
 * lists and the add scratch; frees the old buffers behind the kernels.  Stream-ordered, no synchronisation.  On an
 * allocation failure nothing has changed. */
cudaError_t map_grow(MapBuffers& b, int64_t cap, cudaStream_t st, int* launches) {
    if (cap <= b.cap) return cudaSuccess;
    const MapSizes z = map_sizes(cap, b.max_points);
    MapStore s;
    cudaError_t e = store_alloc(s, z, st);
    if (e != cudaSuccess) return e;
    MapStore old = store_of(b);
    const uint32_t old_slots = b.slots, old_bslots = b.bslots, old_arena_cap = b.arena_cap;
    lv_map_grow_init_kernel<<<kNumSMs * 8, 256, 0, st>>>(s.table, z.slots, s.btable, z.bslots, b.counters);
    store_adopt(b, s, z, cap);
    const VoxelMapRW m = map_rw(b);
    lv_map_rehash_kernel<<<kNumSMs * 8, 256, 0, st>>>(m, old.table, old_slots, old.btable, old_bslots);
    lv_map_arena_copy_kernel<<<kNumSMs * 8, 256, 0, st>>>(old.arena, s.arena, old_arena_cap, b.counters);
    e = cudaGetLastError();
    store_free(old, st);
    if (launches) *launches += 3;
    return e;
}

VoxelMapView map_view(const MapBuffers& b) { return map_view_of(map_rw(b)); }

cudaError_t map_clear(MapBuffers& b, cudaStream_t st, int* launches) {
    lv_map_clear_kernel<<<kNumSMs * 8, 256, 0, st>>>(b.table, b.slots, b.btable, b.bslots, b.counters);
    b.empty = true;
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t map_add(MapBuffers& b, const float* d_xyz, int64_t n, int downsample, cudaStream_t st, int* launches, const MapAddCount& cnt,
                    const UpdateCtrl* to_world) {
    if (n <= 0) return cudaSuccess;
    if (n > b.add_cap) return cudaErrorInvalidValue;
    const VoxelMapRW m = map_rw(b);
    const uint32_t n32 = (uint32_t)n;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    lv_map_begin_kernel<<<1, 32, 0, st>>>(b.counters, n, cnt.n, cnt.min_points, cnt.build_if_empty, cnt.err);
    if (to_world) {
        lv_sweep_to_world_kernel<<<blocks, 256, 0, st>>>(to_world, d_xyz, b.counters + kCtrAddN, b.stage_xyz);
        d_xyz = b.stage_xyz;
        if (launches) *launches += 1;
    }
    lv_map_keys_kernel<<<blocks, 256, 0, st>>>(m, d_xyz, n32, b.skeys, b.svals);
    size_t tmp = b.sort_tmp_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(b.sort_tmp, tmp, b.skeys, b.skeys_alt, b.svals, b.svals_alt, (int)n, 0, b.sort_bits, st);
    if (e != cudaSuccess) return e;
    lv_map_merge_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(m, b.skeys_alt, b.svals_alt, n32, d_xyz, downsample);
    /* touched <= n voxels, dirty <= 27 n: fixed grids striding over the device-side counts */
    uint64_t dil = ((uint64_t)n * 27 + 255) / 256;
    dil = dil < 1 ? 1 : (dil > kNumSMs * 8u ? kNumSMs * 8u : dil);
    lv_map_dilate_kernel<<<(unsigned)dil, 256, 0, st>>>(m);
    uint64_t hal = ((uint64_t)n * 27 + 7) / 8;
    hal = hal < 1 ? 1 : (hal > kNumSMs * 64u ? kNumSMs * 64u : hal);
    lv_map_halo_kernel<<<(unsigned)hal, 256, 0, st>>>(m);
    b.empty = false;
    if (launches) *launches += 5 + 4;   /* + histogram and onesweep passes of the sort (approximate) */
    return cudaGetLastError();
}

/* one thread reads every count before it writes: d_n_out may equal d_n or the gate's count */
__global__ void lv_world_count_kernel(const int64_t* d_n, int64_t n_max, const int64_t* gate_n, int64_t gate_max, int64_t gate_min,
                                      uint32_t* count, int64_t* d_n_out, uint32_t* err) {
    if (threadIdx.x != 0) return;
    int64_t k = device_count(d_n, n_max, err);
    if (gate_n && device_count(gate_n, gate_max, nullptr) < (gate_min > 1 ? gate_min : 1)) k = 0;   /* main.cpp:81 */
    *count = (uint32_t)k;
    *d_n_out = k;
}

cudaError_t launch_sweep_to_world(const UpdateCtrl* d_ctrl, const float* d_xyz, const int64_t* d_n, int64_t n_max, const int64_t* gate_n,
                                  int64_t gate_max, int64_t gate_min, float* d_out, int64_t* d_n_out, uint32_t* count, uint32_t* err,
                                  cudaStream_t st, int* launches) {
    lv_world_count_kernel<<<1, 32, 0, st>>>(d_n, n_max, gate_n, gate_max, gate_min, count, d_n_out, err);
    lv_sweep_to_world_kernel<<<(unsigned)((n_max + 255) / 256), 256, 0, st>>>(d_ctrl, d_xyz, count, d_out);
    if (launches) *launches += 2;
    return cudaGetLastError();
}

/* device counters -> pinned mirror; the caller synchronises the stream before reading b.h_counters */
cudaError_t map_fetch_counters(MapBuffers& b, cudaStream_t st) {
    return cudaMemcpyAsync(b.h_counters, b.counters, sizeof(uint32_t) * kMapCounters, cudaMemcpyDeviceToHost, st);
}

/* all map points in insertion order (ascending id) -> d_out (n x 3 floats); returns the count through *n_out.
 * Synchronises the stream; allocates scratch on the spot (an inspection call, not on the hot path). */
cudaError_t map_points_sorted(MapBuffers& b, float* host_out, int64_t cap, int64_t* n_out, cudaStream_t st) {
    cudaError_t e;
    if ((e = map_fetch_counters(b, st)) != cudaSuccess) return e;
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return e;
    const int64_t n = (int64_t)(int32_t)b.h_counters[kCtrPoints];
    *n_out = n;
    if (n <= 0 || !host_out || cap <= 0) return cudaSuccess;
    DeviceBuf<float4> pts;
    DeviceBuf<uint32_t> ids, idx, ids2, idx2;
    DeviceBuf<float> xyz;
    DeviceBuf<uint8_t> tmp;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, ids.get(), ids2.get(), idx.get(), idx2.get(), (int)n, 0, 32);
    if ((e = pts.reserve(n)) != cudaSuccess || (e = ids.reserve(n)) != cudaSuccess || (e = idx.reserve(n)) != cudaSuccess ||
        (e = ids2.reserve(n)) != cudaSuccess || (e = idx2.reserve(n)) != cudaSuccess || (e = xyz.reserve(3 * (size_t)n)) != cudaSuccess ||
        (e = tmp.reserve(tmp_bytes)) != cudaSuccess)
        return e;
    const VoxelMapRW m = map_rw(b);
    const unsigned blocks = (unsigned)((n + 255) / 256);
    cudaMemsetAsync(b.counters + kCtrGather, 0, sizeof(uint32_t), st);
    lv_map_gather_kernel<<<kNumSMs * 8, 256, 0, st>>>(m, pts, (uint32_t)n);
    lv_map_ids_kernel<<<blocks, 256, 0, st>>>(pts, (uint32_t)n, ids, idx);
    e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, ids.get(), ids2.get(), idx.get(), idx2.get(), (int)n, 0, 32, st);
    lv_map_unpack_kernel<<<blocks, 256, 0, st>>>(pts, idx2, (uint32_t)n, xyz);
    const int64_t m_out = n < cap ? n : cap;
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_out, xyz, sizeof(float) * 3 * (size_t)m_out, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    return e;
}

}  // namespace lv
