/*
 * lv_preloc_global.cu — the kernels of lv_prelocalize_global: the occupancy summary of the map, cell bounds and exact cell
 * scores.  The schedule that decides which cells to launch runs on the host (lv_preloc_bound.h, PrelocSearch).
 *
 *   occ_extent   one thread per block slot: the occupied voxels' extent (atomicMin / atomicMax)
 *   occ_bits     one thread per block slot: every occupied voxel sets its bit in each bitmap level (atomicOr)
 *   bounds       one warp per cell: each lane rotates its points (preloc_rows), forms their voxel boxes over the cell
 *                (preloc_bound_point) and tests them; the warp sums with __reduce_add_sync
 *   exact        one CTA per cell: the rotated points in shared memory as in lv_preloc.cu, one warp per position, the
 *                offset computed in the kernel with preloc_offset, preloc_hit per point; the CTA keeps the best candidate
 *                under the tie rule (a total order, so the result does not depend on which warp finishes first)
 */
#include "lv_internal.h"
#include "lv_preloc_bound.h"

namespace lv {

namespace {

__global__ void occ_extent_kernel(VoxelMapView m, uint32_t bslots, uint32_t* ext) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= bslots) return;
    const uint4 e = m.btable[slot];
    const uint64_t mask = (uint64_t)e.z | ((uint64_t)e.w << 32);
    if ((e.x & e.y) == 0xFFFFFFFFu || !mask) return;
    uint32_t lo[3], hi[3];
    occ_block_range((uint64_t)e.x | ((uint64_t)e.y << 32), mask, lo, hi);
    for (int a = 0; a < 3; ++a) {
        atomicMin(ext + a, lo[a]);
        atomicMax(ext + 3 + a, hi[a]);
    }
}

__global__ void occ_bits_kernel(PrelocOcc o, uint32_t bslots, uint32_t* bits) {
    const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;
    if (slot >= bslots) return;
    const uint4 e = o.map.btable[slot];
    uint64_t mask = (uint64_t)e.z | ((uint64_t)e.w << 32);
    if ((e.x & e.y) == 0xFFFFFFFFu) return;
    const uint32_t bx = e.x & 0x1FFFFFu, by = (uint32_t)(((uint64_t)e.x | ((uint64_t)e.y << 32)) >> 21) & 0x1FFFFFu,
                   bz = (e.y >> 10) & 0x1FFFFFu;
    while (mask) {
        const int v = __ffsll((long long)mask) - 1;
        mask &= mask - 1;
        const uint32_t x = 4 * bx + (v & 3), y = 4 * by + ((v >> 2) & 3), z = 4 * bz + (v >> 4);
        for (int l = o.m0; l <= o.M; ++l) {
            const uint64_t b = occ_bit(o, l, x, y, z);
            atomicOr(bits + o.off[l] + (b >> 5), 1u << (b & 31));
        }
    }
}

__device__ __forceinline__ void load_frame(const float* frames, int64_t h, Rt32& F) {
    LV_UNROLL
    for (int c = 0; c < 9; ++c) F.R[c] = __ldg(frames + 12 * h + c);
    LV_UNROLL
    for (int c = 0; c < 3; ++c) F.t[c] = __ldg(frames + 12 * h + 9 + c);
}

__global__ void __launch_bounds__(kPrelocGlobalThreads) preloc_bounds_kernel(PrelocGlobalArgs a) {
    const int lane = threadIdx.x & 31;
    const int64_t item = (int64_t)blockIdx.x * (kPrelocGlobalThreads / 32) + (threadIdx.x >> 5);
    if (item >= a.count) return;
    const PrelocCell c = a.cells[item];
    Rt32 F;
    load_frame(a.frames, c.h, F);
    int64_t i0, i1, j0, j1;
    preloc_cell_range(c, a.I, &i0, &i1, &j0, &j1);
    float tlo[3], thi[3];
    preloc_cell_t(a.ax, F.t, a.step, i0, i1, j0, j1, tlo, thi);
    uint32_t cnt = 0;
    for (int s = lane; s < a.S; s += 32) {
        const int64_t p = preloc_point_index(s, a.n, a.S);
        float r[3];
        preloc_rows(F, __ldg(a.xyz + 3 * p), __ldg(a.xyz + 3 * p + 1), __ldg(a.xyz + 3 * p + 2), r);
        cnt += (uint32_t)preloc_bound_point(a.occ, r, tlo, thi);
    }
    const uint32_t b = __reduce_add_sync(0xFFFFFFFFu, cnt);
    if (lane == 0) a.bounds[item] = (int32_t)b;
}

__global__ void __launch_bounds__(kPrelocGlobalThreads) preloc_exact_kernel(PrelocGlobalArgs a) {
    extern __shared__ float rows[];                      /* [3][S] */
    __shared__ PrelocBest wbest[kPrelocGlobalThreads / 32];
    const PrelocCell c = a.cells[blockIdx.x];
    const int S = a.S;
    Rt32 F;
    load_frame(a.frames, c.h, F);
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        const int64_t p = preloc_point_index(s, a.n, S);
        float r[3];
        preloc_rows(F, __ldg(a.xyz + 3 * p), __ldg(a.xyz + 3 * p + 1), __ldg(a.xyz + 3 * p + 2), r);
        rows[s] = r[0];
        rows[S + s] = r[1];
        rows[2 * S + s] = r[2];
    }
    __syncthreads();
    int64_t i0, i1, j0, j1;
    preloc_cell_range(c, a.I, &i0, &i1, &j0, &j1);
    const int64_t nj = j1 - j0 + 1, npos = (i1 - i0 + 1) * nj;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    PrelocBest best;
    best.score = -1; best.pad_ = 0; best.tie = 0; best.idx = 0;
    for (int64_t q = warp; q < npos; q += kPrelocGlobalThreads / 32) {
        const int64_t i = i0 + q / nj, j = j0 + q % nj;
        float o[3];
        preloc_offset(a.ax, dmul((double)i, (double)a.step), dmul((double)j, (double)a.step), o);
        const float t[3] = {fadd(F.t[0], o[0]), fadd(F.t[1], o[1]), fadd(F.t[2], o[2])};
        uint32_t cnt = 0;
        for (int s = lane; s < S; s += 32) cnt += (uint32_t)preloc_hit(a.occ.map, rows[s], rows[S + s], rows[2 * S + s], t);
        const uint32_t score = __reduce_add_sync(0xFFFFFFFFu, cnt);
        const PrelocBest b = preloc_best_of((int32_t)score, c.h - a.K, i, j, a.I, a.K);
        if (preloc_better(b, best)) best = b;
    }
    if (lane == 0) wbest[warp] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        PrelocBest b = wbest[0];
        for (int w = 1; w < kPrelocGlobalThreads / 32; ++w)
            if (preloc_better(wbest[w], b)) b = wbest[w];
        a.best[blockIdx.x] = b;
    }
}

}  // namespace

cudaError_t launch_occ_extent(const VoxelMapView& m, uint32_t bslots, uint32_t* ext, cudaStream_t st, int* launches) {
    occ_extent_kernel<<<(bslots + 255) / 256, 256, 0, st>>>(m, bslots, ext);
    *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_occ_bits(const PrelocOcc& o, uint32_t bslots, uint32_t* bits, cudaStream_t st, int* launches) {
    occ_bits_kernel<<<(bslots + 255) / 256, 256, 0, st>>>(o, bslots, bits);
    *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_preloc_bounds(const PrelocGlobalArgs& a, cudaStream_t st, int* launches) {
    const int64_t per = kPrelocGlobalThreads / 32;
    preloc_bounds_kernel<<<(unsigned)((a.count + per - 1) / per), kPrelocGlobalThreads, 0, st>>>(a);
    *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_preloc_exact(const PrelocGlobalArgs& a, cudaStream_t st, int* launches) {
    const cudaError_t e = cudaFuncSetAttribute(preloc_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)(sizeof(float) * 3 * kPrelocMaxPoints));
    if (e != cudaSuccess) return e;
    preloc_exact_kernel<<<(unsigned)a.count, kPrelocGlobalThreads, sizeof(float) * 3 * (size_t)a.S, st>>>(a);
    *launches += 1;
    return cudaGetLastError();
}

}  // namespace lv
