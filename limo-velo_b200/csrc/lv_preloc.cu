/*
 * lv_preloc.cu — the scoring kernel of lv_prelocalize: many candidate start poses probed against the map's block table.
 *
 * Grid: one CTA per (heading, chunk of kPrelocPosPerCta positions), flattened into blockIdx.x.  A CTA gathers the S scored
 * points, applies its heading's rotation once (three dot3f rows per point, 12 B each, kept in shared memory: 48 KB at
 * S = 4096) and then lets each warp take one position offset at a time: every lane adds the translation to its points, probes
 * the block table (16 MB at 1 M map points: L2-resident on an H100) and tests the voxel's occupancy bit; the warp sums with
 * __reduce_add_sync.  Lane 0 writes the score (when asked for) and folds the candidate's selection key into the winner with
 * one atomicMax, so the winner does not depend on the order in which CTAs run.  Arithmetic: lv_preloc.h.
 */
#include "lv_internal.h"
#include "lv_preloc.h"

namespace lv {

namespace {

__global__ void __launch_bounds__(kPrelocThreads) lv_preloc_kernel(PrelocArgs a) {
    extern __shared__ float rows[];                      /* [3][S] */
    const int64_t chunks = (a.positions + kPrelocPosPerCta - 1) / kPrelocPosPerCta;
    const int64_t h = (int64_t)blockIdx.x / chunks;      /* heading index k + K */
    const int64_t q0 = ((int64_t)blockIdx.x % chunks) * kPrelocPosPerCta;
    const int S = a.S;
    Rt32 F;
    LV_UNROLL
    for (int c = 0; c < 9; ++c) F.R[c] = __ldg(a.frames + 12 * h + c);
    LV_UNROLL
    for (int c = 0; c < 3; ++c) F.t[c] = __ldg(a.frames + 12 * h + 9 + c);
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
        const int64_t p = preloc_point_index(s, a.n, S);
        float r[3];
        preloc_rows(F, __ldg(a.xyz + 3 * p), __ldg(a.xyz + 3 * p + 1), __ldg(a.xyz + 3 * p + 2), r);
        rows[s] = r[0];
        rows[S + s] = r[1];
        rows[2 * S + s] = r[2];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t q1 = q0 + kPrelocPosPerCta < a.positions ? q0 + kPrelocPosPerCta : a.positions;
    for (int64_t q = q0 + warp; q < q1; q += kPrelocThreads / 32) {
        const float4 o = __ldg(a.offsets + q);
        const float t[3] = {fadd(F.t[0], o.x), fadd(F.t[1], o.y), fadd(F.t[2], o.z)};
        uint32_t cnt = 0;
        for (int s = lane; s < S; s += 32) cnt += (uint32_t)preloc_hit(a.map, rows[s], rows[S + s], rows[2 * S + s], t);
        const uint32_t score = __reduce_add_sync(0xFFFFFFFFu, cnt);
        if (lane == 0) {
            const int64_t idx = h * a.positions + q;
            if (a.scores) a.scores[idx] = (int32_t)score;
            const int64_t w = 2 * a.I + 1;
            const uint64_t key = preloc_key((int32_t)score, h - a.K, q / w - a.I, q % w - a.I, a.I, idx);
            atomicMax(a.best, (unsigned long long)key);
        }
    }
}

}  // namespace

cudaError_t launch_preloc(const PrelocArgs& a, cudaStream_t st, int* launches) {
    const size_t smem = sizeof(float) * 3 * (size_t)a.S;
    const cudaError_t e = cudaFuncSetAttribute(lv_preloc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               (int)(sizeof(float) * 3 * kPrelocMaxPoints));
    if (e != cudaSuccess) return e;
    const int64_t chunks = (a.positions + kPrelocPosPerCta - 1) / kPrelocPosPerCta;
    lv_preloc_kernel<<<(unsigned)(a.headings * chunks), kPrelocThreads, smem, st>>>(a);
    *launches += 1;
    return cudaGetLastError();
}

}  // namespace lv
