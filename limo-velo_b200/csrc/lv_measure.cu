/*
 * lv_measure.cu — the kernels of one h-evaluation of the measurement model and of the IESKF step.
 *
 * Replaces, per input point, the chain (reference paths relative to the LIMO-Velo tree)
 *   Mapper::match                 src/Modules/Mapper.cpp:40-56       world transform
 *   KD_TREE::Nearest_Search       include/ikd-Tree/ikd_Tree/ikd_Tree.cpp:426-461   exact 5-NN
 *   Plane::Plane / estimate_plane src/Objects/Plane.cpp:19-55, src/Utils/Utils.cpp:32-66
 *   Match::Match                  src/Objects/Match.cpp:18-22
 *   Localizator::calculate_H      src/Modules/Localizator.cpp:29-57
 * the reduction IKFoM performs on its output,
 *   HTH = h_x^T h_x, h_x^T h      esekfom.hpp:1723,1727
 * and the 23x23 algebra between two evaluations (esekfom.hpp:1647-1817, csrc/lv_ieskf.h).
 *
 * Kernels of one evaluation (DESIGN.md 4): lv_reuse_kernel (evaluations after the first: keep the neighbours the
 * exact search provably returns again), lv_search_kernel (exact 5-NN at level 0, thin, 4 or 8 lanes per query),
 * lv_search_rings_kernel (the queries level 0 cannot certify, one warp each), lv_fit_kernel (plane fit, Jacobian
 * row, the 78 + 12 unique normal-equation sums per block in a fixed order; one spare block runs ieskf_prepare),
 * lv_ieskf_step_kernel (one block: reduction of the partials, gain, dx, next frame, loop control).  H (Nm x 12
 * fp64) is never materialised.  Inside an update every kernel is launched with programmatic dependent launch and
 * the whole update is replayed as one CUDA graph (lv_capi.cu).
 *
 * Bound: L2 / HBM gather LATENCY, not bandwidth (algorithmic traffic 72 B per point: 12 B query + 5 x 12 B
 * neighbours); no tensor-core-shaped work.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>

#ifdef LV_STEP_TIMING
__device__ unsigned long long g_probes[2];     /* total hash probes, number of lookups that needed more than 8 */
#ifdef __CUDA_ARCH__
#define LV_PROBE_COUNT() do { atomicAdd(&g_probes[0], 1ull); } while (0)
#endif
#endif
#ifdef LV_STEP_TIMING   /* tuning build only: per-phase clocks of the step kernel */
__device__ long long g_step_clk[64];
#ifdef __CUDA_ARCH__
#define LV_CK(k) do { if (threadIdx.x == 0) g_step_clk[k] = clock64(); } while (0)
#define LV_TK(k) do { g_step_clk[k] = clock64(); } while (0)
#define LV_FK(k) do { if (threadIdx.x == 0 && blockIdx.x == 1) g_step_clk[k] = clock64(); } while (0)
#endif
#endif
#ifndef LV_FK
#define LV_FK(k)
#endif

#include "lv_internal.h"
#include "lv_predict.h"

#ifdef LV_STEP_TIMING   /* tuning build only: wall-clock timeline of the kernels of an update (graph + PDL included) */
__device__ unsigned long long g_tl[5][8][8];   /* [scheduled | past the wait | end (thread 0) | last block past the wait | end (any warp)][evaluation][kind], ns */
__device__ __forceinline__ unsigned long long lv_gt() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define LV_TL_SCHED() const unsigned long long tl_s_ = lv_gt()
#define LV_TL_WORK(c, kind) const int tl_e_ = (c)->n_evals & 7; if (threadIdx.x == 0) { atomicMin(&g_tl[0][tl_e_][kind], tl_s_); const unsigned long long tw_ = lv_gt(); atomicMin(&g_tl[1][tl_e_][kind], tw_); atomicMax(&g_tl[3][tl_e_][kind], tw_); }
#define LV_TL_END(kind) do { if (threadIdx.x == 0) atomicMax(&g_tl[2][tl_e_][kind], lv_gt()); if ((threadIdx.x & 31) == 0) atomicMax(&g_tl[4][tl_e_][kind], lv_gt()); } while (0)
#else
#define LV_TL_SCHED()
#define LV_TL_WORK(c, kind)
#define LV_TL_END(kind)
#endif

namespace lv {

/* the 90 (a, b) products each block accumulates: 78 upper-triangle entries of HTH, then 12 of HTh
 * (b = 12 selects h) */
__constant__ uint8_t c_pair_a[90];
__constant__ uint8_t c_pair_b[90];
/* constant memory is per device: the first handle created on a device copies the table on its own stream and waits for the
 * copy before it marks the device ready, all under the lock, so a handle created at the same time by another thread either
 * waits for that copy or finds it on the device */
static std::mutex g_pairs_mutex;
static bool g_pairs_ready[64] = {false};    /* guarded by g_pairs_mutex */

static cudaError_t init_pairs(cudaStream_t st) {
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) return err;
    if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
    std::lock_guard<std::mutex> lock(g_pairs_mutex);
    if (g_pairs_ready[dev]) return cudaSuccess;
    uint8_t a[90], b[90];
    int e = 0;
    for (int i = 0; i < 12; ++i)
        for (int j = i; j < 12; ++j) { a[e] = (uint8_t)i; b[e] = (uint8_t)j; ++e; }
    for (int i = 0; i < 12; ++i) { a[e] = (uint8_t)i; b[e] = 12; ++e; }
    err = cudaMemcpyToSymbolAsync(c_pair_a, a, sizeof(a), 0, cudaMemcpyHostToDevice, st);
    if (err == cudaSuccess) err = cudaMemcpyToSymbolAsync(c_pair_b, b, sizeof(b), 0, cudaMemcpyHostToDevice, st);
    if (err == cudaSuccess) err = cudaStreamSynchronize(st);       /* a and b live on this stack */
    if (err == cudaSuccess) g_pairs_ready[dev] = true;
    return err;
}

/* Programmatic dependent launch: every kernel of an update lets its successor's blocks be scheduled early
 * (pdl_trigger) and waits for its predecessor's results (pdl_wait) only after a prologue that touches nothing
 * the predecessor writes.  Every path through a kernel executes pdl_wait() and triggers only AFTER it, so
 * "this kernel runs past its wait" implies "its predecessor is complete", and a prologue may read whatever
 * was written two or more kernels ago.  Without the launch attribute both are no-ops. */
#ifdef LV_NO_GRIDDEP   /* diagnosis build: without the instructions every launch must be a plain one (LV_NO_PDL=1) */
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_trigger() {}
#else
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

/* the sweep of this launch: kernel arguments, or the device-side job of a graph replay */
struct JobView { const float* xyz; int n; int n_tiles; };
__device__ __forceinline__ JobView job_view(const MeasureArgs& a) {
    JobView j;
    if (a.job) { j.xyz = a.job->xyz; j.n = a.job->n; j.n_tiles = a.job->n_tiles; }
    else { j.xyz = a.xyz; j.n = a.n; j.n_tiles = a.n_tiles; }
    return j;
}

#define LV_ROW_STRIDE (kMeasureThreads + 4)   /* 132 doubles = 4 (mod 16): the 8 x 4 fragment loads of the fold below are conflict-free */
#define LV_SEARCH_THREADS 128

__device__ __forceinline__ void store_neighbours(const MeasureArgs& a, int qi, const Top5& t) {
    a.nn_a[qi] = make_int4(t.i0, t.i1, t.i2, t.i3);                  /* positions in the arena, -1 = none */
    a.nn_b[qi] = make_int2(t.i4, __float_as_int(t.d4));
}
/* what a later evaluation needs to reuse this answer (lb <= 0: do not) */
__device__ __forceinline__ void store_ref(const MeasureArgs& a, int qi, const float* g, float lb) {
    if (a.ref) a.ref[qi] = make_float4(g[0], g[1], g[2], lb);
}

/*
 * K1 — search, level 0.  G lanes per query, ONE query per lane group, so the grid holds N * G / 32
 * warps and every SM keeps its full complement of warps in flight: the search is a chain of dependent
 * memory round trips (point -> hash slot -> halo bucket) and only resident warps hide them.  The
 * kernel is thin (no plane fit, ~50 registers).  Per group: one hash probe (all lanes, same address),
 * one contiguous scan of the home voxel's halo bucket (a request of the G lanes covers G x 16
 * contiguous bytes), shuffle merge, certification.  Queries level 0 cannot certify (sparse spot, no
 * slot) are appended to a work list for K1b.
 * History: fused with the fit at 127 registers the search phase dominated every 128-query tile; hard
 * queries finished inside the warp that found them serialised many ring searches in one warp (firing
 * order clusters them).
 * Output, 24 B per query: positions of the 5 neighbours and the 5th squared distance.
 */
template <int G, bool LIST>
__global__ void __launch_bounds__(LV_SEARCH_THREADS) lv_search_kernel(const MeasureArgs a) {
    typedef GroupLanes<G> Grp;
    LV_TL_SCHED();
    pdl_wait();                 /* the predecessor (begin / step / reuse kernel) writes the frame and the lists */
    pdl_trigger();
    LV_TL_WORK(a.ctrl, 2);
    /* the search is a chain of dependent round trips (flags -> point -> slot -> bucket): everything that does
     * not depend on an earlier answer is requested up front, the `done` test included */
    const int done = a.ctrl->done;                      /* update already finished (uniform over the grid) */
    const Rt32 T = a.ctrl->frame.lidar_to_world;        /* uniform loads */
    const JobView jb = job_view(a);
    const int n_redo = LIST ? (int)a.hard_count[2] : 0;
    const int slot = (int)(((int64_t)blockIdx.x * LV_SEARCH_THREADS + threadIdx.x) / G);
    const int listed = LIST ? (int)a.redo_list[slot] : 0;   /* redo_list holds max_points entries: always readable */
    if (done) return;
    int qi = slot;
    bool have = slot < jb.n;
    if (LIST) {                 /* only the queries lv_reuse_kernel handed back */
        if ((int)blockIdx.x * (LV_SEARCH_THREADS / G) >= n_redo) return;
        have = slot < n_redo;
        qi = have ? listed : 0;
    }
    float g[3] = {0.f, 0.f, 0.f};
    uint32_t bs = 0, bc = 0, vox[3] = {0u, 0u, 0u};
    int st = 0;                       /* 0 no query / not finite, 1 bucket, 2 no level-0 slot */
    if (have) {
        rt_apply(T, jb.xyz[3 * qi], jb.xyz[3 * qi + 1], jb.xyz[3 * qi + 2], g);   /* Mapper.cpp:51 */
        const bool finite = (fabsf(g[0]) < 1e9f) && (fabsf(g[1]) < 1e9f) && (fabsf(g[2]) < 1e9f);
        if (finite) st = level0_probe(a.map, g[0], g[1], g[2], &bs, &bc, vox) >= 0 ? 1 : 2;
    }
    Top5 t;
    float region = 0.f;
    const bool settled = level0_scan<Grp>(a.map, g[0], g[1], g[2], a.max_d2, bs, bc, st == 1, t, &region, vox);
    if (have && (threadIdx.x & (G - 1)) == 0) {
        store_neighbours(a, qi, t);
        const bool hard = st == 2 || (st == 1 && !settled);
        store_ref(a, qi, g, (st == 1 && settled) ? outsider_bound(t.d5, region) : 0.f);
        if (hard) {
            const uint32_t b = blockIdx.x % kHardBuckets;
            a.hard_list[(size_t)b * a.hard_seg + atomicAdd(a.hard_count + 4 + b, 1u)] = (uint32_t)qi;
        }
    }
    LV_TL_END(2);
}

/*
 * Kv — reuse.  Evaluations after the first of an update: the iterate moved by millimetres, the map not at all.
 * One thread per query re-measures its five stored neighbours from the new world position and keeps them when
 * query_reusable() proves the exact search would return the same five (lv_voxel_search.h); the others go to
 * the redo list and through the search kernels as usual.  Results are identical either way.
 */
__global__ void __launch_bounds__(128) lv_reuse_kernel(const MeasureArgs a) {
    /* Before the wait: everything but the new frame.  The sweep, the stored neighbours (written by the previous
     * evaluation's search kernels, three or more kernels ago) and the map are fetched while the step kernel
     * still runs; after the wait only the frame is missing. */
    LV_TL_SCHED();
    const JobView jb = job_view(a);
    const int qi = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    const bool have = qi < jb.n;
    float p[3] = {0.f, 0.f, 0.f}, q[5][3];
    float ref[4] = {0.f, 0.f, 0.f, 0.f};
    int id[5] = {-1, -1, -1, -1, -1};
    bool cand = false;
    if (have) {
        p[0] = jb.xyz[3 * qi]; p[1] = jb.xyz[3 * qi + 1]; p[2] = jb.xyz[3 * qi + 2];
        const float4 r4 = a.ref[qi];
        const int4 na = a.nn_a[qi];
        const int2 nb = a.nn_b[qi];
        ref[0] = r4.x; ref[1] = r4.y; ref[2] = r4.z; ref[3] = r4.w;
        cand = r4.w > 0.f && nb.x >= 0;
        if (cand) {
            id[0] = na.x; id[1] = na.y; id[2] = na.z; id[3] = na.w; id[4] = nb.x;
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                const float4 v = load_point(a.map.arena + id[k]);
                q[k][0] = v.x; q[k][1] = v.y; q[k][2] = v.z;
            }
        }
    }
    pdl_wait();                 /* the step kernel before us writes the frame and the done flag */
    pdl_trigger();
    LV_TL_WORK(a.ctrl, 1);
    if (a.ctrl->done) return;
    bool redo = false;
    if (have) {
        const Rt32& T = a.ctrl->frame.lidar_to_world;
        float g[3];
        rt_apply(T, p[0], p[1], p[2], g);
        redo = true;
        Top5 t;
        if (cand && query_reusable(ref, g, q, id, a.max_d2, t)) {
            store_neighbours(a, qi, t);
            redo = false;
        }
    }
    /* one atomic per warp */
    const unsigned m = __ballot_sync(0xffffffffu, redo);
    if (m) {
        const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(a.hard_count + 2, (uint32_t)__popc(m));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (redo) a.redo_list[base + (uint32_t)__popc(m & ((1u << lane) - 1u))] = (uint32_t)qi;
    }
    LV_TL_END(1);
}

/* One warp per hard query and a query costs ~10 dependent memory round trips, so the grid gives every hard query of a sweep its
 * own warp (a 65 536-point sweep has ~1 200): 5 blocks of 4 warps are resident per SM (43.5 KB of shared memory
 * each with the per-block reserve: 217 KB of the H100's 228 KB; 96 registers: 61 440 of 65 536). */
enum { kRingsGrid = kNumSMs * 5 };
/*
 * K1b — search beyond ring 1: one WARP per query K1 could not certify (knn5_rings).  The work list
 * length lives on the device; a fixed grid strides over it, so no host round trip is needed.
 */
__global__ void __launch_bounds__(128) lv_search_rings_kernel(const MeasureArgs a) {
    /* flags, frame and job were written two or more kernels ago: safe to fetch while the search still runs
     * (a kernel triggers its successor only after its own wait, so "two kernels ago" is complete by now) */
    LV_TL_SCHED();
    const int done = a.ctrl->done;
    const JobView jb = job_view(a);
    const Rt32 T = a.ctrl->frame.lidar_to_world;
    pdl_wait();                 /* the search kernel's work list and uncertified answers */
    pdl_trigger();
    LV_TL_WORK(a.ctrl, 3);
    if (done) return;
    /* the 32 segment lengths, one per lane, and their prefix sums */
    const int lane = threadIdx.x & 31;
    const uint32_t cnt = a.hard_count[4 + lane];
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += v;
    }
    const uint32_t n_hard = __shfl_sync(0xffffffffu, incl, 31);
    __shared__ RingScratch s_ring[4];                  /* one per warp of the block */
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t h = warp; h < n_hard; h += n_warps) {
        int lo = 0;                                     /* first segment whose inclusive prefix exceeds h */
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const uint32_t v = __shfl_sync(0xffffffffu, incl, lo + step - 1);
            if (v <= h) lo += step;
        }
        const uint32_t before = __shfl_sync(0xffffffffu, incl - cnt, lo);
        const int qi = (int)a.hard_list[(size_t)lo * a.hard_seg + (h - before)];
        float g[3];
        rt_apply(T, jb.xyz[3 * qi], jb.xyz[3 * qi + 1], jb.xyz[3 * qi + 2], g);
        const int2 prev = a.nn_b[qi];   /* level 0's (uncertified) 5th distance bounds the answer from above */
        Top5 u;
        float region = 0.f;
        __syncwarp();
        knn5_rings_warp(a.map, g[0], g[1], g[2], a.max_d2, prev.x >= 0 ? __int_as_float(prev.y) : a.max_d2, u, &region,
                        &s_ring[threadIdx.x >> 5]);
        if ((threadIdx.x & 31) == 0) {
            store_neighbours(a, qi, u);
            store_ref(a, qi, g, outsider_bound(u.d5, region));
        }
    }
    LV_TL_END(3);
}

/*
 * K2 — fit, row, reduce.  One thread per query, one tile = kMeasureThreads queries.
 *   fit + row   gates (Plane.cpp:36-43), 5x3 QR plane fit, residual, Jacobian row
 *   reduce      the 90 unique sums of H^T H and H^T h over the tile, fixed order; H (Nm x 12 fp64) is
 *               never materialised
 */
/* ieskf_prepare() of the iterate being measured, in one spare block (see lv_ieskf.h) */
__device__ __noinline__ void prepare_block(UpdateCtrl* c) {
    __shared__ PrepWork s_prep;
    ExecBlock ex;
    ieskf_prepare(ex, c, &s_prep);
}

__global__ void __launch_bounds__(kMeasureThreads, 4) lv_fit_kernel(const MeasureArgs a) {
    LV_TL_SCHED();
    /* prologue on data written two or more kernels ago (flags, frame, iterate): runs while the searches finish */
    const int done = a.ctrl->done;
    /* with a.prep the grid has one extra block in front; it is dispatched first and is done long before
     * the measurement blocks, so the iterate-only algebra costs the update no time of its own */
    const int n_blocks = a.prep ? (int)gridDim.x - 1 : (int)gridDim.x;
    const int bid = a.prep ? (int)blockIdx.x - 1 : (int)blockIdx.x;
    if (bid < 0) {
        if (!done) prepare_block(a.prep);
        pdl_wait();
        pdl_trigger();
#ifdef LV_STEP_TIMING
        if (threadIdx.x < 32) {   /* tuning build: how many queries this evaluation searched again, how many went to the ring search */
            unsigned v = a.hard_count[4 + threadIdx.x];
            for (int s_ = 16; s_ > 0; s_ >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s_);
            if (threadIdx.x == 0) { g_tl[2][a.ctrl->n_evals & 7][6] = v; g_tl[2][a.ctrl->n_evals & 7][7] = a.hard_count[2]; }
        }
        __syncthreads();
#endif
        /* the searches of this evaluation are over: reset their counters for the next one */
        if (threadIdx.x < kCounters) a.hard_count[threadIdx.x] = 0u;
        return;
    }

    __shared__ Frame s_frame;
    __shared__ double s_rows[16 * LV_ROW_STRIDE];   /* 13 columns of the tile's rows (12 of H, then h), padded to 16 with zeros */
    __shared__ double s_part[4 * 192];              /* per warp: its share of the three 8 x 8 tiles of [H h]^T [H h] */
    for (int i = threadIdx.x; i < 3 * LV_ROW_STRIDE; i += kMeasureThreads) s_rows[13 * LV_ROW_STRIDE + i] = 0.0;

    {   /* the frame of the current iterate: written by the step kernel, broadcast via smem */
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&a.ctrl->frame);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&s_frame);
        for (int i = threadIdx.x; i < (int)(sizeof(Frame) / 4); i += kMeasureThreads) dst[i] = src[i];
    }
    __syncthreads();
    const int tid = threadIdx.x;
    const JobView jb = job_view(a);
    /* the first tile's world points need only the sweep and the frame: transform them before the wait too */
    float g0[3] = {0.f, 0.f, 0.f};
    {
        const int i = bid * kMeasureThreads + tid;
        if (bid < jb.n_tiles && i < jb.n)
            rt_apply(s_frame.lidar_to_world, jb.xyz[3 * i], jb.xyz[3 * i + 1], jb.xyz[3 * i + 2], g0);
    }
    LV_FK(56);
    pdl_wait();                 /* the neighbour lists */
    pdl_trigger();
    LV_TL_WORK(a.ctrl, 4);
    if (done) return;
    LV_FK(57);

    double acc = 0.0;
    int count = 0;

    for (int tile = bid; tile < jb.n_tiles; tile += n_blocks) {
        const int i = tile * kMeasureThreads + tid;
        bool chosen = false;
        double row[12], hval = 0.0;
        if (i < jb.n) {
            float g[3] = {g0[0], g0[1], g0[2]};
            if (tile != bid) rt_apply(s_frame.lidar_to_world, jb.xyz[3 * i], jb.xyz[3 * i + 1], jb.xyz[3 * i + 2], g);
            const int4 na = a.nn_a[i];
            const int2 nb = a.nn_b[i];
            const float d4 = __int_as_float(nb.y);
            float abcd[4] = {0.f, 0.f, 0.f, 0.f};
            float dist = 0.f;
            float q[5][3];
            float dsq[5] = {INFINITY, INFINITY, INFINITY, INFINITY, INFINITY};
            int orig[5] = {-1, -1, -1, -1, -1};
            const bool full = nb.x >= 0;
            if (full) {
                const float4* src = a.map.arena;
                const float4 q0 = load_point(src + na.x), q1 = load_point(src + na.y), q2 = load_point(src + na.z),
                             q3 = load_point(src + na.w), q4 = load_point(src + nb.x);
                q[0][0] = q0.x; q[0][1] = q0.y; q[0][2] = q0.z;
                q[1][0] = q1.x; q[1][1] = q1.y; q[1][2] = q1.z;
                q[2][0] = q2.x; q[2][1] = q2.y; q[2][2] = q2.z;
                q[3][0] = q3.x; q[3][1] = q3.y; q[3][2] = q3.z;
                q[4][0] = q4.x; q[4][1] = q4.y; q[4][2] = q4.z;
                orig[0] = __float_as_int(q0.w); orig[1] = __float_as_int(q1.w); orig[2] = __float_as_int(q2.w);
                orig[3] = __float_as_int(q3.w); orig[4] = __float_as_int(q4.w);
                for (int k = 0; k < 5; ++k) dsq[k] = sq_dist(g[0], g[1], g[2], q[k][0], q[k][1], q[k][2]);
                LV_FK(58);
                canonical_neighbour_order(q, dsq, orig);             /* equidistant neighbours: (distance, x, y, z, id) */
                /* Plane.cpp:36-43: 5 neighbours and the farthest closer than MAX_DIST_PLANE */
                if ((double)d4 < a.gate_d2) {
                    chosen = plane_fit(q, a.planes_threshold, abcd);               /* Plane.cpp:45-55 */
                    if (chosen) {
                        dist = plane_dist(abcd, g);                                /* Match.cpp:21 */
                        jacobian_row(s_frame, g, abcd, dist, a.estimate_extrinsics != 0, row, &hval);
                    } else {
                        abcd[0] = abcd[1] = abcd[2] = abcd[3] = 0.f;
                    }
                }
            }
            if (a.valid) a.valid[i] = chosen ? 1 : 0;
            if (a.g_world) { a.g_world[3 * i] = g[0]; a.g_world[3 * i + 1] = g[1]; a.g_world[3 * i + 2] = g[2]; }
            if (a.nn_idx || a.nn_sqd) {
                for (int k = 0; k < 5; ++k) {
                    if (a.nn_idx) a.nn_idx[5 * i + k] = orig[k];
                    if (a.nn_sqd) a.nn_sqd[5 * i + k] = dsq[k];
                }
            }
            if (a.plane) { for (int k = 0; k < 4; ++k) a.plane[4 * i + k] = abcd[k]; }
            if (a.dist) a.dist[i] = dist;
            if (a.rows) {
                for (int k = 0; k < 12; ++k) a.rows[13 * (size_t)i + k] = chosen ? row[k] : 0.0;
                a.rows[13 * (size_t)i + 12] = chosen ? hval : 0.0;
            }
        }
        LV_FK(59);
        /* stage the row (zeros when rejected), fold the tile into the block's 90 sums */
#pragma unroll
        for (int k = 0; k < 12; ++k) s_rows[k * LV_ROW_STRIDE + tid] = chosen ? row[k] : 0.0;
        s_rows[12 * LV_ROW_STRIDE + tid] = chosen ? hval : 0.0;
        count += __syncthreads_count(chosen ? 1 : 0);
        LV_FK(60);
        {
            /* The tile's 13 x 13 Gram matrix on the fp64 tensor cores (mma.m8n8k4: D = A B + C, A 8x4, B 4x8): 16 x 16 with
             * the padding, three 8 x 8 tiles (00, 01, 11 — it is symmetric), each warp a quarter of the 128 rows.  A lane's A
             * fragment of column-tile I is element (column I*8 + lane/4, row k0 + lane%4) and the B fragment of column-tile J
             * is the same expression with J: two loads feed three MMAs of 256 multiply-adds each.  (The scalar fold — 90
             * threads x 128 x two 8-byte shared loads per multiply-add — waits on the shared-memory wavefronts of all the
             * resident blocks, which reach the fold together; clock64, tools/step_timing.py.) */
            const int lane = tid & 31, w = tid >> 5;
            const double* f0 = s_rows + (lane >> 2) * LV_ROW_STRIDE + 32 * w + (lane & 3);
            const double* f1 = f0 + 8 * LV_ROW_STRIDE;
            double c00a = 0.0, c00b = 0.0, c01a = 0.0, c01b = 0.0, c11a = 0.0, c11b = 0.0;
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                const double a0 = f0[4 * ks], a1 = f1[4 * ks];
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c00a), "+d"(c00b) : "d"(a0), "d"(a0));
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c01a), "+d"(c01b) : "d"(a0), "d"(a1));
                asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c11a), "+d"(c11b) : "d"(a1), "d"(a1));
            }
            double* pt = s_part + w * 192 + (lane >> 2) * 8 + 2 * (lane & 3);   /* C fragment: row lane/4, columns 2 (lane%4), +1 */
            pt[0] = c00a; pt[1] = c00b;
            pt[64] = c01a; pt[65] = c01b;
            pt[128] = c11a; pt[129] = c11b;
        }
        __syncthreads();
        if (tid < 90) {   /* entry (a, b), a <= b: tile 00 / 01 / 11; the warps' shares in warp order */
            const int pa = c_pair_a[tid], pb = c_pair_b[tid];
            const int idx = (pa < 8 ? (pb < 8 ? 0 : 64) : 128) + (pa & 7) * 8 + (pb & 7);
            acc += (s_part[idx] + s_part[192 + idx]) + (s_part[384 + idx] + s_part[576 + idx]);
        }
        __syncthreads();
    }
    LV_FK(61);
    double* out = a.partials + (size_t)bid * kPartialStride;
    if (tid < 90) out[tid] = acc;
    if (tid == 90) out[90] = (double)count;
    /* Pre-reduction: the blocks form groups of kPartialGroup consecutive rows; the block of a group that finishes LAST
     * (a ticket per group) adds the group's rows in row order into one group row.  Which block that is varies, the
     * order of the additions does not, so the result is deterministic; the groups finish at different times and are
     * summed on different SMs while other blocks still work, and the step kernel is left with <= 17 rows instead of
     * kMeasureGridCap (otherwise it pulls ~400 KB of partials through one SM's L2 port). */
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    const int grp = bid / kPartialGroup, r0 = grp * kPartialGroup;
    const int r1 = r0 + kPartialGroup < n_blocks ? r0 + kPartialGroup : n_blocks;
    if (tid == 0) {
        const unsigned ticket = atomicAdd(a.group_tickets + grp, 1u);
        s_last = ticket == (unsigned)(r1 - r0) - 1u ? 1 : 0;
        if (s_last) a.group_tickets[grp] = 0u;          /* nobody else touches it before the next evaluation */
    }
    __syncthreads();
    LV_FK(62);
    if (s_last) {
        __threadfence();
        if (tid < 91) {
            double v[kPartialGroup];
#pragma unroll
            for (int r = 0; r < kPartialGroup; ++r) v[r] = r0 + r < r1 ? __ldcg(a.partials + (size_t)(r0 + r) * kPartialStride + tid) : 0.0;
            double sum = 0.0;
#pragma unroll
            for (int r = 0; r < kPartialGroup; ++r) sum += v[r];
            a.group_rows[(size_t)grp * kPartialStride + tid] = sum;
        }
    }
    LV_FK(63);
    LV_TL_END(4);
}

/* ---- fixed-order reduction of the per-block partials ---------------------------------------- */
/* Warp w of the block owns rows w, w + nwarps, ...; lanes own elements lane, lane+32, lane+64.  Rows are
 * fetched 8 at a time (24 independent loads per lane) and
 * added in row order; then the warp sums are added in warp order.  Deterministic for a given grid. */
__device__ void reduce_partials_block(const double* partials, int n_partials, double* s_tmp /*nwarps*96*/,
                                      double* HTH, double* HTh, int64_t* nm) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    double a0 = 0, a1 = 0, a2 = 0;
    for (int b = warp; b < n_partials; b += 8 * nwarps) {
        double v[8][3];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const int row = b + r * nwarps;
            const double* p = partials + (size_t)row * kPartialStride;
            const bool in = row < n_partials;
            v[r][0] = in ? p[lane] : 0.0;
            v[r][1] = in ? p[lane + 32] : 0.0;
            v[r][2] = in ? p[lane + 64] : 0.0;
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) { a0 += v[r][0]; a1 += v[r][1]; a2 += v[r][2]; }
    }
    s_tmp[warp * 96 + lane] = a0;
    s_tmp[warp * 96 + lane + 32] = a1;
    s_tmp[warp * 96 + lane + 64] = a2;
    __syncthreads();
    if (threadIdx.x < 91) {
        double s = 0;
#pragma unroll 16   /* the loads of a step's 16 warps are issued together, only the additions stay in warp order */
        for (int w = 0; w < nwarps; ++w) s += s_tmp[w * 96 + threadIdx.x];
        const int e = threadIdx.x;
        if (e < 78) {
            const int i = c_pair_a[e], j = c_pair_b[e];
            HTH[i * 12 + j] = s;
            HTH[j * 12 + i] = s;
        } else if (e < 90) {
            HTh[e - 78] = s;
        } else {
            *nm = (int64_t)(s + 0.5);
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kStepThreads) lv_ieskf_step_kernel(UpdateCtrl* c, const IeskfParams prm,
                                                                     const double* partials, int n_partials) {
    /* before the wait: what the previous step (or begin) kernel left, two or more kernels ago */
    static_assert(kStepThreads >= 99 && 2 * kStepThreads >= kN * kN, "one pass for the state, two for P_j");
    LV_TL_SCHED();
    const int t = threadIdx.x;
    const int done = c->done;
    double sv = 0.0;
    if (t < 26) sv = c->x[t];
    else if (t < 52) sv = c->x_prop[t - 26];
    int cv = 0;
    if (t >= 96 && t < 99) cv = t == 96 ? c->n_evals : (t == 97 ? c->t : c->iter);
    pdl_wait();                 /* partials and the prepared P_j / dx_new of the fit kernel */
    pdl_trigger();
    LV_TL_WORK(c, 5);
    if (done) return;
    __shared__ IeskfWork w;
    __shared__ double s_tmp[(kStepThreads / 32) * 96];
    ExecBlock ex;
    LV_CK(0);
    /* ieskf_load(), split: the loads are issued here and parked in shared memory after the reduction, so
     * they are in flight together with the partials */
    const double pj0 = t < kN * kN ? c->P_j[t] : 0.0;
    const double pj1 = t + kStepThreads < kN * kN ? c->P_j[t + kStepThreads] : 0.0;
    if (t >= 52 && t < 75) sv = c->dx_new[t - 52];
    LV_CK(1);
    reduce_partials_block(partials, n_partials, s_tmp, w.HTH, w.HTh, &w.n_matches);
    if (t < kN * kN) w.P[t] = pj0;
    if (t + kStepThreads < kN * kN) w.P[t + kStepThreads] = pj1;
    if (t < 26) w.x[t] = sv;
    else if (t < 52) w.xp[t - 26] = sv;
    else if (t < 75) w.dx_new[t - 52] = sv;
    if (t == 96) { w.n_evals = cv; w.eval_idx = cv < kMaxEvals ? cv : kMaxEvals - 1; }
    if (t == 97) w.t = cv;
    if (t == 98) w.iter = cv;
    __syncthreads();
    LV_CK(2);
    ieskf_step(ex, prm, c, &w);
    LV_TL_END(5);
}

__global__ void __launch_bounds__(kStepThreads) lv_reduce_partials_kernel(const double* partials, int n_partials,
                                                                          double* out) {
    __shared__ double s_tmp[(kStepThreads / 32) * 96];
    __shared__ double HTH[144], HTh[12];
    __shared__ int64_t nm;
    reduce_partials_block(partials, n_partials, s_tmp, HTH, HTh, &nm);
    for (int i = threadIdx.x; i < 144; i += blockDim.x) out[i] = HTH[i];
    if (threadIdx.x < 12) out[144 + threadIdx.x] = HTh[threadIdx.x];
    if (threadIdx.x == 0) out[156] = (double)nm;
}

/* with gate.n the sweep's count comes from device memory (n is then its host-known bound); an update the gate stops finishes
 * here with a status, the state untouched: every later kernel of the update sees done = 1 */
__global__ void __launch_bounds__(256) lv_ieskf_begin_kernel(UpdateCtrl* c, MeasureJob* job, const float* xyz, int n,
                                                             uint32_t* counters, const UpdateGate gate) {
    pdl_trigger();
    if (counters && threadIdx.x < kCounters) counters[threadIdx.x] = 0u;    /* work-list lengths of the measurement kernels */
    const int k = (int)device_count(gate.n, n, gate.words ? &gate.words->err : nullptr);
    if (job && threadIdx.x == 0) {
        job->xyz = xyz;
        job->n = k;
        job->n_tiles = (k + kMeasureThreads - 1) / kMeasureThreads;
    }
    ExecBlock ex;
    ieskf_begin(ex, c);
    if (threadIdx.x == 0) {
        if (gate.n && k < (gate.min_points > 1 ? gate.min_points : 1)) {      /* main.cpp:81 */
            c->status = LV_TOO_FEW_POINTS;
            c->done = 1;
        } else if (gate.map_counters && gate.map_counters[kCtrPoints] == 0u) {  /* Localizator.cpp:24 */
            c->status = LV_EMPTY_MAP;
            c->done = 1;
        } else if (gate.words) {
            gate.words->time_updated = gate.time;                              /* Localizator.cpp:26 */
            gate.words->time_set = 1;
        }
    }
}

/* Localizator::propagate_to (Localizator.cpp:59-75): every IMU sample between two sweeps through esekf::predict, one launch,
 * one thread block; imu = k x 7 doubles (acc, gyro, dt).  The state stays in UpdateCtrl: update -> propagate -> update needs
 * no host round trip. */
__global__ void __launch_bounds__(256) lv_predict_kernel(UpdateCtrl* c, const PredictNoise noise, const double* __restrict__ imu, int k) {
    __shared__ PredictWork w;
    ExecBlock ex;
    LV_PAR(i, kStateLen) w.x[i] = c->x[i];
    LV_PAR(i, kN * kN) w.P[i] = c->P[i];
    ex.sync();
    for (int s = 0; s < k; ++s) predict_step(ex, noise, imu + 7 * s, imu + 7 * s + 3, imu[7 * s + 6], &w);
    LV_PAR(i, kStateLen) c->x[i] = w.x[i];
    LV_PAR(i, kN * kN) c->P[i] = w.P[i];
}

__global__ void lv_set_frame_kernel(UpdateCtrl* c) {
    if (threadIdx.x == 0) {
        make_frame(c->x, &c->frame);
        c->done = 0;
    }
}

__global__ void lv_l2_flush_kernel(uint4* buf, size_t n16) {
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride)
        buf[i] = make_uint4((unsigned)i, 1u, 2u, 3u);
}

/* ---- launchers ------------------------------------------------------------------------------- */
int measure_grid(int n) {
    const int tiles = (n + kMeasureThreads - 1) / kMeasureThreads;
    return tiles < kMeasureGridCap ? (tiles > 0 ? tiles : 1) : kMeasureGridCap;
}

cudaError_t measure_init(cudaStream_t st) { return init_pairs(st); }

/* K1 variant of one launch: lanes per query (4 or 8).
 * 4 lanes per query issue a quarter fewer instructions per query than 8 (the prologue is shared by eight queries of a warp
 * instead of four), which pays when a launch has tens of thousands of queries; 8 lanes have the shorter chain per query (a
 * bucket of 36 points is one batch of loads instead of two), which pays on the short work lists of late evaluations and on
 * small sweeps (tools/timeline.py and bench.py's kernel_ms locate the crossover).  So the choice follows the number of queries the launch can expect:
 * all of them in the first evaluation, ~90 % / 45 % / 12 % in evaluations 2 / 3 / 4 of an update with neighbour reuse (cfg1).
 * LV_SEARCH_GROUP=4|8 overrides for tuning runs and tests (read at every direct launch and when a handle's graph is built). */
static int search_group(const MeasureArgs& a, int eval) {
    const char* e = getenv("LV_SEARCH_GROUP");
    if (e) {
        const int group = atoi(e);
        if (group == 4 || group == 8) return group;
    }
    static const double kRedoShare[4] = {1.0, 0.9, 0.45, 0.12};
    const double share = (eval > 0 && a.ref) ? kRedoShare[eval < 3 ? eval : 3] : 1.0;
    return (double)a.n * share >= 40000.0 ? 4 : 8;
}
static int search_grid(const MeasureArgs& a, int group) {
    const int sgrid = (int)(((int64_t)a.n * group + LV_SEARCH_THREADS - 1) / LV_SEARCH_THREADS);
    return sgrid < 1 ? 1 : sgrid;
}
/* <<<>>> with the programmatic-dependent-launch attribute when `pdl` (see pdl_wait above) */
template <class... Params, class... Args>
static cudaError_t launch_k(void (*kernel)(Params...), unsigned grid, unsigned block, cudaStream_t st, bool pdl, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid, 1, 1);
    cfg.blockDim = dim3(block, 1, 1);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = pdl ? at : nullptr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, Params(args)...);
}

template <bool LIST>
static void launch_search(const MeasureArgs& a, int group, int sgrid, cudaStream_t st, bool pdl) {
    switch (group) {
        case 4: launch_k(lv_search_kernel<4, LIST>, sgrid, LV_SEARCH_THREADS, st, pdl, a); break;
        default: launch_k(lv_search_kernel<8, LIST>, sgrid, LV_SEARCH_THREADS, st, pdl, a); break;
    }
}

cudaError_t launch_measure(const MeasureArgs& a, int grid, cudaStream_t st, const MeasureProbe* probe, int reuse, int pdl) {
    const int group = search_group(a, reuse);          /* reuse = index of the evaluation within its update */
    const int sgrid = search_grid(a, group);
    /* work-list length, a spare word, redo-list length; inside an update with pdl the kernels
     * reset them themselves (begin kernel, fit kernel) so that every node of the update is a kernel */
    if (!pdl) cudaMemsetAsync(a.hard_count, 0, kCounters * sizeof(uint32_t), st);
    if (reuse && a.ref) {
        if (probe) probe->at(probe->ctx, 4);
        launch_k(lv_reuse_kernel, (a.n + 127) / 128 > 0 ? (a.n + 127) / 128 : 1, 128, st, pdl != 0, a);
        if (probe) probe->at(probe->ctx, 0);
        launch_search<true>(a, group, sgrid, st, pdl != 0);
    } else {
        if (probe) probe->at(probe->ctx, 0);
        launch_search<false>(a, group, sgrid, st, pdl != 0);
    }
    static const bool dbg_sync = getenv("LV_DEBUG_SYNC") != nullptr;   /* diagnosis: name the kernel that does not finish */
    if (dbg_sync) { cudaStreamSynchronize(st); fprintf(stderr, "[lv] search done\n"); fflush(stderr); }
    if (probe) probe->at(probe->ctx, 1);
    launch_k(lv_search_rings_kernel, kRingsGrid, 128, st, pdl != 0, a);
    if (dbg_sync) { cudaStreamSynchronize(st); fprintf(stderr, "[lv] search-rings done\n"); fflush(stderr); }
    if (probe) probe->at(probe->ctx, 2);
    launch_k(lv_fit_kernel, grid + (a.prep ? 1 : 0), kMeasureThreads, st, pdl != 0, a);
    if (dbg_sync) { cudaStreamSynchronize(st); fprintf(stderr, "[lv] fit done\n"); fflush(stderr); }
    if (probe) probe->at(probe->ctx, 3);
    return cudaGetLastError();
}
cudaError_t launch_ieskf_begin(UpdateCtrl* c, MeasureJob* job, const float* xyz, int n, uint32_t* counters, const UpdateGate& gate,
                               cudaStream_t st) {
    lv_ieskf_begin_kernel<<<1, 256, 0, st>>>(c, job, xyz, n, counters, gate);
    return cudaGetLastError();
}
const void* ieskf_begin_kernel_ptr() { return (const void*)lv_ieskf_begin_kernel; }
cudaError_t launch_ieskf_step(UpdateCtrl* c, const IeskfParams& prm, const double* partials, int n_partials,
                              cudaStream_t st, int pdl) {
    launch_k(lv_ieskf_step_kernel, 1, kStepThreads, st, pdl != 0, c, prm, partials, n_partials);
    return cudaGetLastError();
}
cudaError_t launch_reduce_partials(const double* partials, int n_partials, double* out, cudaStream_t st) {
    lv_reduce_partials_kernel<<<1, kStepThreads, 0, st>>>(partials, n_partials, out);
    return cudaGetLastError();
}
cudaError_t launch_predict(UpdateCtrl* c, const PredictNoise& noise, const double* d_imu, int k, cudaStream_t st) {
    lv_predict_kernel<<<1, 256, 0, st>>>(c, noise, d_imu, k);
    return cudaGetLastError();
}
cudaError_t launch_set_frame(UpdateCtrl* c, cudaStream_t st) {
    lv_set_frame_kernel<<<1, 32, 0, st>>>(c);
    return cudaGetLastError();
}
cudaError_t launch_l2_flush(void* buf, size_t bytes, cudaStream_t st) {
    lv_l2_flush_kernel<<<kNumSMs * 8, 256, 0, st>>>(reinterpret_cast<uint4*>(buf), bytes / 16);
    return cudaGetLastError();
}

}  // namespace lv

#ifdef LV_STEP_TIMING
extern "C" int lv_debug_step_clocks(long long* out) {
    return (int)cudaMemcpyFromSymbol(out, g_step_clk, sizeof(long long) * 64);
}
extern "C" int lv_debug_probes(unsigned long long* out) {
    cudaDeviceSynchronize();
    int e = (int)cudaMemcpyFromSymbol(out, g_probes, sizeof(unsigned long long) * 2);
    unsigned long long z[2] = {0, 0};
    cudaMemcpyToSymbol(g_probes, z, sizeof(z));
    return e;
}
/* out[5][8][8]; resets the table (starts to ~0, ends to 0) */
extern "C" int lv_debug_timeline(unsigned long long* out) {
    cudaDeviceSynchronize();
    int e = (int)cudaMemcpyFromSymbol(out, g_tl, sizeof(unsigned long long) * 320);
    unsigned long long init[320];
    for (int i = 0; i < 64; ++i) { init[i] = ~0ull; init[64 + i] = ~0ull; init[128 + i] = 0ull; init[192 + i] = 0ull; init[256 + i] = 0ull; }
    cudaMemcpyToSymbol(g_tl, init, sizeof(init));
    return e;
}
#endif
