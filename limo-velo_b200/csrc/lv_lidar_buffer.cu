/*
 * lv_lidar_buffer.cu — Accumulator::BUFFER_L in HBM: Buffer::push (src/Objects/Buffer.cpp:26-28, one message at a time as
 * Accumulator::receive_lidar adds it, src/Modules/Accumulator.cpp:39-48), Accumulator::get (include/Headers/Accumulator.hpp:61-74)
 * and Buffer::clear(t) (Buffer.cpp:66-70).  The index arithmetic, the binary search and the predicates are lv_lidar_buffer.h.
 *
 *   push   a grid copies *d_n points to positions [tail, tail + n) (slot p % cap); the last block to finish advances tail.  When
 *          they do not fit nothing is written and kAsyncLidarFull is raised (the reference's deque has no bound).
 *   get    one block: thread 0 runs the reference's binary search for t2 (its exact probe sequence, which matters on unsorted
 *          content); the block then walks down from that position chunk by chunk until a chunk holds a point with t1 > time (the
 *          walk's break: the highest such position, a max-reduction), counting the points with t2 >= time above it; a second pass
 *          upward compacts them into the output in ascending position, i.e. oldest -> newest as push_front leaves them.
 *   clear  one block walks up from head chunk by chunk until a point fails `t >= time` (the lowest such position, a
 *          min-reduction); head moves there, or to tail.
 *   merge  lv_lidar_merge_device_async: a message from any sensor lands where its times belong (three launches, described
 *          above the merge kernels below).
 * Push, get and clear are one launch each; the counters never leave the device.
 * A ring reserved with lv_lidar_reserve_full carries two more float lanes per slot, intensity and range.  Push, get and move are
 * templates on `Lanes`: the <false> instantiations are the xyz + time kernels as they always were, and the <true> ones copy the
 * lanes in the same loop, slot for slot (lidar_copy_lanes).  Clear reads times only and has one form.
 */
#include <cub/block/block_scan.cuh>

#include "lv_internal.h"
#include "lv_lidar_buffer.h"

namespace lv {

enum { kLidarPushThreads = 256, kLidarBlock = 1024 };

/* the lanes of one launch (Lanes = true): intensity and range of the source and of the destination; a NULL source stores 0 */
struct LaneCopy {
    const float* from_i;
    const float* from_r;
    float* to_i;
    float* to_r;
};

template <bool Lanes>
__global__ void __launch_bounds__(kLidarPushThreads) lv_lidar_push_kernel(float* __restrict__ ring_xyz, double* __restrict__ ring_time, int64_t cap,
                                                                          LidarWords* w, const float* __restrict__ xyz,
                                                                          const double* __restrict__ time, const int64_t* __restrict__ d_n,
                                                                          int64_t n_max, uint32_t* err, LaneCopy lanes) {
    const int64_t head = w->head, tail = w->tail;
    const int64_t n = device_count(d_n, n_max, err);
    const bool fits = lidar_fits(head, tail, n, cap);
    if (fits) {
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
            const int64_t s = lidar_slot(tail + i, cap);
            ring_xyz[3 * s] = xyz[3 * i];
            ring_xyz[3 * s + 1] = xyz[3 * i + 1];
            ring_xyz[3 * s + 2] = xyz[3 * i + 2];
            ring_time[s] = time[i];
            if (Lanes) lidar_copy_lanes(lanes.from_i, lanes.from_r, i, lanes.to_i, lanes.to_r, s);
        }
    }
    /* every thread has read the counters before its block takes a ticket: the last block may move tail */
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&w->ticket, 1u) == gridDim.x - 1) {
            w->ticket = 0;
            if (fits) w->tail = tail + n;
            else if (err) atomicOr(err, kAsyncLidarFull);
        }
    }
}

template <bool Lanes>
__global__ void __launch_bounds__(kLidarBlock) lv_lidar_get_kernel(const float* __restrict__ ring_xyz, const double* __restrict__ ring_time,
                                                                   int64_t cap, LidarWords* w, double t1, double t2, float* __restrict__ xyz,
                                                                   double* __restrict__ time, int64_t n_max, int64_t* d_n_out, uint32_t* err,
                                                                   LaneCopy lanes) {
    typedef cub::BlockScan<int, kLidarBlock> Scan;
    __shared__ typename Scan::TempStorage scan;
    __shared__ long long s_top, s_break;
    const int64_t head = w->head, tail = w->tail;
    if (threadIdx.x == 0) {
        s_top = lidar_window_top(ring_time, cap, head, tail, t2);
        s_break = head - 1;                                      /* no break: the walk runs to content.back() */
    }
    __syncthreads();
    const int64_t top = s_top;
    /* down from the top: the highest position with t1 > time, and the kept points above it */
    int64_t count = 0;
    for (int64_t hi = top; hi >= head; hi -= kLidarBlock) {
        const int64_t p = hi - threadIdx.x;
        const bool in = p >= head;
        const double tp = in ? ring_time[lidar_slot(p, cap)] : 0.0;
        const bool brk = in && lidar_breaks(tp, t1);
        if (brk) atomicMax(&s_break, (long long)p);
        const int found = __syncthreads_or(brk);
        const int64_t b = s_break;
        count += __syncthreads_count(in && p > b && lidar_keeps(tp, t2));
        if (found) break;
    }
    const int64_t lo = s_break + 1;
    if (count > n_max) {                                         /* the window does not fit the caller's buffers */
        if (threadIdx.x == 0) {
            w->window = count;
            w->count = 0;
            if (d_n_out) *d_n_out = 0;
            if (err) atomicOr(err, kAsyncLidarWindow);
        }
        return;
    }
    /* up from the break: compaction in ascending position */
    int64_t base = 0;
    for (int64_t p0 = lo; p0 <= top; p0 += kLidarBlock) {
        const int64_t p = p0 + threadIdx.x;
        const int64_t s = lidar_slot(p, cap);
        const bool in = p <= top;
        const double tp = in ? ring_time[s] : 0.0;
        const int keep = (in && lidar_keeps(tp, t2)) ? 1 : 0;
        int off, total;
        Scan(scan).ExclusiveSum(keep, off, total);
        if (keep) {
            const int64_t o = base + off;
            xyz[3 * o] = ring_xyz[3 * s];
            xyz[3 * o + 1] = ring_xyz[3 * s + 1];
            xyz[3 * o + 2] = ring_xyz[3 * s + 2];
            time[o] = tp;
            if (Lanes) lidar_copy_lanes(lanes.from_i, lanes.from_r, s, lanes.to_i, lanes.to_r, o);
        }
        base += total;
        __syncthreads();                                         /* the scan's storage is reused */
    }
    if (threadIdx.x == 0) {
        w->window = count;
        w->count = count;
        if (d_n_out) *d_n_out = count;
    }
}

__global__ void __launch_bounds__(kLidarBlock) lv_lidar_clear_kernel(const double* __restrict__ ring_time, int64_t cap, LidarWords* w, double t) {
    __shared__ long long s_stop;
    const int64_t head = w->head, tail = w->tail;
    if (threadIdx.x == 0) s_stop = tail;                         /* everything pops */
    __syncthreads();
    for (int64_t p0 = head; p0 < tail; p0 += kLidarBlock) {
        const int64_t p = p0 + threadIdx.x;
        const bool stop = p < tail && !lidar_pops(ring_time[lidar_slot(p, cap)], t);
        if (stop) atomicMin(&s_stop, (long long)p);
        if (__syncthreads_or(stop)) break;
    }
    if (threadIdx.x == 0) w->head = s_stop;
}

/* ---- the time-ordered merge (lv_lidar_buffer.h) ----
 * split   block 0 walks down from tail - 1 chunk by chunk, as get does, to the highest position whose time is <= b[0] (a
 *         max-reduction) and checks the order of T_tail, the positions above it; the other blocks check B's order.  The last block
 *         to finish decides the mode (lidar_merge_mode), raises its flag and leaves split, n and mode in the ring's words.
 * stage   a grid copies T_tail into the overlap scratch, so the write below may overwrite it.
 * write   a grid writes positions [s, tail + n): each thread finds its first output by the merge path of its diagonal, then merges
 *         kMergeItems outputs serially; in the append mode it writes B at [tail, tail + n) as the push does.  The last block
 *         advances tail.
 * Three launches whatever the overlap; stage and write do nothing when the merge is refused. */
enum { kMergeThreads = 256, kMergeItems = 8 };

__global__ void __launch_bounds__(kLidarBlock) lv_lidar_merge_split_kernel(const double* __restrict__ ring_time, int64_t cap, LidarWords* w,
                                                                           const double* __restrict__ time, const int64_t* __restrict__ d_n,
                                                                           int64_t n_max, int64_t reserve, uint32_t* err) {
    __shared__ long long s_split;
    const int64_t head = w->head, tail = w->tail;
    const int64_t n = device_count(d_n, n_max, err);
    int bad = 0;
    if (blockIdx.x == 0) {
        if (threadIdx.x == 0) s_split = n > 0 ? head : tail;    /* an empty message changes nothing: no walk */
        __syncthreads();
        const double b0 = n > 0 ? time[0] : 0.0;
        for (int64_t hi = tail - 1; n > 0 && hi >= head; hi -= kLidarBlock) {
            const int64_t p = hi - threadIdx.x;
            const bool in = p >= head;
            const double tp = in ? ring_time[lidar_slot(p, cap)] : 0.0;
            const bool below = in && lidar_merge_below(tp, b0);
            if (below) atomicMax(&s_split, (long long)(p + 1));
            const int found = __syncthreads_or(below);
            if (in && p >= (int64_t)s_split && !lidar_in_order(tp, p + 1 < tail ? ring_time[lidar_slot(p + 1, cap)] : tp)) bad = 1;
            if (found) break;
        }
    } else {
        const int64_t stride = (int64_t)(gridDim.x - 1) * blockDim.x;
        for (int64_t i = (int64_t)(blockIdx.x - 1) * blockDim.x + threadIdx.x; i < n; i += stride)
            if (!lidar_in_order(time[i], i + 1 < n ? time[i + 1] : time[i])) bad = 1;
    }
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) {
        if (bad) atomicOr(&w->merge_bad, 1u);
        if (blockIdx.x == 0) w->merge_split = s_split;
        __threadfence();
        if (atomicAdd(&w->ticket, 1u) == gridDim.x - 1) {
            __threadfence();
            /* written by other blocks: read past L1 */
            const int64_t split = *(volatile int64_t*)&w->merge_split;
            const bool ordered = *(volatile uint32_t*)&w->merge_bad == 0;
            const uint32_t mode = lidar_merge_mode(head, tail, split, n, cap, reserve, ordered);
            w->merge_bad = 0;
            w->merge_n = n;
            w->merge_mode = mode;
            w->ticket = 0;
            if (err) {
                if (mode == kLidarMergeFull) atomicOr(err, kAsyncLidarFull);
                if (mode == kLidarMergeAppend) atomicOr(err, kAsyncLidarUnsorted);
                if (mode == kLidarMergeOverlap) atomicOr(err, kAsyncLidarOverlap);
            }
        }
    }
}

template <bool Lanes>
__global__ void __launch_bounds__(kMergeThreads) lv_lidar_merge_stage_kernel(const float* __restrict__ ring_xyz, const double* __restrict__ ring_time,
                                                                             int64_t cap, const LidarWords* w, float* __restrict__ a_xyz,
                                                                             double* __restrict__ a_time, LaneCopy lanes) {
    if (w->merge_mode != kLidarMergeWrite) return;
    const int64_t split = w->merge_split, m = w->tail - split;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = lidar_slot(lidar_merge_pos(split, k), cap);
        a_xyz[3 * k] = ring_xyz[3 * s];
        a_xyz[3 * k + 1] = ring_xyz[3 * s + 1];
        a_xyz[3 * k + 2] = ring_xyz[3 * s + 2];
        a_time[k] = ring_time[s];
        if (Lanes) lidar_copy_lanes(lanes.from_i, lanes.from_r, s, lanes.to_i, lanes.to_r, k);
    }
}

/* one point into ring slot s: from the scratch (staged, already in the primary frame) or from the message (through T) */
template <bool Lanes>
__device__ __forceinline__ void merge_store(float* ring_xyz, double* ring_time, int64_t s, const float* xyz, const double* time, int64_t i,
                                            bool transform, const Rt32& T, const float* from_i, const float* from_r, const LaneCopy& lanes) {
    float g[3];
    lidar_merge_xyz(transform, T, xyz, i, g);
    ring_xyz[3 * s] = g[0];
    ring_xyz[3 * s + 1] = g[1];
    ring_xyz[3 * s + 2] = g[2];
    ring_time[s] = time[i];
    if (Lanes) lidar_copy_lanes(from_i, from_r, i, lanes.to_i, lanes.to_r, s);
}

/* lanes: the message's (from_*, NULL: 0) and the ring's (to_*); a_lanes: the scratch's (from_*) */
template <bool Lanes>
__global__ void __launch_bounds__(kMergeThreads) lv_lidar_merge_write_kernel(float* __restrict__ ring_xyz, double* __restrict__ ring_time, int64_t cap,
                                                                             LidarWords* w, const float* __restrict__ a_xyz,
                                                                             const double* __restrict__ a_time, const float* __restrict__ xyz,
                                                                             const double* __restrict__ time, bool transform, Rt32 T,
                                                                             LaneCopy lanes, LaneCopy a_lanes) {
    const uint32_t mode = w->merge_mode;
    const int64_t tail = w->tail, split = w->merge_split, n = w->merge_n;
    const int64_t gthreads = (int64_t)gridDim.x * blockDim.x, t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (mode == kLidarMergeWrite) {
        const int64_t m = tail - split, total = m + n;
        for (int64_t d = t0 * kMergeItems; d < total; d += gthreads * kMergeItems) {
            int64_t i = lidar_merge_path(a_time, m, time, n, d), j = d - i;
            for (int k = 0; k < kMergeItems && d + k < total; ++k) {
                const int64_t s = lidar_slot(lidar_merge_pos(split, d + k), cap);
                if (lidar_merge_takes_a(a_time, m, time, n, i, j))
                    merge_store<Lanes>(ring_xyz, ring_time, s, a_xyz, a_time, i++, false, T, a_lanes.from_i, a_lanes.from_r, lanes);
                else
                    merge_store<Lanes>(ring_xyz, ring_time, s, xyz, time, j++, transform, T, lanes.from_i, lanes.from_r, lanes);
            }
        }
    } else if (mode == kLidarMergeAppend) {
        for (int64_t i = t0; i < n; i += gthreads)
            merge_store<Lanes>(ring_xyz, ring_time, lidar_slot(tail + i, cap), xyz, time, i, transform, T, lanes.from_i, lanes.from_r, lanes);
    }
    /* every thread has read the words before its block takes a ticket: the last block may move tail */
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&w->ticket, 1u) == gridDim.x - 1) {
            w->ticket = 0;
            if (mode == kLidarMergeWrite || mode == kLidarMergeAppend) w->tail = tail + n;
        }
    }
}

/* lv_lidar_reserve: the live positions into a ring of another capacity, each to slot p % new_cap (the counters stay) */
template <bool Lanes>
__global__ void __launch_bounds__(256) lv_lidar_move_kernel(const float* __restrict__ from_xyz, const double* __restrict__ from_time, int64_t from_cap,
                                                            const LidarWords* w, float* __restrict__ xyz, double* __restrict__ time, int64_t cap,
                                                            LaneCopy lanes) {
    const int64_t head = w->head, tail = w->tail;
    for (int64_t p = head + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < tail; p += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = lidar_slot(p, from_cap), b = lidar_slot(p, cap);
        xyz[3 * b] = from_xyz[3 * a];
        xyz[3 * b + 1] = from_xyz[3 * a + 1];
        xyz[3 * b + 2] = from_xyz[3 * a + 2];
        time[b] = from_time[a];
        if (Lanes) lidar_copy_lanes(lanes.from_i, lanes.from_r, a, lanes.to_i, lanes.to_r, b);
    }
}

static unsigned lidar_grid(int64_t n) {
    const int64_t g = (n + kLidarPushThreads - 1) / kLidarPushThreads;
    return (unsigned)(g < 1 ? 1 : (g > 4 * kNumSMs ? 4 * kNumSMs : g));
}

cudaError_t launch_lidar_push(const LidarRing& r, const float* xyz, const double* time, const int64_t* d_n, int64_t n_max, uint32_t* err,
                              cudaStream_t st, int* launches, const float* intensity, const float* range) {
    const LaneCopy lanes{intensity, range, r.intensity, r.range};
    if (r.intensity)
        lv_lidar_push_kernel<true><<<lidar_grid(n_max), kLidarPushThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, xyz, time, d_n, n_max, err, lanes);
    else
        lv_lidar_push_kernel<false><<<lidar_grid(n_max), kLidarPushThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, xyz, time, d_n, n_max, err, lanes);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_lidar_merge(const LidarRing& r, const float* xyz, const double* time, const int64_t* d_n, int64_t n_max, bool transform,
                               const Rt32& T, uint32_t* err, cudaStream_t st, int* launches, const float* intensity, const float* range) {
    /* block 0 walks; the others check the message's order */
    const int64_t check_blocks = (n_max + kLidarBlock - 1) / kLidarBlock;
    const unsigned split_grid = 1 + (unsigned)(check_blocks > 2 * kNumSMs ? 2 * kNumSMs : check_blocks);
    const int64_t tiles = (n_max + r.merge_cap + kMergeItems - 1) / kMergeItems;
    const LaneCopy lanes{intensity, range, r.intensity, r.range};
    lv_lidar_merge_split_kernel<<<split_grid, kLidarBlock, 0, st>>>(r.time, r.cap, r.words, time, d_n, n_max, r.merge_cap, err);
    if (r.intensity) {
        const LaneCopy stage{r.intensity, r.range, r.merge_intensity, r.merge_range};
        const LaneCopy a_lanes{r.merge_intensity, r.merge_range, nullptr, nullptr};
        lv_lidar_merge_stage_kernel<true><<<lidar_grid(r.merge_cap), kMergeThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, r.merge_xyz,
                                                                                            r.merge_time, stage);
        lv_lidar_merge_write_kernel<true><<<lidar_grid(tiles), kMergeThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, r.merge_xyz, r.merge_time,
                                                                                       xyz, time, transform, T, lanes, a_lanes);
    } else {
        lv_lidar_merge_stage_kernel<false><<<lidar_grid(r.merge_cap), kMergeThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, r.merge_xyz,
                                                                                             r.merge_time, LaneCopy{});
        lv_lidar_merge_write_kernel<false><<<lidar_grid(tiles), kMergeThreads, 0, st>>>(r.xyz, r.time, r.cap, r.words, r.merge_xyz,
                                                                                        r.merge_time, xyz, time, transform, T, lanes, LaneCopy{});
    }
    if (launches) *launches += 3;
    return cudaGetLastError();
}

cudaError_t launch_lidar_get(const LidarRing& r, double t1, double t2, float* xyz, double* time, int64_t n_max, int64_t* d_n_out, uint32_t* err,
                             cudaStream_t st, int* launches, float* intensity, float* range) {
    const LaneCopy lanes{r.intensity, r.range, intensity, range};
    if (intensity)
        lv_lidar_get_kernel<true><<<1, kLidarBlock, 0, st>>>(r.xyz, r.time, r.cap, r.words, t1, t2, xyz, time, n_max, d_n_out, err, lanes);
    else
        lv_lidar_get_kernel<false><<<1, kLidarBlock, 0, st>>>(r.xyz, r.time, r.cap, r.words, t1, t2, xyz, time, n_max, d_n_out, err, lanes);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_lidar_clear(const LidarRing& r, double t, cudaStream_t st, int* launches) {
    lv_lidar_clear_kernel<<<1, kLidarBlock, 0, st>>>(r.time, r.cap, r.words, t);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

cudaError_t launch_lidar_move(const LidarRing& from, int64_t live, float* xyz, double* time, int64_t cap, cudaStream_t st, int* launches,
                              float* intensity, float* range) {
    if (live == 0) return cudaSuccess;
    const LaneCopy lanes{from.intensity, from.range, intensity, range};
    if (intensity)
        lv_lidar_move_kernel<true><<<lidar_grid(live), 256, 0, st>>>(from.xyz, from.time, from.cap, from.words, xyz, time, cap, lanes);
    else
        lv_lidar_move_kernel<false><<<lidar_grid(live), 256, 0, st>>>(from.xyz, from.time, from.cap, from.words, xyz, time, cap, lanes);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace lv
