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
 * Each is one launch; the counters never leave the device.
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
