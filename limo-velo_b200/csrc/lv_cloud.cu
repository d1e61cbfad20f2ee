/*
 * lv_cloud.cu — Accumulator::process (src/Modules/Accumulator.cpp:142-151) on the device: the raw `data` of a
 * sensor_msgs/PointCloud2 in HBM -> msg2points (PointCloudProcessor.cpp:24-99) -> temporal_downsample (:101-112) ->
 * sort_points (:114-123), with the per-point arithmetic of lv_wire.h that the host decoder runs too.
 *
 *   flag     every point of the message: xyz from its bytes -> temporal_keep on the raw index
 *   select   cub::DeviceSelect::Flagged: indices of the kept points, in message order
 *   key      every kept point: its absolute time -> an order-preserving u64 key (NaN is flagged: the host sort has no order
 *            for it); the slots past the kept count up to the host-known bound are padded with the largest key
 *   sort     cub::DeviceRadixSort::SortPairs (key, raw index): stable, so equal times stay in message order
 *   gather   every output point: xyz / time / intensity / range decoded again from its bytes, and its raw index
 * The bytes of a kept point are read twice (flag + key, gather), those of a dropped point once (flag).  Every value is
 * assembled from single bytes (lv_wire.h): fields sit at any offset and the message at any address.  Byte offsets are
 * 64-bit: n < 2^31 points of up to 2^31 bytes each.
 *
 * Also Processor::fill's header stamp (PointCloudProcessor.cpp:125-133) of a cloud the publishers send: one block, a max-reduction.
 */
#include <cub/block/block_reduce.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "lv_internal.h"
#include "lv_wire.h"

namespace lv {

__device__ __forceinline__ const uint8_t* cloud_point(const CloudArgs& a, int64_t i) {
    return a.data + (uint64_t)i * (uint64_t)a.layout.point_step;
}

/* std::stable_sort with `<` on doubles: -0.0 and +0.0 are equal (message order), so -0.0 is folded onto +0.0; then the
 * sign-magnitude bits become an unsigned order (negatives reversed, positives above them) */
__device__ __forceinline__ uint64_t time_key(double t) {
    const uint64_t b = (uint64_t)__double_as_longlong(t == 0.0 ? 0.0 : t);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

/* s.count[1] (the NaN flag) is reset here: this kernel runs first */
__global__ void __launch_bounds__(256) lv_cloud_flag_kernel(CloudArgs a, uint8_t* __restrict__ keep, int* __restrict__ count) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) count[1] = 0;
    if (i >= a.n) return;
    const uint8_t* p = cloud_point(a, i);
    const lv_cloud_layout& L = a.layout;
    keep[i] = temporal_keep(i, a.rate, a.min_dist, wire_f32(p + L.off_x), wire_f32(p + L.off_y), wire_f32(p + L.off_z)) ? 1 : 0;
}

__global__ void __launch_bounds__(256) lv_cloud_key_kernel(CloudArgs a, const int32_t* __restrict__ sel, int* __restrict__ count,
                                                           int64_t bound, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                           uint32_t* __restrict__ err) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= bound) return;
    if (j >= count[0]) {                      /* padding: sorts behind every kept point */
        keys[j] = ~0ull;
        vals[j] = 0xffffffffu;
        return;
    }
    const int32_t i = sel[j];
    const double begin = wire_begin_time(a.type, a.layout, a.data, a.n, a.stamp_us, a.stamp_beginning);
    const double t = wire_time(a.type, a.layout, cloud_point(a, i), a.offset_beginning, a.full_rotation_time, begin);
    if (isnan(t)) {
        count[1] = 1;
        if (err) atomicOr(err, kAsyncCloudNaN);
    }
    keys[j] = time_key(t);
    vals[j] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) lv_cloud_gather_kernel(CloudArgs a, const uint32_t* __restrict__ order, const int* __restrict__ count,
                                                              float* __restrict__ xyz, double* __restrict__ time,
                                                              float* __restrict__ intensity, float* __restrict__ range,
                                                              int32_t* __restrict__ idx, int64_t* __restrict__ n_out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0 && n_out) *n_out = count[0];
    if (r >= count[0]) return;
    const uint32_t i = order[r];
    const uint8_t* p = cloud_point(a, i);
    const lv_cloud_layout& L = a.layout;
    const float x = wire_f32(p + L.off_x), y = wire_f32(p + L.off_y), z = wire_f32(p + L.off_z);
    xyz[3 * r] = x; xyz[3 * r + 1] = y; xyz[3 * r + 2] = z;
    const double begin = wire_begin_time(a.type, L, a.data, a.n, a.stamp_us, a.stamp_beginning);
    time[r] = wire_time(a.type, L, p, a.offset_beginning, a.full_rotation_time, begin);
    if (intensity) intensity[r] = wire_intensity(a.type, L, p);
    if (range) range[r] = wire_range(a.type, L, p, x, y, z);
    if (idx) idx[r] = (int32_t)i;
}

int64_t cloud_bound(int64_t n, int rate) { return rate <= 1 ? n : n / rate; }

cudaError_t launch_process_cloud(DownsampleScratch& s, const CloudArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err, cudaStream_t st,
                                 int* launches) {
    const int64_t bound = cloud_bound(a.n, a.rate);
    lv_cloud_flag_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, st>>>(a, s.flags, s.count);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), s.sel.get(), s.count.get(), (int)a.n, st);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((bound + 255) / 256);
    lv_cloud_key_kernel<<<grid, 256, 0, st>>>(a, s.sel, s.count, bound, s.keys64, s.vals, err);
    tmp = s.tmp.size();
    e = cub::DeviceRadixSort::SortPairs(s.tmp, tmp, s.keys64.get(), s.keys64_sorted.get(), s.vals.get(), s.vals_sorted.get(), (int)bound, 0, 64, st);
    if (e != cudaSuccess) return e;
    lv_cloud_gather_kernel<<<grid, 256, 0, st>>>(a, s.vals_sorted, s.count, o.xyz, o.time, o.intensity, o.range, o.idx, d_n_out);
    if (!d_n_out) cudaMemcpyAsync(s.h_count, s.count, 2 * sizeof(int), cudaMemcpyDeviceToHost, st);   /* the synchronous form reads them */
    if (launches) *launches += 6;
    return cudaGetLastError();
}

/* `pcl.header.stamp = 0; for (p : points) stamp = max(stamp, Conversions::sec2Microsec(p.time));` with sec2Microsec =
 * std::round(t * 1e6) converted to uint64 (Utils.cpp:14-16): the product unfused, round half away from zero */
enum { kStampThreads = 1024 };
__global__ void __launch_bounds__(kStampThreads) lv_cloud_stamp_kernel(const double* __restrict__ time, const int64_t* __restrict__ d_n,
                                                                       int64_t n_max, unsigned long long* __restrict__ stamp, uint32_t* err) {
    typedef cub::BlockReduce<unsigned long long, kStampThreads> Reduce;
    __shared__ typename Reduce::TempStorage red;
    const int64_t n = device_count(d_n, n_max, err);
    unsigned long long m = 0;
    for (int64_t i = threadIdx.x; i < n; i += kStampThreads) {
        const unsigned long long us = (unsigned long long)round(dmul(time[i], 1e6));
        m = us > m ? us : m;
    }
    const unsigned long long r = Reduce(red).Reduce(m, cub::Max());
    if (threadIdx.x == 0) *stamp = r;
}

cudaError_t launch_cloud_stamp(const double* d_time, const int64_t* d_n, int64_t n_max, uint64_t* d_stamp_us, uint32_t* err, cudaStream_t st,
                               int* launches) {
    lv_cloud_stamp_kernel<<<1, kStampThreads, 0, st>>>(d_time, d_n, n_max, reinterpret_cast<unsigned long long*>(d_stamp_us), err);
    if (launches) *launches += 1;
    return cudaGetLastError();
}

}  // namespace lv
