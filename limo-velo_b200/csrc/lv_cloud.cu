/*
 * lv_cloud.cu — Accumulator::process (src/Modules/Accumulator.cpp:142-151) on the device: the raw bytes of a LiDAR message in
 * HBM -> msg2points (PointCloudProcessor.cpp:24-99) -> temporal_downsample (:101-112) -> sort_points (:114-123), with the
 * per-point arithmetic of lv_wire.h that the host decoders run too.  One pipeline serves four message formats; a point source
 * (Pc2Source, LivoxSource, VelodyneSource, OusterSource) says where a point's fields are and how its time is computed.
 *
 *   flag     every point of the message: xyz from its bytes -> temporal_keep on the rank
 *   select   cub::DeviceSelect::Flagged: indices of the kept points, in message order
 *   key      every kept point: its absolute time -> an order-preserving u64 key (NaN is flagged: the host sort has no order
 *            for it); the slots past the kept count up to the host-known bound are padded with the largest key
 *   sort     cub::DeviceRadixSort::SortPairs (key, raw index): stable, so equal times stay in message order
 *   gather   every output point: xyz / time / intensity / range decoded again from its bytes, and its raw index
 * sensor_msgs/PointCloud2: the rank is the message index.  livox CustomMsg: msg2points drops points by tag first, so a tag flag
 * and its select come first, and the rank is the position among the tag-kept points (Accumulator.cpp:143-151 decimates the list
 * msg2points returns).  velodyne_msgs/VelodyneScan likewise: a validity flag (return mode, block flags, distance) and its select
 * come first, and the key kernel also checks every packet for a dual return or a stamp that does not convert (the flag kernel
 * resets that word, so the first kernel cannot raise it).  Ouster packets of every UDP profile the same way: a validity flag
 * (column status, measurement id, range) and its select, with no per-packet check: a column's time always converts.  The bytes of a kept point are read twice (flag + key, gather), those
 * of a dropped point once.  Every value is assembled from single bytes (lv_wire.h): fields sit at any offset and the message at any address.  Byte offsets are
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

/* sensor_msgs/PointCloud2: the fields at the layout's offsets; times relative to the header stamp or absolute by LiDAR type */
struct Pc2Source {
    CloudArgs a;
    __device__ __forceinline__ const uint8_t* point(int64_t i) const { return a.data + (uint64_t)i * (uint64_t)a.layout.point_step; }
    __device__ __forceinline__ void xyz(const uint8_t* p, float& x, float& y, float& z) const {
        x = wire_f32(p + a.layout.off_x); y = wire_f32(p + a.layout.off_y); z = wire_f32(p + a.layout.off_z);
    }
    __device__ __forceinline__ double time(const uint8_t* p) const {
        const double begin = wire_begin_time(a.type, a.layout, a.data, a.n, a.stamp_us, a.stamp_beginning);
        return wire_time(a.type, a.layout, p, a.offset_beginning, a.full_rotation_time, begin);
    }
    __device__ __forceinline__ float intensity(const uint8_t* p) const { return wire_intensity(a.type, a.layout, p); }
    __device__ __forceinline__ float range(const uint8_t* p, float x, float y, float z) const { return wire_range(a.type, a.layout, p, x, y, z); }
    __device__ __forceinline__ void check(int64_t, int64_t, int*, uint32_t*) const {}
};

/* livox CustomMsg: 19-byte records, time = timebase + offset_time, intensity = reflectivity, range = |p| */
struct LivoxSource {
    LivoxArgs a;
    __device__ __forceinline__ const uint8_t* point(int64_t i) const { return livox_point(a.data, i); }
    __device__ __forceinline__ void xyz(const uint8_t* p, float& x, float& y, float& z) const {
        x = wire_f32(p + 4); y = wire_f32(p + 8); z = wire_f32(p + 12);
    }
    __device__ __forceinline__ double time(const uint8_t* p) const { return livox_time(a.timebase_ns, p); }
    __device__ __forceinline__ float intensity(const uint8_t* p) const { return livox_reflectivity(p); }
    __device__ __forceinline__ float range(const uint8_t*, float x, float y, float z) const { return wire_norm(x, y, z); }
    __device__ __forceinline__ void check(int64_t, int64_t, int*, uint32_t*) const {}
};

/* velodyne_msgs/VelodyneScan: a point is a slot (its packet and r), decoded through the rotation tables and the calibration */
struct VelodyneSlot {
    const uint8_t* pkt;
    int r;
};
struct VelodyneSource {
    VelodyneArgs a;
    __device__ __forceinline__ VelodyneSlot point(int64_t i) const {
        return {velodyne_packet(a.data, i / kVelodyneSlots), (int)(i % kVelodyneSlots)};
    }
    __device__ __forceinline__ void xyz(const VelodyneSlot& p, float& x, float& y, float& z) const {
        velodyne_xyz(p.pkt, p.r, a.table, a.table + kVelodyneTable, a.cal, x, y, z);
    }
    __device__ __forceinline__ double time(const VelodyneSlot& p) const { return velodyne_time(p.pkt, p.r); }
    __device__ __forceinline__ float intensity(const VelodyneSlot& p) const { return velodyne_reflectivity(p.pkt, p.r); }
    __device__ __forceinline__ float range(const VelodyneSlot&, float x, float y, float z) const { return wire_norm(x, y, z); }
    /* packets k = j, j + stride, ...: a dual-return packet or a stamp that does not convert raises s.count[1] and kAsyncVelodyne */
    __device__ __forceinline__ void check(int64_t j, int64_t stride, int* count, uint32_t* err) const {
        for (int64_t k = j; k < a.n_packets; k += stride) {
            const uint8_t* pkt = velodyne_packet(a.data, k);
            if (velodyne_mode(pkt) == kVelodyneDualReturn || !velodyne_stamp_ok(pkt)) {
                count[1] = 1;
                if (err) atomicOr(err, kAsyncVelodyne);
            }
        }
    }
};

/* ouster packets of any UDP profile: a point is a slot (its column and pixel), decoded through the profile's layout, the column table
 * and the beam terms */
struct OusterSlot {
    const uint8_t* col;
    int p;
};
struct OusterSource {
    OusterArgs a;
    __device__ __forceinline__ OusterSlot point(int64_t i) const {
        return {ouster_column(a.fmt, a.data, i, a.cal.H), (int)(i % a.cal.H)};
    }
    __device__ __forceinline__ void xyz(const OusterSlot& p, float& x, float& y, float& z) const {
        ouster_xyz(a.fmt, p.col, p.p, a.table, a.table + kOusterTable, a.cal, x, y, z);
    }
    __device__ __forceinline__ double time(const OusterSlot& p) const { return ouster_time(p.col); }
    __device__ __forceinline__ float intensity(const OusterSlot& p) const { return ouster_reflectivity(a.fmt, p.col, p.p); }
    __device__ __forceinline__ float range(const OusterSlot& p, float, float, float) const { return ouster_range(a.fmt, p.col, p.p); }
    __device__ __forceinline__ void check(int64_t, int64_t, int*, uint32_t*) const {}
};

/* std::stable_sort with `<` on doubles: -0.0 and +0.0 are equal (message order), so -0.0 is folded onto +0.0; then the
 * sign-magnitude bits become an unsigned order (negatives reversed, positives above them) */
__device__ __forceinline__ uint64_t time_key(double t) {
    const uint64_t b = (uint64_t)__double_as_longlong(t == 0.0 ? 0.0 : t);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

/* temporal_keep on rank j.  rank_sel == NULL: every point of the message, rank = message index.  Otherwise the *n_ranked points
 * rank_sel[0 .. *n_ranked) (the tag-kept ones, in message order), and the slots past them are not kept.
 * s.count[1] (the NaN flag) is reset here: no later kernel of the pipeline runs before this one */
template <class Src>
__global__ void __launch_bounds__(256) lv_cloud_flag_kernel(Src s, const int32_t* __restrict__ rank_sel, const int* __restrict__ n_ranked,
                                                            uint8_t* __restrict__ keep, int* __restrict__ count) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j == 0) count[1] = 0;
    if (j >= s.a.n) return;
    if (rank_sel && j >= *n_ranked) { keep[j] = 0; return; }
    float x, y, z;
    s.xyz(s.point(rank_sel ? rank_sel[j] : j), x, y, z);
    keep[j] = temporal_keep(j, s.a.rate, s.a.min_dist, x, y, z) ? 1 : 0;
}

/* msg2points of a VelodyneScan: the slots that are points (velodyne_slot_valid) */
__global__ void __launch_bounds__(256) lv_velodyne_valid_kernel(VelodyneArgs a, uint8_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    keep[i] = velodyne_slot_valid(velodyne_packet(a.data, i / kVelodyneSlots), (int)(i % kVelodyneSlots)) ? 1 : 0;
}

/* msg2points of ouster packets: the slots that are points (ouster_slot_valid) */
__global__ void __launch_bounds__(256) lv_ouster_valid_kernel(OusterArgs a, uint8_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    keep[i] = ouster_slot_valid(a.fmt, ouster_column(a.fmt, a.data, i, a.cal.H), (int)(i % a.cal.H), a.cal.W) ? 1 : 0;
}

/* msg2points' tag filter of a livox message */
__global__ void __launch_bounds__(256) lv_livox_tag_kernel(LivoxArgs a, uint8_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    keep[i] = livox_tag_keep(livox_point(a.data, i), a.tag_reject_mask) ? 1 : 0;
}

template <class Src>
__global__ void __launch_bounds__(256) lv_cloud_key_kernel(Src s, const int32_t* __restrict__ sel, int* __restrict__ count,
                                                           int64_t bound, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                                                           uint32_t* __restrict__ err) {
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= bound) return;
    s.check(j, bound, count, err);            /* the message's own deferred errors (VelodyneScan: per packet) */
    if (j >= count[0]) {                      /* padding: sorts behind every kept point */
        keys[j] = ~0ull;
        vals[j] = 0xffffffffu;
        return;
    }
    const int32_t i = sel[j];
    const double t = s.time(s.point(i));
    if (isnan(t)) {
        count[1] = 1;
        if (err) atomicOr(err, kAsyncCloudNaN);
    }
    keys[j] = time_key(t);
    vals[j] = (uint32_t)i;
}

template <class Src>
__global__ void __launch_bounds__(256) lv_cloud_gather_kernel(Src s, const uint32_t* __restrict__ order, const int* __restrict__ count,
                                                              float* __restrict__ xyz, double* __restrict__ time,
                                                              float* __restrict__ intensity, float* __restrict__ range,
                                                              int32_t* __restrict__ idx, int64_t* __restrict__ n_out) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0 && n_out) *n_out = count[0];
    if (r >= count[0]) return;
    const uint32_t i = order[r];
    const auto p = s.point(i);
    float x, y, z;
    s.xyz(p, x, y, z);
    xyz[3 * r] = x; xyz[3 * r + 1] = y; xyz[3 * r + 2] = z;
    time[r] = s.time(p);
    if (intensity) intensity[r] = s.intensity(p);
    if (range) range[r] = s.range(p, x, y, z);
    if (idx) idx[r] = (int32_t)i;
}

int64_t cloud_bound(int64_t n, int rate) { return rate <= 1 ? n : n / rate; }

/* select the flagged ranks of `in` into s.sel (s.count[0]), then key, sort and gather them */
template <class Src, class In>
static cudaError_t launch_select_sort_gather(DownsampleScratch& s, const Src& src, In in, const CloudOut& o, int64_t* d_n_out, uint32_t* err,
                                             cudaStream_t st) {
    const int64_t bound = cloud_bound(src.a.n, src.a.rate);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, in, s.flags.get(), s.sel.get(), s.count.get(), (int)src.a.n, st);
    if (e != cudaSuccess) return e;
    const unsigned grid = (unsigned)((bound + 255) / 256);
    lv_cloud_key_kernel<<<grid, 256, 0, st>>>(src, s.sel, s.count, bound, s.keys64, s.vals, err);
    tmp = s.tmp.size();
    e = cub::DeviceRadixSort::SortPairs(s.tmp, tmp, s.keys64.get(), s.keys64_sorted.get(), s.vals.get(), s.vals_sorted.get(), (int)bound, 0, 64, st);
    if (e != cudaSuccess) return e;
    lv_cloud_gather_kernel<<<grid, 256, 0, st>>>(src, s.vals_sorted, s.count, o.xyz, o.time, o.intensity, o.range, o.idx, d_n_out);
    if (!d_n_out) cudaMemcpyAsync(s.h_count, s.count, 2 * sizeof(int), cudaMemcpyDeviceToHost, st);   /* the synchronous form reads them */
    return cudaGetLastError();
}

cudaError_t launch_process_cloud(DownsampleScratch& s, const CloudArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err, cudaStream_t st,
                                 int* launches) {
    const Pc2Source src{a};
    lv_cloud_flag_kernel<<<(unsigned)((a.n + 255) / 256), 256, 0, st>>>(src, nullptr, nullptr, s.flags, s.count);
    const cudaError_t e = launch_select_sort_gather(s, src, cub::CountingInputIterator<int32_t>(0), o, d_n_out, err, st);
    if (e == cudaSuccess && launches) *launches += 6;
    return e;
}

cudaError_t launch_process_livox(DownsampleScratch& s, const LivoxArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err, cudaStream_t st,
                                 int* launches) {
    const LivoxSource src{a};
    const unsigned grid = (unsigned)((a.n + 255) / 256);
    /* the tag-kept indices live in vals_sorted until the second select has read them: the sort writes it only afterwards */
    int32_t* tag_sel = reinterpret_cast<int32_t*>(s.vals_sorted.get());
    lv_livox_tag_kernel<<<grid, 256, 0, st>>>(a, s.flags);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), tag_sel, s.count.get() + 2,
                                               (int)a.n, st);
    if (e != cudaSuccess) return e;
    lv_cloud_flag_kernel<<<grid, 256, 0, st>>>(src, tag_sel, s.count.get() + 2, s.flags, s.count);
    e = launch_select_sort_gather(s, src, static_cast<const int32_t*>(tag_sel), o, d_n_out, err, st);
    if (e == cudaSuccess && launches) *launches += 9;
    return e;
}

cudaError_t launch_process_velodyne(DownsampleScratch& s, const VelodyneArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err,
                                    cudaStream_t st, int* launches) {
    const VelodyneSource src{a};
    const unsigned grid = (unsigned)((a.n + 255) / 256);
    /* as for livox: the msg2points slots live in vals_sorted until the second select has read them */
    int32_t* valid_sel = reinterpret_cast<int32_t*>(s.vals_sorted.get());
    lv_velodyne_valid_kernel<<<grid, 256, 0, st>>>(a, s.flags);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), valid_sel, s.count.get() + 2,
                                               (int)a.n, st);
    if (e != cudaSuccess) return e;
    lv_cloud_flag_kernel<<<grid, 256, 0, st>>>(src, valid_sel, s.count.get() + 2, s.flags, s.count);
    e = launch_select_sort_gather(s, src, static_cast<const int32_t*>(valid_sel), o, d_n_out, err, st);
    if (e == cudaSuccess && launches) *launches += 9;
    return e;
}

cudaError_t launch_process_ouster(DownsampleScratch& s, const OusterArgs& a, const CloudOut& o, int64_t* d_n_out, uint32_t* err,
                                  cudaStream_t st, int* launches) {
    const OusterSource src{a};
    const unsigned grid = (unsigned)((a.n + 255) / 256);
    /* as for livox: the msg2points slots live in vals_sorted until the second select has read them */
    int32_t* valid_sel = reinterpret_cast<int32_t*>(s.vals_sorted.get());
    lv_ouster_valid_kernel<<<grid, 256, 0, st>>>(a, s.flags);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), valid_sel, s.count.get() + 2,
                                               (int)a.n, st);
    if (e != cudaSuccess) return e;
    lv_cloud_flag_kernel<<<grid, 256, 0, st>>>(src, valid_sel, s.count.get() + 2, s.flags, s.count);
    e = launch_select_sort_gather(s, src, static_cast<const int32_t*>(valid_sel), o, d_n_out, err, st);
    if (e == cudaSuccess && launches) *launches += 9;
    return e;
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
