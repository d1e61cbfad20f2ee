/*
 * lv_downsample.cu — the two point-cloud downsamplers in front of the localization path, on the device.
 *
 *   temporal   PointCloudProcessor::temporal_downsample (src/Utils/PointCloudProcessor.cpp:101-112): every
 *              `downsample_rate`-th point of the raw message, and only if farther than `min_dist`.
 *              flag -> select (order kept) -> gather.
 *   voxel grid Compensator::voxelgrid_downsample (src/Modules/Compensator.cpp:148-163) = pcl::VoxelGrid with a
 *              cubic leaf: bounding box -> PCL cell index per point -> stable radix sort -> one centroid per run,
 *              runs in ascending cell index (pcl/filters/impl/voxel_grid.hpp, applyFilter with
 *              downsample_all_data_ = true: CentroidPoint / AccumulatorXYZ: fp32 sum, divided by the count).
 *              PCL's std::sort leaves the order inside a leaf unspecified; here it is input order.
 *              With attribute lanes (lv_voxelgrid_downsample_full) the centroid kernel's <true> instantiation also runs
 *              AccumulatorIntensity (fp32 sum in the same order, / n), and writes what Point(const full_info::Point&)
 *              (Point.cpp:21-25,164-168) makes of the leaf: time 0 (no accumulator) and range = |centroid| (fp32).
 *              Compensator.cpp:161 builds every output point with Point(p), so range is always |output xyz|.
 * Everything stays on the device (the bounding box is consumed by the key kernel, not by the host); the host
 * reads back the output count and one status word.  Streaming integer/byte work: 12 B in per point, 12 B out per
 * leaf, a 32-bit key-value sort between.
 */
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "lv_internal.h"
#include "lv_wire.h"

namespace lv {

struct GridBox {          /* written by the bounding-box kernel, read by the key kernel */
    int mn[3], mx[3];     /* floats in an order-preserving int encoding */
    int overflow;         /* PCL refuses when the cell count exceeds INT32_MAX */
    int64_t n;            /* points of the cloud (<= the host bound the grids and the sort are sized for) */
};

__device__ __forceinline__ int f2ord(float f) { const int i = __float_as_int(f); return i ^ ((i >> 31) & 0x7fffffff); }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i ^ ((i >> 31) & 0x7fffffff)); }

__global__ void lv_ds_box_init_kernel(GridBox* b, const int64_t* d_n, int64_t n_max, uint32_t* err) {
    if (threadIdx.x < 3) { b->mn[threadIdx.x] = 0x7fffffff; b->mx[threadIdx.x] = (int)0x80000000; }
    if (threadIdx.x == 3) b->overflow = 0;
    if (threadIdx.x == 0) b->n = device_count(d_n, n_max, err);
}

__global__ void __launch_bounds__(256) lv_ds_box_kernel(const float* __restrict__ xyz, GridBox* b) {   /* getMinMax3D */
    const int64_t n = b->n;
    int mn[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, mx[3] = {(int)0x80000000, (int)0x80000000, (int)0x80000000};
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const int v = f2ord(xyz[3 * i + a]);
            mn[a] = min(mn[a], v);
            mx[a] = max(mx[a], v);
        }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) {
            mn[a] = min(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], s));
            mx[a] = max(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], s));
        }
        if ((threadIdx.x & 31) == 0) { atomicMin(&b->mn[a], mn[a]); atomicMax(&b->mx[a], mx[a]); }
    }
}

/* voxel_grid.hpp: min_b = floor(min_p * inv), div_b = floor(max_p * inv) - min_b + 1, idx = ijk . (1, div0, div0 div1).
 * Slots [b->n, n_max) get the padding key 0xFFFFFFFF: no cell index reaches it (cells <= INT32_MAX), and the stable sort
 * keeps a real key that ties with it in front, so the first b->n sorted pairs are those of a sort over b->n points. */
__global__ void __launch_bounds__(256) lv_ds_keys_kernel(const float* __restrict__ xyz, int64_t n_max, float inv, GridBox* b,
                                                         uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = b->n;
    if (i >= n && i < n_max) {
        keys[i] = 0xFFFFFFFFu;
        vals[i] = (uint32_t)i;
        return;
    }
    int minb[3], divb[3];
    long long cells = 1;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float lo = ord2f(b->mn[a]), hi = ord2f(b->mx[a]);
        minb[a] = (int)floorf(fmul(lo, inv));
        divb[a] = (int)floorf(fmul(hi, inv)) - minb[a] + 1;
        cells *= (long long)fmul(fsub(hi, lo), inv) + 1;
    }
    if (i == 0 && cells > 2147483647LL) b->overflow = 1;
    if (i >= n) return;
    const int mul[3] = {1, divb[0], divb[0] * divb[1]};
    int idx = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) idx += (int)fsub(floorf(fmul(xyz[3 * i + a], inv)), (float)minb[a]) * mul[a];
    keys[i] = (uint32_t)idx;
    vals[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) lv_ds_heads_kernel(const uint32_t* __restrict__ keys, int64_t n_max, const GridBox* b,
                                                          uint8_t* __restrict__ head) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_max) head[i] = (i < b->n && (i == 0 || keys[i] != keys[i - 1])) ? 1 : 0;
}

/* one thread per leaf: AccumulatorXYZ (xyz += p in sorted order), centroid = xyz / n; Full: the attribute lanes as well */
template <bool Full>
__global__ void __launch_bounds__(256) lv_ds_centroid_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ vals,
                                                             const uint32_t* __restrict__ starts, const int* __restrict__ n_runs,
                                                             const GridBox* __restrict__ b, float* __restrict__ out, VoxelLanes lanes) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    const int runs = *n_runs;
    const int64_t n = b->n;
    if (r >= runs) return;
    const uint32_t s = starts[r], e = r + 1 < runs ? starts[r + 1] : (uint32_t)n;
    float sx = 0.f, sy = 0.f, sz = 0.f;
    float si = 0.f;
    for (uint32_t j = s; j < e; ++j) {
        const uint32_t p = vals[j];
        sx = fadd(sx, xyz[3 * (size_t)p]); sy = fadd(sy, xyz[3 * (size_t)p + 1]); sz = fadd(sz, xyz[3 * (size_t)p + 2]);
        if (Full) si = fadd(si, lanes.intensity[p]);                 /* AccumulatorIntensity */
    }
    const float cnt = (float)(e - s);
    out[3 * (size_t)r] = fdiv(sx, cnt); out[3 * (size_t)r + 1] = fdiv(sy, cnt); out[3 * (size_t)r + 2] = fdiv(sz, cnt);
    if (Full) {
        const float cx = fdiv(sx, cnt), cy = fdiv(sy, cnt), cz = fdiv(sz, cnt);
        if (lanes.intensity_out) lanes.intensity_out[r] = fdiv(si, cnt);
        if (lanes.time_out) lanes.time_out[r] = 0.0;                     /* no accumulator for timestamp: value-initialised */
        if (lanes.range_out) lanes.range_out[r] = wire_norm(cx, cy, cz);   /* set_attributes after set_XYZ: the centroid's norm */
    }
}

/* the output count, and PCL's pass-through: when the cell index overflows, pcl::VoxelGrid::applyFilter warns "Leaf size is too
 * small for the input dataset. Integer indices would overflow." and hands the input on unchanged (Compensator::voxelgrid_downsample
 * carries on with it): the input is copied over the centroids and the count is the input's.  count[0] becomes the output count.
 * Full: time and intensity are passed through as well, and range is |p| of each passed point: Compensator.cpp:161 builds every
 * output point with Point(p), whose set_attributes sets range = this->norm() (Point.cpp:21-25,166-169). */
template <bool Full>
__global__ void __launch_bounds__(256) lv_ds_finish_kernel(const float* __restrict__ xyz, const GridBox* __restrict__ b, int* __restrict__ count,
                                                           float* __restrict__ out, int64_t* __restrict__ n_out, VoxelLanes lanes) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t n = b->n;
    const bool pass = b->overflow && n > 0;
    if (i == 0) {
        const int64_t m = n == 0 ? 0 : (pass ? n : (int64_t)count[0]);
        count[0] = (int)m;
        if (n_out) *n_out = m;
    }
    if (pass && i < 3 * n) out[i] = xyz[i];
    if (Full && pass && i < n) {
        if (lanes.time_out) lanes.time_out[i] = lanes.time[i];
        if (lanes.intensity_out) lanes.intensity_out[i] = lanes.intensity[i];
        if (lanes.range_out) lanes.range_out[i] = wire_norm(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    }
}

/* temporal_downsample: keep = (rate <= 1 or (i + 1) % rate == 0) and min_dist < |p| (lv_wire.h) */
__global__ void __launch_bounds__(256) lv_ds_temporal_flag_kernel(const float* __restrict__ xyz, int64_t n, int rate, double min_dist,
                                                                  uint8_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    keep[i] = temporal_keep(i, rate, min_dist, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]) ? 1 : 0;
}
__global__ void __launch_bounds__(256) lv_ds_gather_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ idx,
                                                           const int* __restrict__ n_sel, float* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= *n_sel) return;
    const size_t p = (size_t)idx[r];
    out[3 * (size_t)r] = xyz[3 * p]; out[3 * (size_t)r + 1] = xyz[3 * p + 1]; out[3 * (size_t)r + 2] = xyz[3 * p + 2];
}

/* ---- scratch + launchers ------------------------------------------------------------------------ */
cudaError_t ds_reserve(DownsampleScratch& s, int64_t n) {
    if (n <= s.cap) return cudaSuccess;
    /* every per-point array is freed before any is reallocated, so the peak stays at the new size */
    s.cap = 0;
    s.keys.reset(); s.keys_sorted.reset(); s.vals.reset(); s.vals_sorted.reset(); s.flags.reset(); s.sel.reset();
    s.keys64.reset(); s.keys64_sorted.reset();
    s.tmp.reset();
    cudaError_t e;
    if ((e = s.box.reserve(1)) != cudaSuccess || (e = s.count.reserve(3)) != cudaSuccess || (e = s.h_count.reserve(2)) != cudaSuccess)
        return e;
    const int64_t cap = n + n / 4 + 1024;
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)cap);
    cub::DeviceSelect::Flagged(nullptr, b, cub::CountingInputIterator<int32_t>(0), (const uint8_t*)nullptr, (int32_t*)nullptr,
                               (int*)nullptr, (int)cap);
    size_t b2 = 0;                            /* the livox front end's second select reads an index array */
    cub::DeviceSelect::Flagged(nullptr, b2, (const int32_t*)nullptr, (const uint8_t*)nullptr, (int32_t*)nullptr, (int*)nullptr, (int)cap);
    b = b > b2 ? b : b2;
    size_t c = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, c, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const uint32_t*)nullptr,
                                    (uint32_t*)nullptr, (int)cap);
    size_t tmp_bytes = (a > b ? a : b);
    tmp_bytes = (tmp_bytes > c ? tmp_bytes : c) + 256;
    if ((e = s.keys.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.keys_sorted.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.vals.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.vals_sorted.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.flags.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.sel.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.keys64.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.keys64_sorted.reserve(cap)) != cudaSuccess) return e;
    if ((e = s.tmp.reserve(tmp_bytes)) != cudaSuccess) return e;
    s.cap = cap;
    return cudaSuccess;
}

cudaError_t launch_voxelgrid(DownsampleScratch& s, const float* d_xyz, const int64_t* d_n, int64_t n_max, float leaf, float* d_out,
                             int64_t* d_n_out, uint32_t* err, cudaStream_t st, int* launches, const VoxelLanes* lanes) {
    const unsigned grid = (unsigned)((n_max + 255) / 256);
    GridBox* box = s.box;
    const float inv = fdiv(1.0f, leaf);
    lv_ds_box_init_kernel<<<1, 32, 0, st>>>(box, d_n, n_max, err);
    lv_ds_box_kernel<<<grid < kNumSMs * 4u ? grid : kNumSMs * 4u, 256, 0, st>>>(d_xyz, box);
    lv_ds_keys_kernel<<<grid, 256, 0, st>>>(d_xyz, n_max, inv, box, s.keys, s.vals);
    size_t tmp = s.tmp.size();
    cudaError_t e = cub::DeviceRadixSort::SortPairs(s.tmp, tmp, s.keys.get(), s.keys_sorted.get(), s.vals.get(), s.vals_sorted.get(), (int)n_max, 0, 32, st);
    if (e != cudaSuccess) return e;
    lv_ds_heads_kernel<<<grid, 256, 0, st>>>(s.keys_sorted, n_max, box, s.flags);
    tmp = s.tmp.size();
    e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), s.sel.get(), s.count.get(), (int)n_max, st);
    if (e != cudaSuccess) return e;
    const uint32_t* starts = reinterpret_cast<const uint32_t*>(s.sel.get());
    const unsigned fgrid = (unsigned)((3 * n_max + 255) / 256);
    if (lanes) {
        lv_ds_centroid_kernel<true><<<grid, 256, 0, st>>>(d_xyz, s.vals_sorted, starts, s.count, box, d_out, *lanes);
        lv_ds_finish_kernel<true><<<fgrid, 256, 0, st>>>(d_xyz, box, s.count, d_out, d_n_out, *lanes);
    } else {
        lv_ds_centroid_kernel<false><<<grid, 256, 0, st>>>(d_xyz, s.vals_sorted, starts, s.count, box, d_out, VoxelLanes());
        lv_ds_finish_kernel<false><<<fgrid, 256, 0, st>>>(d_xyz, box, s.count, d_out, d_n_out, VoxelLanes());
    }
    if (!d_n_out) {                           /* the synchronous form reads the count and the warning flag */
        cudaMemcpyAsync(&s.h_count[0], s.count, sizeof(int), cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(&s.h_count[1], &box->overflow, sizeof(int), cudaMemcpyDeviceToHost, st);
    }
    if (launches) *launches += 11;
    return cudaGetLastError();
}

cudaError_t launch_temporal(DownsampleScratch& s, const float* d_xyz, int64_t n, int rate, double min_dist, float* d_out,
                            int32_t* d_idx_out, cudaStream_t st, int* launches) {
    const unsigned grid = (unsigned)((n + 255) / 256);
    lv_ds_temporal_flag_kernel<<<grid, 256, 0, st>>>(d_xyz, n, rate, min_dist, s.flags);
    size_t tmp = s.tmp.size();
    int32_t* idx = d_idx_out ? d_idx_out : s.sel;
    cudaError_t e = cub::DeviceSelect::Flagged(s.tmp, tmp, cub::CountingInputIterator<int32_t>(0), s.flags.get(), idx, s.count.get(), (int)n, st);
    if (e != cudaSuccess) return e;
    lv_ds_gather_kernel<<<grid, 256, 0, st>>>(d_xyz, idx, s.count, d_out);
    cudaMemcpyAsync(&s.h_count[0], s.count, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (launches) *launches += 4;
    return cudaGetLastError();
}

}  // namespace lv
