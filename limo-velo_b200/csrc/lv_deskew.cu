/*
 * lv_deskew.cu — Compensator::compensate on the GPU (src/Modules/Compensator.cpp:123-146).
 *
 * One thread per point: binary search of the path segment its timestamp falls in, the segment's state integrated
 * to the timestamp with the state's own last controls (State.cpp:103-132), the point carried to the world and back
 * into the LiDAR frame at t2.  The path (a few dozen 176-byte states) is staged in shared memory.  Streaming kernel:
 * 20 B in, 12 B out per point; at sweep sizes it is launch-bound.
 */
#include "lv_deskew.h"
#include "lv_internal.h"

namespace lv {

enum { kDeskewThreads = 256, kMaxPathStates = 256 };

__global__ void __launch_bounds__(kDeskewThreads) lv_deskew_kernel(const lv_state32* path, int ns, const Rt32 back,
                                                                   const float* xyz, const double* t, const int64_t* d_n, int64_t n_max,
                                                                   float* out) {
    __shared__ lv_state32 s_path[kMaxPathStates];
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(path);
        uint32_t* dst = reinterpret_cast<uint32_t*>(s_path);
        const int words = ns * (int)(sizeof(lv_state32) / 4);
        for (int i = threadIdx.x; i < words; i += kDeskewThreads) dst[i] = src[i];
    }
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * kDeskewThreads + threadIdx.x;
    if (i >= device_count(d_n, n_max, nullptr)) return;
    const float p[3] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
    float q[3];
    deskew_point(s_path, ns, back, p, t[i], q);
    out[3 * i] = q[0]; out[3 * i + 1] = q[1]; out[3 * i + 2] = q[2];
}

/* 1 where a timestamp lies outside [t_lo, t_hi] or is smaller than its predecessor (the reference asserts both) */
__global__ void lv_deskew_check_kernel(const double* t, const int64_t* d_n, int64_t n_max, double t_lo, double t_hi, int* bad,
                                       uint32_t* err) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= device_count(d_n, n_max, err)) return;
    const double v = t[i];
    if (!(v >= t_lo && v <= t_hi) || (i > 0 && v < t[i - 1])) {
        *bad = 1;
        if (err) atomicOr(err, kAsyncDeskewPath);
    }
}

int deskew_max_states() { return kMaxPathStates; }

cudaError_t launch_deskew(const lv_state32* d_path, int ns, const lv_state32& Xt2, double t_lo, double t_hi, const float* d_xyz,
                          const double* d_t, const int64_t* d_n, int64_t n_max, float* d_out, int* d_bad, uint32_t* err, cudaStream_t st) {
    const Rt32 back = deskew_back(Xt2);
    const unsigned grid = (unsigned)((n_max + kDeskewThreads - 1) / kDeskewThreads);
    cudaMemsetAsync(d_bad, 0, sizeof(int), st);
    lv_deskew_check_kernel<<<grid, kDeskewThreads, 0, st>>>(d_t, d_n, n_max, t_lo, t_hi, d_bad, err);
    lv_deskew_kernel<<<grid, kDeskewThreads, 0, st>>>(d_path, ns, back, d_xyz, d_t, d_n, n_max, d_out);
    return cudaGetLastError();
}

}  // namespace lv
