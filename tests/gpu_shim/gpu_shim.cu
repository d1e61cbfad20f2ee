/*
 * gpu_shim.cu — TEST-ONLY harness around the filter kernels of liblimovelo_b200.so.
 *
 * It calls the library's own launchers (lv_internal.h: measure_init, launch_reduce_partials, launch_ieskf_step,
 * launch_predict), so the kernels under test are the shipped binary's.  The one piece an update runs inside the fit kernel,
 * ieskf_prepare(), runs here in a one-block kernel compiled from the same header.  Nothing here is reachable from the C ABI
 * of the library: tests/gpu_shim_binding.py loads this file's library with ctypes.
 */
#include <stdint.h>
#include <string.h>

#include <cuda_runtime.h>

#include "../../limo-velo_b200/csrc/lv_internal.h"
#include "../../limo-velo_b200/csrc/lv_predict.h"

using namespace lv;

__global__ void __launch_bounds__(128) gs_prepare_kernel(UpdateCtrl* c) {
    __shared__ PrepWork w;
    ExecBlock ex;                     /* tasks 0..3 need 128 threads */
    ieskf_prepare(ex, c, &w);
}

#define GS_CUDA(call)                             \
    do {                                          \
        cudaError_t e__ = (call);                 \
        if (e__ != cudaSuccess) { rc = (int)e__; goto out; } \
    } while (0)

extern "C" {

/* the layout of one partials row the fit kernel writes: 78 upper-triangle entries of HTH (row-major, j >= i), 12 of HTh, Nm */
void gs_pack_row(const double* HTH, const double* HTh, int64_t nm, double* row) {
    memset(row, 0, sizeof(double) * kPartialStride);
    int e = 0;
    for (int i = 0; i < 12; ++i)
        for (int j = i; j < 12; ++j) row[e++] = HTH[i * 12 + j];
    for (int i = 0; i < 12; ++i) row[e++] = HTh[i];
    row[e] = (double)nm;
}

/*
 * One evaluation on the device.  In: x_prop, P_prop (the update's start), x_cur (the iterate), the loop state iter / t /
 * n_evals, the normal equations.  prm: R, D, limits[23], then max_iter and estimate_extrinsics as doubles.
 * Out: reduced[157] (the packed row after launch_reduce_partials: HTH, HTh, Nm), dx (dx_ of the log entry), x_out (the new
 * iterate), P_out (c->P: the exit block's covariance when done, else P_prop untouched), ints[7] = converged, degenerate,
 * done, status, n_evals, t, iter after the step.  Returns a cudaError_t.
 */
int gs_step(const double* x_prop, const double* P_prop, const double* x_cur, int iter, int t, int n_evals, const double* HTH,
            const double* HTh, int64_t nm, const double* prm_in, double* reduced, double* dx, double* x_out, double* P_out,
            int32_t* ints) {
    int rc = 0;
    UpdateCtrl* c = nullptr;
    double* d_row = nullptr;
    double* d_red = nullptr;
    UpdateCtrl* hc = new UpdateCtrl();
    double row[kPartialStride];
    IeskfParams prm;
    memset(hc, 0, sizeof(*hc));
    memcpy(hc->x_prop, x_prop, sizeof(double) * kStateLen);
    memcpy(hc->P_prop, P_prop, sizeof(double) * kN * kN);
    memcpy(hc->P, P_prop, sizeof(double) * kN * kN);
    memcpy(hc->x, x_cur, sizeof(double) * kStateLen);
    hc->iter = iter;
    hc->t = t;
    hc->n_evals = n_evals;
    prm.R = prm_in[0];
    prm.D = prm_in[1];
    for (int i = 0; i < kN; ++i) prm.limits[i] = prm_in[2 + i];
    prm.max_iter = (int32_t)prm_in[2 + kN];
    prm.estimate_extrinsics = (int32_t)prm_in[3 + kN];
    gs_pack_row(HTH, HTh, nm, row);
    measure_init();
    GS_CUDA(cudaMalloc(&c, sizeof(UpdateCtrl)));
    GS_CUDA(cudaMalloc(&d_row, sizeof(row)));
    GS_CUDA(cudaMalloc(&d_red, sizeof(double) * 160));
    GS_CUDA(cudaMemcpy(c, hc, sizeof(UpdateCtrl), cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(d_row, row, sizeof(row), cudaMemcpyHostToDevice));
    GS_CUDA(launch_reduce_partials(d_row, 1, d_red, 0));
    GS_CUDA(cudaMemcpy(reduced, d_red, sizeof(double) * 157, cudaMemcpyDeviceToHost));
    gs_prepare_kernel<<<1, 128>>>(c);
    GS_CUDA(cudaGetLastError());
    GS_CUDA(launch_ieskf_step(c, prm, d_row, 1, 0, 0));
    GS_CUDA(cudaMemcpy(hc, c, sizeof(UpdateCtrl), cudaMemcpyDeviceToHost));
    {
        const int e = n_evals < kMaxEvals ? n_evals : kMaxEvals - 1;
        memcpy(dx, hc->logs[e].dx, sizeof(double) * kN);
        memcpy(x_out, hc->x, sizeof(double) * kStateLen);
        memcpy(P_out, hc->P, sizeof(double) * kN * kN);
        ints[0] = hc->logs[e].converged;
        ints[1] = hc->logs[e].degenerate;
        ints[2] = hc->done;
        ints[3] = hc->status;
        ints[4] = hc->n_evals;
        ints[5] = hc->t;
        ints[6] = hc->iter;
    }
out:
    cudaFree(c);
    cudaFree(d_row);
    cudaFree(d_red);
    delete hc;
    return rc;
}

/* k IMU samples (k x 7: acc, gyro, dt) through ONE launch_predict; noise = gyr, acc, bias_gyr, bias_acc */
int gs_predict(double* x, double* P, const double* imu, int k, const double* noise) {
    int rc = 0;
    UpdateCtrl* c = nullptr;
    double* d_imu = nullptr;
    UpdateCtrl* hc = new UpdateCtrl();
    const PredictNoise nz = {noise[0], noise[1], noise[2], noise[3]};
    memset(hc, 0, sizeof(*hc));
    memcpy(hc->x, x, sizeof(double) * kStateLen);
    memcpy(hc->P, P, sizeof(double) * kN * kN);
    GS_CUDA(cudaMalloc(&c, sizeof(UpdateCtrl)));
    GS_CUDA(cudaMalloc(&d_imu, sizeof(double) * 7 * (size_t)(k > 0 ? k : 1)));
    GS_CUDA(cudaMemcpy(c, hc, sizeof(UpdateCtrl), cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(d_imu, imu, sizeof(double) * 7 * (size_t)k, cudaMemcpyHostToDevice));
    GS_CUDA(launch_predict(c, nz, d_imu, k, 0));
    GS_CUDA(cudaMemcpy(hc, c, sizeof(UpdateCtrl), cudaMemcpyDeviceToHost));
    memcpy(x, hc->x, sizeof(double) * kStateLen);
    memcpy(P, hc->P, sizeof(double) * kN * kN);
out:
    cudaFree(c);
    cudaFree(d_imu);
    delete hc;
    return rc;
}

}  // extern "C"
