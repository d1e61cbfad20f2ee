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
#include "manifold_ops.h"

using namespace lv;

__global__ void __launch_bounds__(128) gs_prepare_kernel(UpdateCtrl* c) {
    __shared__ PrepWork w;
    ExecBlock ex;                     /* tasks 0..3 need 128 threads */
    ieskf_prepare(ex, c, &w);
}

/* the match stage's per-set arithmetic as lv_fit_kernel runs it, one thread per given set: distances from g, the tie order,
 * the fit, the distance and the row (frame from state x).  q: 15 floats, id: 5 ints per set; out: the reordered ids, abcd,
 * is_plane, dist and 13 doubles (row, then h) whatever is_plane says */
__global__ void gs_fit_sets_kernel(const float* q_in, const float* g_in, const int* id_in, const Frame* fr, float thr, int est, int n,
                                   int* id_out, float* abcd_out, int* ok_out, float* dist_out, double* row_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float q[5][3], d[5], abcd[4];
    int id[5];
    const float g[3] = {g_in[3 * i], g_in[3 * i + 1], g_in[3 * i + 2]};
    for (int k = 0; k < 5; ++k) {
        for (int a = 0; a < 3; ++a) q[k][a] = q_in[15 * i + 3 * k + a];
        d[k] = sq_dist(g[0], g[1], g[2], q[k][0], q[k][1], q[k][2]);
        id[k] = id_in[5 * i + k];
    }
    canonical_neighbour_order(q, d, id);
    const bool ok = plane_fit(q, thr, abcd);
    const float dist = plane_dist(abcd, g);
    double row[12], h;
    jacobian_row(*fr, g, abcd, dist, est != 0, row, &h);
    for (int k = 0; k < 5; ++k) id_out[5 * i + k] = id[k];
    for (int k = 0; k < 4; ++k) abcd_out[4 * i + k] = abcd[k];
    ok_out[i] = ok ? 1 : 0;
    dist_out[i] = dist;
    for (int k = 0; k < 12; ++k) row_out[13 * (size_t)i + k] = row[k];
    row_out[13 * (size_t)i + 12] = h;
}

/* manifold_op (manifold_ops.h) over n rows, one thread per row: the lv_manifold.h functions as the device build runs them */
__global__ void gs_manifold_kernel(const int* op, const double* in, double* out, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    manifold_op(op[i], in + (size_t)kManIn * i, out + (size_t)kManOut * i);
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

/* ---- the map update (lv_map.cu) through the library's own map_alloc / map_add / map_grow / map_clear / map_free, one stream ---- */
struct GsMap {
    MapBuffers b;
    cudaStream_t st = nullptr;
    float* d_xyz = nullptr;      /* the points of one add (add_cap x 3) */
    int64_t* d_n = nullptr;      /* the device count of a MapAddCount add */
};

void* gs_map_create(int64_t max_map_points, int64_t max_points, float voxel_size, float ds) {
    GsMap* g = new GsMap();
    if (cudaStreamCreateWithFlags(&g->st, cudaStreamNonBlocking) != cudaSuccess ||
        map_alloc(g->b, max_map_points, max_points, voxel_size, ds, g->st) != cudaSuccess ||
        cudaMalloc(&g->d_xyz, sizeof(float) * 3 * (size_t)g->b.add_cap) != cudaSuccess || cudaMalloc(&g->d_n, sizeof(int64_t)) != cudaSuccess ||
        map_clear(g->b, g->st, nullptr) != cudaSuccess || cudaStreamSynchronize(g->st) != cudaSuccess) {
        map_free(g->b);
        cudaFree(g->d_xyz);
        cudaFree(g->d_n);
        if (g->st) cudaStreamDestroy(g->st);
        delete g;
        return nullptr;
    }
    return g;
}
/* n points of xyz (host).  dev_count >= 0: the add takes its count from device memory (MapAddCount: clamped to n, none below
 * max(min_points, 1), build_if_empty); dev_count < 0: n on the host, as lv_map_add after its argument checks */
int gs_map_add(void* h, const float* xyz, int64_t n, int downsample, int64_t dev_count, int64_t min_points, int build_if_empty) {
    GsMap* g = static_cast<GsMap*>(h);
    int rc = 0;
    MapAddCount cnt;
    if (n > g->b.add_cap) return (int)cudaErrorInvalidValue;
    if (n > 0) GS_CUDA(cudaMemcpyAsync(g->d_xyz, xyz, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice, g->st));
    if (dev_count >= 0) {
        GS_CUDA(cudaMemcpyAsync(g->d_n, &dev_count, sizeof(int64_t), cudaMemcpyHostToDevice, g->st));
        cnt.n = g->d_n;
        cnt.min_points = min_points;
        cnt.build_if_empty = build_if_empty;
    }
    GS_CUDA(map_add(g->b, g->d_xyz, n, downsample, g->st, nullptr, cnt));
    GS_CUDA(cudaStreamSynchronize(g->st));
out:
    return rc;
}
int gs_map_grow(void* h, int64_t cap) {
    GsMap* g = static_cast<GsMap*>(h);
    int rc = 0;
    GS_CUDA(map_grow(g->b, cap, g->st, nullptr));
    if (g->b.add_cap > 0) {                       /* the add scratch grew with the map */
        cudaFree(g->d_xyz);
        g->d_xyz = nullptr;
        GS_CUDA(cudaMalloc(&g->d_xyz, sizeof(float) * 3 * (size_t)g->b.add_cap));
    }
    GS_CUDA(cudaStreamSynchronize(g->st));
out:
    return rc;
}
int gs_map_clear(void* h) {
    GsMap* g = static_cast<GsMap*>(h);
    int rc = 0;
    GS_CUDA(map_clear(g->b, g->st, nullptr));
    GS_CUDA(cudaStreamSynchronize(g->st));
out:
    return rc;
}
/* dims = {voxel slots, block slots, arena capacity, list capacity, add capacity}; counters = the kMapCounters device words */
int gs_map_dims(void* h, int64_t* dims, uint32_t* counters) {
    GsMap* g = static_cast<GsMap*>(h);
    int rc = 0;
    dims[0] = g->b.slots;
    dims[1] = g->b.bslots;
    dims[2] = g->b.arena_cap;
    dims[3] = g->b.list_cap;
    dims[4] = g->b.add_cap;
    GS_CUDA(cudaMemcpy(counters, g->b.counters, sizeof(uint32_t) * kMapCounters, cudaMemcpyDeviceToHost));
out:
    return rc;
}
/* both tables, arena[0, arena_top) and the first n_touched / n_dirty entries of the lists (the caller takes them from the counters) */
int gs_map_dump(void* h, uint32_t* table, uint32_t* btable, float* arena, uint32_t arena_top, uint32_t* touched, uint32_t n_touched,
                uint32_t* dirty, uint32_t n_dirty) {
    GsMap* g = static_cast<GsMap*>(h);
    int rc = 0;
    GS_CUDA(cudaMemcpy(table, g->b.table, sizeof(uint4) * 2 * (size_t)g->b.slots, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(btable, g->b.btable, sizeof(uint4) * (size_t)g->b.bslots, cudaMemcpyDeviceToHost));
    if (arena_top > g->b.arena_cap) return (int)cudaErrorInvalidValue;
    GS_CUDA(cudaMemcpy(arena, g->b.arena, sizeof(float4) * (size_t)arena_top, cudaMemcpyDeviceToHost));
    if (n_touched > g->b.list_cap || n_dirty > g->b.list_cap) return (int)cudaErrorInvalidValue;
    GS_CUDA(cudaMemcpy(touched, g->b.touched, sizeof(uint32_t) * (size_t)n_touched, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(dirty, g->b.dirty, sizeof(uint32_t) * (size_t)n_dirty, cudaMemcpyDeviceToHost));
out:
    return rc;
}
void gs_map_free(void* h) {
    GsMap* g = static_cast<GsMap*>(h);
    if (!g) return;
    map_free(g->b);
    cudaFree(g->d_xyz);
    cudaFree(g->d_n);
    cudaStreamDestroy(g->st);
    delete g;
}

/* gs_fit_sets_kernel on n sets (host arrays in and out; shapes there); returns a cudaError_t */
int gs_fit_sets(const float* q, const float* g, const int* id, const double* x, float thr, int est, int n, int* id_out, float* abcd,
                int* ok, float* dist, double* rows) {
    int rc = 0;
    Frame fr;
    make_frame(x, &fr);
    float *dq = nullptr, *dg = nullptr, *dabcd = nullptr, *ddist = nullptr;
    int *did = nullptr, *dido = nullptr, *dok = nullptr;
    double* drows = nullptr;
    Frame* dfr = nullptr;
    GS_CUDA(cudaMalloc(&dq, sizeof(float) * 15 * (size_t)n));
    GS_CUDA(cudaMalloc(&dg, sizeof(float) * 3 * (size_t)n));
    GS_CUDA(cudaMalloc(&did, sizeof(int) * 5 * (size_t)n));
    GS_CUDA(cudaMalloc(&dido, sizeof(int) * 5 * (size_t)n));
    GS_CUDA(cudaMalloc(&dabcd, sizeof(float) * 4 * (size_t)n));
    GS_CUDA(cudaMalloc(&dok, sizeof(int) * (size_t)n));
    GS_CUDA(cudaMalloc(&ddist, sizeof(float) * (size_t)n));
    GS_CUDA(cudaMalloc(&drows, sizeof(double) * 13 * (size_t)n));
    GS_CUDA(cudaMalloc(&dfr, sizeof(Frame)));
    GS_CUDA(cudaMemcpy(dq, q, sizeof(float) * 15 * (size_t)n, cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(dg, g, sizeof(float) * 3 * (size_t)n, cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(did, id, sizeof(int) * 5 * (size_t)n, cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(dfr, &fr, sizeof(Frame), cudaMemcpyHostToDevice));
    gs_fit_sets_kernel<<<(unsigned)((n + 127) / 128), 128>>>(dq, dg, did, dfr, thr, est, n, dido, dabcd, dok, ddist, drows);
    GS_CUDA(cudaGetLastError());
    GS_CUDA(cudaMemcpy(id_out, dido, sizeof(int) * 5 * (size_t)n, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(abcd, dabcd, sizeof(float) * 4 * (size_t)n, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(ok, dok, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(dist, ddist, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    GS_CUDA(cudaMemcpy(rows, drows, sizeof(double) * 13 * (size_t)n, cudaMemcpyDeviceToHost));
out:
    cudaFree(dq); cudaFree(dg); cudaFree(did); cudaFree(dido); cudaFree(dabcd); cudaFree(dok); cudaFree(ddist); cudaFree(drows);
    cudaFree(dfr);
    return rc;
}

/* gs_manifold_kernel on n rows (host arrays: op[n], in[n x kManIn], out[n x kManOut]); returns a cudaError_t */
int gs_manifold(const int* op, const double* in, double* out, int n) {
    int rc = 0;
    int* dop = nullptr;
    double *din = nullptr, *dout = nullptr;
    GS_CUDA(cudaMalloc(&dop, sizeof(int) * (size_t)n));
    GS_CUDA(cudaMalloc(&din, sizeof(double) * kManIn * (size_t)n));
    GS_CUDA(cudaMalloc(&dout, sizeof(double) * kManOut * (size_t)n));
    GS_CUDA(cudaMemcpy(dop, op, sizeof(int) * (size_t)n, cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemcpy(din, in, sizeof(double) * kManIn * (size_t)n, cudaMemcpyHostToDevice));
    GS_CUDA(cudaMemset(dout, 0, sizeof(double) * kManOut * (size_t)n));
    gs_manifold_kernel<<<(unsigned)((n + 127) / 128), 128>>>(dop, din, dout, n);
    GS_CUDA(cudaGetLastError());
    GS_CUDA(cudaMemcpy(out, dout, sizeof(double) * kManOut * (size_t)n, cudaMemcpyDeviceToHost));
out:
    cudaFree(dop); cudaFree(din); cudaFree(dout);
    return rc;
}

}  // extern "C"
