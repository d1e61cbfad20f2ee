/*
 * tests/cpu_shim_buffer/buffer.cpp — TEST-ONLY host build of the device LiDAR buffer's index arithmetic (lv_lidar_buffer.h).
 *
 * A ring of `cap` slots with the head / tail counters of lv_lidar_buffer.cu, driven serially through the header's functions:
 * the same slot mapping, the same binary search probe for probe, the same break / keep / pop predicates.  The kernels reduce
 * over chunks what this walks one position at a time: the break is the highest position at or below the top for which
 * lidar_breaks holds, the clear stops at the lowest position for which lidar_pops fails.  Not part of the product.
 */
#include <vector>

#include "../../limo-velo_b200/csrc/lv_lidar_buffer.h"

using namespace lv;

struct ShimRing {
    int64_t cap, head = 0, tail = 0;
    std::vector<float> xyz;
    std::vector<double> time;
};

extern "C" {

ShimRing* shim_lidar_create(int64_t cap) {
    ShimRing* r = new ShimRing();
    r->cap = cap;
    r->xyz.assign(3 * (size_t)cap, 0.f);
    r->time.assign((size_t)cap, 0.0);
    return r;
}
void shim_lidar_destroy(ShimRing* r) { delete r; }
int64_t shim_lidar_size(const ShimRing* r) { return r->tail - r->head; }
int64_t shim_lidar_tail(const ShimRing* r) { return r->tail; }
/* the times of content[0], content[1], ... (newest inserted first) */
void shim_lidar_content(const ShimRing* r, double* time) {
    for (int64_t k = 0; k < r->tail - r->head; ++k) time[k] = r->time[lidar_slot(lidar_pos(r->tail, k), r->cap)];
}

/* 1: appended; 0: they do not fit, the ring is unchanged */
int shim_lidar_push(ShimRing* r, const float* xyz, const double* time, int64_t n) {
    if (!lidar_fits(r->head, r->tail, n, r->cap)) return 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t s = lidar_slot(r->tail + i, r->cap);
        for (int c = 0; c < 3; ++c) r->xyz[3 * s + c] = xyz[3 * i + c];
        r->time[s] = time[i];
    }
    r->tail += n;
    return 1;
}

/* the window's size; its points are written (ascending position) only when it fits n_max */
int64_t shim_lidar_get(const ShimRing* r, double t1, double t2, float* xyz, double* time, int64_t n_max) {
    const int64_t top = lidar_window_top(r->time.data(), r->cap, r->head, r->tail, t2);
    int64_t brk = r->head - 1;
    for (int64_t p = top; p >= r->head; --p)
        if (lidar_breaks(r->time[lidar_slot(p, r->cap)], t1)) { brk = p; break; }
    int64_t count = 0;
    for (int64_t p = brk + 1; p <= top; ++p) count += lidar_keeps(r->time[lidar_slot(p, r->cap)], t2) ? 1 : 0;
    if (count > n_max) return count;
    int64_t o = 0;
    for (int64_t p = brk + 1; p <= top; ++p) {
        const int64_t s = lidar_slot(p, r->cap);
        if (!lidar_keeps(r->time[s], t2)) continue;
        for (int c = 0; c < 3; ++c) xyz[3 * o + c] = r->xyz[3 * s + c];
        time[o++] = r->time[s];
    }
    return count;
}

void shim_lidar_clear(ShimRing* r, double t) {
    int64_t stop = r->tail;
    for (int64_t p = r->head; p < r->tail; ++p)
        if (!lidar_pops(r->time[lidar_slot(p, r->cap)], t)) { stop = p; break; }
    r->head = stop;
}

}  // extern "C"
