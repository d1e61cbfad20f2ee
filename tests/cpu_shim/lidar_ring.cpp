/*
 * tests/cpu_shim/lidar_ring.cpp — TEST-ONLY host build of the device LiDAR buffer (lv_lidar_buffer.h).
 *
 * A ring of `cap` slots with the head / tail counters of lv_lidar_buffer.cu, xyz, time and, once it has them, the intensity /
 * range lanes of lv_lidar_reserve_full, driven serially through the header's functions as the push / get / move kernels use them:
 * the same slot mapping, the same binary search probe for probe, the same break / keep / pop predicates, and lidar_copy_lanes for
 * every lane copy (a source without lanes stores 0).  The kernels reduce over chunks what this walks one position at a time: the
 * break is the highest position at or below the top for which lidar_breaks holds, the clear stops at the lowest position for which
 * lidar_pops fails.  A ring created without lanes, pushed and read with NULL lanes, is the plain xyz + time buffer.  Not part of
 * the product.
 */
#include <vector>

#include "../../limo-velo_b200/csrc/lv_lidar_buffer.h"

using namespace lv;

struct ShimRing {
    int64_t cap, head = 0, tail = 0;
    bool lanes = false;
    std::vector<float> xyz, intensity, range;
    std::vector<double> time;
};

extern "C" {

ShimRing* shim_lidar_create(int64_t cap, int lanes) {
    ShimRing* r = new ShimRing();
    r->cap = cap;
    r->lanes = lanes != 0;
    r->xyz.assign(3 * (size_t)cap, 0.f);
    r->time.assign((size_t)cap, 0.0);
    if (r->lanes) { r->intensity.assign((size_t)cap, -1.f); r->range.assign((size_t)cap, -1.f); }
    return r;
}
void shim_lidar_destroy(ShimRing* r) { delete r; }
int64_t shim_lidar_size(const ShimRing* r) { return r->tail - r->head; }
/* the times of content[0], content[1], ... (newest inserted first) */
void shim_lidar_content(const ShimRing* r, double* time) {
    for (int64_t k = 0; k < r->tail - r->head; ++k) time[k] = r->time[lidar_slot(lidar_pos(r->tail, k), r->cap)];
}

/* lv_lidar_reserve (lanes = 0: keep the ring's) / lv_lidar_reserve_full (lanes = 1): the live positions into new arrays, slot
 * p % new_cap; 0 when more points are live than fit */
int shim_lidar_reserve(ShimRing* r, int64_t cap, int lanes) {
    if (r->tail - r->head > cap) return 0;
    ShimRing n;
    n.cap = cap;
    n.lanes = lanes || r->lanes;
    n.xyz.assign(3 * (size_t)cap, 0.f);
    n.time.assign((size_t)cap, 0.0);
    if (n.lanes) { n.intensity.assign((size_t)cap, -1.f); n.range.assign((size_t)cap, -1.f); }
    for (int64_t p = r->head; p < r->tail; ++p) {
        const int64_t a = lidar_slot(p, r->cap), b = lidar_slot(p, cap);
        for (int c = 0; c < 3; ++c) n.xyz[3 * b + c] = r->xyz[3 * a + c];
        n.time[b] = r->time[a];
        if (n.lanes)
            lidar_copy_lanes(r->lanes ? r->intensity.data() : nullptr, r->lanes ? r->range.data() : nullptr, a, n.intensity.data(),
                             n.range.data(), b);
    }
    r->cap = cap;
    r->lanes = n.lanes;
    r->xyz.swap(n.xyz);
    r->time.swap(n.time);
    r->intensity.swap(n.intensity);
    r->range.swap(n.range);
    return 1;
}

/* 1: appended; 0: they do not fit, the ring is unchanged.  intensity / range NULL: the plain push (lanes, if any, get 0) */
int shim_lidar_push(ShimRing* r, const float* xyz, const double* time, const float* intensity, const float* range, int64_t n) {
    if (!lidar_fits(r->head, r->tail, n, r->cap)) return 0;
    for (int64_t i = 0; i < n; ++i) {
        const int64_t s = lidar_slot(r->tail + i, r->cap);
        for (int c = 0; c < 3; ++c) r->xyz[3 * s + c] = xyz[3 * i + c];
        r->time[s] = time[i];
        if (r->lanes) lidar_copy_lanes(intensity, range, i, r->intensity.data(), r->range.data(), s);
    }
    r->tail += n;
    return 1;
}

/* the window's size; its points are written (ascending position) only when it fits n_max, and their lanes too when intensity /
 * range are non-NULL (a ring with lanes only), as in launch_lidar_get */
int64_t shim_lidar_get(const ShimRing* r, double t1, double t2, float* xyz, double* time, float* intensity, float* range, int64_t n_max) {
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
        time[o] = r->time[s];
        if (intensity) lidar_copy_lanes(r->intensity.data(), r->range.data(), s, intensity, range, o);
        ++o;
    }
    return count;
}

void shim_lidar_clear(ShimRing* r, double t) {
    int64_t stop = r->tail;
    for (int64_t p = r->head; p < r->tail; ++p)
        if (!lidar_pops(r->time[lidar_slot(p, r->cap)], t)) { stop = p; break; }
    r->head = stop;
}

/* content[k] (newest inserted first) with its lanes (0 on a ring without them) */
void shim_lidar_content_full(const ShimRing* r, float* xyz, double* time, float* intensity, float* range) {
    for (int64_t k = 0; k < r->tail - r->head; ++k) {
        const int64_t s = lidar_slot(lidar_pos(r->tail, k), r->cap);
        for (int c = 0; c < 3; ++c) xyz[3 * k + c] = r->xyz[3 * s + c];
        time[k] = r->time[s];
        intensity[k] = r->lanes ? r->intensity[s] : 0.f;
        range[k] = r->lanes ? r->range[s] : 0.f;
    }
}

/* lv_lidar_merge_device_async with a merge reserve of `reserve` points.  T: 12 floats or NULL; intensity / range NULL: the plain
 * form.  Returns the mode (kLidarMerge*). */
int shim_lidar_merge(ShimRing* r, const float* xyz, const double* time, const float* intensity, const float* range, int64_t n, const float* T,
                     int64_t reserve) {
    const int64_t head = r->head, tail = r->tail, cap = r->cap;
    int64_t split = tail;
    bool ordered = true;
    if (n > 0) {
        split = head;
        for (int64_t p = tail - 1; p >= head; --p)
            if (lidar_merge_below(r->time[lidar_slot(p, cap)], time[0])) { split = p + 1; break; }
        for (int64_t p = split; p < tail; ++p)
            ordered = ordered && lidar_in_order(r->time[lidar_slot(p, cap)], r->time[lidar_slot(p + 1 < tail ? p + 1 : p, cap)]);
        for (int64_t i = 0; i < n; ++i) ordered = ordered && lidar_in_order(time[i], time[i + 1 < n ? i + 1 : i]);
    }
    const uint32_t mode = lidar_merge_mode(head, tail, split, n, cap, reserve, ordered);
    Rt32 rt{};
    if (T) {
        for (int k = 0; k < 9; ++k) rt.R[k] = T[k];
        for (int k = 0; k < 3; ++k) rt.t[k] = T[9 + k];
    }
    const float* from_i = r->lanes ? intensity : nullptr;
    const float* from_r = r->lanes ? range : nullptr;
    auto store = [&](int64_t s, const float* px, const double* pt, int64_t i, bool transform, const float* li, const float* lr) {
        lidar_merge_xyz(transform, rt, px, i, &r->xyz[3 * s]);
        r->time[s] = pt[i];
        if (r->lanes) lidar_copy_lanes(li, lr, i, r->intensity.data(), r->range.data(), s);
    };
    if (mode == kLidarMergeWrite) {
        const int64_t m = tail - split;
        std::vector<float> a_xyz(3 * (size_t)m), a_i((size_t)m), a_r((size_t)m);
        std::vector<double> a_time((size_t)m);
        for (int64_t k = 0; k < m; ++k) {
            const int64_t s = lidar_slot(lidar_merge_pos(split, k), cap);
            for (int c = 0; c < 3; ++c) a_xyz[3 * k + c] = r->xyz[3 * s + c];
            a_time[k] = r->time[s];
            if (r->lanes) lidar_copy_lanes(r->intensity.data(), r->range.data(), s, a_i.data(), a_r.data(), k);
        }
        for (int64_t o = 0; o < m + n; ++o) {
            const int64_t i = lidar_merge_path(a_time.data(), m, time, n, o), j = o - i;
            const int64_t s = lidar_slot(lidar_merge_pos(split, o), cap);
            if (lidar_merge_takes_a(a_time.data(), m, time, n, i, j)) store(s, a_xyz.data(), a_time.data(), i, false, a_i.data(), a_r.data());
            else store(s, xyz, time, j, T != nullptr, from_i, from_r);
        }
    } else if (mode == kLidarMergeAppend) {
        for (int64_t i = 0; i < n; ++i) store(lidar_slot(tail + i, cap), xyz, time, i, T != nullptr, from_i, from_r);
    }
    if (mode == kLidarMergeWrite || mode == kLidarMergeAppend) r->tail = tail + n;
    return (int)mode;
}

}  // extern "C"
