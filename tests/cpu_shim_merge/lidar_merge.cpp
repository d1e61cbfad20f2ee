/*
 * tests/cpu_shim_merge/lidar_merge.cpp — TEST-ONLY host build of the time-ordered merge of the device LiDAR buffer
 * (lv_lidar_buffer.h, lv_lidar_merge_device_async).
 *
 * The ring, its push, get and clear are tests/cpu_shim/lidar_ring.cpp, compiled here unchanged, so the merge runs on the same ring
 * the buffer's host build drives.  The merge uses the header's walk predicate, order rule, mode, merge path and transform: the walk
 * one position at a time, the order of T_tail and B, the mode, then T_tail staged and every output found by the merge path of its
 * own diagonal (the kernel finds one per kMergeItems outputs and merges the rest serially).  Not part of the product.
 */
#include "../cpu_shim/lidar_ring.cpp"

extern "C" {

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
