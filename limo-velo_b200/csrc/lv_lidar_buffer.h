/*
 * lv_lidar_buffer.h — index arithmetic of the device LiDAR buffer: Accumulator::BUFFER_L (include/Headers/Accumulator.hpp:3)
 * with Buffer::push / clear(t) (src/Objects/Buffer.cpp:26-28,66-70) and Accumulator::get (Accumulator.hpp:61-74).
 *
 * The reference keeps a std::deque<Point> that Buffer::push grows at the FRONT: content[0] is the newest point inserted, and
 * across messages the order is arrival order, not time order.  The device keeps a ring of `cap` slots and two monotonically
 * increasing 64-bit counters head <= tail: position p (head <= p < tail) lives in slot p % cap, and
 *
 *     content[k] = ring[tail - 1 - k],   size = tail - head,   content.back() = ring[head].
 *
 * Everything here compiles for the device (lv_lidar_buffer.cu) and for the host (tests/cpu_shim/lidar_ring.cpp, test-only), so the
 * kernels and the host build share the probe sequence of the binary search, the predicates of the walk and of clear, and the
 * rules of the time-ordered merge.  Comparisons are written exactly as in the reference, so a NaN point time behaves as it does there.
 */
#ifndef LV_LIDAR_BUFFER_H_
#define LV_LIDAR_BUFFER_H_

#include <stdint.h>

#include "lv_hd.h"
#include "lv_point_math.h"

namespace lv {

/* the largest ring: the reference's indices are `int`, and (low + high) of its binary search must not overflow */
enum : int64_t { kLidarMaxCapacity = (int64_t)1 << 30 };

LV_HD int64_t lidar_slot(int64_t p, int64_t cap) { return p % cap; }
/* ring position of content[k] */
LV_HD int64_t lidar_pos(int64_t tail, int64_t k) { return tail - 1 - k; }
/* Buffer::push of n points keeps the ring's content only if they fit */
LV_HD bool lidar_fits(int64_t head, int64_t tail, int64_t n, int64_t cap) { return tail + n - head <= cap; }

/* Algorithms::binary_search(content, t, desc = true) (include/Headers/Utils.hpp:9-23), probe for probe: on content that is
 * not sorted (a late or overlapping message) the answer depends on exactly which elements it reads */
LV_HD int64_t lidar_binary_search(const double* time, int64_t cap, int64_t head, int64_t tail, double t) {
    int64_t low = 0, high = (tail - head) - 1;
    while (high >= low) {
        const int64_t mid = (low + high) / 2;
        (time[lidar_slot(lidar_pos(tail, mid), cap)] < t) ? high = mid - 1 : low = mid + 1;
    }
    if (--high < 0) return 0;
    return high;
}

/* Accumulator::get: the walk starts at k_t2 = max(0, binary_search(content, t2)), i.e. at this ring position; on an empty
 * buffer it is head - 1 (nothing to walk) */
LV_HD int64_t lidar_window_top(const double* time, int64_t cap, int64_t head, int64_t tail, double t2) {
    int64_t k = lidar_binary_search(time, cap, head, tail, t2);
    if (k < 0) k = 0;
    return lidar_pos(tail, k);
}
/* `if (t1 > cnt.time) break;` — the walk goes from the top to lower positions: it stops at the highest position <= top
 * for which this holds */
LV_HD bool lidar_breaks(double time, double t1) { return t1 > time; }
/* `if (t2 >= cnt.time) result.push_front(cnt);` — kept points come out in ascending position (oldest inserted first) */
LV_HD bool lidar_keeps(double time, double t2) { return t2 >= time; }
/* Buffer::clear(t): `while (size > 0 and t >= back().time) pop_back();` — head advances to the lowest position for which
 * this fails (a NaN time stops it, as it stops the loop) */
LV_HD bool lidar_pops(double time, double t) { return t >= time; }

/* The attribute lanes of a ring reserved with lv_lidar_reserve_full: the reference's BUFFER_L holds whole Points, and push / get
 * copy their intensity and range with xyz and time (Accumulator.hpp:61-74, Point.cpp:21-35).  One lane copy of element a of a
 * source into element b of a destination; a source without lanes (NULL) gives 0: a plain push onto a ring with lanes, or
 * lv_lidar_reserve_full over points that arrived before the ring had lanes. */
LV_HD void lidar_copy_lanes(const float* from_i, const float* from_r, int64_t a, float* to_i, float* to_r, int64_t b) {
    to_i[b] = from_i ? from_i[a] : 0.f;
    to_r[b] = from_r ? from_r[a] : 0.f;
}

/* ---- the time-ordered merge of one message (lv_lidar_merge_device_async): several sensors into one buffer ----------------------
 * L is the live content by ascending position, B the message's n points with times b[0, n).  The split s is one past the highest
 * live position whose time is <= b[0] (head when there is none), found by walking down from tail - 1; T_tail = positions [s, tail).
 * When T_tail and B are each in order (lidar_in_order on every element and its successor), positions [s, tail + n) become
 * std::merge(T_tail, B) by time, ring points first on equal times, and positions below s do not move: the message lands where its
 * times belong.  When B starts no earlier than the newest live point, s = tail and the merge is the plain push.  Otherwise (a NaN
 * time, a batch that is not time-sorted, a ring that a plain push left unsorted) B is appended as the plain push does and the
 * caller is told.  An empty B changes nothing. */
/* the walk's predicate: position p lies below the split */
LV_HD bool lidar_merge_below(double time, double b0) { return time <= b0; }
/* a followed by b is in order: neither is NaN and b is not less than a.  Element i of a run is checked against its successor, the
 * last one against itself, so a lone NaN is caught too. */
LV_HD bool lidar_in_order(double a, double b) { return a == a && b == b && !(b < a); }

/* what a merge does, decided once the split and the order are known; the two refusals leave the ring unchanged */
enum : uint32_t {
    kLidarMergeWrite = 0,        /* std::merge onto [s, tail + n)                                                    */
    kLidarMergeAppend = 1,       /* not in order: appended as the plain push, kAsyncLidarUnsorted                      */
    kLidarMergeFull = 2,         /* refused: the n points do not fit the ring, kAsyncLidarFull                          */
    kLidarMergeOverlap = 3       /* refused: T_tail holds more points than the merge reserve, kAsyncLidarOverlap      */
};
LV_HD uint32_t lidar_merge_mode(int64_t head, int64_t tail, int64_t split, int64_t n, int64_t cap, int64_t reserve, bool ordered) {
    if (!lidar_fits(head, tail, n, cap)) return kLidarMergeFull;
    if (!ordered) return kLidarMergeAppend;
    if (tail - split > reserve) return kLidarMergeOverlap;
    return kLidarMergeWrite;
}

/* the merge-path split of diagonal d: of the first d outputs of std::merge(a[0, m), b[0, n)) (a first on equal times), how many
 * come from a.  A binary search over the diagonal, so any output can be found without merging what comes before it. */
LV_HD int64_t lidar_merge_path(const double* a, int64_t m, const double* b, int64_t n, int64_t d) {
    int64_t lo = d > n ? d - n : 0, hi = d < m ? d : m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) / 2;
        if (!(b[d - 1 - mid] < a[mid])) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
/* output i + j of the merge is a[i] (true) or b[j] (false), with i of them from a before it */
LV_HD bool lidar_merge_takes_a(const double* a, int64_t m, const double* b, int64_t n, int64_t i, int64_t j) {
    return i < m && (j >= n || !(b[j] < a[i]));
}
/* the ring position of output o (T_tail's k-th point is staged at scratch index k, the position s + k) */
LV_HD int64_t lidar_merge_pos(int64_t split, int64_t o) { return split + o; }

/* point i of a message into the primary LiDAR's frame: rt_apply (RotTransl * Point, fp32 unfused), or the input bits unchanged
 * when there is no transform (no identity multiply: 0 * inf and -0.0 would change bits) */
LV_HD void lidar_merge_xyz(bool transform, const Rt32& T, const float* xyz, int64_t i, float* out) {
    if (transform) {
        rt_apply(T, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], out);
    } else {
        out[0] = xyz[3 * i];
        out[1] = xyz[3 * i + 1];
        out[2] = xyz[3 * i + 2];
    }
}

}  // namespace lv
#endif
