/*
 * lv_preloc.h — the arithmetic of lv_prelocalize (a start pose in a saved map), host+device.
 *
 * A brute-force search over position and heading about the gravity axis: every candidate pose scores the number of sweep
 * points whose world point lands in a voxel that holds map points (the occupancy bit of the block table, lv_voxel_map.h).
 * The host builds one frame per heading (preloc_heading_frame) and one offset per position (preloc_offset); the kernel
 * (lv_preloc.cu) only reads those tables and the map.  For heading 0 and offset 0 the world points are those of
 * lv_match_all at the base state (rt_apply of make_frame's lidar_to_world), bit for bit.
 *
 * tests/cpu_shim/preloc.cpp runs these functions serially on the host.
 */
#ifndef LV_PRELOC_H_
#define LV_PRELOC_H_

#include "lv_voxel_map.h"

namespace lv {

enum { kPrelocMaxPoints = 4096 };
#define LV_PRELOC_MAX_CANDIDATES ((int64_t)1 << 24)

/* half-width in grid steps: floor(range / step + 1e-9) (the 1e-9 keeps an exact multiple that rounds just below) */
LV_HD double preloc_half(float range, float step) { return floor((double)range / (double)step + 1e-9); }

/* rotation axis g = grav / |grav| and the position axes u, v: u = normalize(e - (e.g) g), v = g x u, with e the world x axis,
 * or the y axis when |g_x| > 0.9 */
struct PrelocAxes {
    double g[3], u[3], v[3];
};
LV_HD PrelocAxes preloc_axes(const double* x) {
    PrelocAxes a;
    const double* gr = x + kGrav;
    const double gn = sqrt(dot3d(gr[0], gr[1], gr[2], gr[0], gr[1], gr[2]));
    for (int c = 0; c < 3; ++c) a.g[c] = gr[c] / gn;
    double e[3] = {1.0, 0.0, 0.0};
    if (fabs(a.g[0]) > 0.9) { e[0] = 0.0; e[1] = 1.0; }
    const double eg = dot3d(e[0], e[1], e[2], a.g[0], a.g[1], a.g[2]);
    double w[3];
    for (int c = 0; c < 3; ++c) w[c] = dsub(e[c], dmul(eg, a.g[c]));
    const double wn = sqrt(dot3d(w[0], w[1], w[2], w[0], w[1], w[2]));
    for (int c = 0; c < 3; ++c) a.u[c] = w[c] / wn;
    a.v[0] = dsub(dmul(a.g[1], a.u[2]), dmul(a.g[2], a.u[1]));
    a.v[1] = dsub(dmul(a.g[2], a.u[0]), dmul(a.g[0], a.u[2]));
    a.v[2] = dsub(dmul(a.g[0], a.u[1]), dmul(a.g[1], a.u[0]));
    return a;
}

/* q(g, theta): the rotation by theta about g, right-hand rule, (x, y, z, w) */
LV_HD Quatd preloc_quat(const PrelocAxes& a, double theta) {
    const double half = dmul(0.5, theta);
    const double s = sin(half), c = cos(half);
    Quatd q;
    q.x = dmul(s, a.g[0]); q.y = dmul(s, a.g[1]); q.z = dmul(s, a.g[2]); q.w = c;
    return q;
}

/* the state of heading theta before the position offset: rot' = q(g, theta) (x) rot, vel' = R(g, theta) vel, every other
 * field as in x.  theta == 0 keeps x as it is (so the base candidate is the base state bit for bit). */
LV_HD void preloc_rotate_state(const double* x, const PrelocAxes& a, double theta, double* out) {
    for (int i = 0; i < kStateLen; ++i) out[i] = x[i];
    if (theta == 0.0) return;
    const Quatd q = preloc_quat(a, theta);
    store_quat(out + kRot, quat_mul(q, load_quat(x + kRot)));
    const Mat3d R = quat_to_rot(q);
    const double* v = x + kVel;
    for (int r = 0; r < 3; ++r) out[kVel + r] = dot3d(R.m[3 * r], R.m[3 * r + 1], R.m[3 * r + 2], v[0], v[1], v[2]);
}

/* the fp64 position offset a u + b v (products, then the sum) */
LV_HD void preloc_offset_d(const PrelocAxes& ax, double a, double b, double* o) {
    for (int c = 0; c < 3; ++c) o[c] = dadd(dmul(a, ax.u[c]), dmul(b, ax.v[c]));
}
/* ... and the fp32 offset the world points move by */
LV_HD void preloc_offset(const PrelocAxes& ax, double a, double b, float* o) {
    double d[3];
    preloc_offset_d(ax, a, b, d);
    for (int c = 0; c < 3; ++c) o[c] = (float)d[c];
}

/* the candidate state: preloc_rotate_state, then pos' = pos + (a u + b v) in fp64 */
LV_HD void preloc_candidate(const double* x, const PrelocAxes& ax, double theta, double a, double b, double* out) {
    preloc_rotate_state(x, ax, theta, out);
    double d[3];
    preloc_offset_d(ax, a, b, d);
    for (int c = 0; c < 3; ++c) out[kPos + c] = dadd(x[kPos + c], d[c]);
}

/* F_k = make_frame(x with rot', vel').lidar_to_world: the LiDAR-to-world transform of heading theta at the base position */
LV_HD Rt32 preloc_heading_frame(const double* x, const PrelocAxes& ax, double theta) {
    double xr[kStateLen];
    preloc_rotate_state(x, ax, theta, xr);
    Frame f;
    make_frame(xr, &f);
    return f.lidar_to_world;
}

/* index into the sweep of scored point s of S (of n): floor(s n / S) */
LV_HD int64_t preloc_point_index(int64_t s, int64_t n, int64_t S) { return s * n / S; }

/* the three rows of F.R applied to p (dot3f, as rt_apply) */
LV_HD void preloc_rows(const Rt32& F, float px, float py, float pz, float* r) {
    r[0] = dot3f(F.R[0], F.R[1], F.R[2], px, py, pz);
    r[1] = dot3f(F.R[3], F.R[4], F.R[5], px, py, pz);
    r[2] = dot3f(F.R[6], F.R[7], F.R[8], px, py, pz);
}

/* 1 when the world point r + t (t = fadd(F.t, offset)) lies in a voxel that holds map points.  A coordinate that is not
 * below 1e9 in magnitude (or NaN) never scores: the map stores no such point (map_point_key). */
LV_HD int preloc_hit(const VoxelMapView& m, float rx, float ry, float rz, const float* t) {
    const float wx = fadd(rx, t[0]), wy = fadd(ry, t[1]), wz = fadd(rz, t[2]);
    if (!(fabsf(wx) < 1e9f && fabsf(wy) < 1e9f && fabsf(wz) < 1e9f)) return 0;
    const uint32_t bx = voxel_coord(m.grid, wx), by = voxel_coord(m.grid, wy), bz = voxel_coord(m.grid, wz);
    const uint64_t mask = block_find(m, voxel_key(bx >> 2, by >> 2, bz >> 2));
    return (int)((mask >> block_bit(bx, by, bz)) & 1ull);
}

/* The selection key of a candidate: the highest key wins.  Score first; then the smaller |k|, then the smaller i^2 + j^2 (packed
 * as |k| (2 I^2 + 1) + i^2 + j^2, which stays below (2K+1)(2I+1)^2 <= 2^24), then the smaller linear index (< 2^24). */
LV_HD uint64_t preloc_key(int32_t score, int64_t k, int64_t i, int64_t j, int64_t I, int64_t idx) {
    const uint64_t ak = (uint64_t)(k < 0 ? -k : k);
    const uint64_t tie = ak * (uint64_t)(2 * I * I + 1) + (uint64_t)(i * i + j * j);
    return ((uint64_t)(uint32_t)score << 48) | ((0xFFFFFFull - tie) << 24) | (0xFFFFFFull - (uint64_t)idx);
}
LV_HD int64_t preloc_key_index(uint64_t key) { return (int64_t)(0xFFFFFFull - (key & 0xFFFFFFull)); }
LV_HD int32_t preloc_key_score(uint64_t key) { return (int32_t)(key >> 48); }

}  // namespace lv
#endif
