/*
 * lv_deskew.h — State arithmetic of the Compensator, host+device (single precision like the reference).
 *
 *   state_add_imu     State::operator+= -> update -> propagate_f   src/Objects/State.cpp:73-75,103-132
 *   so3_exp_f         SO3Math::Exp<float, float>                    include/Headers/Utils.hpp:28-54
 *   deskew_point      the body of Compensator::compensate           src/Modules/Compensator.cpp:131-142
 *
 * fp32 arithmetic is unfused (lv_hd.h) and 3-term products are summed like the rest of the fp32 geometry
 * (lv_point_math.h); sinf / cosf are the platform's (CUDA's differ from glibc's in the last ulp, which is why
 * this stage is held to a tolerance, not to bit-exactness: tests/test_gpu_frontend.py).
 */
#ifndef LV_DESKEW_H_
#define LV_DESKEW_H_

#include "../../include/limovelo_b200.h"
#include "lv_point_math.h"

namespace lv {

LV_HD void m3mul_f(const float* A, const float* B, float* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[i * 3 + j] = dot3f(A[i * 3], A[i * 3 + 1], A[i * 3 + 2], B[j], B[3 + j], B[6 + j]);
}

LV_HD void so3_exp_f(const float* av, float dt, float* E) {
    const float n = fsqrt(fadd(fadd(fmul(av[0], av[0]), fmul(av[1], av[1])), fmul(av[2], av[2])));
    for (int i = 0; i < 9; ++i) E[i] = (i % 4 == 0) ? 1.f : 0.f;
    if (!((double)n > 0.0000001)) return;
    const float r[3] = {fdiv(av[0], n), fdiv(av[1], n), fdiv(av[2], n)};
    const float K[9] = {0.f, -r[2], r[1], r[2], 0.f, -r[0], -r[1], r[0], 0.f};
    const float ang = fmul(n, dt);
    const float sn = sinf(ang), c1 = (float)(1.0 - (double)cosf(ang));
    float cK[9], KK[9];
    for (int i = 0; i < 9; ++i) cK[i] = fmul(c1, K[i]);
    m3mul_f(cK, K, KK);
    for (int i = 0; i < 9; ++i) E[i] = fadd(fadd(E[i], fmul(sn, K[i])), KK[i]);
}

LV_HD void state_propagate(lv_state32* s, const float* a, const float* w, float dt) {   /* State.cpp:103-120 */
    float wb[3], ab[3], E[9], Rn[9], Rab[3];
    for (int i = 0; i < 3; ++i) { wb[i] = fsub(w[i], s->bw[i]); ab[i] = fsub(a[i], s->ba[i]); }
    so3_exp_f(wb, dt, E);
    m3mul_f(s->R, E, Rn);
    for (int i = 0; i < 3; ++i) Rab[i] = dot3f(s->R[i * 3], s->R[i * 3 + 1], s->R[i * 3 + 2], ab[0], ab[1], ab[2]);
    float vn[3], pn[3];
    for (int i = 0; i < 3; ++i) {
        const float acc = fsub(Rab[i], s->g[i]);
        vn[i] = fadd(s->vel[i], fmul(acc, dt));
        pn[i] = fadd(s->pos[i], fadd(fmul(s->vel[i], dt), fmul(fmul(fmul(0.5f, acc), dt), dt)));
    }
    for (int i = 0; i < 9; ++i) s->R[i] = Rn[i];
    for (int i = 0; i < 3; ++i) { s->vel[i] = vn[i]; s->pos[i] = pn[i]; }
}

LV_HD void state_add_imu(lv_state32* s, const float* a, const float* w, double time) {  /* State.cpp:122-132 */
    const float dt = (float)(time - s->time);
    state_propagate(s, a, w, dt);
    s->time = time;
    for (int i = 0; i < 3; ++i) {
        s->a[i] = fadd(fmul(0.5f, s->a[i]), fmul(0.5f, a[i]));
        s->w[i] = fadd(fmul(0.5f, s->w[i]), fmul(0.5f, w[i]));
    }
}

LV_HD Rt32 state_rt(const lv_state32& s) {       /* RotTransl(const State&) (RotTransl.cpp:19-22) */
    Rt32 r;
    for (int i = 0; i < 9; ++i) r.R[i] = s.R[i];
    for (int i = 0; i < 3; ++i) r.t[i] = s.pos[i];
    return r;
}
LV_HD Rt32 state_il(const lv_state32& s) {       /* State::I_Rt_L (State.cpp:64-69) */
    Rt32 r;
    for (int i = 0; i < 9; ++i) r.R[i] = s.RLI[i];
    for (int i = 0; i < 3; ++i) r.t[i] = s.tLI[i];
    return r;
}
/* Xt2.I_Rt_L().inv() * Xt2.inv()  (Compensator.cpp:139) */
LV_HD Rt32 deskew_back(const lv_state32& Xt2) { return rt_mul(rt_inv(state_il(Xt2)), rt_inv(state_rt(Xt2))); }

/* index s of the path segment Compensator::compensate assigns a (time-sorted) point to: the first s with
 * t <= path[s + 1].time (the while loop of Compensator.cpp:130-131 moves on when t > path[s + 1].time) */
LV_HD int deskew_segment(const lv_state32* path, int ns, double t) {
    int lo = 0, hi = ns - 2;            /* answer in [0, ns - 2] */
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (t <= path[mid + 1].time) hi = mid; else lo = mid + 1;
    }
    return lo;
}

LV_HD void deskew_point(const lv_state32* path, int ns, const Rt32& back, const float* p, double t, float* out) {
    lv_state32 X = path[deskew_segment(path, ns, t)];
    const float a[3] = {X.a[0], X.a[1], X.a[2]}, w[3] = {X.w[0], X.w[1], X.w[2]};
    state_add_imu(&X, a, w, t);                                   /* Compensator.cpp:133-134 */
    float g[3];
    rt_apply(rt_mul(state_rt(X), state_il(X)), p[0], p[1], p[2], g);   /* :137 */
    rt_apply(back, g[0], g[1], g[2], out);                        /* :138 */
}

}  // namespace lv
#endif
