/*
 * lv_oracle.cpp — CPU oracle: restatement of LIMO-Velo's Localizator::correct path.
 *
 * TEST INFRASTRUCTURE ONLY (see lv_oracle.h).  Never linked into the product.
 * Compile with -ffp-contract=off: the reference is built "-std=c++14 -O3" for
 * baseline x86-64 (CMakeLists.txt:8,16), i.e. without FMA contraction.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference; esekfom.hpp = include/IKFoM/IKFoM_toolkit/esekfom/esekfom.hpp,
 * mtk/... = include/IKFoM/IKFoM_toolkit/mtk/...).
 */
#include "lv_oracle.h"

#include <dlfcn.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <unordered_map>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------
// small fixed-size helpers (row-major)
// ------------------------------------------------------------------------------------------
typedef double M3[9];

inline void mat3_mul(const double* A, const double* B, double* C) {
    double T[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            T[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
    memcpy(C, T, sizeof(T));
}
inline void mat3_T(const double* A, double* B) {
    double T[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[i * 3 + j] = A[j * 3 + i];
    memcpy(B, T, sizeof(T));
}
inline void mat3_vec(const double* A, const double* v, double* r) {
    double t[3];
    for (int i = 0; i < 3; ++i) t[i] = A[i * 3 + 0] * v[0] + A[i * 3 + 1] * v[1] + A[i * 3 + 2] * v[2];
    r[0] = t[0]; r[1] = t[1]; r[2] = t[2];
}
// mtk/src/mtkmath.hpp:176-183
inline void hat(const double* v, double* H) {
    H[0] = 0;     H[1] = -v[2]; H[2] = v[1];
    H[3] = v[2];  H[4] = 0;     H[5] = -v[0];
    H[6] = -v[1]; H[7] = v[0];  H[8] = 0;
}
const double kTol = 1e-11;  // MTK::tolerance<double>, mtkmath.hpp:122

// Eigen::Quaternion::toRotationMatrix (q = x,y,z,w)
void quat_to_rot(const double* q, double* R) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2 * x, ty = 2 * y, tz = 2 * z;
    const double twx = tx * w, twy = ty * w, twz = tz * w;
    const double txx = tx * x, txy = ty * x, txz = tz * x;
    const double tyy = ty * y, tyz = tz * y, tzz = tz * z;
    R[0] = 1 - (tyy + tzz); R[1] = txy - twz;       R[2] = txz + twy;
    R[3] = txy + twz;       R[4] = 1 - (txx + tzz); R[5] = tyz - twx;
    R[6] = txz - twy;       R[7] = tyz + twx;       R[8] = 1 - (txx + tyy);
}
// Eigen quaternion product a*b
void quat_mul(const double* a, const double* b, double* r) {
    const double ax = a[0], ay = a[1], az = a[2], aw = a[3];
    const double bx = b[0], by = b[1], bz = b[2], bw = b[3];
    double t[4];
    t[3] = aw * bw - ax * bx - ay * by - az * bz;
    t[0] = aw * bx + ax * bw + ay * bz - az * by;
    t[1] = aw * by + ay * bw + az * bx - ax * bz;
    t[2] = aw * bz + az * bw + ax * by - ay * bx;
    memcpy(r, t, sizeof(t));
}
// Eigen Quaternion(Matrix3) (quat_product / QuaternionBase::operator=(MatrixBase))
void rot_to_quat(const double* R, double* q) {
    double t = R[0] + R[4] + R[8];
    if (t > 0) {
        t = std::sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (R[7] - R[5]) * t;
        q[1] = (R[2] - R[6]) * t;
        q[2] = (R[3] - R[1]) * t;
    } else {
        int i = 0;
        if (R[4] > R[0]) i = 1;
        if (R[8] > R[i * 3 + i]) i = 2;
        int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(R[i * 3 + i] - R[j * 3 + j] - R[k * 3 + k] + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (R[k * 3 + j] - R[j * 3 + k]) * t;
        q[j] = (R[j * 3 + i] + R[i * 3 + j]) * t;
        q[k] = (R[k * 3 + i] + R[i * 3 + k]) * t;
    }
}

// mtkmath.hpp:142-174
void cos_sinc_sqrt(double x2, double* c, double* s) {
    static const double taylor_0_bound = std::numeric_limits<double>::epsilon();
    static const double taylor_2_bound = std::sqrt(taylor_0_bound);
    static const double taylor_n_bound = std::sqrt(taylor_2_bound);
    if (x2 >= taylor_n_bound) {
        double x = std::sqrt(x2);
        *c = std::cos(x);
        *s = std::sin(x) / x;
        return;
    }
    static const double inv[] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
    double cosi = 1., sinc = 1;
    double term = -1 / 2. * x2;
    for (int i = 0; i < 3; ++i) {
        cosi += term;
        term *= inv[2 * i];
        sinc += term;
        term *= -inv[2 * i + 1] * x2;
    }
    *c = cosi;
    *s = sinc;
}
// MTK::exp (mtkmath.hpp:249-256) producing a quaternion: SO3::exp (SOn.hpp:284-288) passes scale/2
void so3_exp(const double* v, double scale_half, double* q) {
    double norm2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    double c, s;
    cos_sinc_sqrt(scale_half * scale_half * norm2, &c, &s);
    double mult = s * scale_half;
    q[0] = mult * v[0]; q[1] = mult * v[1]; q[2] = mult * v[2]; q[3] = c;
}
// SO3::log via MTK::log(scale=2, plus_minus_periodicity=true) (SOn.hpp:293-297, mtkmath.hpp:268-288)
void so3_log(const double* q, double* r) {
    double nv = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    if (nv < kTol) nv = kTol;
    double s = 2.0 / nv * std::atan(nv / q[3]);
    r[0] = s * q[0]; r[1] = s * q[1]; r[2] = s * q[2];
}
// mtkmath.hpp:235-247
void A_matrix(const double* v, double* A) {
    double sq = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    double norm = std::sqrt(sq);
    for (int i = 0; i < 9; ++i) A[i] = (i % 4 == 0) ? 1.0 : 0.0;
    if (norm < kTol) return;
    double H[9], HH[9];
    hat(v, H);
    mat3_mul(H, H, HH);
    double a = (1 - std::cos(norm)) / sq, b = (1 - std::sin(norm) / norm) / sq;
    for (int i = 0; i < 9; ++i) A[i] += a * H[i] + b * HH[i];
}

// S2 with length 98090/10000, S2_typ = 1 (use-ikfom.hpp:8; S2.hpp:97-118)
const double kS2Len = 98090.0 / 10000.0;
// S2.hpp:215-231 (typ 1 branch), Bx is 3x2 row-major
void S2_Bx(const double* v, double* B) {
    const double L = kS2Len;
    if (v[0] + L > kTol) {
        B[0] = -v[1];                          B[1] = -v[2];
        B[2] = L - v[1] * v[1] / (L + v[0]);   B[3] = -v[2] * v[1] / (L + v[0]);
        B[4] = -v[2] * v[1] / (L + v[0]);      B[5] = L - v[2] * v[2] / (L + v[0]);
        for (int i = 0; i < 6; ++i) B[i] /= L;
    } else {
        for (int i = 0; i < 6; ++i) B[i] = 0;
        B[1 * 2 + 1] = -1;
        B[2 * 2 + 0] = 1;
    }
}
// S2.hpp:136-142
void S2_boxplus(double* v, const double* d2) {
    double B[6];
    S2_Bx(v, B);
    double Bu[3] = {B[0] * d2[0] + B[1] * d2[1], B[2] * d2[0] + B[3] * d2[1], B[4] * d2[0] + B[5] * d2[1]};
    double q[4], R[9];
    so3_exp(Bu, 0.5, q);
    quat_to_rot(q, R);
    mat3_vec(R, v, v);
}
// S2.hpp:144-167   res = this [-] other
void S2_boxminus(const double* v, const double* o, double* res) {
    double H[9], hv[3];
    hat(v, H);
    mat3_vec(H, o, hv);
    double v_sin = std::sqrt(hv[0] * hv[0] + hv[1] * hv[1] + hv[2] * hv[2]);
    double v_cos = v[0] * o[0] + v[1] * o[1] + v[2] * o[2];
    double theta = std::atan2(v_sin, v_cos);
    if (v_sin < kTol) {
        if (std::fabs(theta) > kTol) { res[0] = 3.1415926; res[1] = 0; }
        else { res[0] = 0; res[1] = 0; }
        return;
    }
    double B[6], Ho[9], t[3];
    S2_Bx(o, B);
    hat(o, Ho);
    mat3_vec(Ho, v, t);
    double f = theta / v_sin;
    // Bx^T (2x3) * t
    res[0] = f * (B[0] * t[0] + B[2] * t[1] + B[4] * t[2]);
    res[1] = f * (B[1] * t[0] + B[3] * t[1] + B[5] * t[2]);
}
// S2.hpp:259-264  Nx (2x3) = 1/L^2 * Bx^T * hat(vec)
void S2_Nx_yy(const double* v, double* N) {
    double B[6], H[9];
    S2_Bx(v, B);
    hat(v, H);
    for (int i = 0; i < 2; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += B[k * 2 + i] * H[k * 3 + j];
            N[i * 3 + j] = 1 / kS2Len / kS2Len * s;
        }
}
// S2.hpp:266-280  Mx (3x2); note scalar(1/2) == 0 -> exp_delta = identity
void S2_Mx(const double* v, const double* d2, double* Mx) {
    double B[6], H[9];
    S2_Bx(v, B);
    hat(v, H);
    double nd = std::sqrt(d2[0] * d2[0] + d2[1] * d2[1]);
    if (nd < kTol) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 2; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += H[i * 3 + k] * B[k * 2 + j];
                Mx[i * 2 + j] = -s;
            }
        return;
    }
    double Bu[3] = {B[0] * d2[0] + B[1] * d2[1], B[2] * d2[0] + B[3] * d2[1], B[4] * d2[0] + B[5] * d2[1]};
    double q[4], E[9], A[9], At[9], T1[9], T2[9];
    so3_exp(Bu, 0.0 /* scalar(1/2) is integer division: esekfom quirk 2 */, q);
    quat_to_rot(q, E);
    A_matrix(Bu, A);
    mat3_T(A, At);
    mat3_mul(E, H, T1);
    mat3_mul(T1, At, T2);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 2; ++j) {
            double s = 0;
            for (int k = 0; k < 3; ++k) s += T2[i * 3 + k] * B[k * 2 + j];
            Mx[i * 2 + j] = -s;
        }
}

// state field offsets in the flat 26-double layout
enum { S_POS = 0, S_ROT = 3, S_OFFR = 7, S_OFFT = 11, S_VEL = 14, S_BG = 17, S_BA = 20, S_GRAV = 23 };

// mtk/build_manifold.hpp:192-194 with the per-type boxplus (SOn.hpp:233-236, S2.hpp:136-142, vect.hpp:117-119)
void state_boxplus(double* x, const double* d) {
    for (int i = 0; i < 3; ++i) x[S_POS + i] += d[0 + i];
    double q[4];
    so3_exp(d + 3, 0.5, q);
    quat_mul(x + S_ROT, q, x + S_ROT);
    so3_exp(d + 6, 0.5, q);
    quat_mul(x + S_OFFR, q, x + S_OFFR);
    for (int i = 0; i < 3; ++i) x[S_OFFT + i] += d[9 + i];
    for (int i = 0; i < 3; ++i) x[S_VEL + i] += d[12 + i];
    for (int i = 0; i < 3; ++i) x[S_BG + i] += d[15 + i];
    for (int i = 0; i < 3; ++i) x[S_BA + i] += d[18 + i];
    S2_boxplus(x + S_GRAV, d + 21);
}
// build_manifold.hpp:198-200 ; res = x [-] y
void state_boxminus(const double* x, const double* y, double* d) {
    for (int i = 0; i < 3; ++i) d[0 + i] = x[S_POS + i] - y[S_POS + i];
    double yc[4], r[4];
    yc[0] = -y[S_ROT]; yc[1] = -y[S_ROT + 1]; yc[2] = -y[S_ROT + 2]; yc[3] = y[S_ROT + 3];
    quat_mul(yc, x + S_ROT, r);
    so3_log(r, d + 3);
    yc[0] = -y[S_OFFR]; yc[1] = -y[S_OFFR + 1]; yc[2] = -y[S_OFFR + 2]; yc[3] = y[S_OFFR + 3];
    quat_mul(yc, x + S_OFFR, r);
    so3_log(r, d + 6);
    for (int i = 0; i < 3; ++i) d[9 + i] = x[S_OFFT + i] - y[S_OFFT + i];
    for (int i = 0; i < 3; ++i) d[12 + i] = x[S_VEL + i] - y[S_VEL + i];
    for (int i = 0; i < 3; ++i) d[15 + i] = x[S_BG + i] - y[S_BG + i];
    for (int i = 0; i < 3; ++i) d[18 + i] = x[S_BA + i] - y[S_BA + i];
    S2_boxminus(x + S_GRAV, y + S_GRAV, d + 21);
}

// ------------------------------------------------------------------------------------------
// dense algebra: partial-pivot LU inverse (Eigen fixed-size inverse() for n>4 is
// PartialPivLU::inverse) and a cyclic Jacobi eigen-solver for the symmetric 6x6 block.
// ------------------------------------------------------------------------------------------
void inverse_n(const double* A, int n, double* Ainv) {
    std::vector<double> lu(A, A + n * n);
    std::vector<int> perm(n);
    for (int i = 0; i < n; ++i) perm[i] = i;
    for (int k = 0; k < n; ++k) {
        int piv = k;
        double best = std::fabs(lu[k * n + k]);
        for (int i = k + 1; i < n; ++i)
            if (std::fabs(lu[i * n + k]) > best) { best = std::fabs(lu[i * n + k]); piv = i; }
        if (piv != k) {
            for (int j = 0; j < n; ++j) std::swap(lu[k * n + j], lu[piv * n + j]);
            std::swap(perm[k], perm[piv]);
        }
        double d = lu[k * n + k];
        for (int i = k + 1; i < n; ++i) {
            double f = lu[i * n + k] / d;
            lu[i * n + k] = f;
            for (int j = k + 1; j < n; ++j) lu[i * n + j] -= f * lu[k * n + j];
        }
    }
    // solve LU X = P I column by column
    std::vector<double> col(n);
    for (int c = 0; c < n; ++c) {
        for (int i = 0; i < n; ++i) col[i] = (perm[i] == c) ? 1.0 : 0.0;
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < i; ++j) col[i] -= lu[i * n + j] * col[j];
        for (int i = n - 1; i >= 0; --i) {
            for (int j = i + 1; j < n; ++j) col[i] -= lu[i * n + j] * col[j];
            col[i] /= lu[i * n + i];
        }
        for (int i = 0; i < n; ++i) Ainv[i * n + c] = col[i];
    }
}

// cyclic Jacobi for symmetric n x n; eigenvalues ascending, eigenvectors = columns of V,
// sign-normalised so that the largest-magnitude component of each vector is positive.
void sym_eig(const double* Ain, int n, double* evals, double* V) {
    std::vector<double> A(Ain, Ain + n * n);
    for (int i = 0; i < n * n; ++i) V[i] = (i % (n + 1) == 0) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0;
        for (int i = 0; i < n; ++i)
            for (int j = i + 1; j < n; ++j) off += A[i * n + j] * A[i * n + j];
        double diag = 0;
        for (int i = 0; i < n; ++i) diag += A[i * n + i] * A[i * n + i];
        if (off <= 1e-30 * diag || off == 0.0) break;
        for (int p = 0; p < n; ++p)
            for (int q = p + 1; q < n; ++q) {
                double apq = A[p * n + q];
                if (apq == 0.0) continue;
                double theta = (A[q * n + q] - A[p * n + p]) / (2 * apq);
                double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1));
                double c = 1 / std::sqrt(t * t + 1), s = t * c;
                for (int k = 0; k < n; ++k) {
                    double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; ++k) {
                    double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; ++k) {
                    double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s * vkq;
                    V[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
    std::vector<int> order(n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return A[a * n + a] < A[b * n + b]; });
    std::vector<double> Vs(n * n);
    for (int j = 0; j < n; ++j) {
        int src = order[j];
        evals[j] = A[src * n + src];
        int imax = 0;
        for (int k = 1; k < n; ++k)
            if (std::fabs(V[k * n + src]) > std::fabs(V[imax * n + src])) imax = k;
        double sg = V[imax * n + src] < 0 ? -1.0 : 1.0;
        for (int k = 0; k < n; ++k) Vs[k * n + j] = sg * V[k * n + src];
    }
    memcpy(V, Vs.data(), sizeof(double) * n * n);
}

// ------------------------------------------------------------------------------------------
// fp32 geometry: State / RotTransl / Plane / Match (all single precision in the reference)
// ------------------------------------------------------------------------------------------
struct Rt32 { float R[9]; float t[3]; };

inline void m3mul_f(const float* A, const float* B, float* C) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            C[i * 3 + j] = (A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j]) + A[i * 3 + 2] * B[2 * 3 + j];
}
inline void m3vec_f(const float* A, const float* v, float* r) {
    for (int i = 0; i < 3; ++i) r[i] = (A[i * 3 + 0] * v[0] + A[i * 3 + 1] * v[1]) + A[i * 3 + 2] * v[2];
}
// RotTransl operator* (RotTransl.cpp:36-41): (R1 R2, R1 t2 + t1)
inline Rt32 rt_mul(const Rt32& a, const Rt32& b) {
    Rt32 r;
    m3mul_f(a.R, b.R, r.R);
    float t[3];
    m3vec_f(a.R, b.t, t);
    for (int i = 0; i < 3; ++i) r.t[i] = t[i] + a.t[i];
    return r;
}
// RotTransl::inv (RotTransl.cpp:29-34): (R^T, -R^T t)
inline Rt32 rt_inv(const Rt32& a) {
    Rt32 r;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r.R[i * 3 + j] = a.R[j * 3 + i];
    float nR[9];
    for (int i = 0; i < 9; ++i) nR[i] = -r.R[i];
    m3vec_f(nR, a.t, r.t);
    return r;
}
// RotTransl * Point (RotTransl.cpp:43-48)
inline void rt_apply(const Rt32& a, const float* p, float* g) {
    float t[3];
    m3vec_f(a.R, p, t);
    for (int i = 0; i < 3; ++i) g[i] = t[i] + a.t[i];
}

struct State32 {
    Rt32 X;     // (R, pos)
    Rt32 IL;    // (RLI, tLI)  State::I_Rt_L()
};
// State(const state_ikfom&, double) (State.cpp:51-62): double -> float casts
State32 make_state32(const double* x) {
    State32 s;
    double R[9];
    quat_to_rot(x + S_ROT, R);
    for (int i = 0; i < 9; ++i) s.X.R[i] = (float)R[i];
    for (int i = 0; i < 3; ++i) s.X.t[i] = (float)x[S_POS + i];
    quat_to_rot(x + S_OFFR, R);
    for (int i = 0; i < 9; ++i) s.IL.R[i] = (float)R[i];
    for (int i = 0; i < 3; ++i) s.IL.t[i] = (float)x[S_OFFT + i];
    return s;
}

// --- Eigen 3.3 ColPivHouseholderQR<Matrix<float,Dynamic,Dynamic>>::solve restated for 5x3 --------------
// (Utils.cpp:47).  Sequential summation; Eigen's SIMD packet order is not reproducible here.
void colpiv_qr_solve_5x3(const float A_in[5][3], const float b_in[5], float x_out[3]) {
    const int rows = 5, cols = 3, size = 3;
    float qr[5][3];
    memcpy(qr, A_in, sizeof(qr));
    float hCoeffs[3];
    int transp[3];
    float normsUpdated[3], normsDirect[3];
    const float eps = std::numeric_limits<float>::epsilon();
    for (int k = 0; k < cols; ++k) {
        float s = 0;
        for (int i = 0; i < rows; ++i) s += qr[i][k] * qr[i][k];
        normsDirect[k] = std::sqrt(s);
        normsUpdated[k] = normsDirect[k];
    }
    float maxn = std::max(normsUpdated[0], std::max(normsUpdated[1], normsUpdated[2]));
    const float threshold_helper = (maxn * eps) * (maxn * eps) / (float)rows;
    const float norm_downdate_threshold = std::sqrt(eps);
    int nonzero_pivots = size;
    for (int k = 0; k < size; ++k) {
        int big = k;
        for (int j = k + 1; j < cols; ++j)
            if (normsUpdated[j] > normsUpdated[big]) big = j;
        float big_sq = normsUpdated[big] * normsUpdated[big];
        if (nonzero_pivots == size && big_sq < threshold_helper * (float)(rows - k)) nonzero_pivots = k;
        transp[k] = big;
        if (k != big) {
            for (int i = 0; i < rows; ++i) std::swap(qr[i][k], qr[i][big]);
            std::swap(normsUpdated[k], normsUpdated[big]);
            std::swap(normsDirect[k], normsDirect[big]);
        }
        // makeHouseholderInPlace on qr[k..rows-1][k]
        float tailSq = 0;
        for (int i = k + 1; i < rows; ++i) tailSq += qr[i][k] * qr[i][k];
        float c0 = qr[k][k], beta, tau;
        if (tailSq <= std::numeric_limits<float>::min()) {
            tau = 0;
            beta = c0;
            for (int i = k + 1; i < rows; ++i) qr[i][k] = 0;
        } else {
            beta = std::sqrt(c0 * c0 + tailSq);
            if (c0 >= 0) beta = -beta;
            for (int i = k + 1; i < rows; ++i) qr[i][k] = qr[i][k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        qr[k][k] = beta;
        hCoeffs[k] = tau;
        // applyHouseholderOnTheLeft to the bottom-right corner (rows-k) x (cols-k-1)
        if (tau != 0) {
            for (int j = k + 1; j < cols; ++j) {
                float tmp = 0;
                for (int i = k + 1; i < rows; ++i) tmp += qr[i][k] * qr[i][j];
                tmp += qr[k][j];
                qr[k][j] -= tau * tmp;
                for (int i = k + 1; i < rows; ++i) qr[i][j] -= tau * qr[i][k] * tmp;
            }
        }
        // column-norm downdate
        for (int j = k + 1; j < cols; ++j) {
            if (normsUpdated[j] != 0) {
                float temp = std::fabs(qr[k][j]) / normsUpdated[j];
                temp = (1.0f + temp) * (1.0f - temp);
                temp = temp < 0 ? 0 : temp;
                float r = normsUpdated[j] / normsDirect[j];
                float temp2 = temp * (r * r);
                if (temp2 <= norm_downdate_threshold) {
                    float s = 0;
                    for (int i = k + 1; i < rows; ++i) s += qr[i][j] * qr[i][j];
                    normsDirect[j] = std::sqrt(s);
                    normsUpdated[j] = normsDirect[j];
                } else {
                    normsUpdated[j] *= std::sqrt(temp);
                }
            }
        }
    }
    // column permutation from the transpositions
    int perm[3] = {0, 1, 2};
    for (int k = 0; k < size; ++k) std::swap(perm[k], perm[transp[k]]);
    // c = Q^T b : apply H_0, H_1, ... H_{nonzero-1} in order
    float c[5];
    memcpy(c, b_in, sizeof(c));
    x_out[0] = x_out[1] = x_out[2] = 0;
    if (nonzero_pivots == 0) return;
    for (int k = 0; k < nonzero_pivots; ++k) {
        float tau = hCoeffs[k];
        if (tau == 0) continue;
        float tmp = 0;
        for (int i = k + 1; i < rows; ++i) tmp += qr[i][k] * c[i];
        tmp += c[k];
        c[k] -= tau * tmp;
        for (int i = k + 1; i < rows; ++i) c[i] -= tau * qr[i][k] * tmp;
    }
    // back substitution on the leading nonzero_pivots x nonzero_pivots upper triangle
    for (int i = nonzero_pivots - 1; i >= 0; --i) {
        float s = c[i];
        for (int j = i + 1; j < nonzero_pivots; ++j) s -= qr[i][j] * c[j];
        c[i] = s / qr[i][i];
    }
    for (int i = 0; i < nonzero_pivots; ++i) x_out[perm[i]] = c[i];
}

// R3Math::estimate_plane (Utils.cpp:32-57) + is_plane (Utils.cpp:59-66)
bool plane_fit(const float pts[5][3], float threshold, float abcd[4]) {
    float b[5] = {-1.f, -1.f, -1.f, -1.f, -1.f};
    float nv[3];
    colpiv_qr_solve_5x3(pts, b, nv);
    float n = std::sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
    abcd[0] = nv[0] / n;
    abcd[1] = nv[1] / n;
    abcd[2] = nv[2] / n;
    abcd[3] = (float)(1.0 / n);
    for (int j = 0; j < 5; ++j) {
        float res = abcd[0] * pts[j][0] + abcd[1] * pts[j][1] + abcd[2] * pts[j][2] + abcd[3];
        if (std::fabs(res) > threshold) return false;
    }
    return true;
}

// ------------------------------------------------------------------------------------------
// Map: point store + exact kNN backends
// ------------------------------------------------------------------------------------------
inline float calc_dist(const float* a, const float* b) {  // ikd_Tree.cpp:1682-1687
    float dist = 0.0f;
    dist = (a[0] - b[0]) * (a[0] - b[0]) + (a[1] - b[1]) * (a[1] - b[1]) + (a[2] - b[2]) * (a[2] - b[2]);
    return dist;
}

struct HeapItem { float d; int idx; float x; };
// PointType_CMP::operator< (ikd_Tree.h:109-115)
inline bool heap_less(const HeapItem& a, const HeapItem& b) {
    if (std::fabs(a.d - b.d) < 1e-10) return a.x < b.x;
    return a.d < b.d;
}
struct TopK {   // bounded max-heap semantics of MANUAL_HEAP as used by Search()
    int k, n;
    HeapItem it[16];
    explicit TopK(int k_) : k(k_), n(0) {}
    float top() const { return it[0].d; }
    void push(const HeapItem& h) {
        it[n++] = h;
        std::push_heap(it, it + n, heap_less);
    }
    void pop() {
        std::pop_heap(it, it + n, heap_less);
        --n;
    }
    void offer(float d, int idx, float x) {   // ikd_Tree.cpp:1087-1093
        if (n < k || d < top()) {
            if (n >= k) pop();
            push(HeapItem{d, idx, x});
        }
    }
};

struct KdNode { int pt; int axis; int left, right; float lo[3], hi[3]; };

struct KdTree {
    std::vector<KdNode> nodes;
    const float* P = nullptr;
    int root = -1;
    int build_rec(std::vector<int>& ids, int l, int r) {   // ikd_Tree.cpp:679-733
        if (l > r) return -1;
        int mid = (l + r) >> 1;
        float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
        for (int i = l; i <= r; ++i)
            for (int a = 0; a < 3; ++a) {
                mn[a] = std::min(mn[a], P[3 * ids[i] + a]);
                mx[a] = std::max(mx[a], P[3 * ids[i] + a]);
            }
        int axis = 0;
        for (int a = 1; a < 3; ++a)
            if (mx[a] - mn[a] > mx[axis] - mn[axis]) axis = a;
        const float* Pp = P;
        std::nth_element(ids.begin() + l, ids.begin() + mid, ids.begin() + r + 1,
                         [Pp, axis](int a, int b) { return Pp[3 * a + axis] < Pp[3 * b + axis]; });
        int me = (int)nodes.size();
        nodes.push_back(KdNode());
        nodes[me].pt = ids[mid];
        nodes[me].axis = axis;
        for (int a = 0; a < 3; ++a) { nodes[me].lo[a] = mn[a]; nodes[me].hi[a] = mx[a]; }
        int L = build_rec(ids, l, mid - 1);
        int R = build_rec(ids, mid + 1, r);
        nodes[me].left = L;
        nodes[me].right = R;
        return me;
    }
    void build(const float* pts, const std::vector<int>& alive) {
        P = pts;
        nodes.clear();
        nodes.reserve(alive.size());
        std::vector<int> ids(alive);
        root = build_rec(ids, 0, (int)ids.size() - 1);
    }
    float box_dist(int n, const float* q) const {   // ikd_Tree.cpp:1690-1708
        if (n < 0) return INFINITY;
        float d = 0;
        for (int a = 0; a < 3; ++a) {
            if (q[a] < nodes[n].lo[a]) d += (q[a] - nodes[n].lo[a]) * (q[a] - nodes[n].lo[a]);
            if (q[a] > nodes[n].hi[a]) d += (q[a] - nodes[n].hi[a]) * (q[a] - nodes[n].hi[a]);
        }
        return d;
    }
    void search(int n, const float* q, TopK& h) const {   // ikd_Tree.cpp:1062-1243 (max_dist = INF)
        if (n < 0) return;
        const KdNode& nd = nodes[n];
        h.offer(calc_dist(q, P + 3 * nd.pt), nd.pt, P[3 * nd.pt]);
        float dl = box_dist(nd.left, q), dr = box_dist(nd.right, q);
        int first = nd.left, second = nd.right;
        float d1 = dl, d2 = dr;
        if (dr < dl) { first = nd.right; second = nd.left; d1 = dr; d2 = dl; }
        if (first >= 0 && (h.n < h.k || d1 < h.top())) search(first, q, h);
        if (second >= 0 && (h.n < h.k || d2 < h.top())) search(second, q, h);
    }
};

// verbatim reference ikd-Tree (oracle/_ref/libikdtree_ref.so, built by oracle/Makefile from the
// sources under /root/reference — optional backend)
struct RefIkd {
    void* lib = nullptr;
    void* (*create)(float, float, float) = nullptr;
    void (*destroy)(void*) = nullptr;
    void (*build)(void*, const float*, int64_t) = nullptr;
    int (*add)(void*, const float*, int64_t, int) = nullptr;
    int (*size)(void*) = nullptr;
    int (*nearest)(void*, const float*, int, float*, float*) = nullptr;
    int64_t (*flatten)(void*, float*, int64_t) = nullptr;
    bool load() {
        if (lib) return true;
        const char* env = getenv("LVO_REF_IKDTREE");
        std::string path = env ? env : "";
        if (path.empty()) {
            Dl_info info;
            if (dladdr((void*)&calc_dist, &info) && info.dli_fname) {
                std::string me = info.dli_fname;
                size_t p = me.find_last_of('/');
                path = (p == std::string::npos ? std::string(".") : me.substr(0, p)) + "/_ref/libikdtree_ref.so";
            }
        }
        lib = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
        if (!lib) return false;
        create = (void* (*)(float, float, float))dlsym(lib, "refikd_create");
        destroy = (void (*)(void*))dlsym(lib, "refikd_destroy");
        build = (void (*)(void*, const float*, int64_t))dlsym(lib, "refikd_build");
        add = (int (*)(void*, const float*, int64_t, int))dlsym(lib, "refikd_add_points");
        size = (int (*)(void*))dlsym(lib, "refikd_size");
        nearest = (int (*)(void*, const float*, int, float*, float*))dlsym(lib, "refikd_nearest");
        flatten = (int64_t (*)(void*, float*, int64_t))dlsym(lib, "refikd_flatten");
        return create && destroy && build && add && size && nearest && flatten;
    }
};
RefIkd g_ref;

double g_knn_s = 0, g_total_s = 0;
int g_threads = 1;   /* OpenMP team of the match loop (Mapper.cpp:45-46: MP_PROC_NUM) */
inline double now_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

struct lvo_map {
    int backend = LVO_KNN_KDTREE;
    std::vector<float> pts;          // all points ever inserted (xyz)
    std::vector<uint8_t> alive;
    int64_t n_alive = 0;
    // voxel index for the Add_Points downsample rule
    std::unordered_map<uint64_t, std::vector<int>> vox;
    // kNN structures (rebuilt lazily after a change)
    mutable bool dirty = true;
    mutable KdTree kd;
    mutable std::vector<int> alive_ids;
    void* ref = nullptr;             // verbatim ikd-Tree instance
};

namespace {
const float kDownsampleSize = 0.2f;  // KD_TREE<Point>(0.3, 0.6, 0.2) (Mapper.cpp:65)

/* 21 bits per axis, wrapped: cells 2^21 apart (419 km) share a bucket, which the exact box test of lvo_map_add filters out;
 * unmasked, a coordinate beyond +-209 km spilled into the next field and one point could be found through two keys */
inline uint64_t vox_key(int ix, int iy, int iz) {
    const uint64_t m = 0x1FFFFF;
    return (((uint64_t)(uint32_t)(ix + (1 << 20)) & m) << 42) | (((uint64_t)(uint32_t)(iy + (1 << 20)) & m) << 21) |
           ((uint64_t)(uint32_t)(iz + (1 << 20)) & m);
}
inline int vox_idx(float v) { return (int)std::floor(v / kDownsampleSize); }

void map_insert_point(lvo_map* m, const float* p) {
    int id = (int)(m->pts.size() / 3);
    m->pts.push_back(p[0]); m->pts.push_back(p[1]); m->pts.push_back(p[2]);
    m->alive.push_back(1);
    m->n_alive++;
    m->vox[vox_key(vox_idx(p[0]), vox_idx(p[1]), vox_idx(p[2]))].push_back(id);
    m->dirty = true;
}

void map_prepare(const lvo_map* m) {
    if (!m->dirty) return;
    m->alive_ids.clear();
    int64_t n = (int64_t)m->alive.size();
    for (int64_t i = 0; i < n; ++i)
        if (m->alive[i]) m->alive_ids.push_back((int)i);
    if (m->backend == LVO_KNN_KDTREE) m->kd.build(m->pts.data(), m->alive_ids);
    m->dirty = false;
}

// Neighbours PointType_CMP leaves unordered (distances within 1e-10 and equal x) come off the heap in whatever order the
// walk left them.  They are put in (y, z, point id) order, the product's fixed choice, so that the plane fit sees one row
// order; the (distance, x) order of the comparator is kept.
void tie_order(int found, int32_t* idx, float* sqd, float* nn) {
    auto before = [&](int a, int b) {
        for (int c = 0; c < 3; ++c)
            if (nn[3 * a + c] != nn[3 * b + c]) return nn[3 * a + c] < nn[3 * b + c];
        return idx[a] < idx[b];
    };
    auto swap_next = [&](int i) {
        std::swap(idx[i], idx[i + 1]);
        std::swap(sqd[i], sqd[i + 1]);
        for (int c = 0; c < 3; ++c) std::swap(nn[3 * i + c], nn[3 * (i + 1) + c]);
    };
    // exact ties first, so that the non-transitive 1e-10 pass below starts from an order that depends only on the set
    for (int pass = 0; pass + 1 < found; ++pass)
        for (int i = 0; i + 1 < found; ++i)
            if (sqd[i + 1] == sqd[i] && before(i + 1, i)) swap_next(i);
    for (int pass = 0; pass + 1 < found; ++pass)
        for (int i = 0; i + 1 < found; ++i)
            if (std::fabs(sqd[i + 1] - sqd[i]) < 1e-10 && before(i + 1, i)) swap_next(i);
}

int map_knn(const lvo_map* m, const float* g, int k, int32_t* idx, float* sqd, float* nn) {
    if (k > 16) k = 16;
    if (m->backend == LVO_KNN_REF_IKDTREE) {
        float pts[16 * 3], d[16];
        int found = g_ref.nearest(m->ref, g, k, pts, d);
        for (int i = 0; i < found; ++i) {
            if (idx) idx[i] = -1;
            if (sqd) sqd[i] = d[i];
            if (nn) { nn[3 * i] = pts[3 * i]; nn[3 * i + 1] = pts[3 * i + 1]; nn[3 * i + 2] = pts[3 * i + 2]; }
        }
        if (idx && sqd && nn) tie_order(found, idx, sqd, nn);
        return found;
    }
    map_prepare(m);
    TopK h(k);
    if (m->backend == LVO_KNN_BRUTE) {
        for (int id : m->alive_ids) h.offer(calc_dist(g, &m->pts[3 * id]), id, m->pts[3 * id]);
    } else {
        m->kd.search(m->kd.root, g, h);
    }
    int found = h.n;
    // Nearest_Search pops the max-heap and inserts at the front -> ascending (ikd_Tree.cpp:452-459)
    for (int i = found - 1; i >= 0; --i) {
        HeapItem it = h.it[0];
        h.pop();
        if (idx) idx[i] = it.idx;
        if (sqd) sqd[i] = it.d;
        if (nn) { nn[3 * i] = m->pts[3 * it.idx]; nn[3 * i + 1] = m->pts[3 * it.idx + 1]; nn[3 * i + 2] = m->pts[3 * it.idx + 2]; }
    }
    if (idx && sqd && nn) tie_order(found, idx, sqd, nn);
    return found;
}

struct MatchOut {
    bool chosen;
    float g[3];
    float abcd[4];
    float dist;
    int32_t nn_idx[5];
    float nn_sqd[5];
};

// Mapper::match_plane (Mapper.cpp:82-90) + Plane::Plane (Plane.cpp:19-25) + Match::Match (Match.cpp:18-22)
void match_point(const lvo_map* m, const lvo_params* prm, const Rt32& T, const float* p, MatchOut* o) {
    rt_apply(T, p, o->g);   // X * X.I_Rt_L() * p  (Mapper.cpp:51)
    float nn[5 * 3];
    for (int i = 0; i < 5; ++i) { o->nn_idx[i] = -1; o->nn_sqd[i] = INFINITY; }
    o->abcd[0] = o->abcd[1] = o->abcd[2] = o->abcd[3] = 0;
    o->dist = 0;
    double t0 = g_threads == 1 ? now_s() : 0.0;
    int found = map_knn(m, o->g, 5, o->nn_idx, o->nn_sqd, nn);
    if (g_threads == 1) g_knn_s += now_s() - t0;
    o->chosen = false;
    if (found < 5) return;                                                         // Plane.cpp:36-38
    if (!((double)o->nn_sqd[4] < prm->max_dist_plane * prm->max_dist_plane)) return;   // Plane.cpp:40-43
    float pts[5][3];
    memcpy(pts, nn, sizeof(pts));
    o->chosen = plane_fit(pts, prm->planes_threshold, o->abcd);                    // Plane.cpp:45-55
    if (!o->chosen) { o->abcd[0] = o->abcd[1] = o->abcd[2] = o->abcd[3] = 0; return; }
    o->dist = o->abcd[0] * o->g[0] + o->abcd[1] * o->g[1] + o->abcd[2] * o->g[2] + o->abcd[3];   // Plane.cpp:27-29
}

// one row of Localizator::calculate_H (Localizator.cpp:36-56)
void h_row(const double* x, const State32& S, const lvo_params* prm, const MatchOut& mt, double* row12, double* hval) {
    // p_lidar = S.I_Rt_L().inv() * S.inv() * match.point   (RotTransl * RotTransl first, then * Point)
    Rt32 Tinv = rt_mul(rt_inv(S.IL), rt_inv(S.X));
    float p_lidar[3], p_imu[3];
    rt_apply(Tinv, mt.g, p_lidar);
    rt_apply(S.IL, p_lidar, p_imu);
    double Rq[9], Rinv[9], RLq[9], RLinv[9];
    double qc[4] = {-x[S_ROT], -x[S_ROT + 1], -x[S_ROT + 2], x[S_ROT + 3]};
    quat_to_rot(qc, Rinv);
    double qlc[4] = {-x[S_OFFR], -x[S_OFFR + 1], -x[S_OFFR + 2], x[S_OFFR + 3]};
    quat_to_rot(qlc, RLinv);
    (void)Rq; (void)RLq;
    double n[3] = {(double)mt.abcd[0], (double)mt.abcd[1], (double)mt.abcd[2]};
    double C[3], RC[3];
    mat3_vec(Rinv, n, C);
    mat3_vec(RLinv, C, RC);
    double pl[3] = {(double)p_lidar[0], (double)p_lidar[1], (double)p_lidar[2]};
    double pi[3] = {(double)p_imu[0], (double)p_imu[1], (double)p_imu[2]};
    double B[3] = {pl[1] * RC[2] - pl[2] * RC[1], pl[2] * RC[0] - pl[0] * RC[2], pl[0] * RC[1] - pl[1] * RC[0]};
    double A[3] = {pi[1] * C[2] - pi[2] * C[1], pi[2] * C[0] - pi[0] * C[2], pi[0] * C[1] - pi[1] * C[0]};
    for (int i = 0; i < 12; ++i) row12[i] = 0;
    row12[0] = mt.abcd[0]; row12[1] = mt.abcd[1]; row12[2] = mt.abcd[2];
    row12[3] = A[0]; row12[4] = A[1]; row12[5] = A[2];
    if (prm->estimate_extrinsics) {
        row12[6] = B[0]; row12[7] = B[1]; row12[8] = B[2];
        row12[9] = C[0]; row12[10] = C[1]; row12[11] = C[2];
    }
    *hval = -(double)mt.dist;
}

Rt32 total_transform(const State32& S) { return rt_mul(S.X, S.IL); }   // State * RotTransl (State.cpp:83-85)

// measurement reduced to what the IESKF consumes
int measure_reduced(const lvo_map* m, const double* x, const lvo_params* prm, const float* xyz, int64_t n,
                    double* HTH, double* HTh, int64_t* nm) {
    State32 S = make_state32(x);
    Rt32 T = total_transform(S);
    for (int i = 0; i < 144; ++i) HTH[i] = 0;
    for (int i = 0; i < 12; ++i) HTh[i] = 0;
    int64_t cnt = 0;
    if (m->backend != LVO_KNN_REF_IKDTREE) map_prepare(m);
    // Mapper::match runs this loop under "#pragma omp parallel for" with MP_PROC_NUM threads and a racy
    // shared push_back (Mapper.cpp:45-53); here every thread keeps private sums (order-insensitive to
    // ~1e-12 relative) that are added in thread order.
#pragma omp parallel num_threads(g_threads)
    {
        double hth[144] = {0}, hthv[12] = {0};
        int64_t c_local = 0;
#pragma omp for schedule(static)
        for (int64_t i = 0; i < n; ++i) {
            MatchOut mt;
            match_point(m, prm, T, xyz + 3 * i, &mt);
            if (!mt.chosen) continue;
            double row[12], h;
            h_row(x, S, prm, mt, row, &h);
            for (int a = 0; a < 12; ++a) {
                for (int b = 0; b < 12; ++b) hth[a * 12 + b] += row[a] * row[b];
                hthv[a] += row[a] * h;
            }
            ++c_local;
        }
#pragma omp for ordered schedule(static, 1)
        for (int t = 0; t < g_threads; ++t) {
#pragma omp ordered
            {
                for (int a = 0; a < 144; ++a) HTH[a] += hth[a];
                for (int a = 0; a < 12; ++a) HTh[a] += hthv[a];
                cnt += c_local;
            }
        }
    }
    *nm = cnt;
    return LVO_OK;
}

// ------------------------------------------------------------------------------------------
// IESKF update (esekfom.hpp:1620-1823), n = 23, measurement block 12
// ------------------------------------------------------------------------------------------
const int N = LVO_DOF;
inline double& PP(double* P, int i, int j) { return P[i * N + j]; }

// P[idx:idx+d, :] = J * P[idx:idx+d, :]  then  P[:, idx:idx+d] = P[:, idx:idx+d] * J^T   (esekfom.hpp:1667-1672)
void apply_block_both(double* P, int idx, int d, const double* J /*d x d row-major*/) {
    double t[3];
    for (int i = 0; i < N; ++i) {
        for (int a = 0; a < d; ++a) {
            double s = 0;
            for (int b = 0; b < d; ++b) s += J[a * d + b] * PP(P, idx + b, i);
            t[a] = s;
        }
        for (int a = 0; a < d; ++a) PP(P, idx + a, i) = t[a];
    }
    for (int i = 0; i < N; ++i) {
        for (int a = 0; a < d; ++a) {
            double s = 0;
            for (int b = 0; b < d; ++b) s += PP(P, i, idx + b) * J[a * d + b];
            t[a] = s;
        }
        for (int a = 0; a < d; ++a) PP(P, i, idx + a) = t[a];
    }
}

// one evaluation, esekfom.hpp:1647-1762 (valid only for Nm >= 23, i.e. the "else" branch :1720-1729)
void ieskf_step(const double* x_prop, const double* P_prop, const double* x_cur, const lvo_params* prm,
                const double* HTH, const double* HTh, double* dx_out, double* x_new, double* P_now,
                double* Kx /*23x12*/, int* converged) {
    double dx[N], dx_new[N];
    state_boxminus(x_cur, x_prop, dx);                                 // :1652
    memcpy(dx_new, dx, sizeof(dx));
    memcpy(P_now, P_prop, sizeof(double) * N * N);                     // :1655
    const int so3_idx[2] = {3, 6};
    for (int b = 0; b < 2; ++b) {                                      // :1659-1674
        int idx = so3_idx[b];
        double A[9], J[9];
        A_matrix(dx + idx, A);
        mat3_T(A, J);
        double t[3];
        mat3_vec(J, dx_new + idx, t);
        dx_new[idx] = t[0]; dx_new[idx + 1] = t[1]; dx_new[idx + 2] = t[2];
        apply_block_both(P_now, idx, 3, J);
    }
    {                                                                   // :1676-1697 (S2 @21)
        int idx = 21;
        double Nx[6], Mx[6], J[4];
        S2_Nx_yy(x_cur + S_GRAV, Nx);
        S2_Mx(x_prop + S_GRAV, dx + idx, Mx);
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 2; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += Nx[i * 3 + k] * Mx[k * 2 + j];
                J[i * 2 + j] = s;
            }
        double t0 = J[0] * dx_new[idx] + J[1] * dx_new[idx + 1];
        double t1 = J[2] * dx_new[idx] + J[3] * dx_new[idx + 1];
        dx_new[idx] = t0; dx_new[idx + 1] = t1;
        apply_block_both(P_now, idx, 2, J);
    }
    // :1722-1729
    std::vector<double> T(N * N), Tinv(N * N), Pinv(N * N);
    for (int i = 0; i < N * N; ++i) T[i] = P_now[i] / prm->lidar_noise;
    inverse_n(T.data(), N, Tinv.data());
    for (int i = 0; i < 12; ++i)
        for (int j = 0; j < 12; ++j) Tinv[i * N + j] += HTH[i * 12 + j];
    inverse_n(Tinv.data(), N, Pinv.data());
    double K_h[N];
    for (int i = 0; i < N; ++i) {
        double s = 0;
        for (int k = 0; k < 12; ++k) s += Pinv[i * N + k] * HTh[k];
        K_h[i] = s;
        for (int j = 0; j < 12; ++j) {
            double s2 = 0;
            for (int k = 0; k < 12; ++k) s2 += Pinv[i * N + k] * HTH[k * 12 + j];
            Kx[i * 12 + j] = s2;
        }
    }
    // :1733  dx_ = K_h + (K_x - I) dx_new
    double dx_[N];
    for (int i = 0; i < N; ++i) {
        double s = 0;
        for (int j = 0; j < 12; ++j) s += Kx[i * 12 + j] * dx_new[j];
        dx_[i] = K_h[i] + s - dx_new[i];
    }
    // :1736-1744 degeneracy
    double A6[36], ev[6], V[36];
    for (int i = 0; i < 6; ++i)
        for (int j = 0; j < 6; ++j) A6[i * 6 + j] = HTH[i * 12 + j];
    sym_eig(A6, 6, ev, V);
    double prod = 1;
    for (int i = 0; i < 6; ++i) prod *= ev[i];
    if (prod < 1e-20)
        for (int i = 0; i < 36; ++i) V[i] = (i % 7 == 0) ? 1.0 : 0.0;
    double sel[36];
    memcpy(sel, V, sizeof(sel));
    bool any_masked = false;
    for (int j = 0; j < 6; ++j)
        if (ev[j] < prm->degeneracy_threshold) {
            for (int c = 0; c < 6; ++c) sel[j * 6 + c] = 0;
            any_masked = true;
        }
    double dnd[N];
    memcpy(dnd, dx_, sizeof(dnd));
    if (any_masked) {
        double Vinv[36], t[6], r[6];
        inverse_n(V, 6, Vinv);
        for (int i = 0; i < 6; ++i) {
            double s = 0;
            for (int j = 0; j < 6; ++j) s += sel[i * 6 + j] * dx_[j];
            t[i] = s;
        }
        for (int i = 0; i < 6; ++i) {
            double s = 0;
            for (int j = 0; j < 6; ++j) s += Vinv[i * 6 + j] * t[j];
            r[i] = s;
        }
        for (int i = 0; i < 6; ++i) dnd[i] = r[i];
    }
    memcpy(x_new, x_cur, sizeof(double) * LVO_STATE_LEN);
    state_boxplus(x_new, dnd);                                          // :1747
    *converged = 1;
    for (int i = 0; i < N; ++i)
        if (std::fabs(dx_[i]) > prm->limits[i]) { *converged = 0; break; }   // :1748-1756
    memcpy(dx_out, dx_, sizeof(dx_));
}

// exit block, esekfom.hpp:1764-1817
void ieskf_finish(const double* x_prop, const double* x_new, const double* dx_, const double* P_now_in,
                  const double* Kx_in, double* P_out) {
    std::vector<double> P(P_now_in, P_now_in + N * N), L(P_now_in, P_now_in + N * N);
    std::vector<double> Kx(Kx_in, Kx_in + N * 12);
    const int so3_idx[2] = {3, 6};
    double t[3];
    for (int b = 0; b < 2; ++b) {
        int idx = so3_idx[b];
        double A[9], J[9];
        A_matrix(dx_ + idx, A);
        mat3_T(A, J);
        for (int i = 0; i < N; ++i) {    // L rows = J * P rows
            for (int a = 0; a < 3; ++a) {
                double s = 0;
                for (int c = 0; c < 3; ++c) s += J[a * 3 + c] * P[(idx + c) * N + i];
                t[a] = s;
            }
            for (int a = 0; a < 3; ++a) L[(idx + a) * N + i] = t[a];
        }
        for (int i = 0; i < 12; ++i) {
            for (int a = 0; a < 3; ++a) {
                double s = 0;
                for (int c = 0; c < 3; ++c) s += J[a * 3 + c] * Kx[(idx + c) * 12 + i];
                t[a] = s;
            }
            for (int a = 0; a < 3; ++a) Kx[(idx + a) * 12 + i] = t[a];
        }
        for (int i = 0; i < N; ++i) {
            for (int a = 0; a < 3; ++a) {
                double s = 0;
                for (int c = 0; c < 3; ++c) s += L[i * N + idx + c] * J[a * 3 + c];
                t[a] = s;
            }
            for (int a = 0; a < 3; ++a) L[i * N + idx + a] = t[a];
            for (int a = 0; a < 3; ++a) {
                double s = 0;
                for (int c = 0; c < 3; ++c) s += P[i * N + idx + c] * J[a * 3 + c];
                t[a] = s;
            }
            for (int a = 0; a < 3; ++a) P[i * N + idx + a] = t[a];
        }
    }
    {
        int idx = 21;
        double Nx[6], Mx[6], J[4];
        S2_Nx_yy(x_new + S_GRAV, Nx);
        S2_Mx(x_prop + S_GRAV, dx_ + idx, Mx);
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 2; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += Nx[i * 3 + k] * Mx[k * 2 + j];
                J[i * 2 + j] = s;
            }
        for (int i = 0; i < N; ++i) {
            double a0 = J[0] * P[idx * N + i] + J[1] * P[(idx + 1) * N + i];
            double a1 = J[2] * P[idx * N + i] + J[3] * P[(idx + 1) * N + i];
            L[idx * N + i] = a0; L[(idx + 1) * N + i] = a1;
        }
        for (int i = 0; i < 12; ++i) {
            double a0 = J[0] * Kx[idx * 12 + i] + J[1] * Kx[(idx + 1) * 12 + i];
            double a1 = J[2] * Kx[idx * 12 + i] + J[3] * Kx[(idx + 1) * 12 + i];
            Kx[idx * 12 + i] = a0; Kx[(idx + 1) * 12 + i] = a1;
        }
        for (int i = 0; i < N; ++i) {
            double a0 = L[i * N + idx] * J[0] + L[i * N + idx + 1] * J[1];
            double a1 = L[i * N + idx] * J[2] + L[i * N + idx + 1] * J[3];
            L[i * N + idx] = a0; L[i * N + idx + 1] = a1;
            double b0 = P[i * N + idx] * J[0] + P[i * N + idx + 1] * J[1];
            double b1 = P[i * N + idx] * J[2] + P[i * N + idx + 1] * J[3];
            P[i * N + idx] = b0; P[i * N + idx + 1] = b1;
        }
    }
    for (int i = 0; i < N; ++i)                                         // :1817
        for (int j = 0; j < N; ++j) {
            double s = 0;
            for (int k = 0; k < 12; ++k) s += Kx[i * 12 + k] * P[k * N + j];
            P_out[i * N + j] = L[i * N + j] - s;
        }
}

}  // namespace

// ==========================================================================================
// C API
// ==========================================================================================
extern "C" {

lvo_map* lvo_map_create(int backend) {
    if (backend == LVO_KNN_REF_IKDTREE && !g_ref.load()) return nullptr;
    lvo_map* m = new lvo_map();
    m->backend = backend;
    if (backend == LVO_KNN_REF_IKDTREE) m->ref = g_ref.create(0.3f, 0.6f, 0.2f);   // Mapper.cpp:65
    return m;
}
void lvo_map_destroy(lvo_map* m) {
    if (!m) return;
    if (m->ref) g_ref.destroy(m->ref);
    delete m;
}
int lvo_map_build(lvo_map* m, const float* xyz, int64_t n) {
    if (!m || n <= 0) return LVO_BAD_ARG;
    m->pts.clear(); m->alive.clear(); m->vox.clear(); m->n_alive = 0;
    m->pts.reserve(3 * n);
    for (int64_t i = 0; i < n; ++i) map_insert_point(m, xyz + 3 * i);
    if (m->ref) g_ref.build(m->ref, xyz, n);
    return LVO_OK;
}
// KD_TREE::Add_Points (ikd_Tree.cpp:478-573), single-threaded semantics
int lvo_map_add(lvo_map* m, const float* xyz, int64_t n, int downsample) {
    if (!m) return LVO_BAD_ARG;
    if (n <= 0) return LVO_OK;                       // Mapper.cpp:23
    if (m->n_alive == 0) return lvo_map_build(m, xyz, n);   // Mapper.cpp:26
    if (m->ref) g_ref.add(m->ref, xyz, n, downsample);
    for (int64_t i = 0; i < n; ++i) {
        const float* p = xyz + 3 * i;
        if (!downsample) { map_insert_point(m, p); continue; }
        const float ds = kDownsampleSize;
        float bmin[3], bmax[3], mid[3];
        for (int a = 0; a < 3; ++a) {
            bmin[a] = std::floor(p[a] / ds) * ds;
            bmax[a] = bmin[a] + ds;
            mid[a] = (float)(bmin[a] + (bmax[a] - bmin[a]) / 2.0);
        }
        // Search_by_range: half-open box test on the stored coordinates (ikd_Tree.cpp:1262)
        std::vector<int> storage;
        int cx = vox_idx(p[0]), cy = vox_idx(p[1]), cz = vox_idx(p[2]);
        for (int dx = -1; dx <= 1; ++dx)
            for (int dy = -1; dy <= 1; ++dy)
                for (int dz = -1; dz <= 1; ++dz) {
                    auto it = m->vox.find(vox_key(cx + dx, cy + dy, cz + dz));
                    if (it == m->vox.end()) continue;
                    for (int id : it->second) {
                        if (!m->alive[id]) continue;
                        const float* q = &m->pts[3 * id];
                        if (bmin[0] <= q[0] && bmax[0] > q[0] && bmin[1] <= q[1] && bmax[1] > q[1] && bmin[2] <= q[2] && bmax[2] > q[2])
                            storage.push_back(id);
                    }
                }
        float min_dist = calc_dist(p, mid);
        int best = -1;   // -1 = the new point
        for (int id : storage) {
            float d = calc_dist(&m->pts[3 * id], mid);
            if (d < min_dist) { min_dist = d; best = id; }
        }
        // same_point(new, downsample_result) (ikd_Tree.cpp:1676-1679)
        bool same = (best < 0);
        if (!same) {
            const float* q = &m->pts[3 * best];
            same = std::fabs(p[0] - q[0]) < 1e-6 && std::fabs(p[1] - q[1]) < 1e-6 && std::fabs(p[2] - q[2]) < 1e-6;
        }
        if (storage.size() > 1 || same) {
            float keep[3];
            const float* src = best < 0 ? p : &m->pts[3 * best];
            keep[0] = src[0]; keep[1] = src[1]; keep[2] = src[2];
            for (int id : storage) { m->alive[id] = 0; m->n_alive--; }
            map_insert_point(m, keep);
            m->dirty = true;
        }
    }
    return LVO_OK;
}
int64_t lvo_map_size(const lvo_map* m) {
    if (!m) return 0;
    if (m->ref) return g_ref.size(m->ref);
    return m->n_alive;
}
int64_t lvo_map_points(const lvo_map* m, float* out, int64_t cap) {
    if (!m) return 0;
    if (m->ref) return g_ref.flatten(m->ref, out, cap);
    int64_t k = 0, n = (int64_t)m->alive.size();
    for (int64_t i = 0; i < n; ++i)
        if (m->alive[i]) {
            if (k < cap) { out[3 * k] = m->pts[3 * i]; out[3 * k + 1] = m->pts[3 * i + 1]; out[3 * k + 2] = m->pts[3 * i + 2]; }
            ++k;
        }
    return k;
}
int lvo_knn(const lvo_map* m, const float g[3], int k, int32_t* idx, float* sqd, float* nn_xyz) {
    if (!m || lvo_map_size(m) == 0) return 0;
    return map_knn(m, g, k, idx, sqd, nn_xyz);
}

int lvo_match_all(const lvo_map* m, const double* x, const lvo_params* prm, const float* xyz, int64_t n,
                  uint8_t* valid, int32_t* nn_idx, float* nn_sqd, float* plane, float* dist, float* g_world) {
    if (!m || lvo_map_size(m) == 0) return LVO_EMPTY_MAP;
    State32 S = make_state32(x);
    Rt32 T = total_transform(S);
    for (int64_t i = 0; i < n; ++i) {
        MatchOut mt;
        match_point(m, prm, T, xyz + 3 * i, &mt);
        if (valid) valid[i] = mt.chosen ? 1 : 0;
        if (nn_idx) memcpy(nn_idx + 5 * i, mt.nn_idx, sizeof(mt.nn_idx));
        if (nn_sqd) memcpy(nn_sqd + 5 * i, mt.nn_sqd, sizeof(mt.nn_sqd));
        if (plane) memcpy(plane + 4 * i, mt.abcd, sizeof(mt.abcd));
        if (dist) dist[i] = mt.dist;
        if (g_world) memcpy(g_world + 3 * i, mt.g, sizeof(mt.g));
    }
    return LVO_OK;
}

int lvo_measure(const lvo_map* m, const double* x, const lvo_params* prm, const float* xyz, int64_t n,
                double* h_x, double* h, int64_t* nm) {
    if (!m || lvo_map_size(m) == 0) { *nm = 0; return LVO_EMPTY_MAP; }
    State32 S = make_state32(x);
    Rt32 T = total_transform(S);
    std::vector<double> rows;
    std::vector<double> hs;
    for (int64_t i = 0; i < n; ++i) {
        MatchOut mt;
        match_point(m, prm, T, xyz + 3 * i, &mt);
        if (!mt.chosen) continue;
        double row[12], hv;
        h_row(x, S, prm, mt, row, &hv);
        rows.insert(rows.end(), row, row + 12);
        hs.push_back(hv);
    }
    int64_t cnt = (int64_t)hs.size();
    *nm = cnt;
    for (int64_t i = 0; i < cnt; ++i) {
        if (h) h[i] = hs[i];
        if (h_x)
            for (int c = 0; c < 12; ++c) h_x[c * cnt + i] = rows[12 * i + c];   // column-major Nm x 12
    }
    return LVO_OK;
}

int lvo_measure_reduced(const lvo_map* m, const double* x, const lvo_params* prm, const float* xyz, int64_t n,
                        double* HTH, double* HTh, int64_t* nm) {
    if (!m || lvo_map_size(m) == 0) { *nm = 0; return LVO_EMPTY_MAP; }
    return measure_reduced(m, x, prm, xyz, n, HTH, HTh, nm);
}

int lvo_update_step(const double* x_prop, const double* P_prop, const double* x_cur, const lvo_params* prm,
                    const double* HTH, const double* HTh, double* dx_out, double* x_new, double* P_now,
                    double* Kx_out, int32_t* converged) {
    int c = 0;
    ieskf_step(x_prop, P_prop, x_cur, prm, HTH, HTh, dx_out, x_new, P_now, Kx_out, &c);
    *converged = c;
    return LVO_OK;
}
int lvo_update_finish(const double* x_prop, const double* x_new, const double* dx, const double* P_now,
                      const double* Kx, double* P_out) {
    ieskf_finish(x_prop, x_new, dx, P_now, Kx, P_out);
    return LVO_OK;
}

int lvo_update_iterated(const lvo_map* m, double* x, double* P, const lvo_params* prm, const float* xyz,
                        int64_t n, lvo_iter_log* logs, int32_t* n_evals) {
    *n_evals = 0;
    if (!m || lvo_map_size(m) == 0) return LVO_EMPTY_MAP;              // Localizator.cpp:24
    double t_begin = now_s();
    g_knn_s = 0;
    double x_prop[LVO_STATE_LEN], P_prop[N * N];
    memcpy(x_prop, x, sizeof(x_prop));
    memcpy(P_prop, P, sizeof(P_prop));
    int t = 0;
    const int maximum_iter = prm->max_num_iters;
    int status = LVO_OK;
    for (int i = -1; i < maximum_iter; ++i) {                           // esekfom.hpp:1634
        lvo_iter_log* lg = &logs[*n_evals];
        measure_reduced(m, x, prm, xyz, n, lg->HTH, lg->HTh, &lg->n_matches);
        if (lg->n_matches < N) {                                        // esekfom.hpp:1701-1709: undefined in
            status = LVO_TOO_FEW_MATCHES;                               // the reference (quirk 4) -> stop
            break;
        }
        double dx_[N], x_new[LVO_STATE_LEN], P_now[N * N], Kx[N * 12];
        int conv = 0;
        ieskf_step(x_prop, P_prop, x, prm, lg->HTH, lg->HTh, dx_, x_new, P_now, Kx, &conv);
        memcpy(x, x_new, sizeof(x_new));
        if (conv) t++;
        if (!t && i == maximum_iter - 2) conv = 1;                      // :1759-1762
        lg->converged = conv;
        memcpy(lg->dx, dx_, sizeof(dx_));
        memcpy(lg->x_after, x, sizeof(double) * LVO_STATE_LEN);
        (*n_evals)++;
        if (t > 1 || i == maximum_iter - 1) {                           // :1764
            ieskf_finish(x_prop, x, dx_, P_now, Kx, P);
            break;
        }
    }
    g_total_s = now_s() - t_begin;
    return status;
}

// esekf::predict (esekfom.hpp:279-384) with f, df_dx, df_dw of use-ikfom.cpp:49-90
int lvo_predict(double* x, double* P, const double acc[3], const double gyro[3], double dt,
                double cov_gyro, double cov_acc, double cov_bias_gyro, double cov_bias_acc) {
    const int M = 24, PN = 12;
    double R[9];
    quat_to_rot(x + S_ROT, R);
    // get_f (use-ikfom.cpp:49-61) in the 24-dim flattened layout: pos0 rot3 offR6 offT9 vel12 bg15 ba18 grav21
    double f[M] = {0};
    double omega[3], a_b[3], a_in[3];
    for (int i = 0; i < 3; ++i) { omega[i] = gyro[i] - x[S_BG + i]; a_b[i] = acc[i] - x[S_BA + i]; }
    mat3_vec(R, a_b, a_in);
    for (int i = 0; i < 3; ++i) {
        f[i] = x[S_VEL + i];
        f[i + 3] = omega[i];
        f[i + 12] = a_in[i] + x[S_GRAV + i];
    }
    // df_dx (24x23) (use-ikfom.cpp:63-79)
    std::vector<double> fx(M * N, 0.0), fw(M * PN, 0.0);
    for (int i = 0; i < 3; ++i) fx[(0 + i) * N + 12 + i] = 1.0;
    double Ha[9], RH[9];
    hat(a_b, Ha);
    mat3_mul(R, Ha, RH);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            fx[(12 + i) * N + 3 + j] = -RH[i * 3 + j];
            fx[(12 + i) * N + 18 + j] = -R[i * 3 + j];
        }
    double zero2[2] = {0, 0}, gm[6];
    S2_Mx(x + S_GRAV, zero2, gm);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 2; ++j) fx[(12 + i) * N + 21 + j] = gm[i * 2 + j];
    for (int i = 0; i < 3; ++i) fx[(3 + i) * N + 15 + i] = -1.0;
    // df_dw (24x12) (use-ikfom.cpp:82-90)
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) fw[(12 + i) * PN + 3 + j] = -R[i * 3 + j];
    for (int i = 0; i < 3; ++i) {
        fw[(3 + i) * PN + 0 + i] = -1.0;
        fw[(15 + i) * PN + 6 + i] = 1.0;
        fw[(18 + i) * PN + 9 + i] = 1.0;
    }
    double x_before[LVO_STATE_LEN];
    memcpy(x_before, x, sizeof(x_before));
    // x_.oplus(f_, dt) (build_manifold.hpp:195-197): vect += dt*v ; SO3 *= exp(v, dt) ; S2.oplus(v, dt)
    for (int i = 0; i < 3; ++i) x[S_POS + i] += dt * f[0 + i];
    {
        double q[4];
        so3_exp(f + 3, dt / 2, q);
        quat_mul(x + S_ROT, q, x + S_ROT);
        so3_exp(f + 6, dt / 2, q);
        quat_mul(x + S_OFFR, q, x + S_OFFR);
    }
    for (int i = 0; i < 3; ++i) x[S_OFFT + i] += dt * f[9 + i];
    for (int i = 0; i < 3; ++i) x[S_VEL + i] += dt * f[12 + i];
    for (int i = 0; i < 3; ++i) x[S_BG + i] += dt * f[15 + i];
    for (int i = 0; i < 3; ++i) x[S_BA + i] += dt * f[18 + i];
    {   // S2::oplus (S2.hpp:129-134)
        double q[4], Rq[9];
        so3_exp(f + 21, dt / 2, q);
        quat_to_rot(q, Rq);
        mat3_vec(Rq, x + S_GRAV, x + S_GRAV);
    }
    // F_x1, f_x_final, f_w_final (esekfom.hpp:289-368)
    std::vector<double> F1(N * N, 0.0), fxf(N * N, 0.0), fwf(N * PN, 0.0);
    for (int i = 0; i < N; ++i) F1[i * N + i] = 1.0;
    // vect states: (idx, dim, dof): pos(0,0) offT(9,9) vel(12,12) bg(15,15) ba(18,18)
    const int vidx[5] = {0, 9, 12, 15, 18};
    for (int v = 0; v < 5; ++v)
        for (int j = 0; j < 3; ++j) {
            for (int i = 0; i < N; ++i) fxf[(vidx[v] + j) * N + i] = fx[(vidx[v] + j) * N + i];
            for (int i = 0; i < PN; ++i) fwf[(vidx[v] + j) * PN + i] = fw[(vidx[v] + j) * PN + i];
        }
    const int sidx[2] = {3, 6};
    for (int b = 0; b < 2; ++b) {
        int idx = sidx[b], dim = sidx[b];
        double seg[3] = {-1 * f[dim] * dt, -1 * f[dim + 1] * dt, -1 * f[dim + 2] * dt};
        // res = exp(seg, scalar(1/2)) == identity (quirk 2) -> F_x1 block = I
        double A[9];
        A_matrix(seg, A);
        for (int i = 0; i < N; ++i) {
            double c[3] = {fx[(dim)*N + i], fx[(dim + 1) * N + i], fx[(dim + 2) * N + i]}, r[3];
            mat3_vec(A, c, r);
            for (int a = 0; a < 3; ++a) fxf[(idx + a) * N + i] = r[a];
        }
        for (int i = 0; i < PN; ++i) {
            double c[3] = {fw[(dim)*PN + i], fw[(dim + 1) * PN + i], fw[(dim + 2) * PN + i]}, r[3];
            mat3_vec(A, c, r);
            for (int a = 0; a < 3; ++a) fwf[(idx + a) * PN + i] = r[a];
        }
    }
    {   // S2 state idx 21, dim 21
        int idx = 21, dim = 21;
        double seg[3] = {f[dim] * dt, f[dim + 1] * dt, f[dim + 2] * dt};
        double Nx[6], Mx[6], z2[2] = {0, 0};
        S2_Nx_yy(x + S_GRAV, Nx);
        S2_Mx(x_before + S_GRAV, z2, Mx);
        // res = identity (scalar(1/2) == 0): F_x1 block = Nx * Mx
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 2; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += Nx[i * 3 + k] * Mx[k * 2 + j];
                F1[(idx + i) * N + idx + j] = s;
            }
        double Hb[9], A[9], At[9], T1[9];
        hat(x_before + S_GRAV, Hb);
        A_matrix(seg, A);
        mat3_T(A, At);
        mat3_mul(Hb, At, T1);
        double rt[6];   // -Nx * T1  (2x3)
        for (int i = 0; i < 2; ++i)
            for (int j = 0; j < 3; ++j) {
                double s = 0;
                for (int k = 0; k < 3; ++k) s += Nx[i * 3 + k] * T1[k * 3 + j];
                rt[i * 3 + j] = -s;
            }
        for (int i = 0; i < N; ++i)
            for (int a = 0; a < 2; ++a)
                fxf[(idx + a) * N + i] = rt[a * 3 + 0] * fx[(dim)*N + i] + rt[a * 3 + 1] * fx[(dim + 1) * N + i] + rt[a * 3 + 2] * fx[(dim + 2) * N + i];
        for (int i = 0; i < PN; ++i)
            for (int a = 0; a < 2; ++a)
                fwf[(idx + a) * PN + i] = rt[a * 3 + 0] * fw[(dim)*PN + i] + rt[a * 3 + 1] * fw[(dim + 1) * PN + i] + rt[a * 3 + 2] * fw[(dim + 2) * PN + i];
    }
    // F_x1 += f_x_final*dt ; P = F P F^T + (dt fw) Q (dt fw)^T  (esekfom.hpp:379-381)
    for (int i = 0; i < N * N; ++i) F1[i] += fxf[i] * dt;
    double Q[PN];   // diagonal (Localizator.cpp:164-168)
    for (int i = 0; i < 3; ++i) { Q[i] = cov_gyro; Q[3 + i] = cov_acc; Q[6 + i] = cov_bias_gyro; Q[9 + i] = cov_bias_acc; }
    std::vector<double> FP(N * N, 0.0), Pn(N * N, 0.0);
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) {
            double s = 0;
            for (int k = 0; k < N; ++k) s += F1[i * N + k] * P[k * N + j];
            FP[i * N + j] = s;
        }
    for (int i = 0; i < N; ++i)
        for (int j = 0; j < N; ++j) {
            double s = 0;
            for (int k = 0; k < N; ++k) s += FP[i * N + k] * F1[j * N + k];
            double w = 0;
            for (int k = 0; k < PN; ++k) w += (dt * fwf[i * PN + k]) * Q[k] * (dt * fwf[j * PN + k]);
            Pn[i * N + j] = s + w;
        }
    memcpy(P, Pn.data(), sizeof(double) * N * N);
    return LVO_OK;
}

// Localizator::init_IKFoM_state (Localizator.cpp:135-153)
int lvo_init_state(double* x, double* P, const float q_imu[4], const float g0[3], const float RLI_yaml[9],
                   const float tLI[3]) {
    for (int i = 0; i < LVO_STATE_LEN; ++i) x[i] = 0;
    for (int i = 0; i < 4; ++i) x[S_ROT + i] = (double)q_imu[i];
    // S2(-gravity) normalised to the S2 length (S2.hpp:124-127)
    double g[3] = {-(double)g0[0], -(double)g0[1], -(double)g0[2]};
    double n = std::sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
    for (int i = 0; i < 3; ++i) x[S_GRAV + i] = g[i] / n * kS2Len;
    // column-major Map of the row-major YAML list, no transpose (Localizator.cpp:140, quirk 10)
    double Rm[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) Rm[i * 3 + j] = (double)RLI_yaml[j * 3 + i];
    rot_to_quat(Rm, x + S_OFFR);
    for (int i = 0; i < 3; ++i) x[S_OFFT + i] = (double)tLI[i];
    for (int i = 0; i < N * N; ++i) P[i] = 0;
    for (int i = 0; i < N; ++i) P[i * N + i] = 1.0;
    for (int i = 6; i < 12; ++i) P[i * N + i] = 0.00001;
    for (int i = 15; i < 18; ++i) P[i * N + i] = 0.0001;
    for (int i = 18; i < 21; ++i) P[i * N + i] = 0.001;
    for (int i = 21; i < 23; ++i) P[i * N + i] = 0.00001;
    return LVO_OK;
}

void lvo_boxplus(double* x, const double* d23) { state_boxplus(x, d23); }
void lvo_boxminus(const double* x, const double* y, double* d23) { state_boxminus(x, y, d23); }
void lvo_quat_to_rot(const double q[4], double R[9]) { quat_to_rot(q, R); }
void lvo_plane_fit(const float* pts5, float threshold, float abcd[4], int* is_plane) {
    float pts[5][3];
    memcpy(pts, pts5, sizeof(pts));
    *is_plane = plane_fit(pts, threshold, abcd) ? 1 : 0;
}
void lvo_inverse(const double* A, int n, double* Ainv) { inverse_n(A, n, Ainv); }
void lvo_sym_eig6(const double* A, double* evals, double* evecs) { sym_eig(A, 6, evals, evecs); }
void lvo_last_timing(double* knn_s, double* total_s) { *knn_s = g_knn_s; *total_s = g_total_s; }
void lvo_set_threads(int n) { g_threads = n < 1 ? 1 : n; }

}  // extern "C"

// ------------------------------------------------------------------------------------------
// Deskew: State arithmetic and Compensator (fp32; SURVEY 8f row 2).  PARITY UNPINNED: the reference's Compensator
// needs ROS/PCL/Eigen and cannot be built here, and its tests hold no vectors for it; this follows the source
// text line by line (summation order of 3-term products as in the fp32 geometry above).
// ------------------------------------------------------------------------------------------
namespace {
// SO3Math::Exp<float, float> (Utils.hpp:28-54)
void so3_exp_f(const float* av, float dt, float* E) {
    const float n = sqrtf((av[0] * av[0] + av[1] * av[1]) + av[2] * av[2]);
    for (int i = 0; i < 9; ++i) E[i] = (i % 4 == 0) ? 1.f : 0.f;
    if (!((double)n > 0.0000001)) return;
    const float r[3] = {av[0] / n, av[1] / n, av[2] / n};
    const float K[9] = {0.f, -r[2], r[1], r[2], 0.f, -r[0], -r[1], r[0], 0.f};
    const float ang = n * dt;
    const float sn = sinf(ang), c1 = (float)(1.0 - (double)cosf(ang));
    float cK[9], KK[9];
    for (int i = 0; i < 9; ++i) cK[i] = c1 * K[i];
    m3mul_f(cK, K, KK);
    for (int i = 0; i < 9; ++i) E[i] = (E[i] + sn * K[i]) + KK[i];
}
// State::propagate_f (State.cpp:103-120)
void propagate_f(lvo_state32* s, const float* a, const float* w, float dt) {
    float wb[3], ab[3], E[9], Rn[9], Rab[3];
    for (int i = 0; i < 3; ++i) { wb[i] = w[i] - s->bw[i]; ab[i] = a[i] - s->ba[i]; }
    so3_exp_f(wb, dt, E);
    m3mul_f(s->R, E, Rn);
    m3vec_f(s->R, ab, Rab);
    float vn[3], pn[3];
    for (int i = 0; i < 3; ++i) {
        const float acc = Rab[i] - s->g[i];
        vn[i] = s->vel[i] + acc * dt;
        pn[i] = s->pos[i] + (s->vel[i] * dt + ((0.5f * acc) * dt) * dt);
    }
    memcpy(s->R, Rn, sizeof(Rn));
    for (int i = 0; i < 3; ++i) { s->vel[i] = vn[i]; s->pos[i] = pn[i]; }
}
}  // namespace

extern "C" {

void lvo_state_from_ikfom(const double* x, double time, const float a[3], const float w[3],
                          const float initial_gravity[3], lvo_state32* out) {
    memset(out, 0, sizeof(*out));
    const State32 s = make_state32(x);
    memcpy(out->R, s.X.R, sizeof(out->R));
    memcpy(out->RLI, s.IL.R, sizeof(out->RLI));
    for (int i = 0; i < 3; ++i) {
        out->pos[i] = s.X.t[i];
        out->tLI[i] = s.IL.t[i];
        out->vel[i] = (float)x[S_VEL + i];
        out->bw[i] = (float)x[S_BG + i];
        out->ba[i] = (float)x[S_BA + i];
        out->g[i] = initial_gravity[i];     /* State() reads Config.initial_gravity and nothing overwrites it */
        out->a[i] = a[i];
        out->w[i] = w[i];
    }
    out->time = time;
}

void lvo_state_add_imu(lvo_state32* s, const float a[3], const float w[3], double time) {
    const float dt = (float)(time - s->time);       /* State.cpp:124 */
    propagate_f(s, a, w, dt);
    s->time = time;
    for (int i = 0; i < 3; ++i) {                   /* State.cpp:130-131: (double)0.5 * float vector, cast to float */
        s->a[i] = 0.5f * s->a[i] + 0.5f * a[i];
        s->w[i] = 0.5f * s->w[i] + 0.5f * w[i];
    }
}

int lvo_upsample(const lvo_state32* states, int ns, const float* imu_a, const float* imu_w, const double* imu_t, int ni,
                 lvo_state32* out, int cap) {
    int s = 0, u = 0, no = 0;
    auto push = [&](const lvo_state32& v) { if (no < cap) out[no] = v; ++no; };
    lvo_state32 cur = states[0];
    while (s < ns - 1) {
        push(states[s]);
        while (u < ni && imu_t[u] < states[s + 1].time) {
            lvo_state_add_imu(&cur, imu_a + 3 * u, imu_w + 3 * u, imu_t[u]);
            ++u;
            push(cur);
        }
        cur = states[s++];          /* Compensator.cpp:98: the state BEFORE the increment (reference quirk) */
    }
    if (u >= ni) u = ni - 1;
    push(states[ns - 1]);
    cur = states[ns - 1];
    while (cur.time < imu_t[ni - 1] && u < ni) {
        lvo_state_add_imu(&cur, imu_a + 3 * u, imu_w + 3 * u, imu_t[u]);
        ++u;
        push(cur);
    }
    return no;
}

void lvo_get_t2(const lvo_state32* states, int ns, double t2, lvo_state32* out) {
    int s = ns - 1;
    while (t2 < states[s].time) --s;
    *out = states[s];
    const float a[3] = {out->a[0], out->a[1], out->a[2]}, w[3] = {out->w[0], out->w[1], out->w[2]};
    lvo_state_add_imu(out, a, w, t2);
}

int64_t lvo_compensate(const lvo_state32* states, int ns, const lvo_state32* Xt2, const float* xyz, const double* t,
                       int64_t n, float* xyz_out) {
    Rt32 X2, IL2;
    memcpy(X2.R, Xt2->R, sizeof(X2.R)); memcpy(X2.t, Xt2->pos, sizeof(X2.t));
    memcpy(IL2.R, Xt2->RLI, sizeof(IL2.R)); memcpy(IL2.t, Xt2->tLI, sizeof(IL2.t));
    const Rt32 back = rt_mul(rt_inv(IL2), rt_inv(X2));          /* Xt2.I_Rt_L().inv() * Xt2.inv() */
    int64_t p = 0, no = 0;
    for (int s = 0; s < ns - 1; ++s) {
        while (p < n && states[s].time <= t[p] && t[p] <= states[s + 1].time) {
            lvo_state32 Xtp = states[s];
            const float a[3] = {Xtp.a[0], Xtp.a[1], Xtp.a[2]}, w[3] = {Xtp.w[0], Xtp.w[1], Xtp.w[2]};
            lvo_state_add_imu(&Xtp, a, w, t[p]);
            Rt32 X, IL;
            memcpy(X.R, Xtp.R, sizeof(X.R)); memcpy(X.t, Xtp.pos, sizeof(X.t));
            memcpy(IL.R, Xtp.RLI, sizeof(IL.R)); memcpy(IL.t, Xtp.tLI, sizeof(IL.t));
            float g[3];
            rt_apply(rt_mul(X, IL), xyz + 3 * p, g);            /* Xtp * Xtp.I_Rt_L() * p */
            rt_apply(back, g, xyz_out + 3 * no);
            ++no;
            ++p;
        }
    }
    return no;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// Downsampling (SURVEY 8f row 3).  PARITY UNPINNED for the voxel grid: PCL is not in this image; the
// restatement follows pcl/filters/impl/voxel_grid.hpp (1.8-1.12: applyFilter, downsample_all_data_ = true ->
// CentroidPoint -> AccumulatorXYZ) as called from Compensator.cpp:148-163.
// ------------------------------------------------------------------------------------------
#include <algorithm>
#include <limits>

extern "C" {

int64_t lvo_temporal_downsample(const float* xyz, int64_t n, int rate, double min_dist, int32_t* idx_out) {
    int64_t no = 0;
    int ds_counter = 0;
    for (int64_t i = 0; i < n; ++i) {
        const bool keep = rate <= 1 || (++ds_counter % rate == 0);              /* PointCloudProcessor.cpp:107 */
        const float* p = xyz + 3 * i;
        const float nrm = sqrtf((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2]);     /* Eigen Vector3f::norm() */
        if (keep && min_dist < (double)nrm) idx_out[no++] = (int32_t)i;         /* :108 */
    }
    return no;
}

int64_t lvo_voxelgrid_downsample(const float* xyz, int64_t n, float leaf, float* xyz_out, int64_t cap) {
    if (n <= 0) return 0;
    const float inv = 1.0f / leaf;                                             /* inverse_leaf_size_ = 1 / leaf_size_ */
    float mn[3] = {std::numeric_limits<float>::max(), std::numeric_limits<float>::max(), std::numeric_limits<float>::max()};
    float mx[3] = {-mn[0], -mn[0], -mn[0]};
    for (int64_t i = 0; i < n; ++i)                                            /* getMinMax3D */
        for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], xyz[3 * i + a]); mx[a] = std::max(mx[a], xyz[3 * i + a]); }
    int64_t d[3];
    for (int a = 0; a < 3; ++a) d[a] = (int64_t)((mx[a] - mn[a]) * inv) + 1;
    if (d[0] * d[1] * d[2] > (int64_t)std::numeric_limits<int32_t>::max()) return -1;
    int minb[3], divb[3];
    for (int a = 0; a < 3; ++a) {
        minb[a] = (int)floorf(mn[a] * inv);
        divb[a] = (int)floorf(mx[a] * inv) - minb[a] + 1;
    }
    const int mul[3] = {1, divb[0], divb[0] * divb[1]};
    std::vector<std::pair<unsigned, int64_t>> iv((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
        int idx = 0;
        for (int a = 0; a < 3; ++a) idx += (int)(floorf(xyz[3 * i + a] * inv) - (float)minb[a]) * mul[a];
        iv[(size_t)i] = std::make_pair((unsigned)idx, i);
    }
    std::stable_sort(iv.begin(), iv.end(), [](const std::pair<unsigned, int64_t>& a, const std::pair<unsigned, int64_t>& b) { return a.first < b.first; });
    int64_t no = 0;
    for (size_t i = 0; i < iv.size();) {
        size_t j = i;
        float s[3] = {0.f, 0.f, 0.f};
        while (j < iv.size() && iv[j].first == iv[i].first) {                 /* AccumulatorXYZ: xyz += p */
            for (int a = 0; a < 3; ++a) s[a] += xyz[3 * iv[j].second + a];
            ++j;
        }
        const float cnt = (float)(j - i);
        if (no < cap)
            for (int a = 0; a < 3; ++a) xyz_out[3 * no + a] = s[a] / cnt;     /* xyz / n */
        ++no;
        i = j;
    }
    return no;
}

}  // extern "C"
