/*
 * manifold_ops.h — TEST-ONLY dispatcher over the functions of limo-velo_b200/csrc/lv_manifold.h, one input row at a time.
 *
 * tests/gpu_shim runs it in a kernel (one thread per row, the device build of the header) and tests/cpu_shim in a host loop
 * (the g++ build), so the same rows go through both builds.  A row is kManIn doubles in and kManOut doubles out; the op code
 * says what they hold (tests/manifold_cases.py packs and unpacks them).
 */
#ifndef LV_TEST_MANIFOLD_OPS_H_
#define LV_TEST_MANIFOLD_OPS_H_

#include "../../limo-velo_b200/csrc/lv_manifold.h"

namespace lv {

enum { kManIn = 64, kManOut = 32 };
enum ManOp {
    kOpCosSinc = 0,      /* x2                -> cos, sinc                  */
    kOpSo3Exp = 1,       /* v[3], half        -> q (x, y, z, w)             */
    kOpSo3Log = 2,       /* q[4]              -> v[3]                       */
    kOpAMatrix = 3,      /* v[3]              -> A (3x3 row-major)          */
    kOpS2Bx = 4,         /* v[3]              -> Bx (3x2 row-major)         */
    kOpS2Boxplus = 5,    /* v[3], d0, d1      -> v [+] d                    */
    kOpS2Boxminus = 6,   /* v[3], o[3]        -> v [-] o                    */
    kOpS2Nx = 7,         /* v[3]              -> Nx (2x3 row-major)         */
    kOpS2Mx = 8,         /* v[3], d0, d1      -> Mx (3x2 row-major)         */
    kOpRotToQuat = 9,    /* R (3x3 row-major) -> q                          */
    kOpQuatToRot = 10,   /* q[4]              -> R                          */
    kOpBoxplus = 11,     /* x[26], d[23]      -> x [+] d                    */
    kOpBoxminus = 12,    /* x[26], y[26]      -> x [-] y                    */
};

LV_HD void manifold_op(int op, const double* in, double* out) {
    switch (op) {
    case kOpCosSinc: cos_sinc_sqrt(in[0], out, out + 1); break;
    case kOpSo3Exp: store_quat(out, so3_exp(load_vec3(in), in[3])); break;
    case kOpSo3Log: store_vec3(out, so3_log(load_quat(in))); break;
    case kOpAMatrix: {
        const Mat3d A = A_matrix(load_vec3(in));
        for (int i = 0; i < 9; ++i) out[i] = A.m[i];
        break;
    }
    case kOpS2Bx: s2_Bx(load_vec3(in), out); break;
    case kOpS2Boxplus: store_vec3(out, s2_boxplus(load_vec3(in), in[3], in[4])); break;
    case kOpS2Boxminus: s2_boxminus(load_vec3(in), load_vec3(in + 3), out); break;
    case kOpS2Nx: s2_Nx_yy(load_vec3(in), out); break;
    case kOpS2Mx: s2_Mx(load_vec3(in), in[3], in[4], out); break;
    case kOpRotToQuat: {
        Mat3d R;
        for (int i = 0; i < 9; ++i) R.m[i] = in[i];
        store_quat(out, rot_to_quat(R));
        break;
    }
    case kOpQuatToRot: {
        const Mat3d R = quat_to_rot(load_quat(in));
        for (int i = 0; i < 9; ++i) out[i] = R.m[i];
        break;
    }
    case kOpBoxplus:
        for (int i = 0; i < kStateLen; ++i) out[i] = in[i];
        state_boxplus(out, in + kStateLen);
        break;
    case kOpBoxminus: state_boxminus(in, in + kStateLen, out); break;
    default: break;
    }
}

}  // namespace lv
#endif
