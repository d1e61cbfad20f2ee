"""ctypes binding of tests/gpu_shim/liblv_gpushim.so (TEST-ONLY: the library's filter kernels launched one at a time)."""
import ctypes as C
import os

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gpu_shim")
_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(os.path.join(_DIR, "liblv_gpushim.so"))
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int32)
        L.gs_step.argtypes = [dp, dp, dp, C.c_int, C.c_int, C.c_int, dp, dp, C.c_int64, dp, dp, dp, dp, dp, ip]
        L.gs_predict.argtypes = [dp, dp, dp, C.c_int, dp]
        L.gs_pack_row.argtypes = [dp, dp, C.c_int64, dp]
        _lib = L
    return _lib


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _a(v):
    return np.ascontiguousarray(v, np.float64)


def pack_row(HTH, HTh, nm):
    row = np.zeros(96)
    lib().gs_pack_row(_d(_a(HTH)), _d(_a(HTh)), int(nm), _d(row))
    return row


def step(x_prop, P_prop, x_cur, HTH, HTh, nm, R, D, limits, max_iter, estimate_extrinsics=1, it=-1, t=0, n_evals=0):
    """one lv_ieskf_step_kernel evaluation (after ieskf_prepare); returns a dict"""
    prm = _a(np.concatenate([[R, D], np.asarray(limits, np.float64), [max_iter, estimate_extrinsics]]))
    reduced, dx, x, P, ints = np.zeros(157), np.zeros(23), np.zeros(26), np.zeros((23, 23)), np.zeros(7, np.int32)
    rc = lib().gs_step(_d(_a(x_prop)), _d(_a(P_prop)), _d(_a(x_cur)), int(it), int(t), int(n_evals), _d(_a(HTH)), _d(_a(HTh)),
                       int(nm), _d(prm), _d(reduced), _d(dx), _d(x), _d(P), ints.ctypes.data_as(C.POINTER(C.c_int32)))
    assert rc == 0, "CUDA error %d" % rc
    return dict(reduced=reduced, dx=dx, x=x, P=P, converged=int(ints[0]), degenerate=int(ints[1]), done=int(ints[2]),
                status=int(ints[3]), n_evals=int(ints[4]), t=int(ints[5]), iter=int(ints[6]))


def predict(x, P, acc, gyro, dt, noise):
    """k samples through ONE launch_predict (no batching)"""
    acc, gyro, dt = np.asarray(acc).reshape(-1, 3), np.asarray(gyro).reshape(-1, 3), np.asarray(dt).reshape(-1)
    imu = _a(np.concatenate([acc, gyro, dt[:, None]], axis=1))
    x, P = _a(x).copy(), _a(P).reshape(23, 23).copy()
    rc = lib().gs_predict(_d(x), _d(P), _d(imu), len(dt), _d(_a(noise)))
    assert rc == 0, "CUDA error %d" % rc
    return x, P
