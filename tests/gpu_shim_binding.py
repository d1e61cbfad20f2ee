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
        vp = C.c_void_p
        L.gs_map_create.restype = vp
        L.gs_map_create.argtypes = [C.c_int64, C.c_int64, C.c_float, C.c_float]
        L.gs_map_add.argtypes = [vp, vp, C.c_int64, C.c_int, C.c_int64, C.c_int64, C.c_int]
        L.gs_map_grow.argtypes = [vp, C.c_int64]
        L.gs_map_clear.argtypes = [vp]
        L.gs_map_dims.argtypes = [vp, vp, vp]
        L.gs_map_dump.argtypes = [vp, vp, vp, vp, C.c_uint32, vp, C.c_uint32, vp, C.c_uint32]
        L.gs_map_free.argtypes = [vp]
        L.gs_manifold.argtypes = [vp, vp, vp, C.c_int]
        L.gs_fit_sets.argtypes = [vp, vp, vp, vp, C.c_float, C.c_int, C.c_int, vp, vp, vp, vp, vp]
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


def manifold(ops, rows):
    """the lv_manifold.h functions on the device, one thread per row (tests/gpu_shim/manifold_ops.h: ops[n] op codes,
    rows n x 64 inputs); returns n x 32 outputs"""
    ops = np.ascontiguousarray(ops, np.int32)
    rows = np.ascontiguousarray(rows, np.float64).reshape(len(ops), 64)
    out = np.zeros((len(ops), 32))
    rc = lib().gs_manifold(ops.ctypes.data, rows.ctypes.data, out.ctypes.data, len(ops))
    assert rc == 0, "CUDA error %d" % rc
    return out


class GsMap:
    """the device map through the library's own map_alloc / map_add / map_grow / map_clear (one stream, synchronised per call)"""

    def __init__(self, max_map_points, max_points, voxel_size, ds=0.2):
        self.L = lib()
        self.k = min(3, max(1, int(np.floor(float(np.float32(voxel_size)) / float(np.float32(ds)) + 0.5))))   # map_alloc's k
        self.h = self.L.gs_map_create(int(max_map_points), int(max_points), float(voxel_size), float(ds))
        assert self.h, "map_alloc failed"

    def close(self):
        if self.h:
            self.L.gs_map_free(C.c_void_p(self.h))
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, xyz, downsample=True, count=None, min_points=0, build_if_empty=False):
        """map_add of xyz; count: the add's count in device memory (MapAddCount)"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        rc = self.L.gs_map_add(C.c_void_p(self.h), xyz.ctypes.data, xyz.shape[0], int(downsample),
                               -1 if count is None else int(count), int(min_points), int(build_if_empty))
        assert rc == 0, "CUDA error %d" % rc

    def grow(self, cap):
        rc = self.L.gs_map_grow(C.c_void_p(self.h), int(cap))
        assert rc == 0, "CUDA error %d" % rc

    def clear(self):
        rc = self.L.gs_map_clear(C.c_void_p(self.h))
        assert rc == 0, "CUDA error %d" % rc

    def dims(self):
        d, ctr = np.zeros(5, np.int64), np.zeros(16, np.uint32)
        rc = self.L.gs_map_dims(C.c_void_p(self.h), d.ctypes.data, ctr.ctypes.data)
        assert rc == 0, "CUDA error %d" % rc
        return d, ctr

    def dump(self):
        import map_ref
        d, ctr = self.dims()
        slots, bslots, list_cap = int(d[0]), int(d[1]), int(d[3])
        top = int(ctr[map_ref.CTR_ARENA_TOP])
        nt, nd = min(int(ctr[map_ref.CTR_TOUCHED]), list_cap), min(int(ctr[map_ref.CTR_DIRTY]), list_cap)
        table, btable = np.zeros((slots, 8), np.uint32), np.zeros((bslots, 4), np.uint32)
        arena, touched, dirty = np.zeros((max(top, 1), 4), np.uint32), np.zeros(max(nt, 1), np.uint32), np.zeros(max(nd, 1), np.uint32)
        rc = self.L.gs_map_dump(C.c_void_p(self.h), table.ctypes.data, btable.ctypes.data, arena.ctypes.data, top,
                                touched.ctypes.data, nt, dirty.ctypes.data, nd)
        assert rc == 0, "CUDA error %d" % rc
        return map_ref.Dump(table, btable, arena[:top], ctr, touched[:nt], dirty[:nd], self.k)
