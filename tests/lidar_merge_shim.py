"""ctypes binding of tests/cpu_shim_merge/liblv_mergeshim.so (TEST-ONLY host build of the LiDAR buffer's time-ordered merge,
on the ring of tests/cpu_shim/lidar_ring.cpp)."""
import ctypes as C
import os
import subprocess

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpu_shim_merge")
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _DIR])
        L = C.CDLL(os.path.join(_DIR, "liblv_mergeshim.so"))
        vp, i64, dp, fp = C.c_void_p, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_float)
        L.shim_lidar_create.restype = vp
        L.shim_lidar_create.argtypes = [i64, C.c_int]
        L.shim_lidar_destroy.argtypes = [vp]
        L.shim_lidar_destroy.restype = None
        L.shim_lidar_size.argtypes = [vp]
        L.shim_lidar_size.restype = i64
        L.shim_lidar_push.argtypes = [vp, fp, dp, fp, fp, i64]
        L.shim_lidar_get.argtypes = [vp, C.c_double, C.c_double, fp, dp, fp, fp, i64]
        L.shim_lidar_get.restype = i64
        L.shim_lidar_clear.argtypes = [vp, C.c_double]
        L.shim_lidar_clear.restype = None
        L.shim_lidar_content_full.argtypes = [vp, fp, dp, fp, fp]
        L.shim_lidar_content_full.restype = None
        L.shim_lidar_merge.argtypes = [vp, fp, dp, fp, fp, i64, fp, i64]
        _lib = L
    return _lib
