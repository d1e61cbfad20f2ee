"""limovelo_b200 — Python (ctypes) access to liblimovelo_b200.so for tests and benchmarks.

The product is the C-ABI shared library (include/limovelo_b200.h) built from csrc/ (CUDA, sm_90a)
and host/ (C++); this module only marshals numpy arrays into it.  There is no Python or CPU
implementation behind it: if the library is missing, loading raises, and without a CUDA device
every compute call returns LV_ERR_CUDA (raised as RuntimeError here).

The directory name contains a hyphen, so import it through `__graft_entry__.load_package()`
(registers it as module `limovelo_b200`).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LV_LIB_PATH") or os.path.join(_HERE, "liblimovelo_b200.so")   # LV_LIB_PATH: variant builds of tools/
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "limovelo_b200.h")

STATE_LEN, DOF, MAX_EVALS = 26, 23, 8
OK, EMPTY_MAP, TOO_FEW_MATCHES, ERR_ARG, ERR_CUDA, ERR_CAPACITY, ERR_IO, TOO_FEW_POINTS = range(8)
STATUS_NAMES = ["LV_OK", "LV_EMPTY_MAP", "LV_TOO_FEW_MATCHES", "LV_ERR_ARG", "LV_ERR_CUDA", "LV_ERR_CAPACITY",
                "LV_ERR_IO", "LV_TOO_FEW_POINTS"]


class Params(C.Structure):
    _fields_ = [
        ("MAX_NUM_ITERS", C.c_int32), ("NUM_MATCH_POINTS", C.c_int32), ("estimate_extrinsics", C.c_int32),
        ("print_degeneracy_values", C.c_int32), ("MAX_DIST_PLANE", C.c_double), ("PLANES_THRESHOLD", C.c_float),
        ("pad0_", C.c_float), ("LiDAR_noise", C.c_double), ("degeneracy_threshold", C.c_double),
        ("LIMITS", C.c_double * DOF),
        ("covariance_gyroscope", C.c_double), ("covariance_acceleration", C.c_double),
        ("covariance_bias_gyroscope", C.c_double), ("covariance_bias_acceleration", C.c_double),
        ("initial_gravity", C.c_float * 3), ("I_Translation_L", C.c_float * 3), ("I_Rotation_L", C.c_float * 9),
        ("map_downsample_size", C.c_float), ("voxel_size", C.c_float), ("device", C.c_int32),
        ("pad1_", C.c_int32), ("max_map_points", C.c_int64), ("max_points", C.c_int64),
        ("stream", C.c_void_p),
    ]


class IterLog(C.Structure):
    _fields_ = [("n_matches", C.c_int64), ("converged", C.c_int32), ("degenerate", C.c_int32),
                ("HTH", C.c_double * 144), ("HTh", C.c_double * 12), ("dx", C.c_double * DOF),
                ("x_after", C.c_double * STATE_LEN)]


class Profile(C.Structure):
    _fields_ = [("measure_ms", C.c_double), ("solve_ms", C.c_double), ("build_ms", C.c_double),
                ("measure_launches", C.c_int64), ("solve_launches", C.c_int64), ("build_launches", C.c_int64),
                ("total_launches", C.c_int64), ("idle_ms", C.c_double), ("idle_launches", C.c_int64),
                ("search_ms", C.c_double), ("search_upper_ms", C.c_double), ("fit_ms", C.c_double),
                ("reuse_ms", C.c_double), ("search_first_ms", C.c_double), ("search_first_launches", C.c_int64)]


class MapInfo(C.Structure):
    """struct lv_map_info: capacity, usage and growth of the device map"""
    _fields_ = [("capacity_points", C.c_int64), ("voxel_slots", C.c_int64), ("block_slots", C.c_int64),
                ("arena_entries", C.c_int64), ("add_capacity", C.c_int64), ("bytes", C.c_int64),
                ("points", C.c_int64), ("slots_used", C.c_int64), ("blocks_used", C.c_int64), ("arena_top", C.c_int64),
                ("growths", C.c_int64), ("growth_limit", C.c_int64), ("host_waits", C.c_int64),
                ("error_flags", C.c_uint32), ("pad_", C.c_uint32)]


class LidarInfo(C.Structure):
    """struct lv_lidar_info: fill state of the LiDAR buffer"""
    _fields_ = [("points", C.c_int64), ("capacity", C.c_int64), ("oldest_time", C.c_double), ("newest_time", C.c_double)]


class PrelocParams(C.Structure):
    """lv_preloc_params: the window lv_prelocalize searches"""
    _fields_ = [("radius", C.c_float), ("step", C.c_float), ("yaw_range", C.c_float), ("yaw_step", C.c_float),
                ("max_points", C.c_int32), ("pad_", C.c_int32)]


class PrelocResult(C.Structure):
    """lv_preloc_result: the winning candidate"""
    _fields_ = [("x", C.c_double * STATE_LEN), ("candidates", C.c_int64), ("index", C.c_int64), ("k", C.c_int32),
                ("i", C.c_int32), ("j", C.c_int32), ("score", C.c_int32), ("points", C.c_int32), ("pad_", C.c_int32)]


class PrelocStats(C.Structure):
    """lv_preloc_stats: the work of one lv_prelocalize_global call"""
    _fields_ = [("candidates", C.c_int64), ("cells_bounded", C.c_int64), ("candidates_scored", C.c_int64), ("probes", C.c_int64),
                ("launches", C.c_int32), ("pad_", C.c_int32)]


def preloc_count(radius, step, yaw_range, yaw_step, max_points=2048):
    """the number of candidates of a window, -1 for invalid parameters (no GPU needed)"""
    return int(lib().lv_preloc_count(C.byref(PrelocParams(radius, step, yaw_range, yaw_step, max_points, 0))))


def pcd_write(path, xyz):
    """the points (m x 3, float32) as a binary PCD v0.7 file with fields x y z"""
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    _check(lib().lv_pcd_write(str(path).encode(), _f(xyz), xyz.shape[0]))


def pcd_read(path):
    """the finite x y z points of an ascii or binary PCD file, in file order (m x 3, float32)"""
    L, n = lib(), C.c_int64(0)
    _check(L.lv_pcd_read(str(path).encode(), None, 0, C.byref(n)))
    out = np.zeros((max(n.value, 1), 3), np.float32)
    _check(L.lv_pcd_read(str(path).encode(), _f(out), n.value, C.byref(n)))
    return out[:n.value]


def build(verbose=False):
    """Compile liblimovelo_b200.so in-tree with nvcc for sm_90a (works without a GPU)."""
    cmd = ["make", "-C", _HERE, "-j8"]
    if not verbose:
        cmd.insert(1, "-s")
    subprocess.check_call(cmd)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("liblimovelo_b200.so is not built (run __graft_entry__.build()); there is no fallback")
    L = C.CDLL(LIB_PATH)
    dp, fp, vp = C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_void_p
    i64, i32p = C.c_int64, C.POINTER(C.c_int32)
    L.lv_default_params.argtypes = [C.POINTER(Params)]
    L.lv_default_params.restype = None
    L.lv_params_from_yaml.argtypes = [C.c_char_p, C.POINTER(Params)]
    L.lv_create.argtypes = [C.POINTER(Params), C.POINTER(vp)]
    L.lv_destroy.argtypes = [vp]
    L.lv_destroy.restype = None
    L.lv_last_error.restype = C.c_char_p
    L.lv_version.restype = C.c_char_p
    L.lv_result_bytes.restype = C.c_int64
    L.lv_map_build.argtypes = [vp, fp, i64]
    L.lv_map_add.argtypes = [vp, fp, i64, C.c_int]
    L.lv_map_size.argtypes = [vp]
    L.lv_map_size.restype = i64
    L.lv_map_exists.argtypes = [vp]
    L.lv_map_points.argtypes = [vp, fp, i64]
    L.lv_map_points.restype = i64
    L.lv_map_build_device.argtypes = [vp, vp, i64]
    L.lv_map_add_device.argtypes = [vp, vp, i64, C.c_int]
    L.lv_map_status.argtypes = [vp]
    L.lv_map_add_sweep_device.argtypes = [vp, vp, i64, C.c_int]
    L.lv_map_add_last_sweep.argtypes = [vp, C.c_int]
    if hasattr(L, "lv_map_reserve"):   # map growth; absent from older builds that tools/ab_bench.py may load via LV_LIB_PATH
        L.lv_map_reserve.argtypes = [vp, i64]
        L.lv_map_set_growth.argtypes = [vp, i64]
        L.lv_map_info.argtypes = [vp, C.POINTER(MapInfo)]
    L.lv_measure.argtypes = [vp, dp, fp, i64, dp, dp, C.POINTER(i64)]
    L.lv_measure_reduced.argtypes = [vp, dp, fp, i64, dp, dp, C.POINTER(i64)]
    L.lv_match_all.argtypes = [vp, dp, fp, i64, C.POINTER(C.c_uint8), i32p, fp, fp, fp, fp]
    L.lv_last_neighbours.argtypes = [vp, i64, i32p]
    L.lv_set_state.argtypes = [vp, dp, dp]
    L.lv_get_state.argtypes = [vp, dp, dp]
    L.lv_init_state.argtypes = [vp, fp]
    L.lv_predict.argtypes = [vp, dp, dp, C.c_double]
    L.lv_propagate_device.argtypes = [vp, dp, dp, dp, C.c_int32]
    L.lv_init_state_host.argtypes = [C.POINTER(Params), fp, dp, dp]
    L.lv_predict_host.argtypes = [C.POINTER(Params), dp, dp, C.c_double, dp, dp]
    L.lv_correct.argtypes = [vp, fp, i64, C.c_double, C.POINTER(IterLog), i32p, dp, dp]
    L.lv_correct_device.argtypes = [vp, vp, i64, C.c_double]
    L.lv_last_logs.argtypes = [vp, C.POINTER(IterLog), i32p]
    L.lv_last_time_updated.argtypes = [vp]
    L.lv_last_time_updated.restype = C.c_double
    L.lv_host_alloc.argtypes = [i64]
    L.lv_host_alloc.restype = vp
    L.lv_host_free.argtypes = [vp]
    L.lv_host_free.restype = None
    L.lv_device_alloc.argtypes = [vp, i64]
    L.lv_device_alloc.restype = vp
    L.lv_device_free.argtypes = [vp, vp]
    L.lv_device_free.restype = None
    L.lv_memcpy_h2d.argtypes = [vp, vp, vp, i64]
    L.lv_memcpy_d2h.argtypes = [vp, vp, vp, i64]
    L.lv_process_cloud_device.argtypes = [vp, C.c_int, C.POINTER(CloudLayout), vp, i64, i64, C.c_uint64, C.c_int, C.c_int,
                                          C.c_double, C.c_int32, C.c_double, vp, vp, vp, vp, vp, C.POINTER(i64)]
    if hasattr(L, "lv_async_status"):   # the stream-ordered tick; absent from older builds that tools/ab_bench.py may load
        L.lv_process_cloud_device_async.argtypes = [vp, C.c_int, C.POINTER(CloudLayout), vp, i64, i64, C.c_uint64, C.c_int, C.c_int,
                                                    C.c_double, C.c_int32, C.c_double, vp, vp, vp, vp, vp, vp]
        L.lv_compensate_device_async.argtypes = [vp, vp, C.c_int32, vp, vp, vp, vp, i64, vp]
        L.lv_voxelgrid_downsample_device_async.argtypes = [vp, vp, vp, i64, C.c_float, vp, vp]
        L.lv_correct_device_async.argtypes = [vp, vp, vp, i64, i64, C.c_double]
        L.lv_async_status.argtypes = [vp]
    if hasattr(L, "lv_lidar_reserve"):   # the LiDAR buffer; absent from older builds that tools/ab_bench.py may load
        L.lv_lidar_reserve.argtypes = [vp, i64]
        L.lv_lidar_push_device_async.argtypes = [vp, vp, vp, vp, i64]
        L.lv_lidar_get_points_device_async.argtypes = [vp, C.c_double, C.c_double, vp, vp, i64, vp]
        L.lv_lidar_get_points_device.argtypes = [vp, C.c_double, C.c_double, vp, vp, i64, C.POINTER(i64)]
        L.lv_lidar_clear_async.argtypes = [vp, C.c_double]
        L.lv_lidar_info.argtypes = [vp, C.POINTER(LidarInfo)]
    if hasattr(L, "lv_sweep_to_world_device_async"):   # the tick's output and mapping step; absent from older builds
        L.lv_sweep_to_world_device_async.argtypes = [vp, vp, vp, i64, vp, vp]
        L.lv_map_add_device_async.argtypes = [vp, vp, vp, i64, C.c_int]
    if hasattr(L, "lv_lidar_reserve_full"):   # full points (intensity, range) through the tick; absent from older builds
        L.lv_lidar_reserve_full.argtypes = [vp, i64]
        L.lv_lidar_push_full_device_async.argtypes = [vp, vp, vp, vp, vp, vp, i64]
        L.lv_lidar_get_points_full_device_async.argtypes = [vp, C.c_double, C.c_double, vp, vp, vp, vp, i64, vp]
        L.lv_voxelgrid_downsample_full.argtypes = [vp, vp, vp, vp, i64, C.c_float, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_voxelgrid_downsample_full_device_async.argtypes = [vp, vp, vp, vp, vp, i64, C.c_float, vp, vp, vp, vp, vp]
        L.lv_cloud_stamp_device_async.argtypes = [vp, vp, vp, i64, vp]
    if hasattr(L, "lv_process_livox_device"):   # the Livox front end; absent from older builds
        L.lv_livox_to_points.argtypes = [vp, i64, i64, C.c_uint64, C.c_uint8, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_livox_device.argtypes = [vp, vp, i64, i64, C.c_uint64, C.c_uint8, C.c_int32, C.c_double, vp, vp, vp, vp, vp,
                                              C.POINTER(i64)]
        L.lv_process_livox_device_async.argtypes = [vp, vp, i64, i64, C.c_uint64, C.c_uint8, C.c_int32, C.c_double, vp, vp, vp, vp, vp, vp]
        L.lv_bag_parse_livox.argtypes = [vp, i64, C.POINTER(LivoxView)]
    if hasattr(L, "lv_process_velodyne_device"):   # the Velodyne packet front end; absent from older builds
        cp = C.POINTER(VelodyneCalibration)
        L.lv_velodyne_default_calibration.argtypes = [C.c_int, cp]
        L.lv_velodyne_to_points.argtypes = [vp, i64, i64, cp, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_velodyne_device.argtypes = [vp, vp, i64, i64, cp, C.c_int32, C.c_double, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_velodyne_device_async.argtypes = [vp, vp, i64, i64, cp, C.c_int32, C.c_double, vp, vp, vp, vp, vp, vp]
        L.lv_bag_parse_velodyne_scan.argtypes = [vp, i64, C.POINTER(VelodyneView)]
    if hasattr(L, "lv_process_ouster_device"):   # the Ouster packet front end; absent from older builds
        cp = C.POINTER(OusterCalibration)
        L.lv_ouster_calibration_from_json.argtypes = [C.c_char_p, i64, cp]
        L.lv_ouster_to_points.argtypes = [vp, i64, i64, cp, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_ouster_device.argtypes = [vp, vp, i64, i64, cp, C.c_int32, C.c_double, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_ouster_device_async.argtypes = [vp, vp, i64, i64, cp, C.c_int32, C.c_double, vp, vp, vp, vp, vp, vp]
        L.lv_bag_parse_ouster_packet.argtypes = [vp, i64, C.POINTER(OusterPacketView)]
        L.lv_ouster_imu_packet.argtypes = [vp, i64, C.POINTER(ImuSample)]
    if hasattr(L, "lv_process_ouster_packets_device"):   # the Ouster UDP profiles of firmware 2.2+; absent from older builds
        cp = C.POINTER(OusterCalibration)
        L.lv_ouster_sensor_from_json.argtypes = [C.c_char_p, i64, cp, C.POINTER(C.c_int)]
        L.lv_ouster_packets_to_points.argtypes = [vp, i64, i64, cp, C.c_int, vp, vp, vp, vp, vp, C.POINTER(i64)]
        L.lv_process_ouster_packets_device.argtypes = [vp, vp, i64, i64, cp, C.c_int, C.c_int32, C.c_double, vp, vp, vp, vp, vp,
                                                       C.POINTER(i64)]
        L.lv_process_ouster_packets_device_async.argtypes = [vp, vp, i64, i64, cp, C.c_int, C.c_int32, C.c_double, vp, vp, vp, vp,
                                                             vp, vp]
    if hasattr(L, "lv_lidar_reserve_merge"):   # the time-ordered merge of several LiDARs; absent from older builds
        L.lv_lidar_reserve_merge.argtypes = [vp, i64]
        L.lv_lidar_merge_device_async.argtypes = [vp, vp, vp, vp, i64, fp]
        L.lv_lidar_merge_full_device_async.argtypes = [vp, vp, vp, vp, vp, vp, i64, fp]
    if hasattr(L, "lv_prelocalize"):   # start pose search and PCD files; absent from older builds
        L.lv_preloc_count.argtypes = [C.POINTER(PrelocParams)]
        L.lv_preloc_count.restype = i64
        L.lv_prelocalize.argtypes = [vp, vp, i64, C.POINTER(PrelocParams), C.POINTER(PrelocResult), i32p]
        L.lv_pcd_write.argtypes = [C.c_char_p, fp, i64]
        L.lv_pcd_read.argtypes = [C.c_char_p, fp, i64, C.POINTER(i64)]
    if hasattr(L, "lv_prelocalize_global"):   # the whole-map start pose search; absent from older builds
        L.lv_prelocalize_global.argtypes = [vp, vp, i64, C.POINTER(PrelocParams), C.POINTER(PrelocResult), C.POINTER(PrelocStats)]
        L.lv_map_extent.argtypes = [vp, dp, dp]
    L.lv_synchronize.argtypes = [vp]
    L.lv_profile_enable.argtypes = [vp, C.c_int]
    L.lv_profile_get.argtypes = [vp, C.POINTER(Profile), C.c_int]
    L.lv_flush_l2.argtypes = [vp]
    _lib = L
    return L


SYNTH_LIB_PATH = os.path.join(_HERE, "liblv_synth.so")
_synth = None


def synth_lib():
    """liblv_synth.so (include/lv_synth.h): the synthetic reader + the YAML reader, plain C++ — a process that only
    needs inputs (bench.py's CPU reference arm) never loads the CUDA library."""
    global _synth
    if _synth is not None:
        return _synth
    if not os.path.exists(SYNTH_LIB_PATH):
        raise RuntimeError("liblv_synth.so is not built (run __graft_entry__.build())")
    L = C.CDLL(SYNTH_LIB_PATH)
    dp, fp, vp, i64 = C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_void_p, C.c_int64
    L.lv_default_params.argtypes = [C.POINTER(Params)]
    L.lv_default_params.restype = None
    L.lv_params_from_yaml.argtypes = [C.c_char_p, C.POINTER(Params)]
    L.lv_init_state_host.argtypes = [C.POINTER(Params), fp, dp, dp]
    L.lv_synth_world_create.argtypes = [C.c_uint64, i64]
    L.lv_synth_world_create.restype = vp
    L.lv_synth_world_destroy.argtypes = [vp]
    L.lv_synth_world_destroy.restype = None
    L.lv_synth_world_map.argtypes = [vp, fp, i64]
    L.lv_synth_world_map.restype = i64
    L.lv_synth_world_extent.argtypes = [vp]
    L.lv_synth_world_extent.restype = C.c_double
    L.lv_synth_pose.argtypes = [vp, C.c_double, C.POINTER(Params), dp]
    L.lv_synth_pose.restype = None
    L.lv_synth_sweep.argtypes = [vp, dp, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
                                 C.c_uint64, fp]
    L.lv_synth_sweep.restype = i64
    _synth = L
    return L


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def default_params(_L=None, **over):
    p = Params()
    (_L or lib()).lv_default_params(C.byref(p))
    for k, v in over.items():
        cur = getattr(p, k)
        if hasattr(cur, "__len__"):
            for i, x in enumerate(v):
                cur[i] = x
        else:
            setattr(p, k, v)
    return p


def params_from_yaml(path, _L=None, **over):
    """lv_params from a LIMO-Velo YAML (+ field overrides).  _L: the library providing the reader (default: the product's;
    liblv_synth.so carries the same reader for processes that must not load the CUDA library)"""
    p = default_params(_L)
    st = (_L or lib()).lv_params_from_yaml(str(path).encode(), C.byref(p))
    if st != OK:
        raise RuntimeError("lv_params_from_yaml(%s) -> %s" % (path, STATUS_NAMES[st]))
    for k, v in over.items():
        setattr(p, k, v)
    return p


CONFIG_DIR = os.path.join(_HERE, "config")


def _check(st, allow=()):
    if st != OK and st not in allow:
        raise RuntimeError("%s: %s" % (STATUS_NAMES[st], lib().lv_last_error().decode()))
    return st


def _logs_to_py(logs, n):
    out = []
    for i in range(n):
        lg = logs[i]
        out.append(dict(n_matches=int(lg.n_matches), converged=int(lg.converged), degenerate=int(lg.degenerate),
                        HTH=np.array(lg.HTH[:]).reshape(12, 12), HTh=np.array(lg.HTh[:]),
                        dx=np.array(lg.dx[:]), x_after=np.array(lg.x_after[:])))
    return out


class State32(C.Structure):
    """lv_state32: `State` of the reference (Objects.hpp:97-120), single precision"""
    _fields_ = [("R", C.c_float * 9), ("pos", C.c_float * 3), ("vel", C.c_float * 3), ("bw", C.c_float * 3),
                ("ba", C.c_float * 3), ("g", C.c_float * 3), ("RLI", C.c_float * 9), ("tLI", C.c_float * 3),
                ("a", C.c_float * 3), ("w", C.c_float * 3), ("time", C.c_double)]

    def as_tuple(self):
        return tuple(np.array(getattr(self, k)[:], dtype=np.float32).tobytes() for k, _ in self._fields_[:-1]) + (self.time,)


def _f3(v):
    return (C.c_float * 3)(*[float(t) for t in v])


def state_from_ikfom(params, x, time, a, w):
    """State(const state_ikfom&, double) (State.cpp:40-62)"""
    out = State32()
    lib().lv_state_from_ikfom(C.byref(params), _d(np.ascontiguousarray(x, np.float64)), C.c_double(time), _f3(a), _f3(w),
                              C.byref(out))
    return out


def state_add_imu(state, a, w, time):
    """State::operator+=(IMU) on a copy"""
    out = State32.from_buffer_copy(state)
    lib().lv_state_add_imu(C.byref(out), _f3(a), _f3(w), C.c_double(time))
    return out


def compensator_upsample(states, imu_a, imu_w, imu_t):
    """Compensator::upsample: list of State32 + IMU arrays -> the integrated path (list of State32)"""
    ns, ni = len(states), len(imu_t)
    arr = (State32 * ns)(*states)
    a = np.ascontiguousarray(imu_a, np.float32).reshape(ni, 3)
    w = np.ascontiguousarray(imu_w, np.float32).reshape(ni, 3)
    t = np.ascontiguousarray(imu_t, np.float64)
    cap = ns + ni + 8
    out = (State32 * cap)()
    lib().lv_compensator_upsample.restype = C.c_int32
    n = lib().lv_compensator_upsample(arr, ns, _f(a), _f(w), _d(t), ni, out, cap)
    assert n <= cap
    return [State32.from_buffer_copy(out[i]) for i in range(n)]


def compensator_get_t2(path, t2):
    arr = (State32 * len(path))(*path)
    out = State32()
    lib().lv_compensator_get_t2(arr, len(path), C.c_double(t2), C.byref(out))
    return out


class CloudLayout(C.Structure):
    _fields_ = [("point_step", C.c_int32), ("off_x", C.c_int32), ("off_y", C.c_int32), ("off_z", C.c_int32),
                ("off_intensity", C.c_int32), ("off_time", C.c_int32), ("off_range", C.c_int32)]


LIDAR_TYPES = {"velodyne": 0, "hesai": 1, "ouster": 2, "custom": 3}


def _transform12(T):
    """a rigid transform as lv_lidar_merge_device_async takes it: None, or 12 floats (R row-major, then t)"""
    if T is None:
        return None
    return (C.c_float * 12)(*np.ascontiguousarray(T, np.float32).reshape(12).tolist())


def cloud_layout(lidar, dtype):
    """lv_cloud_layout of a numpy structured dtype with the fields of `lidar`'s point struct"""
    f = dtype.fields
    tname = {"velodyne": "time", "ouster": "t"}.get(lidar, "timestamp")
    iname = "reflectivity" if lidar == "ouster" else "intensity"
    return CloudLayout(dtype.itemsize, f["x"][1], f["y"][1], f["z"][1], f[iname][1], f[tname][1],
                       f["range"][1] if "range" in f else 0)


def pointcloud2_to_points(lidar, pts, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time):
    """PointCloudProcessor::msg2points on a numpy structured array (its buffer is the message's `data`)"""
    pts = np.ascontiguousarray(pts)
    lay = cloud_layout(lidar, pts.dtype)
    n = len(pts)
    xyz, t = np.zeros((n, 3), np.float32), np.zeros(n, np.float64)
    inten, rng = np.zeros(n, np.float32), np.zeros(n, np.float32)
    _check(lib().lv_pointcloud2_to_points(LIDAR_TYPES[lidar], C.byref(lay), pts.ctypes.data_as(C.POINTER(C.c_uint8)), C.c_int64(n),
                                         C.c_uint64(header_stamp_us), int(stamp_beginning), int(offset_beginning),
                                         C.c_double(full_rotation_time), _f(xyz), _d(t), _f(inten), _f(rng)))
    return xyz, t, inten, rng


def time_sort_indices(t):
    t = np.ascontiguousarray(t, np.float64)
    idx = np.zeros(len(t), np.int32)
    _check(lib().lv_time_sort_indices(_d(t), C.c_int64(len(t)), idx.ctypes.data_as(C.POINTER(C.c_int32))))
    return idx


# livox_ros_driver(2)/CustomMsg: one 19-byte record per point (include/limovelo_b200.h)
LIVOX_RECORD = np.dtype({"names": ["offset_time", "x", "y", "z", "reflectivity", "tag", "line"],
                         "formats": ["<u4", "<f4", "<f4", "<f4", "u1", "u1", "u1"], "offsets": [0, 4, 8, 12, 16, 17, 18], "itemsize": 19})


class LivoxView(C.Structure):
    _fields_ = [("stamp_sec", C.c_uint32), ("stamp_nsec", C.c_uint32), ("timebase", C.c_uint64), ("point_num", C.c_uint32),
                ("lidar_id", C.c_uint8), ("n_points", C.c_int64), ("data", C.c_void_p), ("data_bytes", C.c_int64)]


def bag_parse_livox(msg):
    """lv_bag_parse_livox on a serialised CustomMsg (bytes): returns (LivoxView, the records as a LIVOX_RECORD array)"""
    v = LivoxView()
    buf = C.create_string_buffer(bytes(msg), len(msg))
    _check(lib().lv_bag_parse_livox(buf, len(msg), C.byref(v)))
    off = v.data - C.addressof(buf) if v.n_points else 0
    return v, np.frombuffer(buf.raw[off:off + v.data_bytes], LIVOX_RECORD).copy()


def livox_to_points(records, timebase_ns, tag_reject_mask):
    """msg2points of a Livox message on the host (records: LIVOX_RECORD array, or its raw bytes): returns (xyz, time, intensity,
    range, index in the message) of the tag-kept points, in message order"""
    raw = np.ascontiguousarray(np.frombuffer(np.ascontiguousarray(records).tobytes(), np.uint8))
    n = len(raw) // 19
    out = (np.empty((n, 3), np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.int32))
    m = C.c_int64(0)
    _check(lib().lv_livox_to_points(raw.ctypes.data_as(C.c_void_p), len(raw), n, C.c_uint64(timebase_ns), int(tag_reject_mask),
                                    *(a.ctypes.data_as(C.c_void_p) for a in out), C.byref(m)))
    return tuple(a[:m.value].copy() for a in out)


# velodyne_msgs/VelodyneScan of a VLP-16 / Puck Hi-Res: packets of 1214 bytes, 384 slots each (include/limovelo_b200.h)
VELODYNE_PACKET = 1214
VELODYNE_SLOTS = 384
VELODYNE_MODELS = {"vlp16": 0, "puck_hires": 1}


class VelodyneCalibration(C.Structure):
    _fields_ = [("vert_correction", C.c_double * 16), ("rot_correction", C.c_double * 16), ("dist_correction", C.c_double * 16),
                ("vert_offset_correction", C.c_double * 16), ("horiz_offset_correction", C.c_double * 16)]


class VelodyneView(C.Structure):
    _fields_ = [("stamp_sec", C.c_uint32), ("stamp_nsec", C.c_uint32), ("n_packets", C.c_int64), ("packets", C.c_void_p),
                ("data_bytes", C.c_int64)]


def velodyne_calibration(model="vlp16"):
    """lv_velodyne_default_calibration: the nominal calibration of "vlp16" or "puck_hires" (a VelodyneCalibration)"""
    cal = VelodyneCalibration()
    _check(lib().lv_velodyne_default_calibration(VELODYNE_MODELS[model], C.byref(cal)))
    return cal


def bag_parse_velodyne_scan(msg):
    """lv_bag_parse_velodyne_scan on a serialised VelodyneScan (bytes): returns (VelodyneView, the packets as uint8 bytes)"""
    v = VelodyneView()
    buf = C.create_string_buffer(bytes(msg), len(msg))
    _check(lib().lv_bag_parse_velodyne_scan(buf, len(msg), C.byref(v)))
    off = v.packets - C.addressof(buf) if v.n_packets else 0
    return v, np.frombuffer(buf.raw[off:off + v.data_bytes], np.uint8).copy()


def velodyne_to_points(packets, cal):
    """msg2points of a VelodyneScan on the host (packets: their bytes, 1214 per packet): returns (xyz, time, intensity, range, slot)
    of the points, in slot order"""
    raw = np.ascontiguousarray(np.frombuffer(bytes(memoryview(packets)), np.uint8))
    k = len(raw) // VELODYNE_PACKET
    n = VELODYNE_SLOTS * k
    out = (np.empty((n, 3), np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.int32))
    m = C.c_int64(0)
    _check(lib().lv_velodyne_to_points(raw.ctypes.data_as(C.c_void_p), len(raw), k, C.byref(cal),
                                       *(a.ctypes.data_as(C.c_void_p) for a in out), C.byref(m)))
    return tuple(a[:m.value].copy() for a in out)


# ouster_ros/PacketMsg of an Ouster: packets of 16 columns in one of four lidar UDP profiles (include/limovelo_b200.h, lv_ouster_profile)
OUSTER_COLUMNS = 16
OUSTER_IMU_PACKET = 48
OUSTER_LEGACY, OUSTER_RNG19_RFL8_SIG16_NIR16, OUSTER_RNG19_RFL8_SIG16_NIR16_DUAL, OUSTER_RNG15_RFL8_NIR8 = range(4)
OUSTER_PROFILES = {"LEGACY": OUSTER_LEGACY, "RNG19_RFL8_SIG16_NIR16": OUSTER_RNG19_RFL8_SIG16_NIR16,
                   "RNG19_RFL8_SIG16_NIR16_DUAL": OUSTER_RNG19_RFL8_SIG16_NIR16_DUAL, "RNG15_RFL8_NIR8": OUSTER_RNG15_RFL8_NIR8}
_OUSTER_PIXEL_BYTES = {OUSTER_RNG19_RFL8_SIG16_NIR16: 12, OUSTER_RNG19_RFL8_SIG16_NIR16_DUAL: 16, OUSTER_RNG15_RFL8_NIR8: 4}


def ouster_packet_bytes(H, profile=OUSTER_LEGACY):
    """bytes per lidar packet: 16 (20 + 12 H) for LEGACY, 32 + 16 (12 + s H) + 32 for the others (s: the profile's pixel bytes)"""
    if profile == OUSTER_LEGACY:
        return OUSTER_COLUMNS * (20 + 12 * H)
    return 64 + OUSTER_COLUMNS * (12 + _OUSTER_PIXEL_BYTES[profile] * H)


class OusterCalibration(C.Structure):
    _fields_ = [("columns_per_frame", C.c_int32), ("pixels_per_column", C.c_int32), ("beam_altitude_angles", C.c_double * 128),
                ("beam_azimuth_angles", C.c_double * 128), ("lidar_origin_to_beam_origin_mm", C.c_double)]


class OusterPacketView(C.Structure):
    _fields_ = [("data", C.c_void_p), ("bytes", C.c_int64)]


class ImuSample(C.Structure):
    """lv_imu_sample: what Accumulator::receive_imu reads"""
    _fields_ = [("stamp_sec", C.c_uint32), ("stamp_nsec", C.c_uint32), ("orientation", C.c_double * 4),
                ("angular_velocity", C.c_double * 3), ("linear_acceleration", C.c_double * 3)]


def ouster_calibration(W, altitude_deg, azimuth_deg, origin_mm=0.0):
    """an OusterCalibration from W (columns per frame) and the per-beam angles in degrees (H = their count)"""
    cal = OusterCalibration()
    cal.columns_per_frame, cal.pixels_per_column = int(W), len(altitude_deg)
    for p, (a, z) in enumerate(zip(altitude_deg, azimuth_deg)):
        cal.beam_altitude_angles[p], cal.beam_azimuth_angles[p] = float(a), float(z)
    cal.lidar_origin_to_beam_origin_mm = float(origin_mm)
    return cal


def ouster_calibration_from_json(text):
    """lv_ouster_calibration_from_json on the sensor metadata (str or bytes): an OusterCalibration"""
    raw = text.encode() if isinstance(text, str) else bytes(text)
    cal = OusterCalibration()
    _check(lib().lv_ouster_calibration_from_json(raw, len(raw), C.byref(cal)))
    return cal


def ouster_sensor_from_json(text):
    """lv_ouster_sensor_from_json on the sensor metadata (str or bytes): (OusterCalibration, profile)"""
    raw = text.encode() if isinstance(text, str) else bytes(text)
    cal, profile = OusterCalibration(), C.c_int(-1)
    _check(lib().lv_ouster_sensor_from_json(raw, len(raw), C.byref(cal), C.byref(profile)))
    return cal, profile.value


def bag_parse_ouster_packet(msg):
    """lv_bag_parse_ouster_packet on a serialised PacketMsg (bytes): the packet's bytes"""
    v = OusterPacketView()
    buf = C.create_string_buffer(bytes(msg), len(msg))
    _check(lib().lv_bag_parse_ouster_packet(buf, len(msg), C.byref(v)))
    off = v.data - C.addressof(buf) if v.bytes else 0
    return buf.raw[off:off + v.bytes]


def ouster_imu_packet(pkt):
    """lv_ouster_imu_packet on the 48 bytes of an IMU packet: an ImuSample"""
    raw = bytes(pkt)
    s = ImuSample()
    _check(lib().lv_ouster_imu_packet(raw, len(raw), C.byref(s)))
    return s


def ouster_to_points(packets, cal, profile=OUSTER_LEGACY):
    """msg2points of Ouster packets of a lidar UDP profile on the host (packets: their bytes): returns (xyz, time, intensity, range,
    slot) of the points, in slot order"""
    raw = np.ascontiguousarray(np.frombuffer(bytes(memoryview(packets)), np.uint8))
    k = len(raw) // ouster_packet_bytes(cal.pixels_per_column, profile)
    n = OUSTER_COLUMNS * cal.pixels_per_column * k
    out = (np.empty((n, 3), np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32), np.empty(n, np.int32))
    m = C.c_int64(0)
    _check(lib().lv_ouster_packets_to_points(raw.ctypes.data_as(C.c_void_p), len(raw), k, C.byref(cal), int(profile),
                                             *(a.ctypes.data_as(C.c_void_p) for a in out), C.byref(m)))
    return tuple(a[:m.value].copy() for a in out)


def init_state_host(params, q_imu=(0, 0, 0, 1)):
    """Localizator::init_IKFoM_state on the host (no GPU needed)."""
    x, P = np.zeros(STATE_LEN), np.zeros((DOF, DOF))
    q = np.ascontiguousarray(q_imu, dtype=np.float32)
    _check(lib().lv_init_state_host(C.byref(params), _f(q), _d(x), _d(P)))
    return x, P


def predict_host(params, x, P, acc, gyro, dt):
    """Localizator::propagate -> esekf::predict on the host (no GPU needed)."""
    x = np.array(x, dtype=np.float64).copy()
    P = np.array(P, dtype=np.float64).reshape(DOF, DOF).copy()
    acc = np.ascontiguousarray(acc, dtype=np.float64)
    gyro = np.ascontiguousarray(gyro, dtype=np.float64)
    _check(lib().lv_predict_host(C.byref(params), _d(acc), _d(gyro), float(dt), _d(x), _d(P)))
    return x, P


class Localizer:
    """One lv_handle: the Localizator + Mapper pair of one sequence on one GPU."""

    def __init__(self, params):
        self.L = lib()
        self.params = params
        self.h = C.c_void_p()
        _check(self.L.lv_create(C.byref(params), C.byref(self.h)))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.lv_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # Mapper
    def map_build(self, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        return _check(self.L.lv_map_build(self.h, _f(xyz), xyz.shape[0]))

    def map_add(self, xyz, downsample=True):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        return _check(self.L.lv_map_add(self.h, _f(xyz), xyz.shape[0], int(downsample)))

    def map_add_device(self, d_xyz, n, downsample=True):
        """Mapper::add from a device buffer; asynchronous (no host round trip)"""
        return _check(self.L.lv_map_add_device(self.h, C.c_void_p(d_xyz), int(n), int(downsample)))

    def propagate_device(self, acc, gyro, dt):
        """Localizator::propagate_to on the device: k IMU samples (k x 3, k x 3, k), one launch, the state stays in HBM"""
        acc = np.ascontiguousarray(acc, np.float64).reshape(-1, 3)
        gyro = np.ascontiguousarray(gyro, np.float64).reshape(-1, 3)
        dt = np.ascontiguousarray(dt, np.float64).reshape(-1)
        assert len(acc) == len(gyro) == len(dt)
        return _check(self.L.lv_propagate_device(self.h, _d(acc), _d(gyro), _d(dt), len(dt)))

    def map_add_sweep_device(self, d_xyz_lidar, n, downsample=True):
        """main.cpp:99-105 on the device: the LiDAR-frame sweep, transformed by the filter's current state, joins the map"""
        return _check(self.L.lv_map_add_sweep_device(self.h, C.c_void_p(d_xyz_lidar), int(n), int(downsample)))

    def map_add_last_sweep(self, downsample=True):
        return _check(self.L.lv_map_add_last_sweep(self.h, int(downsample)))

    def map_status(self):
        """synchronises; raises on LV_ERR_CAPACITY (device map out of table / arena space)"""
        return _check(self.L.lv_map_status(self.h))

    def map_size(self):
        return int(self.L.lv_map_size(self.h))

    def map_reserve(self, points):
        """grow the map now to a capacity of at least `points` points (asynchronous; no-op below the capacity)"""
        return _check(self.L.lv_map_reserve(self.h, int(points)))

    def map_set_growth(self, max_points):
        """let the map grow by itself before an add that may not fit, up to a capacity of max_points points (0: off)"""
        return _check(self.L.lv_map_set_growth(self.h, int(max_points)))

    def map_info(self):
        """capacity, usage (device counters) and growth of the map as a dict; synchronises"""
        out = MapInfo()
        _check(self.L.lv_map_info(self.h, C.byref(out)))
        return {k: getattr(out, k) for k, _ in MapInfo._fields_ if k != "pad_"}

    def map_points(self):
        n = self.map_size()
        out = np.zeros((max(n, 1), 3), np.float32)
        k = self.L.lv_map_points(self.h, _f(out), n)
        return out[:k]

    # operator boundary
    def measure_reduced(self, x, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        x = np.ascontiguousarray(x, dtype=np.float64)
        HTH, HTh, nm = np.zeros((12, 12)), np.zeros(12), C.c_int64(0)
        st = _check(self.L.lv_measure_reduced(self.h, _d(x), _f(xyz), xyz.shape[0], _d(HTH), _d(HTh), C.byref(nm)),
                    allow=(EMPTY_MAP,))
        return st, HTH, HTh, nm.value

    def measure(self, x, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        x = np.ascontiguousarray(x, dtype=np.float64)
        n = xyz.shape[0]
        hx, h, nm = np.zeros(12 * n), np.zeros(n), C.c_int64(0)
        st = _check(self.L.lv_measure(self.h, _d(x), _f(xyz), n, _d(hx), _d(h), C.byref(nm)), allow=(EMPTY_MAP,))
        k = nm.value
        return st, hx[:12 * k].reshape(12, k).T.copy(), h[:k].copy()

    def match_all(self, x, xyz):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
        x = np.ascontiguousarray(x, dtype=np.float64)
        n = xyz.shape[0]
        out = dict(valid=np.zeros(n, np.uint8), nn_idx=np.zeros((n, 5), np.int32), nn_sqd=np.zeros((n, 5), np.float32),
                   plane=np.zeros((n, 4), np.float32), dist=np.zeros(n, np.float32), g=np.zeros((n, 3), np.float32))
        st = _check(self.L.lv_match_all(self.h, _d(x), _f(xyz), n, out["valid"].ctypes.data_as(C.POINTER(C.c_uint8)),
                                        out["nn_idx"].ctypes.data_as(C.POINTER(C.c_int32)), _f(out["nn_sqd"]),
                                        _f(out["plane"]), _f(out["dist"]), _f(out["g"])), allow=(EMPTY_MAP,))
        out["status"] = st
        return out

    def last_neighbours(self, n):
        """map point ids (n x 5) of the neighbours the last evaluation handed to the plane fit"""
        out = np.zeros((n, 5), np.int32)
        _check(self.L.lv_last_neighbours(self.h, C.c_int64(n), out.ctypes.data_as(C.POINTER(C.c_int32))), allow=(EMPTY_MAP,))
        return out

    def prelocalize(self, d_xyz, n, radius, step, yaw_range, yaw_step, max_points, scores=False):
        """lv_prelocalize: search the window of positions and headings around the filter's state for the pose at which most of
        the n sweep points (device buffer, LiDAR frame) land in occupied map voxels, and move the state there.  Returns
        (status, result dict); with scores=True the dict holds every candidate's score as scores[k + K, i + I, j + I]."""
        prm = PrelocParams(radius, step, yaw_range, yaw_step, max_points, 0)
        res = PrelocResult()
        cnt = self.L.lv_preloc_count(C.byref(prm))
        buf = np.zeros(max(cnt, 1) if scores else 1, np.int32)
        st = _check(self.L.lv_prelocalize(self.h, C.c_void_p(d_xyz), int(n), C.byref(prm), C.byref(res),
                                          buf.ctypes.data_as(C.POINTER(C.c_int32)) if scores else None), allow=(EMPTY_MAP,))
        out = {k: getattr(res, k) for k, _ in PrelocResult._fields_ if k not in ("x", "pad_")}
        out["x"] = np.array(res.x[:])
        if scores and st == OK:
            I = int(np.floor(float(np.float32(radius)) / float(np.float32(step)) + 1e-9))
            out["scores"] = buf.reshape(-1, 2 * I + 1, 2 * I + 1)
        return st, out

    def prelocalize_global(self, d_xyz, n, radius, step, yaw_range, yaw_step, max_points):
        """lv_prelocalize_global: the same search, winner and effect as prelocalize, pruned by an exact upper bound, for windows
        of up to 2^40 candidates (a whole map).  Returns (status, result dict, stats dict)."""
        prm = PrelocParams(radius, step, yaw_range, yaw_step, max_points, 0)
        res, stats = PrelocResult(), PrelocStats()
        st = _check(self.L.lv_prelocalize_global(self.h, C.c_void_p(d_xyz), int(n), C.byref(prm), C.byref(res), C.byref(stats)),
                    allow=(EMPTY_MAP,))
        out = {k: getattr(res, k) for k, _ in PrelocResult._fields_ if k not in ("x", "pad_")}
        out["x"] = np.array(res.x[:])
        return st, out, {k: getattr(stats, k) for k, _ in PrelocStats._fields_ if k != "pad_"}

    def map_extent(self):
        """(lo, hi): the world-frame box of the occupied voxels' faces (m); raises on an empty map"""
        lo, hi = np.zeros(3), np.zeros(3)
        _check(self.L.lv_map_extent(self.h, _d(lo), _d(hi)))
        return lo, hi

    # Localizator
    def set_state(self, x, P):
        x = np.ascontiguousarray(x, dtype=np.float64)
        P = np.ascontiguousarray(P, dtype=np.float64)
        _check(self.L.lv_set_state(self.h, _d(x), _d(P)))

    def get_state(self):
        x, P = np.zeros(STATE_LEN), np.zeros((DOF, DOF))
        _check(self.L.lv_get_state(self.h, _d(x), _d(P)))
        return x, P

    def init_state(self, q_imu=(0, 0, 0, 1)):
        q = np.ascontiguousarray(q_imu, dtype=np.float32)
        _check(self.L.lv_init_state(self.h, _f(q)))

    def predict(self, acc, gyro, dt):
        acc = np.ascontiguousarray(acc, dtype=np.float64)
        gyro = np.ascontiguousarray(gyro, dtype=np.float64)
        _check(self.L.lv_predict(self.h, _d(acc), _d(gyro), float(dt)))

    def correct(self, xyz, time=0.0, raw_ptr=None, n=None):
        """Localizator::correct.  xyz: numpy (host) array, or raw_ptr/n for a pinned host buffer."""
        if raw_ptr is None:
            xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
            ptr, n = _f(xyz), xyz.shape[0]
        else:
            ptr = C.cast(raw_ptr, C.POINTER(C.c_float))
        logs = (IterLog * MAX_EVALS)()
        ne = C.c_int32(0)
        x, P = np.zeros(STATE_LEN), np.zeros((DOF, DOF))
        st = _check(self.L.lv_correct(self.h, ptr, n, float(time), logs, C.byref(ne), _d(x), _d(P)),
                    allow=(EMPTY_MAP, TOO_FEW_MATCHES))
        return st, x, P, _logs_to_py(logs, ne.value)

    def compensate(self, path, Xt2, xyz, t):
        """Compensator::compensate (deskew) on host buffers: returns the points in the LiDAR frame at t2"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        t = np.ascontiguousarray(t, np.float64)
        out = np.empty_like(xyz)
        arr = (State32 * len(path))(*path)
        _check(self.L.lv_compensate(self.h, arr, len(path), C.byref(Xt2), _f(xyz), _d(t), C.c_int64(xyz.shape[0]), _f(out)))
        return out

    def compensate_device(self, path, Xt2, d_xyz, d_t, n, d_out):
        arr = (State32 * len(path))(*path)
        return _check(self.L.lv_compensate_device(self.h, arr, len(path), C.byref(Xt2), C.c_void_p(d_xyz), C.c_void_p(d_t),
                                                  C.c_int64(n), C.c_void_p(d_out)))

    def temporal_downsample(self, xyz, rate, min_dist):
        """PointCloudProcessor::temporal_downsample: returns (kept points, their indices)"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        out, idx, n = np.empty_like(xyz), np.empty(xyz.shape[0], np.int32), C.c_int64(0)
        _check(self.L.lv_temporal_downsample(self.h, _f(xyz), C.c_int64(xyz.shape[0]), C.c_int32(rate), C.c_double(min_dist),
                                             _f(out), idx.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n)))
        return out[:n.value].copy(), idx[:n.value].copy()

    def voxelgrid_downsample(self, xyz, leaf):
        """Compensator::voxelgrid_downsample (pcl::VoxelGrid centroids)"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        out, n = np.empty_like(xyz), C.c_int64(0)
        _check(self.L.lv_voxelgrid_downsample(self.h, _f(xyz), C.c_int64(xyz.shape[0]), C.c_float(leaf), _f(out), C.byref(n)))
        return out[:n.value].copy()

    def voxelgrid_downsample_full(self, xyz, time, intensity, leaf):
        """Compensator::voxelgrid_downsample of full points (full_info::Point through pcl::VoxelGrid): returns (xyz, time, intensity,
        range) of the leaves: the xyz centroids, time 0, the mean intensity and the centroid's norm (on an overflow: the input's xyz,
        time and intensity, and each point's norm)"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        n = xyz.shape[0]
        ins = (np.ascontiguousarray(time, np.float64), np.ascontiguousarray(intensity, np.float32))
        assert all(a.shape == (n,) for a in ins)
        out = (np.empty_like(xyz), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32))
        m = C.c_int64(0)
        _check(self.L.lv_voxelgrid_downsample_full(self.h, *(a.ctypes.data_as(C.c_void_p) for a in (xyz,) + ins), C.c_int64(n), C.c_float(leaf),
                                                   *(a.ctypes.data_as(C.c_void_p) for a in out), C.byref(m)))
        return tuple(a[:m.value].copy() for a in out)

    def voxelgrid_downsample_device(self, d_xyz, n, leaf, d_out):
        m = C.c_int64(0)
        _check(self.L.lv_voxelgrid_downsample_device(self.h, C.c_void_p(d_xyz), C.c_int64(n), C.c_float(leaf), C.c_void_p(d_out),
                                                     C.byref(m)))
        return m.value

    def process_cloud_device(self, lidar, layout, d_data, data_bytes, n, header_stamp_us, stamp_beginning, offset_beginning,
                             full_rotation_time, downsample_rate, min_dist, d_xyz, d_time, d_intensity=None, d_range=None,
                             d_idx=None):
        """Accumulator::process on message bytes already in device memory (raw pointers); returns the points kept"""
        m = C.c_int64(0)
        _check(self.L.lv_process_cloud_device(self.h, LIDAR_TYPES[lidar], C.byref(layout), C.c_void_p(d_data), int(data_bytes), int(n),
                                              int(header_stamp_us), int(stamp_beginning), int(offset_beginning),
                                              float(full_rotation_time), int(downsample_rate), float(min_dist), C.c_void_p(d_xyz),
                                              C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx),
                                              C.byref(m)))
        return m.value

    def process_cloud(self, lidar, pts, header_stamp_us, stamp_beginning, offset_beginning, full_rotation_time, downsample_rate,
                      min_dist):
        """Accumulator::process on a numpy structured array (its buffer is the message's `data`): uploads it, returns
        (xyz, time, intensity, range, index in the message) of the kept points in time order"""
        pts = np.ascontiguousarray(pts)
        n = len(pts)
        out = (np.empty((n, 3), np.float32), np.empty(n, np.float64), np.empty(n, np.float32), np.empty(n, np.float32),
               np.empty(n, np.int32))
        bufs = [self.device_alloc(max(pts.nbytes, 1))] + [self.device_alloc(max(a.nbytes, 1)) for a in out]
        try:
            _check(self.L.lv_memcpy_h2d(self.h, bufs[0], pts.ctypes.data_as(C.c_void_p), pts.nbytes))
            m = self.process_cloud_device(lidar, cloud_layout(lidar, pts.dtype), bufs[0], pts.nbytes, n, header_stamp_us,
                                          stamp_beginning, offset_beginning, full_rotation_time, downsample_rate, min_dist, *bufs[1:])
            return tuple(self.download(d, a[:m]) for a, d in zip(out, bufs[1:]))
        finally:
            for d in bufs:
                self.device_free(d)

    def process_livox_device(self, d_data, data_bytes, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist, d_xyz, d_time,
                             d_intensity=None, d_range=None, d_idx=None):
        """Accumulator::process on the records of a Livox message already in device memory (raw pointers); returns the points kept"""
        m = C.c_int64(0)
        _check(self.L.lv_process_livox_device(self.h, C.c_void_p(d_data), int(data_bytes), int(n), C.c_uint64(timebase_ns), int(tag_reject_mask),
                                              int(downsample_rate), float(min_dist), C.c_void_p(d_xyz), C.c_void_p(d_time),
                                              C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx), C.byref(m)))
        return m.value

    def process_livox(self, records, timebase_ns, tag_reject_mask, downsample_rate, min_dist):
        """Accumulator::process on a Livox message's records (LIVOX_RECORD array): uploads them, returns (xyz, time, intensity, range,
        index in the message) of the kept points in time order"""
        raw = np.frombuffer(np.ascontiguousarray(records).tobytes(), np.uint8)
        n = len(raw) // 19
        out = (np.empty((n, 3), np.float32), np.empty(n, np.float64), np.empty(n, np.float32), np.empty(n, np.float32),
               np.empty(n, np.int32))
        bufs = [self.device_alloc(max(raw.nbytes, 1))] + [self.device_alloc(max(a.nbytes, 1)) for a in out]
        try:
            _check(self.L.lv_memcpy_h2d(self.h, bufs[0], raw.ctypes.data_as(C.c_void_p), raw.nbytes))
            m = self.process_livox_device(bufs[0], raw.nbytes, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist, *bufs[1:])
            return tuple(self.download(d, a[:m]) for a, d in zip(out, bufs[1:]))
        finally:
            for d in bufs:
                self.device_free(d)

    def process_velodyne_device(self, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_intensity=None,
                                d_range=None, d_idx=None):
        """Accumulator::process on the packets of a VelodyneScan already in device memory (raw pointers); returns the points kept"""
        m = C.c_int64(0)
        _check(self.L.lv_process_velodyne_device(self.h, C.c_void_p(d_packets), int(data_bytes), int(n_packets), C.byref(cal),
                                                 int(downsample_rate), float(min_dist), C.c_void_p(d_xyz), C.c_void_p(d_time),
                                                 C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx), C.byref(m)))
        return m.value

    def process_velodyne(self, packets, cal, downsample_rate, min_dist):
        """Accumulator::process on a VelodyneScan's packets (their bytes): uploads them, returns (xyz, time, intensity, range, slot)
        of the kept points in time order"""
        raw = np.frombuffer(bytes(memoryview(packets)), np.uint8)
        k = len(raw) // VELODYNE_PACKET
        n = VELODYNE_SLOTS * k
        out = (np.empty((n, 3), np.float32), np.empty(n, np.float64), np.empty(n, np.float32), np.empty(n, np.float32),
               np.empty(n, np.int32))
        bufs = [self.device_alloc(max(raw.nbytes, 1))] + [self.device_alloc(max(a.nbytes, 1)) for a in out]
        try:
            _check(self.L.lv_memcpy_h2d(self.h, bufs[0], raw.ctypes.data_as(C.c_void_p), raw.nbytes))
            m = self.process_velodyne_device(bufs[0], raw.nbytes, k, cal, downsample_rate, min_dist, *bufs[1:])
            return tuple(self.download(d, a[:m]) for a, d in zip(out, bufs[1:]))
        finally:
            for d in bufs:
                self.device_free(d)

    def process_ouster_device(self, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_intensity=None,
                              d_range=None, d_idx=None, profile=OUSTER_LEGACY):
        """Accumulator::process on Ouster packets of a lidar UDP profile already in device memory (raw pointers); returns the points
        kept"""
        m = C.c_int64(0)
        _check(self.L.lv_process_ouster_packets_device(self.h, C.c_void_p(d_packets), int(data_bytes), int(n_packets), C.byref(cal),
                                                       int(profile), int(downsample_rate), float(min_dist), C.c_void_p(d_xyz),
                                                       C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range),
                                                       C.c_void_p(d_idx), C.byref(m)))
        return m.value

    def process_ouster(self, packets, cal, downsample_rate, min_dist, profile=OUSTER_LEGACY):
        """Accumulator::process on Ouster packets of a lidar UDP profile (their bytes): uploads them, returns (xyz, time, intensity,
        range, slot) of the kept points in time order"""
        raw = np.frombuffer(bytes(memoryview(packets)), np.uint8)
        k = len(raw) // ouster_packet_bytes(cal.pixels_per_column, profile)
        n = OUSTER_COLUMNS * cal.pixels_per_column * k
        out = (np.empty((n, 3), np.float32), np.empty(n, np.float64), np.empty(n, np.float32), np.empty(n, np.float32),
               np.empty(n, np.int32))
        bufs = [self.device_alloc(max(raw.nbytes, 1))] + [self.device_alloc(max(a.nbytes, 1)) for a in out]
        try:
            _check(self.L.lv_memcpy_h2d(self.h, bufs[0], raw.ctypes.data_as(C.c_void_p), raw.nbytes))
            m = self.process_ouster_device(bufs[0], raw.nbytes, k, cal, downsample_rate, min_dist, *bufs[1:], profile=profile)
            return tuple(self.download(d, a[:m]) for a, d in zip(out, bufs[1:]))
        finally:
            for d in bufs:
                self.device_free(d)

    def download(self, d_ptr, out):
        """copy device memory into the contiguous numpy array `out` (its whole size); returns out"""
        if out.nbytes:
            _check(self.L.lv_memcpy_d2h(self.h, out.ctypes.data_as(C.c_void_p), C.c_void_p(d_ptr), out.nbytes))
        return out

    def correct_buffers(self):
        """preallocated outputs for correct_raw (benchmarks: keeps numpy / ctypes construction out of the timed call)"""
        return dict(logs=(IterLog * MAX_EVALS)(), ne=C.c_int32(0), x=np.zeros(STATE_LEN), P=np.zeros((DOF, DOF)))

    def correct_raw(self, raw_ptr, n, buf, time=0.0):
        """lv_correct on a host pointer, nothing else: returns the status; unpack `buf` with correct_unpack"""
        return self.L.lv_correct(self.h, C.cast(raw_ptr, C.POINTER(C.c_float)), n, float(time), buf["logs"],
                                 C.byref(buf["ne"]), _d(buf["x"]), _d(buf["P"]))

    @staticmethod
    def correct_unpack(buf):
        return buf["x"].copy(), buf["P"].copy(), _logs_to_py(buf["logs"], buf["ne"].value)

    def correct_device(self, d_ptr, n, time=0.0):
        return _check(self.L.lv_correct_device(self.h, d_ptr, n, float(time)), allow=(EMPTY_MAP,))

    # the tick without a host wait: counts live in device memory (int64 at d_n / d_n_out), nothing synchronises
    def process_cloud_device_async(self, lidar, layout, d_data, data_bytes, n, header_stamp_us, stamp_beginning, offset_beginning,
                                   full_rotation_time, downsample_rate, min_dist, d_xyz, d_time, d_n_out, d_intensity=None,
                                   d_range=None, d_idx=None):
        """lv_process_cloud_device with the count of kept points written to d_n_out"""
        return _check(self.L.lv_process_cloud_device_async(
            self.h, LIDAR_TYPES[lidar], C.byref(layout), C.c_void_p(d_data), int(data_bytes), int(n), int(header_stamp_us),
            int(stamp_beginning), int(offset_beginning), float(full_rotation_time), int(downsample_rate), float(min_dist),
            C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx),
            C.c_void_p(d_n_out)))

    def process_livox_device_async(self, d_data, data_bytes, n, timebase_ns, tag_reject_mask, downsample_rate, min_dist, d_xyz, d_time,
                                   d_n_out, d_intensity=None, d_range=None, d_idx=None):
        """lv_process_livox_device with the count of kept points written to d_n_out"""
        return _check(self.L.lv_process_livox_device_async(
            self.h, C.c_void_p(d_data), int(data_bytes), int(n), C.c_uint64(timebase_ns), int(tag_reject_mask), int(downsample_rate),
            float(min_dist), C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx),
            C.c_void_p(d_n_out)))

    def process_velodyne_device_async(self, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_n_out,
                                      d_intensity=None, d_range=None, d_idx=None):
        """lv_process_velodyne_device with the count of kept points written to d_n_out"""
        return _check(self.L.lv_process_velodyne_device_async(
            self.h, C.c_void_p(d_packets), int(data_bytes), int(n_packets), C.byref(cal), int(downsample_rate), float(min_dist),
            C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx),
            C.c_void_p(d_n_out)))

    def process_ouster_device_async(self, d_packets, data_bytes, n_packets, cal, downsample_rate, min_dist, d_xyz, d_time, d_n_out,
                                    d_intensity=None, d_range=None, d_idx=None, profile=OUSTER_LEGACY):
        """lv_process_ouster_packets_device with the count of kept points written to d_n_out"""
        return _check(self.L.lv_process_ouster_packets_device_async(
            self.h, C.c_void_p(d_packets), int(data_bytes), int(n_packets), C.byref(cal), int(profile), int(downsample_rate),
            float(min_dist), C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_range), C.c_void_p(d_idx),
            C.c_void_p(d_n_out)))

    def compensate_device_async(self, path, Xt2, d_xyz, d_t, d_n, n_max, d_out):
        """lv_compensate_device over the *d_n points"""
        arr = (State32 * len(path))(*path)
        return _check(self.L.lv_compensate_device_async(self.h, arr, len(path), C.byref(Xt2), C.c_void_p(d_xyz), C.c_void_p(d_t),
                                                        C.c_void_p(d_n), int(n_max), C.c_void_p(d_out)))

    def voxelgrid_downsample_device_async(self, d_xyz, d_n, n_max, leaf, d_out, d_n_out):
        """lv_voxelgrid_downsample_device over the *d_n points; the leaf count goes to d_n_out"""
        return _check(self.L.lv_voxelgrid_downsample_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_n), int(n_max), C.c_float(leaf),
                                                                  C.c_void_p(d_out), C.c_void_p(d_n_out)))

    def voxelgrid_downsample_full_async(self, d_xyz, d_time, d_intensity, d_n, n_max, leaf, d_out, d_time_out, d_intensity_out,
                                        d_range_out, d_n_out):
        """lv_voxelgrid_downsample_device_async of full points: the leaves' xyz, time 0, mean intensity and centroid norm (an output
        lane may be None)"""
        return _check(self.L.lv_voxelgrid_downsample_full_device_async(
            self.h, C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity), C.c_void_p(d_n), int(n_max),
            C.c_float(leaf), C.c_void_p(d_out), C.c_void_p(d_time_out), C.c_void_p(d_intensity_out), C.c_void_p(d_range_out),
            C.c_void_p(d_n_out)))

    def cloud_stamp_async(self, d_time, d_n, n_max, d_stamp_us):
        """the published cloud's header stamp (max of round(t * 1e6), uint64 microseconds) of the *d_n times into d_stamp_us"""
        return _check(self.L.lv_cloud_stamp_device_async(self.h, C.c_void_p(d_time), C.c_void_p(d_n), int(n_max), C.c_void_p(d_stamp_us)))

    def correct_device_async(self, d_ptr, d_n, n_max, min_points, time=0.0):
        """Localizator::correct on the *d_n points behind main.cpp:81's MAX_POINTS2MATCH gate; LV_EMPTY_MAP while the host knows the
        map is empty, else LV_OK (the update's own status is fetched later, e.g. by last_logs)"""
        return _check(self.L.lv_correct_device_async(self.h, C.c_void_p(d_ptr), C.c_void_p(d_n), int(n_max), int(min_points),
                                                     float(time)), allow=(EMPTY_MAP,))

    def sweep_to_world_async(self, d_xyz_lidar, d_n, n_max, d_xyz_world, d_n_out):
        """Xt2 * Xt2.I_Rt_L() * the *d_n points with the filter state on the device; the count goes to d_n_out (0 on a gated tick)"""
        return _check(self.L.lv_sweep_to_world_device_async(self.h, C.c_void_p(d_xyz_lidar), C.c_void_p(d_n), int(n_max),
                                                            C.c_void_p(d_xyz_world), C.c_void_p(d_n_out)))

    def map_add_device_async(self, d_xyz, d_n, n_max, downsample=True):
        """Mapper::add of the *d_n world-frame points of a device buffer (built un-downsampled on an empty map)"""
        return _check(self.L.lv_map_add_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_n), int(n_max), int(downsample)))

    def async_status(self):
        """the deferred errors of the async calls (cleared by the call): returns (status, lv_last_error text); synchronises"""
        st = self.L.lv_async_status(self.h)
        return st, (self.L.lv_last_error().decode() if st != OK else "")

    # the LiDAR buffer (Accumulator::BUFFER_L) in HBM: raw device pointers, counts as int64 in device memory
    def lidar_reserve(self, capacity):
        """size the buffer for `capacity` points (the live points stay, in order); synchronises"""
        return _check(self.L.lv_lidar_reserve(self.h, int(capacity)))

    def lidar_push_async(self, d_xyz, d_time, d_n, n_max):
        """Accumulator::receive_lidar's push of the *d_n processed points (e.g. lv_process_cloud_device_async's output)"""
        return _check(self.L.lv_lidar_push_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_n), int(n_max)))

    def lidar_reserve_full(self, capacity):
        """size the buffer for `capacity` full points (xyz, time, intensity, range); synchronises"""
        return _check(self.L.lv_lidar_reserve_full(self.h, int(capacity)))

    def lidar_push_full_async(self, d_xyz, d_time, d_intensity, d_range, d_n, n_max):
        """lidar_push_async with the points' intensity and range (a buffer reserved with lidar_reserve_full)"""
        return _check(self.L.lv_lidar_push_full_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity),
                                                             C.c_void_p(d_range), C.c_void_p(d_n), int(n_max)))

    def lidar_reserve_merge(self, overlap_points):
        """room for `overlap_points` buffered points that one merge may move; synchronises"""
        return _check(self.L.lv_lidar_reserve_merge(self.h, int(overlap_points)))

    def lidar_merge_async(self, d_xyz, d_time, d_n, n_max, T=None):
        """lv_lidar_merge_device_async: the *d_n points by time into the buffer, through T (12 floats: R row-major, then t) from the
        sensor's frame into the primary LiDAR's, or unchanged (T None)"""
        return _check(self.L.lv_lidar_merge_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_n), int(n_max),
                                                         _transform12(T)))

    def lidar_merge_full_async(self, d_xyz, d_time, d_intensity, d_range, d_n, n_max, T=None):
        """lidar_merge_async with the points' intensity and range (a buffer reserved with lidar_reserve_full)"""
        return _check(self.L.lv_lidar_merge_full_device_async(self.h, C.c_void_p(d_xyz), C.c_void_p(d_time), C.c_void_p(d_intensity),
                                                              C.c_void_p(d_range), C.c_void_p(d_n), int(n_max), _transform12(T)))

    def lidar_get_points_full_async(self, t1, t2, d_xyz, d_time, d_intensity, d_range, n_max, d_n_out):
        """lidar_get_points_async with the window's intensity and range"""
        return _check(self.L.lv_lidar_get_points_full_device_async(self.h, float(t1), float(t2), C.c_void_p(d_xyz), C.c_void_p(d_time),
                                                                   C.c_void_p(d_intensity), C.c_void_p(d_range), int(n_max),
                                                                   C.c_void_p(d_n_out)))

    def lidar_get_points_async(self, t1, t2, d_xyz, d_time, n_max, d_n_out):
        """Accumulator::get_points(t1, t2) into device buffers of n_max points; the count goes to d_n_out"""
        return _check(self.L.lv_lidar_get_points_device_async(self.h, float(t1), float(t2), C.c_void_p(d_xyz), C.c_void_p(d_time),
                                                              int(n_max), C.c_void_p(d_n_out)))

    def lidar_get_points(self, t1, t2, d_xyz, d_time, n_max):
        """the same, synchronising: returns the count (raises on a window above n_max)"""
        n = C.c_int64(0)
        _check(self.L.lv_lidar_get_points_device(self.h, float(t1), float(t2), C.c_void_p(d_xyz), C.c_void_p(d_time), int(n_max),
                                                 C.byref(n)))
        return n.value

    def lidar_clear_async(self, t):
        """Accumulator::clear_lidar(t)"""
        return _check(self.L.lv_lidar_clear_async(self.h, float(t)))

    def lidar_info(self):
        """points, capacity, oldest_time, newest_time of the buffer as a dict; synchronises"""
        out = LidarInfo()
        _check(self.L.lv_lidar_info(self.h, C.byref(out)))
        return {k: getattr(out, k) for k, _ in LidarInfo._fields_}

    def last_time_updated(self):
        return float(self.L.lv_last_time_updated(self.h))

    def result_bytes(self):
        return int(self.L.lv_result_bytes())

    def last_logs(self):
        logs = (IterLog * MAX_EVALS)()
        ne = C.c_int32(0)
        st = _check(self.L.lv_last_logs(self.h, logs, C.byref(ne)), allow=(TOO_FEW_MATCHES, TOO_FEW_POINTS, EMPTY_MAP))
        return st, _logs_to_py(logs, ne.value)

    # utilities
    def device_alloc(self, nbytes):
        p = self.L.lv_device_alloc(self.h, nbytes)
        if not p:
            raise RuntimeError("lv_device_alloc failed")
        return p

    def device_free(self, p):
        self.L.lv_device_free(self.h, p)

    def upload(self, arr):
        arr = np.ascontiguousarray(arr)
        p = self.device_alloc(arr.nbytes)
        _check(self.L.lv_memcpy_h2d(self.h, p, arr.ctypes.data_as(C.c_void_p), arr.nbytes))
        return p

    def synchronize(self):
        _check(self.L.lv_synchronize(self.h))

    def profile_enable(self, on=True):
        _check(self.L.lv_profile_enable(self.h, int(on)))

    def profile(self, reset=True):
        p = Profile()
        _check(self.L.lv_profile_get(self.h, C.byref(p), int(reset)))
        return {k: getattr(p, k) for k, _ in Profile._fields_}

    def flush_l2(self):
        _check(self.L.lv_flush_l2(self.h))


class PinnedBuffer:
    """Pinned host memory (lv_host_alloc) viewed as a numpy float32 array."""

    def __init__(self, shape):
        self.L = lib()
        n = int(np.prod(shape))
        self.ptr = self.L.lv_host_alloc(n * 4)
        if not self.ptr:
            raise RuntimeError("lv_host_alloc failed (no CUDA device?)")
        self.array = np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_float)), shape=(n,)).reshape(shape)

    def free(self):
        if self.ptr:
            self.L.lv_host_free(self.ptr)
            self.ptr = None


class SynthWorld:
    """Seeded synthetic world + LiDAR ray caster (liblv_synth.so, limo-velo_b200/host/lv_synth.cpp)."""

    def __init__(self, seed, m):
        self.L = synth_lib()
        self.w = self.L.lv_synth_world_create(int(seed), int(m))
        if not self.w:
            raise RuntimeError("lv_synth_world_create failed")
        self.m = int(m)

    def __del__(self):
        try:
            if self.w:
                self.L.lv_synth_world_destroy(self.w)
                self.w = None
        except Exception:
            pass

    def map(self):
        out = np.zeros((self.m, 3), np.float32)
        n = self.L.lv_synth_world_map(self.w, _f(out), self.m)
        return out[:n]

    def extent(self):
        return float(self.L.lv_synth_world_extent(self.w))

    def pose(self, s, params):
        x = np.zeros(STATE_LEN)
        self.L.lv_synth_pose(self.w, float(s), C.byref(params), _d(x))
        return x

    def sweep(self, x, rings=64, azimuths=1024, elev=(-24.8, 2.0), min_dist=4.0, range_sigma=0.02, seed=0, out=None):
        x = np.ascontiguousarray(x, dtype=np.float64)
        if out is None:
            out = np.zeros((rings * azimuths, 3), np.float32)
        n = self.L.lv_synth_sweep(self.w, _d(x), rings, azimuths, elev[0], elev[1], min_dist, range_sigma, int(seed),
                                  _f(out))
        assert n == rings * azimuths
        return out
