"""ctypes binding of tests/cpu_shim/liblv_cpushim.so (TEST-ONLY host build of the product headers): the map, search and
filter (shim.cpp), the LiDAR buffer and its time-ordered merge (lidar_ring.cpp), the start-pose searches (preloc.cpp) and the buffer and event owners over
a fake CUDA runtime (buffers.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_DIR = os.path.join(_HERE, "cpu_shim")


class ShimParams(C.Structure):
    _fields_ = [("max_iter", C.c_int32), ("estimate_extrinsics", C.c_int32), ("max_dist_plane", C.c_double),
                ("planes_threshold", C.c_float), ("voxel_size", C.c_float), ("R", C.c_double), ("D", C.c_double),
                ("limits", C.c_double * 23)]


class IterLog(C.Structure):
    _fields_ = [("n_matches", C.c_int64), ("converged", C.c_int32), ("degenerate", C.c_int32),
                ("HTH", C.c_double * 144), ("HTh", C.c_double * 12), ("dx", C.c_double * 23),
                ("x_after", C.c_double * 26)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", _DIR])
        L = C.CDLL(os.path.join(_DIR, "liblv_cpushim.so"))
        L.shim_map_create.restype = C.c_void_p
        L.shim_map_create.argtypes = [C.POINTER(C.c_float), C.c_int64, C.c_float, C.c_double]
        L.shim_map_create_cap.restype = C.c_void_p
        L.shim_map_create_cap.argtypes = [C.POINTER(C.c_float), C.c_int64, C.c_int64, C.c_float]
        L.shim_map_destroy.argtypes = [C.c_void_p]
        L.shim_map_add.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int64, C.c_int]
        L.shim_map_size.argtypes = [C.c_void_p]
        L.shim_map_size.restype = C.c_int64
        L.shim_map_error.argtypes = [C.c_void_p]
        L.shim_map_error.restype = C.c_uint32
        L.shim_map_points.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int64]
        L.shim_map_points.restype = C.c_int64
        L.shim_map_check.argtypes = [C.c_void_p]
        L.shim_map_dims.argtypes = [C.c_void_p] * 3
        L.shim_map_dump.argtypes = [C.c_void_p] * 6
        L.shim_map_grow.argtypes = [C.c_void_p, C.c_int64]
        L.shim_map_grow.restype = None
        L.shim_map_counter.argtypes = [C.c_void_p, C.c_int]
        L.shim_map_counter.restype = C.c_uint32
        assert L.shim_sizeof_iterlog() == C.sizeof(IterLog)

        vp, i64, f, dp, fp, i32p = C.c_void_p, C.c_int64, C.c_float, C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int32)
        L.shim_lidar_create.restype = vp
        L.shim_lidar_create.argtypes = [i64, C.c_int]
        L.shim_lidar_destroy.argtypes = [vp]
        L.shim_lidar_destroy.restype = None
        L.shim_lidar_size.argtypes = [vp]
        L.shim_lidar_size.restype = i64
        L.shim_lidar_content.argtypes = [vp, dp]
        L.shim_lidar_content.restype = None
        L.shim_lidar_reserve.argtypes = [vp, i64, C.c_int]
        L.shim_lidar_push.argtypes = [vp, fp, dp, fp, fp, i64]
        L.shim_lidar_get.argtypes = [vp, C.c_double, C.c_double, fp, dp, fp, fp, i64]
        L.shim_lidar_get.restype = i64
        L.shim_lidar_clear.argtypes = [vp, C.c_double]
        L.shim_lidar_clear.restype = None
        L.shim_lidar_content_full.argtypes = [vp, fp, dp, fp, fp]
        L.shim_lidar_content_full.restype = None
        L.shim_lidar_merge.argtypes = [vp, fp, dp, fp, fp, i64, fp, i64]

        L.shim_preloc_scores.argtypes = [dp, fp, i64, fp, i64, f, f, f, f, f, f, C.c_int32, i32p, fp, fp]
        L.shim_preloc_scores.restype = i64
        L.shim_preloc_candidate.argtypes = [dp, f, f, C.c_int32, C.c_int32, C.c_int32, dp]
        L.shim_preloc_candidate.restype = None
        L.shim_preloc_axes.argtypes = [dp, dp]
        L.shim_preloc_axes.restype = None
        L.shim_pg_bounds.argtypes = [dp, fp, i64, fp, i64, f, f, f, f, i64, i64, i64, i32p, i64, i32p]
        L.shim_pg_search.argtypes = [dp, fp, i64, fp, i64, f, f, f, f, f, f, C.c_int32, C.c_int, C.POINTER(i64), C.POINTER(i64)]
        L.shim_pg_extent.argtypes = [fp, i64, f, f, C.POINTER(C.c_uint32), i32p]
        L.shim_pg_top_level.argtypes = [i64, i64]

        L.shim_manifold.argtypes = [vp, vp, vp, C.c_int]
        L.shim_manifold.restype = None
        L.shim_buf_fail_at.argtypes = [i64]
        L.shim_buf_fail_at.restype = None
        L.shim_buf_counts.argtypes = [C.POINTER(i64)]
        L.shim_buf_counts.restype = None
        L.shim_buf_new.argtypes = [C.c_int]
        L.shim_buf_new.restype = vp
        L.shim_buf_move_new.argtypes = [vp]
        L.shim_buf_move_new.restype = vp
        L.shim_buf_move_assign.argtypes = [vp, vp]
        L.shim_buf_move_assign.restype = None
        L.shim_buf_reserve.argtypes = [vp, i64]
        L.shim_buf_size.argtypes = [vp]
        L.shim_buf_size.restype = i64
        L.shim_buf_ptr.argtypes = [vp]
        L.shim_buf_ptr.restype = C.c_size_t
        for fn in (L.shim_buf_reset, L.shim_buf_delete, L.shim_event_delete):
            fn.argtypes = [vp]
            fn.restype = None
        L.shim_event_new.restype = vp
        L.shim_event_create.argtypes = [vp]
        L.shim_event_handle.argtypes = [vp]
        L.shim_event_handle.restype = C.c_size_t
        _lib = L
    return _lib


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _d(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def make_params(oprm, voxel_size=0.5):
    """from an oracle Params struct"""
    p = ShimParams()
    p.max_iter = oprm.max_num_iters
    p.estimate_extrinsics = oprm.estimate_extrinsics
    p.max_dist_plane = oprm.max_dist_plane
    p.planes_threshold = oprm.planes_threshold
    p.voxel_size = voxel_size
    p.R = oprm.lidar_noise
    p.D = oprm.degeneracy_threshold
    for i in range(23):
        p.limits[i] = oprm.limits[i]
    return p


class ShimMap:
    def __init__(self, xyz, cell=0.5, max_dist=2.0, capacity=0):
        """capacity: map points to size the tables for (default: the build); isolated points need 27 table slots each"""
        self.L = lib()
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        self.k = min(3, max(1, int(np.floor(float(np.float32(cell)) / float(np.float32(0.2)) + 0.5))))   # map_alloc's k
        self.h = self.L.shim_map_create_cap(_f(xyz), xyz.shape[0], int(capacity), C.c_float(cell))

    def __del__(self):
        try:
            self.L.shim_map_destroy(C.c_void_p(self.h))
        except Exception:
            pass

    def add(self, xyz, downsample=True):
        """Mapper::add on an existing map (KD_TREE::Add_Points), through the product's map_merge_run / dilate / halo"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        self.L.shim_map_add(C.c_void_p(self.h), _f(xyz), xyz.shape[0], int(downsample))

    def size(self):
        return int(self.L.shim_map_size(C.c_void_p(self.h)))

    def error(self):
        return int(self.L.shim_map_error(C.c_void_p(self.h)))

    def points(self):
        n = self.size()
        out = np.zeros((max(n, 1), 3), np.float32)
        k = self.L.shim_map_points(C.c_void_p(self.h), _f(out), n)
        assert k == n
        return out[:n]

    def check(self):
        """0 when every halo bucket equals the concatenation of its 27 own extents, flags are clear, blocks are marked"""
        return int(self.L.shim_map_check(C.c_void_p(self.h)))

    def dump(self):
        """the layout as it stands: map_ref.Dump of both tables, arena[0, arena_top), counters and the last add's lists"""
        import map_ref
        dims, ctr = np.zeros(4, np.uint32), np.zeros(16, np.uint32)
        self.L.shim_map_dims(C.c_void_p(self.h), dims.ctypes.data_as(C.c_void_p), ctr.ctypes.data_as(C.c_void_p))
        slots, bslots, top, list_cap = (int(v) for v in dims)
        table, btable = np.zeros((slots, 8), np.uint32), np.zeros((bslots, 4), np.uint32)
        arena = np.zeros((max(top, 1), 4), np.uint32)
        touched = np.zeros(max(1, min(int(ctr[map_ref.CTR_TOUCHED]), list_cap)), np.uint32)
        dirty = np.zeros(max(1, min(int(ctr[map_ref.CTR_DIRTY]), list_cap)), np.uint32)
        self.L.shim_map_dump(C.c_void_p(self.h), *(a.ctypes.data_as(C.c_void_p) for a in (table, btable, arena, touched, dirty)))
        return map_ref.Dump(table, btable, arena[:top], ctr, touched[:min(int(ctr[map_ref.CTR_TOUCHED]), list_cap)],
                            dirty[:min(int(ctr[map_ref.CTR_DIRTY]), list_cap)], self.k)

    def match_all(self, x, prm, xyz, rows=False):
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        x = np.ascontiguousarray(x, np.float64)
        n = xyz.shape[0]
        out = dict(valid=np.zeros(n, np.uint8), nn_idx=np.zeros((n, 5), np.int32), nn_sqd=np.zeros((n, 5), np.float32),
                   plane=np.zeros((n, 4), np.float32), dist=np.zeros(n, np.float32), g=np.zeros((n, 3), np.float32),
                   rows=np.zeros((n, 13), np.float64))
        self.L.shim_match_all(C.c_void_p(self.h), _d(x), C.byref(prm), _f(xyz), C.c_int64(n),
                              out["valid"].ctypes.data_as(C.c_void_p), out["nn_idx"].ctypes.data_as(C.c_void_p),
                              _f(out["nn_sqd"]), _f(out["plane"]), _f(out["dist"]), _f(out["g"]), _d(out["rows"]))
        return out

    def query_stats(self, x, xyz, max_dist=2.0):
        """per query: level (0 settled at level 0, 1 home bucket but not certified, 2 no level-0 slot) and home bucket size"""
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        n = xyz.shape[0]
        level, scanned = np.zeros(n, np.int32), np.zeros(n, np.int32)
        self.L.shim_query_stats(C.c_void_p(self.h), _d(np.ascontiguousarray(x, np.float64)), _f(xyz), C.c_int64(n),
                                C.c_double(max_dist), level.ctypes.data_as(C.c_void_p), scanned.ctypes.data_as(C.c_void_p))
        return level, scanned

    def reuse_check(self, x0, x1, xyz, max_dist=2.0):
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        n = xyz.shape[0]
        reused, same = np.zeros(n, np.uint8), np.zeros(n, np.uint8)
        self.L.shim_reuse_check(C.c_void_p(self.h), _d(np.ascontiguousarray(x0, np.float64)),
                                _d(np.ascontiguousarray(x1, np.float64)), C.c_double(max_dist), _f(xyz), C.c_int64(n),
                                reused.ctypes.data_as(C.c_void_p), same.ctypes.data_as(C.c_void_p))
        return reused.astype(bool), same.astype(bool)

    def update(self, x, P, prm, xyz):
        xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
        x = np.array(x, np.float64).copy()
        P = np.array(P, np.float64).reshape(23, 23).copy()
        logs = (IterLog * 8)()
        ne = C.c_int32(0)
        st = self.L.shim_update(C.c_void_p(self.h), _d(x), _d(P), C.byref(prm), _f(xyz), C.c_int64(xyz.shape[0]), logs,
                                C.byref(ne))
        out = []
        for i in range(ne.value):
            lg = logs[i]
            out.append(dict(n_matches=int(lg.n_matches), converged=int(lg.converged), degenerate=int(lg.degenerate),
                            HTH=np.array(lg.HTH[:]).reshape(12, 12), HTh=np.array(lg.HTh[:]), dx=np.array(lg.dx[:]),
                            x_after=np.array(lg.x_after[:])))
        return st, x, P, out


def step(x_prop, P_prop, x_cur, prm, HTH, HTh, nm, it, t_in):
    L = lib()
    a = lambda v: np.ascontiguousarray(v, np.float64)
    x_prop, P_prop, x_cur, HTH, HTh = a(x_prop), a(P_prop), a(x_cur), a(HTH), a(HTh)
    dx, x_new, P_out, done = np.zeros(23), np.zeros(26), np.zeros((23, 23)), C.c_int32(0)
    st = L.shim_step(_d(x_prop), _d(P_prop), _d(x_cur), C.byref(prm), _d(HTH), _d(HTh), C.c_int64(nm), C.c_int(it),
                     C.c_int(t_in), _d(dx), _d(x_new), _d(P_out), C.byref(done))
    return st, dx, x_new, P_out, done.value


def boxplus(x, d):
    x = np.array(x, np.float64).copy()
    lib().shim_boxplus(_d(x), _d(np.ascontiguousarray(d, np.float64)))
    return x


def boxminus(x, y):
    d = np.zeros(23)
    lib().shim_boxminus(_d(np.ascontiguousarray(x, np.float64)), _d(np.ascontiguousarray(y, np.float64)), _d(d))
    return d


def manifold(ops, rows):
    """tests/gpu_shim_binding.manifold on the host build: the lv_manifold.h functions over rows (manifold_ops.h)"""
    ops = np.ascontiguousarray(ops, np.int32)
    rows = np.ascontiguousarray(rows, np.float64).reshape(len(ops), 64)
    out = np.zeros((len(ops), 32))
    lib().shim_manifold(ops.ctypes.data, rows.ctypes.data, out.ctypes.data, len(ops))
    return out


def plane_fit(pts5, thr):
    pts5 = np.ascontiguousarray(pts5, np.float32).reshape(5, 3)
    abcd = np.zeros(4, np.float32)
    ok = C.c_int(0)
    lib().shim_plane_fit(_f(pts5), C.c_float(thr), _f(abcd), C.byref(ok))
    return abcd, bool(ok.value)


def fit_sets(q, g, ids, x, thr, est=True, L=None):
    """the per-set arithmetic of the fit kernel on n given sets (q: n x 5 x 3, g: n x 3, ids: n x 5): the tie order, the fit,
    the distance and the row.  L: this module's library (host build) or gpu_shim_binding's (the device)."""
    q = np.ascontiguousarray(q, np.float32).reshape(-1, 15)
    n = q.shape[0]
    g = np.ascontiguousarray(g, np.float32).reshape(n, 3)
    ids = np.ascontiguousarray(ids, np.int32).reshape(n, 5)
    out = dict(ids=np.zeros((n, 5), np.int32), plane=np.zeros((n, 4), np.float32), ok=np.zeros(n, np.int32),
               dist=np.zeros(n, np.float32), rows=np.zeros((n, 13)))
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    fn = lib().shim_fit_sets if L is None else L.gs_fit_sets
    rc = fn(vp(q), vp(g), vp(ids), vp(np.ascontiguousarray(x, np.float64)), C.c_float(thr), int(est), int(n), vp(out["ids"]),
            vp(out["plane"]), vp(out["ok"]), vp(out["dist"]), vp(out["rows"]))
    assert L is None or rc == 0, "CUDA error %d" % rc
    return out
