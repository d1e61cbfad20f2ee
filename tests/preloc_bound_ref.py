"""lv_prelocalize_global's cell bound restated in numpy, and calls into its host build (tests/cpu_shim/preloc.cpp).

The restatement takes the voxel code of tests/preloc_ref.py: for each cell it forms every scored point's world point at the
cell's four corner candidates (the offsets a u + b v in fp64, rounded to fp32, fadd(F.t, o), fadd(row, t)), takes the
per-axis minimum and maximum of their voxel coordinates as the point's voxel box, and counts the points whose box holds an
occupied voxel, exactly (a summed-volume table over the occupied voxels).  It does not use the header's route (the corner
offsets' range first, then one fadd per end), so equal results also say that the route is monotone as DESIGN.md §5e argues."""
import ctypes as C

import numpy as np

import preloc_ref as R
import shim_binding

f32 = np.float32


class Occupancy:
    """the occupied voxels of a map (biased voxel coordinates) as a summed-volume table: exact box counts"""

    def __init__(self, map_xyz, ds, k):
        keys = R.occupancy(map_xyz, ds, k)
        v = np.stack([keys & 0x1FFFFF, (keys >> 21) & 0x1FFFFF, (keys >> 42) & 0x1FFFFF], axis=1).astype(np.int64)
        self.keys = keys
        self.lo = v.min(axis=0)
        self.hi = v.max(axis=0)
        dims = self.hi - self.lo + 1
        grid = np.zeros(dims + 1, np.int32)             # a zero plane in front of each axis
        rel = v - self.lo + 1
        grid[rel[:, 0], rel[:, 1], rel[:, 2]] = 1
        self.sat = grid.cumsum(0).cumsum(1).cumsum(2)

    def count(self, lo, hi):
        """occupied voxels in the boxes [lo, hi] (n x 3, inclusive)"""
        a = np.clip(np.asarray(lo, np.int64) - self.lo, -1, self.hi - self.lo + 1)
        b = np.clip(np.asarray(hi, np.int64) - self.lo, -1, self.hi - self.lo)
        a = np.maximum(a, 0)
        empty = np.any(b < a, axis=1)
        b = np.maximum(b, a - 1)
        S = self.sat
        x0, y0, z0 = a[:, 0], a[:, 1], a[:, 2]
        x1, y1, z1 = b[:, 0] + 1, b[:, 1] + 1, b[:, 2] + 1
        c = (S[x1, y1, z1] - S[x0, y1, z1] - S[x1, y0, z1] - S[x1, y1, z0]
             + S[x0, y0, z1] + S[x0, y1, z0] + S[x1, y0, z0] - S[x0, y0, z0])
        return np.where(empty, 0, c)


def cell_range(cell, I):
    """(i0, i1, j0, j1) of a cell (h, l, ci, cj), clipped at the window's edge"""
    _, l, ci, cj = cell
    W, s = 2 * I + 1, 1 << l
    return ci * s - I, min((ci + 1) * s, W) - 1 - I, cj * s - I, min((cj + 1) * s, W) - 1 - I


class Scene:
    """one base state, sweep subset and map: frames, rows and occupancy computed once"""

    def __init__(self, x, xyz, map_xyz, ds, voxel_size, step, yaw_step, I, K, S):
        self.x, self.ds, self.step, self.I, self.K, self.S = x, ds, step, I, K, S
        self.k = R.voxel_k(ds, voxel_size)
        self.occ = Occupancy(map_xyz, ds, self.k)
        self.g, self.u, self.v = R.axes(x)
        p = np.asarray(xyz, np.float32)[R.subset(len(xyz), S)]
        self.rows, self.t = [], []
        for h in range(2 * K + 1):
            Rm, t = R.lidar_to_world(R.rotate_state(x, self.g, float(h - K) * float(f32(yaw_step))))
            self.rows.append(np.stack([R.dot3f(Rm[r, 0], Rm[r, 1], Rm[r, 2], p[:, 0], p[:, 1], p[:, 2]) for r in range(3)], axis=1))
            self.t.append(t)

    def world(self, h, i, j):
        """the S world points of candidate (h - K, i, j)"""
        o = np.array(R.offset64(self.u, self.v, float(i) * float(f32(self.step)), float(j) * float(f32(self.step))),
                     np.float64).astype(np.float32)
        return self.rows[h] + (self.t[h] + o)

    def bound(self, cell):
        """points whose voxel box over the cell holds an occupied voxel (the coordinates here are far below 1e9)"""
        h = cell[0]
        i0, i1, j0, j1 = cell_range(cell, self.I)
        vox = np.stack([R.voxels(self.world(h, i, j), self.ds, self.k) for i in (i0, i1) for j in (j0, j1)])
        return int((self.occ.count(vox.min(axis=0), vox.max(axis=0)) > 0).sum())

    def exact_max(self, cell):
        """the highest exact score over the cell's candidates (preloc_ref's score: occupied voxel, stored coordinates)"""
        h = cell[0]
        i0, i1, j0, j1 = cell_range(cell, self.I)
        best = 0
        for i in range(i0, i1 + 1):
            for j in range(j0, j1 + 1):
                w = self.world(h, i, j)
                hit = np.isin(R.keys(R.voxels(w, self.ds, self.k)), self.occ.keys) & R.stored(w)
                best = max(best, int(hit.sum()))
        return best


# ---- the host build of csrc/lv_preloc_bound.h -------------------------------------------------------------------------------
def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def host_bounds(x, xyz, map_xyz, ds, voxel_size, step, yaw_step, I, K, S, cells):
    x = np.ascontiguousarray(x, np.float64)
    xyz = np.ascontiguousarray(xyz, np.float32)
    mp = np.ascontiguousarray(map_xyz, np.float32)
    cells = np.ascontiguousarray(cells, np.int32).reshape(-1, 4)
    out = np.zeros(len(cells), np.int32)
    L = shim_binding.lib()
    st = L.shim_pg_bounds(x.ctypes.data_as(C.POINTER(C.c_double)), _fp(xyz), len(xyz), _fp(mp), len(mp), ds, voxel_size, step,
                          yaw_step, I, K, S, cells.ctypes.data_as(C.POINTER(C.c_int32)), len(cells),
                          out.ctypes.data_as(C.POINTER(C.c_int32)))
    assert st == 0
    return out


STATS = ("candidates", "cells_bounded", "candidates_scored", "probes", "launches")


def host_search(x, xyz, map_xyz, ds, voxel_size, radius, step, yaw_range, yaw_step, max_points, prune=True):
    """(winner's linear index, its score, stats dict) of the host build"""
    x = np.ascontiguousarray(x, np.float64)
    xyz = np.ascontiguousarray(xyz, np.float32)
    mp = np.ascontiguousarray(map_xyz, np.float32)
    best = np.zeros(3, np.int64)
    stats = np.zeros(5, np.int64)
    L = shim_binding.lib()
    st = L.shim_pg_search(x.ctypes.data_as(C.POINTER(C.c_double)), _fp(xyz), len(xyz), _fp(mp), len(mp), ds, voxel_size, radius,
                          step, yaw_range, yaw_step, max_points, int(prune), best.ctypes.data_as(C.POINTER(C.c_int64)),
                          stats.ctypes.data_as(C.POINTER(C.c_int64)))
    assert st == 0
    return int(best[2]), int(best[0]), dict(zip(STATS, (int(s) for s in stats)))


def host_extent(map_xyz, ds, voxel_size):
    """(lo, hi) biased voxel coordinates of the occupied voxels and the bitmap levels (m0, M) of the host build"""
    mp = np.ascontiguousarray(map_xyz, np.float32)
    ext = np.zeros(6, np.uint32)
    lev = np.zeros(2, np.int32)
    L = shim_binding.lib()
    assert L.shim_pg_extent(_fp(mp), len(mp), ds, voxel_size, ext.ctypes.data_as(C.POINTER(C.c_uint32)),
                            lev.ctypes.data_as(C.POINTER(C.c_int32))) == 0
    return ext[:3].astype(np.int64), ext[3:].astype(np.int64), (int(lev[0]), int(lev[1]))
