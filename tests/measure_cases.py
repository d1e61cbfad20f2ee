"""Cases and bars for the rows of H / h and their normal equations (tests/test_measure_mp.py, tests/test_gpu_measure.py).

Row bars.  The product's world point and frame are fp32 (lv_point_math.h, as in the reference's State casts), the rest of the
row is fp64.  With u = 2^-24 and s = |g| + |pos| + |T_LI| + |p| (metres), counting every fp32 rounding in norm:
  * an fp32 rotation is the fp64 one rounded entry by entry, or two such composed by 3-term dot products: off by <= 15 u in
    Frobenius norm; an fp32 transform R v + t then adds <= 6 u |v| + 2 u |t| of its own rounding;
  * g = (R R_LI) p + (R T_LI + pos)                               off by <= 21 u |p| + 24 u |T_LI| + 2 u |pos|  <= 24 u s
  * p_lidar = (R_LI^T R^T) g - (R_LI^T R^T pos + R_LI^T T_LI)     g's error + 21 u |g| + 24 u (|pos| + |T_LI|)  <= 48 u s
  * p_imu = R_LI p_lidar + T_LI                                  p_lidar's error + 21 u |p| + 2 u |T_LI|         <= 72 u s
A and B are those points crossed with fp64 vectors of norm |n| ~ 1, C and n are exact to fp64, so every entry of a row is off
by at most C_ROW u s.  h = -(n . g + D) in fp32: g's error plus 4 roundings of terms bounded by |g| and |D|, at most
C_H u (s + |D|).  Far from the origin s is ~1e6 m, and the rotational columns legitimately lose centimetres of lever arm.
"""
import math

import numpy as np
import mpmath

import geometry as geo
import measure_mp as M

U32 = 2.0 ** -24
U64 = 2.0 ** -53
C_ROW = 72
C_H = 28


# ---- scenes ---------------------------------------------------------------------------------------------------------------
def large_extrinsic(O, sc):
    """the xaloc scene re-expressed in a LiDAR frame 30 degrees and (0.5, -0.3, 1.2) m from the configured one: the same world
    points (so the same matches), state x_prop with that extrinsic"""
    axis = np.array([1.0, 2.0, -1.0]) / math.sqrt(6.0)
    q = np.concatenate([math.sin(math.radians(15)) * axis, [math.cos(math.radians(15))]])
    t = np.array([0.5, -0.3, 1.2])
    x = np.array(sc.x_prop, np.float64).copy()
    R0, t0 = O.quat_to_rot(x[7:11]), x[11:14].copy()
    x[7:11], x[11:14] = q, t
    R1 = O.quat_to_rot(q)
    p_imu = sc.sweep.astype(np.float64) @ R0.T + t0
    return x, ((p_imu - t) @ R1).astype(np.float32)


def far_scenes(lv):
    """tests/geometry.py's sweep-built scene at (2e5, -3e5, 50) and (4.3e5, 0, 0)"""
    return [geo.sweep_built(lv, o) for o in geo.FAR_OFFSETS]


# ---- rows against the 50-digit rows ---------------------------------------------------------------------------------------
def row_errors(x, xyz, plane, rows, est):
    """per matched point: the largest |row entry - exact| / (C_ROW u s) and |h - exact| / (C_H u (s + |D|)), and the largest
    row error in metres.  rows: n x 13 (12 of H, then h) of the points xyz with planes `plane`."""
    x = np.asarray(x, np.float64)
    scale0 = float(np.linalg.norm(x[0:3]) + np.linalg.norm(x[11:14]))
    r_row, r_h, worst = np.zeros(len(xyz)), np.zeros(len(xyz)), 0.0
    for i in range(len(xyz)):
        ex, hx = M.rows_exact(x, xyz[i], plane[i], est)
        g = M.world_point(x, xyz[i])
        s = scale0 + float(mpmath.sqrt(g[0] ** 2 + g[1] ** 2 + g[2] ** 2)) + float(np.linalg.norm(xyz[i].astype(np.float64)))
        e = max(abs(float(mpmath.mpf(float(rows[i, k])) - ex[k])) for k in range(12))
        r_row[i] = e / (C_ROW * U32 * s)
        r_h[i] = abs(float(mpmath.mpf(float(rows[i, 12])) - hx)) / (C_H * U32 * (s + abs(float(plane[i][3]))))
        worst = max(worst, e)
    return r_row, r_h, worst


def fd_gap(x, xyz, plane, est):
    """the largest |rows_exact - rows_fd| over the points"""
    gap = mpmath.mpf(0)
    for i in range(len(xyz)):
        a, _ = M.rows_exact(x, xyz[i], plane[i], est)
        b = M.rows_fd(x, xyz[i], plane[i], est)
        gap = max(gap, max(abs(a[k] - b[k]) for k in range(12)))
    return float(gap)


# ---- exact normal equations -----------------------------------------------------------------------------------------------
def _two_prod(a, b):
    """a * b = p + e exactly (Dekker's product with Veltkamp's split; no overflow or underflow at these magnitudes)"""
    p = a * b
    sa, sb = a * 134217729.0, b * 134217729.0
    ah, bh = sa - (sa - a), sb - (sb - b)
    al, bl = a - ah, b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def gram_diffs(rows, HTH, HTh):
    """|HTH_ij - sum_k H_ki H_kj| and sum_k |H_ki H_kj| for the upper triangle (i <= j; column 12 is HTh, h as column 12), as
    two 12 x 13 arrays with zeros below.  The sums are exact: every product is split into two doubles without error, and the
    difference of the device's value with their sum is correctly rounded by math.fsum."""
    H = np.ascontiguousarray(rows, np.float64).reshape(-1, 13)
    got = np.concatenate([np.asarray(HTH).reshape(12, 12), np.asarray(HTh).reshape(12, 1)], axis=1)
    diff, mag = np.zeros((12, 13)), np.zeros((12, 13))
    for i in range(12):
        for j in range(i, 13):
            p, e = _two_prod(H[:, i], H[:, j])
            diff[i, j] = abs(math.fsum([float(got[i, j])] + (-p).tolist() + (-e).tolist()))
            mag[i, j] = math.fsum(np.abs(p).tolist() + (np.sign(p) * e).tolist())     # |p + e| = |p| + sign(p) e
    return diff, mag


def gram_errors(rows, HTH, HTh, gamma):
    """entry-wise |HTH - exact| / (gamma u64 sum_k |H_ki H_kj|) of gram_diffs; an entry whose bar is zero must be exactly
    zero (ratio inf otherwise)"""
    diff, mag = gram_diffs(rows, HTH, HTh)
    bar = gamma * U64 * mag
    out = np.where(bar > 0, diff / np.where(bar > 0, bar, 1.0), 0.0)
    out[(bar == 0) & (diff != 0)] = math.inf
    return out


def fold_gamma(n, threads=128, grid_cap=528, group=32, step_warps=16):
    """gamma(n) of lv_fit_kernel + reduce_partials_block on an n-point sweep: |HTH_ij - exact| <= gamma u64 sum_k |H_ki H_kj|.
    Every value is a sum of products along one tree; with d the largest number of roundings from a product to the root,
    the error is at most d u / (1 - d u) times the sum of the absolute terms.  Along the tree, per product:
      1    the product itself;
      31   the MMA chain of one warp: 32 rows of the tile in 8 k-steps of 4 (at most one rounding per product and per
           addition, whether the DMMA rounds per step or once per fragment);
      2    the four warp shares, (s0 + s1) + (s2 + s3);
      T    the block's tiles, tile, tile + grid, ... added to its accumulator (T = ceil(tiles / grid));
      31   the group's up to 32 block rows in row order;
      then reduce_partials_block over the G <= 17 group rows: each of its 16 warps adds its ceil(G / 16) rows in row order,
      and the warp sums are added in warp order, 15 roundings past the first.
    The additions that start from an exact zero are not counted."""
    tiles = max(1, -(-n // threads))
    grid = min(tiles, grid_cap)
    T = -(-tiles // grid)
    G = -(-grid // group)
    d = 1 + 31 + 2 + T + 31 + (-(-G // step_warps)) + (step_warps - 1)
    return d / (1.0 - d * U64)
