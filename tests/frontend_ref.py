"""The front end of a tick, restated independently: deskew in 50-digit arithmetic (mpmath), the PCL voxel grid and the
temporal decimator in numpy with every fp32 operation spelled out.

Written from the reference's text, not from the product's headers or the oracle (oracle/lv_oracle.cpp), so that it checks
both.  Line numbers cite the reference:
  State.cpp:94-121        State::propagate_f / State::update (the state integrated to a point's stamp)
  Utils.hpp:28-54         SO3Math::Exp (Rodrigues, identity when |w - bw| <= 1e-7)
  RotTransl.cpp:29-48     RotTransl::inv (R^T, -R^T t), RotTransl * RotTransl, RotTransl * Point
  Compensator.cpp:53-61   get_t2;  :123-146 compensate (linear segment walk);  :148-163 voxelgrid_downsample
  PointCloudProcessor.cpp:101-112  temporal_downsample
and pcl/filters/impl/voxel_grid.hpp (VoxelGrid::applyFilter with downsample_all_data_ = true: CentroidPoint ->
AccumulatorXYZ, a fp32 running sum divided by the count).

States are any ctypes structure with the lv_state32 fields (R, pos, vel, bw, ba, g, RLI, tLI, a, w: float; time: double).
"""
import math

import mpmath
import numpy as np
from mpmath import mp

mp.dps = 50

U32 = 2.0 ** -24                 # unit roundoff of fp32
INT32_MAX = 2 ** 31 - 1


# ---- deskew (Compensator::compensate) in 50 digits ----------------------------------------------------------------------
def _v(a):
    return [mpmath.mpf(float(x)) for x in a]


def _mm(A, B):                   # 3x3 row-major lists
    return [sum((A[3 * i + k] * B[3 * k + j] for k in range(3)), mpmath.mpf(0)) for i in range(3) for j in range(3)]


def _mv(A, v):
    return [A[3 * i] * v[0] + A[3 * i + 1] * v[1] + A[3 * i + 2] * v[2] for i in range(3)]


def _T(A):
    return [A[3 * j + i] for i in range(3) for j in range(3)]


def _rt_mul(a, b):               # RotTransl.cpp:36-41: (R1 R2, R1 t2 + t1)
    return _mm(a[0], b[0]), [x + y for x, y in zip(_mv(a[0], b[1]), a[1])]


def _rt_inv(a):                  # RotTransl.cpp:29-34: (R^T, -R^T t); the transpose, not the inverse of an fp32 matrix
    Rt = _T(a[0])
    return Rt, [-x for x in _mv(Rt, a[1])]


def _rt_apply(a, p):             # RotTransl.cpp:43-48
    return [x + y for x, y in zip(_mv(a[0], p), a[1])]


def so3_exp(wb, dt):
    """the rotating branch of SO3Math::Exp (Utils.hpp:28-54) for the exact vector wb over the exact dt"""
    n = mpmath.sqrt(wb[0] ** 2 + wb[1] ** 2 + wb[2] ** 2)
    r = [x / n for x in wb]
    K = [0, -r[2], r[1], r[2], 0, -r[0], -r[1], r[0], 0]
    K = [mpmath.mpf(x) for x in K]
    KK = _mm(K, K)
    s, c1 = mpmath.sin(n * dt), 1 - mpmath.cos(n * dt)
    return [(1 if i % 4 == 0 else 0) + s * K[i] + c1 * KK[i] for i in range(9)]


def _fp32_norm_gt(wb32):
    """the reference evaluates |w - bw| > 1e-7 on its fp32 vector: the branch is decided in fp32, the rest is exact"""
    w = np.asarray(wb32, np.float32)
    n = np.sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2], dtype=np.float32)
    return float(n) > 0.0000001


def propagate_exact(X, t):
    """State X integrated to time t with its own last controls (Compensator.cpp:133-134 -> State.cpp:112-115, 94-110):
    returns (R, pos) exactly.  dt = t - X.time without rounding."""
    dt = mpmath.mpf(t) - mpmath.mpf(X.time)
    R, pos, vel, g = _v(X.R), _v(X.pos), _v(X.vel), _v(X.g)
    w, bw, a, ba = _v(X.w), _v(X.bw), _v(X.a), _v(X.ba)
    wb = [x - y for x, y in zip(w, bw)]
    wb32 = np.float32(X.w[:]) - np.float32(X.bw[:])
    Rn = _mm(R, so3_exp(wb, dt)) if _fp32_norm_gt(wb32) else R
    acc = [x - y for x, y in zip(_mv(R, [x - y for x, y in zip(a, ba)]), g)]
    pn = [pos[i] + vel[i] * dt + acc[i] * dt * dt / 2 for i in range(3)]
    return Rn, pn


def back_transform(Xt2):
    """Xt2.I_Rt_L().inv() * Xt2.inv() (Compensator.cpp:138)"""
    return _rt_mul(_rt_inv((_v(Xt2.RLI), _v(Xt2.tLI))), _rt_inv((_v(Xt2.R), _v(Xt2.pos))))


def deskew_point(X, back, p, t):
    """one point through Compensator.cpp:133-138 from state X (the start of its segment): exact (q, g) as mpf triples"""
    R, pos = propagate_exact(X, t)
    g = _rt_apply(_rt_mul((R, pos), (_v(X.RLI), _v(X.tLI))), _v(p))
    return _rt_apply(back, g), g


def segments(path, t):
    """the linear walk of Compensator.cpp:130-131: segment of every (sorted) stamp; -1 where the walk drops a point"""
    seg = np.full(len(t), -1, np.int64)
    p = 0
    for s in range(len(path) - 1):
        while p < len(t) and path[s].time <= t[p] <= path[s + 1].time:
            seg[p] = s
            p += 1
    return seg


def compensate(path, Xt2, xyz, t, seg=None):
    """Compensator::compensate in 50 digits.  Returns (q: float64 n x 3 rounded from the exact values, the segment of every
    point by the reference's walk, M: the largest magnitude of every point's chain).  `seg` forces the segment of every point
    (for the separation of neighbouring segments); default: the walk."""
    walk = segments(path, t)
    assert (walk >= 0).all(), "the path must surround every stamp"
    seg = walk if seg is None else np.asarray(seg)
    back = back_transform(Xt2)
    out, gmax = np.empty((len(t), 3)), np.empty(len(t))
    for i in range(len(t)):
        q, g = deskew_point(path[int(seg[i])], back, xyz[i], float(t[i]))
        out[i] = [float(v) for v in q]
        gmax[i] = max(abs(float(v)) for v in g)
    return out, walk, chain_magnitude(path, Xt2, xyz, seg, gmax)


def chain_magnitude(path, Xt2, xyz, seg, gmax):
    """M of the tolerance: the largest magnitude in a point's fp32 chain (|p|, |pos| of its state and of Xt2, |g|)"""
    pos = np.array([np.abs(np.float64(path[int(s)].pos[:])).max() for s in seg])
    M = np.maximum(np.abs(np.asarray(xyz, np.float64)).max(axis=1), pos)
    return np.maximum(np.maximum(M, np.abs(np.float64(Xt2.pos[:])).max()), gmax)


# ---- voxel grid (pcl::VoxelGrid::applyFilter) in numpy fp32 ---------------------------------------------------------------
f32 = np.float32


def _wrap32(v):
    v = int(v) & 0xFFFFFFFF
    return v - (1 << 32) if v >= (1 << 31) else v


def voxel_cells(xyz, leaf):
    """the per-point cell index and the grid of voxel_grid.hpp (applyFilter): returns dict(overflow, key (uint32 per point,
    the int32 index with its wrap, as PCL stores it in cloud_point_index_idx), ijk, minb, divb, d)."""
    xyz = np.ascontiguousarray(xyz, f32).reshape(-1, 3)
    inv = f32(1) / f32(leaf)                                   # inverse_leaf_size_ = 1 / leaf_size_ (fp32)
    mn, mx = xyz.min(axis=0), xyz.max(axis=0)                  # getMinMax3D (the sign of a zero cannot reach an index)
    d = [int((f32(mx[a] - mn[a]) * inv).astype(np.int64)) + 1 for a in range(3)]      # dx, dy, dz: int64 truncation
    assert d[0] * d[1] * d[2] < 2 ** 63, "outside the domain: PCL's int64 product would wrap"
    if d[0] * d[1] * d[2] > INT32_MAX:                         # "Leaf size is too small ... Integer indices would overflow"
        return dict(overflow=True, d=d)
    minb = [int(np.floor(f32(mn[a] * inv))) for a in range(3)]
    divb = [int(np.floor(f32(mx[a] * inv))) - minb[a] + 1 for a in range(3)]
    mul = [1, divb[0], _wrap32(divb[0] * divb[1])]            # divb_mul_ (Vector4i: int32 products)
    ijk = np.empty((len(xyz), 3), np.int64)
    for a in range(3):
        fl = np.floor(xyz[:, a] * inv)                         # std::floor(float) stays fp32
        diff = fl - f32(minb[a])                               # fp32 subtraction: inexact once |x * inv| > 2^24
        assert diff.dtype == f32
        ijk[:, a] = diff.astype(np.int64)
    assert (np.abs(ijk) < 2 ** 31).all()
    idx = ijk[:, 0] * mul[0] + ijk[:, 1] * mul[1] + ijk[:, 2] * mul[2]   # exact, then the int32 wrap of the C sum
    key = (idx & 0xFFFFFFFF).astype(np.uint32)                 # static_cast<unsigned int>(idx)
    return dict(overflow=False, key=key, ijk=ijk, minb=minb, divb=divb, d=d, mul=mul)


def _seq_sums(pts, starts, counts):
    """fp32 running sums x += p per leaf in the order given (AccumulatorXYZ), starting from +0"""
    out = np.zeros((len(starts), 3), f32)
    small = counts <= 64
    si, sc = starts[small], counts[small]
    acc = np.zeros((len(si), 3), f32)
    for k in range(int(sc.max()) if len(sc) else 0):
        m = sc > k
        acc[m] = acc[m] + pts[si[m] + k]
    out[small] = acc
    for r in np.nonzero(~small)[0]:
        seg = np.concatenate([np.zeros((1, 3), f32), pts[starts[r]:starts[r] + counts[r]]])
        out[r] = np.add.accumulate(seg, axis=0, dtype=f32)[-1]   # strictly sequential, unlike np.sum
    return out


def voxelgrid(xyz, leaf, exact=False):
    """pcl::VoxelGrid<PointT>::filter with a cubic leaf.  Returns dict(out: the centroids (fp32, ascending key, input order
    inside a leaf: std::sort of PCL leaves that order unspecified; the stable sort pins it), count per leaf, key per leaf,
    overflow; with exact=True also mean: the exact mean of every leaf (math.fsum / count, float64)).  On overflow PCL warns
    and the output is the input."""
    xyz = np.ascontiguousarray(xyz, f32).reshape(-1, 3)
    c = voxel_cells(xyz, leaf)
    if c["overflow"]:
        return dict(out=xyz.copy(), overflow=True, count=None, key=None, d=c["d"])
    order = np.argsort(c["key"], kind="stable")
    ks = c["key"][order]
    head = np.ones(len(ks), bool)
    head[1:] = ks[1:] != ks[:-1]
    starts = np.nonzero(head)[0]
    counts = np.diff(np.append(starts, len(ks)))
    sums = _seq_sums(xyz[order], starts, counts)
    out = sums / counts.astype(f32)[:, None]                  # xyz / n: n (size_t) converted to float, fp32 division
    assert out.dtype == f32
    res = dict(out=out, overflow=False, count=counts, key=ks[starts], order=order, starts=starts, d=c["d"],
               divb=c["divb"], minb=c["minb"], cells=c)
    if exact:
        p64 = xyz[order].astype(np.float64)
        res["mean"] = np.array([[math.fsum(p64[s:s + n, a]) / n for a in range(3)] for s, n in zip(starts, counts)])
    return res


# ---- temporal decimator (PointCloudProcessor::temporal_downsample) --------------------------------------------------------
def temporal(xyz, rate, min_dist):
    """indices kept: keep_point = rate <= 1 or ++ds_counter % rate == 0 (the counter counts every point), and
    min_dist < p.norm() (a strict <, double against the fp32 norm)"""
    xyz = np.ascontiguousarray(xyz, f32).reshape(-1, 3)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    nrm = np.sqrt((x * x + y * y) + z * z)
    assert nrm.dtype == f32
    i = np.arange(1, len(xyz) + 1)
    keep = np.ones(len(xyz), bool) if rate <= 1 else (i % rate == 0)
    keep &= min_dist < nrm.astype(np.float64)
    return np.nonzero(keep)[0].astype(np.int32)


def fp32_norm(p):
    p = np.asarray(p, f32)
    return np.sqrt((p[0] * p[0] + p[1] * p[1]) + p[2] * p[2])
