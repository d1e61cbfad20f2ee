"""lv_prelocalize restated in numpy, and calls into its host build (tests/cpu_shim/preloc.cpp).

The restatement follows the definition in include/limovelo_b200.h, not the header's code: the rotation matrices from the
quaternions in fp64 (Python floats, the products and sums in Eigen's toRotationMatrix order), cast to fp32 and composed in fp32
like State / RotTransl (make_frame's lidar_to_world), the world point w = fadd(dot3f(R row, p), fadd(t, o)), its voxel
floor(floor(w / ds) / k) per axis, and occupancy as the set of voxels that hold a stored map point."""
import ctypes as C
import math

import numpy as np

import shim_binding

f32 = np.float32
BIAS = 1 << 20
KPOS, KROT, KOFFR, KOFFT, KVEL, KGRAV = 0, 3, 7, 11, 14, 23


def quat_to_rot(q):
    """Eigen toRotationMatrix, q = (x, y, z, w), every product and sum rounded in double"""
    x, y, z, w = (float(t) for t in q)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    return [[1.0 - (tyy + tzz), txy - twz, txz + twy],
            [txy + twz, 1.0 - (txx + tzz), tyz - twx],
            [txz - twy, tyz + twx, 1.0 - (txx + tyy)]]


def quat_mul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz)


def dot3f(a0, a1, a2, b0, b1, b2):
    return (f32(a0) * f32(b0) + f32(a1) * f32(b1)) + f32(a2) * f32(b2)


def axes(x):
    g = [float(t) for t in x[KGRAV:KGRAV + 3]]
    gn = math.sqrt((g[0] * g[0] + g[1] * g[1]) + g[2] * g[2])
    g = [t / gn for t in g]
    e = [0.0, 1.0, 0.0] if abs(g[0]) > 0.9 else [1.0, 0.0, 0.0]
    eg = (e[0] * g[0] + e[1] * g[1]) + e[2] * g[2]
    w = [e[c] - eg * g[c] for c in range(3)]
    wn = math.sqrt((w[0] * w[0] + w[1] * w[1]) + w[2] * w[2])
    u = [t / wn for t in w]
    v = [g[1] * u[2] - g[2] * u[1], g[2] * u[0] - g[0] * u[2], g[0] * u[1] - g[1] * u[0]]
    return g, u, v


def rotate_state(x, g, theta):
    """rot' = q(g, theta) (x) rot, vel' = R(g, theta) vel; theta 0 keeps x"""
    out = np.array(x, np.float64)
    if theta == 0.0:
        return out
    half = 0.5 * theta
    s, c = math.sin(half), math.cos(half)
    q = (s * g[0], s * g[1], s * g[2], c)
    out[KROT:KROT + 4] = quat_mul(q, tuple(float(t) for t in x[KROT:KROT + 4]))
    R = quat_to_rot(q)
    vel = [float(t) for t in x[KVEL:KVEL + 3]]
    out[KVEL:KVEL + 3] = [(R[r][0] * vel[0] + R[r][1] * vel[1]) + R[r][2] * vel[2] for r in range(3)]
    return out


def offset64(u, v, a, b):
    return [a * u[c] + b * v[c] for c in range(3)]


def candidate(x, step, yaw_step, k, i, j):
    g, u, v = axes(x)
    out = rotate_state(x, g, float(k) * float(f32(yaw_step)))
    o = offset64(u, v, float(i) * float(f32(step)), float(j) * float(f32(step)))
    out[KPOS:KPOS + 3] = [float(x[KPOS + c]) + o[c] for c in range(3)]
    return out


def lidar_to_world(x):
    """make_frame(x).lidar_to_world: X = (R(rot), pos), IL = (R(offset_R_L_I), offset_T_L_I) in fp32, X * IL"""
    XR = np.array(quat_to_rot(x[KROT:KROT + 4]), np.float32)
    XT = np.array(x[KPOS:KPOS + 3], np.float64).astype(np.float32)
    LR = np.array(quat_to_rot(x[KOFFR:KOFFR + 4]), np.float32)
    LT = np.array(x[KOFFT:KOFFT + 3], np.float64).astype(np.float32)
    R = np.zeros((3, 3), np.float32)
    t = np.zeros(3, np.float32)
    for r in range(3):
        for c in range(3):
            R[r, c] = dot3f(XR[r, 0], XR[r, 1], XR[r, 2], LR[0, c], LR[1, c], LR[2, c])
        t[r] = dot3f(XR[r, 0], XR[r, 1], XR[r, 2], LT[0], LT[1], LT[2]) + XT[r]
    return R, t


def voxel_k(ds, voxel_size):
    k = int(math.floor(float(f32(voxel_size)) / float(f32(ds)) + 0.5))
    return min(max(k, 1), 3)


def voxels(w, ds, k):
    """biased voxel coordinates (n x 3 int64) of fp32 points, as voxel_coord"""
    cell = np.floor(w.astype(np.float32) / f32(ds)).astype(np.int64)
    return np.clip(cell // k + BIAS, 0, 0x1FFFFF)


def keys(vx):
    return vx[:, 0] | (vx[:, 1] << 21) | (vx[:, 2] << 42)


def stored(w):
    return np.all(np.abs(w) < f32(1e9), axis=1)


def occupancy(map_xyz, ds, k):
    m = np.asarray(map_xyz, np.float32)
    m = m[stored(m)]
    return np.unique(keys(voxels(m, ds, k)))


def subset(n, S):
    return (np.arange(S, dtype=np.int64) * n) // S


def grid(radius, step, yaw_range, yaw_step):
    I = int(math.floor(float(f32(radius)) / float(f32(step)) + 1e-9))
    K = int(math.floor(float(f32(yaw_range)) / float(f32(yaw_step)) + 1e-9))
    return I, K


def world_points(x, xyz, S, radius, step, yaw_range, yaw_step):
    """every candidate's world points: (2K+1, (2I+1)^2, S, 3) float32, in linear index order"""
    I, K = grid(radius, step, yaw_range, yaw_step)
    W = 2 * I + 1
    g, u, v = axes(x)
    p = np.asarray(xyz, np.float32)[subset(len(xyz), S)]
    off = np.array([[offset64(u, v, float(i) * float(f32(step)), float(j) * float(f32(step)))
                     for j in range(-I, I + 1)] for i in range(-I, I + 1)], np.float64).reshape(W * W, 3).astype(np.float32)
    out = np.zeros((2 * K + 1, W * W, S, 3), np.float32)
    for k in range(-K, K + 1):
        R, t = lidar_to_world(rotate_state(x, g, float(k) * float(f32(yaw_step))))
        rows = np.stack([dot3f(R[r, 0], R[r, 1], R[r, 2], p[:, 0], p[:, 1], p[:, 2]) for r in range(3)], axis=1)
        tt = (t[None, :] + off)                                   # fadd(F.t, o)
        out[k + K] = rows[None, :, :] + tt[:, None, :]
    return out


def score_all(x, xyz, map_xyz, ds, voxel_size, radius, step, yaw_range, yaw_step, max_points):
    """(scores in linear index order, hits (C, S) bool, world points)"""
    S = min(len(xyz), max_points)
    k = voxel_k(ds, voxel_size)
    occ = occupancy(map_xyz, ds, k)
    w = world_points(x, xyz, S, radius, step, yaw_range, yaw_step).reshape(-1, S, 3)
    flat = w.reshape(-1, 3)
    hit = np.isin(keys(voxels(flat, ds, k)), occ) & stored(flat)
    hit = hit.reshape(-1, S)
    return hit.sum(axis=1).astype(np.int32), hit, w


def winner(scores, I, K):
    """arg max under the tie rule: score, then smaller |k|, then smaller i^2 + j^2, then smaller index"""
    W = 2 * I + 1
    idx = np.arange(len(scores), dtype=np.int64)
    k = idx // (W * W) - K
    i = (idx % (W * W)) // W - I
    j = idx % W - I
    order = np.lexsort((idx, i * i + j * j, np.abs(k), -scores.astype(np.int64)))
    return int(order[0])


def at_face(w, ds):
    """per point: a coordinate within an ulp of a cell face (its cell changes one ulp away)"""
    w = np.asarray(w, np.float32)
    lo = np.floor(np.nextafter(w, np.float32(-np.inf)) / f32(ds))
    hi = np.floor(np.nextafter(w, np.float32(np.inf)) / f32(ds))
    return np.any(lo != hi, axis=-1)


# ---- the host build of csrc/lv_preloc.h -------------------------------------------------------------------------------------
def host_scores(x, xyz, map_xyz, ds, voxel_size, radius, step, yaw_range, yaw_step, max_points):
    """(scores, winner index, frames, offsets) of the host build"""
    I, K = grid(radius, step, yaw_range, yaw_step)
    W = 2 * I + 1
    x = np.ascontiguousarray(x, np.float64)
    xyz = np.ascontiguousarray(xyz, np.float32)
    mp = np.ascontiguousarray(map_xyz, np.float32)
    scores = np.zeros((2 * K + 1) * W * W, np.int32)
    frames = np.zeros((2 * K + 1, 12), np.float32)
    offs = np.zeros((W * W, 3), np.float32)
    fpt = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    L = shim_binding.lib()
    best = L.shim_preloc_scores(x.ctypes.data_as(C.POINTER(C.c_double)), fpt(xyz), len(xyz), fpt(mp), len(mp), ds, voxel_size,
                                radius, step, yaw_range, yaw_step, max_points, scores.ctypes.data_as(C.POINTER(C.c_int32)),
                                fpt(frames), fpt(offs))
    return scores, int(best), frames, offs


def host_candidate(x, step, yaw_step, k, i, j):
    x = np.ascontiguousarray(x, np.float64)
    out = np.zeros(26)
    shim_binding.lib().shim_preloc_candidate(x.ctypes.data_as(C.POINTER(C.c_double)), step, yaw_step, k, i, j,
                                             out.ctypes.data_as(C.POINTER(C.c_double)))
    return out
