"""Seeded inputs for the front end of a tick (deskew, voxel grid, temporal decimator), built to reach the places where the
kernels can differ from the reference.  Every generator checks, through the restatement (frontend_ref), that its case takes
the path it is built for.  States are the oracle's State32 (same layout as the product's lv.State32)."""
import math
from fractions import Fraction

import numpy as np

import frontend_ref as F

f32 = np.float32

# the deskew bar: e_gpu <= e_oracle + K * u32 * M (see test_gpu_frontend.py for where K comes from)
K = 8
SEPARATION = 1e3                 # inconsistent paths: a neighbouring segment moves every point by >= 1e3 x the bar


# ---- deskew -------------------------------------------------------------------------------------------------------------
def _rot(rng, scale):
    v = rng.normal(0, 1, 3)
    v *= scale / np.linalg.norm(v)
    th = np.linalg.norm(v)
    if th == 0:
        return np.eye(3)
    k = v / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + math.sin(th) * Kx + (1 - math.cos(th)) * Kx @ Kx


def make_state(O, R, pos, vel, time, a, w, bw=(1e-3, -2e-3, 5e-4), ba=(0.02, 0.01, -0.03), g=(0, 0, 9.81),
               RLI=np.eye(3), tLI=(0, 0, 0)):
    s = O.State32()
    s.R[:] = [float(f32(x)) for x in np.ravel(R)]
    s.RLI[:] = [float(f32(x)) for x in np.ravel(RLI)]
    for name, v in (("pos", pos), ("vel", vel), ("bw", bw), ("ba", ba), ("g", g), ("tLI", tLI), ("a", a), ("w", w)):
        getattr(s, name)[:] = [float(f32(x)) for x in v]
    s.time = float(time)
    return s


def random_path(O, rng, ns, t0=10.0, span=0.11, pos0=(0.0, 0.0, 0.0), jump=0.0, gyro=0.5, vary_extrinsics=True,
                times=None, identity=False):
    """ns states over [t0, t0 + span]: 15 m/s along x, a yawing vehicle, IMU-like controls.  jump > 0 displaces every state by
    `jump` m in a random direction: the states are then not integrations of each other (an inconsistent path)."""
    if times is None:
        times = t0 + np.sort(np.concatenate([[0.0, span], rng.uniform(0, span, ns - 2)]))
    path = []
    R = _rot(rng, 0.3)
    for k in range(ns):
        dt = times[k] - times[0]
        pos = np.asarray(pos0) + np.array([15.0, 0.3, -0.1]) * dt
        if jump:
            d = rng.normal(0, 1, 3)
            pos = pos + jump * d / np.linalg.norm(d)
        bw = rng.normal(0, 1e-3, 3).astype(f32)
        w = bw.copy() if identity else bw + np.array([0.02, -0.01, gyro]) + rng.normal(0, 0.01, 3)
        a = np.array([0.3, -0.2, 9.8]) + rng.normal(0, 0.05, 3)
        RLI, tLI = (_rot(rng, 0.05) @ np.diag([1.0, -1.0, -1.0]), rng.normal(0, 0.3, 3)) if vary_extrinsics else (np.eye(3), (0, 0, 0))
        path.append(make_state(O, _rot(rng, 0.05 * k) @ R, pos, [15.0, 0.3, -0.1], times[k], a, w, bw=bw, RLI=RLI, tLI=tLI))
    return path


def lidar_points(rng, n, r=(1.0, 20.0)):
    d = rng.normal(0, 1, (n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (d * rng.uniform(r[0], r[1], (n, 1))).astype(f32)


def stamps_uniform(rng, path, n):
    t = np.sort(rng.uniform(path[0].time, path[-1].time, n))
    if n >= 2:
        t[0], t[-1] = path[0].time, path[-1].time
    return t


def stamps_on_states(path):
    """every state time, and one double-ulp either side (inside the path)"""
    ts = []
    for s in path:
        ts += [np.nextafter(s.time, -np.inf), s.time, np.nextafter(s.time, np.inf)]
    t = np.array(sorted(ts))
    return t[(t >= path[0].time) & (t <= path[-1].time)]


def _case(O, name, path, xyz, t, t2=None, inconsistent=False):
    t2 = path[-1].time - 0.004 if t2 is None else t2
    Xt2 = O.get_t2(path, t2)
    seg = F.segments(path, t)
    assert (seg >= 0).all() and len(path) >= 2
    return dict(name=name, path=path, Xt2=Xt2, xyz=np.ascontiguousarray(xyz, f32), t=np.ascontiguousarray(t, np.float64),
                seg=seg, inconsistent=inconsistent)


def deskew_separation(c, exact=None):
    """the inconsistent-path proof: for every point, the exact result from a neighbouring segment lies at least
    SEPARATION x the bar (K u32 M, doubled for e_oracle) away from the result from its own segment"""
    path, seg = c["path"], c["seg"]
    q, _, M = F.compensate(path, c["Xt2"], c["xyz"], c["t"]) if exact is None else exact
    bar = 2 * K * F.U32 * M
    sep = np.full(len(seg), np.inf)
    for d in (-1, 1):
        alt = np.clip(seg + d, 0, len(path) - 2)
        m = alt != seg
        if m.any():
            qa, _, _ = F.compensate(path, c["Xt2"], c["xyz"][m], c["t"][m], seg=alt[m])
            sep[m] = np.minimum(sep[m], np.abs(qa - q[m]).max(axis=1))
    assert (sep >= SEPARATION * bar).all(), (c["name"], (sep / bar).min())
    return sep / bar


DESKEW_NAMES = ["ns2", "ns3", "ns255", "ns256", "upsampled100Hz", "upsampled400Hz", "upsampled1000Hz", "upsampled2000Hz",
                "on_state_times", "duplicate_state_times", "one_stamp", "ros_epoch", "identity_branch", "just_above_identity",
                "large_rotation", "far_2e5_-3e5_50", "far_4.3e5"]


def deskew_cases(O, rng_seed=20261015):
    """the families the kernel is checked on (n kept small: every point is evaluated in 50 digits)"""
    rng = np.random.default_rng(rng_seed)
    out = []
    for ns in (2, 3, 255, 256):
        p = random_path(O, rng, ns, jump=0.0 if ns == 2 else 0.15)
        out.append(_case(O, "ns%d" % ns, p, lidar_points(rng, 300), stamps_uniform(rng, p, 300), inconsistent=ns > 2))
    for hz in (100, 400, 1000, 2000):
        st = random_path(O, rng, 4, span=0.1)
        imu_t = np.arange(st[0].time + 0.2 / hz, st[-1].time + 1.5 / hz, 1.0 / hz)
        imu_a = (np.array([0.3, -0.2, 9.8]) + rng.normal(0, 0.05, (len(imu_t), 3))).astype(f32)
        imu_w = (np.array([0.02, -0.01, 0.5]) + rng.normal(0, 0.01, (len(imu_t), 3))).astype(f32)
        p = O.upsample(st, imu_a, imu_w, imu_t)
        assert 4 < len(p) <= 256
        out.append(_case(O, "upsampled%dHz" % hz, p, lidar_points(rng, 300), stamps_uniform(rng, p, 300)))
    p = random_path(O, rng, 12, jump=0.15)
    t = stamps_on_states(p)
    out.append(_case(O, "on_state_times", p, lidar_points(rng, len(t)), t, inconsistent=True))
    tm = 10.0 + np.array([0, 0.02, 0.02, 0.05, 0.05, 0.05, 0.08, 0.11])
    p = random_path(O, rng, len(tm), times=tm, jump=0.15)
    t = np.sort(np.concatenate([tm, rng.uniform(tm[0], tm[-1], 100)]))
    out.append(_case(O, "duplicate_state_times", p, lidar_points(rng, len(t)), t, inconsistent=True))
    p = random_path(O, rng, 6, jump=0.15)
    out.append(_case(O, "one_stamp", p, lidar_points(rng, 200), np.full(200, p[3].time), inconsistent=True))
    p = random_path(O, rng, 6, t0=1.7e9, jump=0.15)
    t = np.concatenate([stamps_on_states(p), stamps_uniform(rng, p, 100)])
    out.append(_case(O, "ros_epoch", p, lidar_points(rng, len(t)), np.sort(t), inconsistent=True))
    # the identity branch of SO3Math::Exp: no sinf / cosf anywhere, so the kernel must equal the oracle bit for bit.  Near the
    # origin with slow points, so that the 0.5 acc dt^2 term is a large share of every coordinate
    p = random_path(O, rng, 5, span=0.2, identity=True, gyro=0.0, vary_extrinsics=False)
    for s in p:
        s.pos[:] = [0.0, 0.0, 0.0]; s.vel[:] = [0.0, 0.0, 0.0]; s.g[:] = [0.0, 0.0, 0.0]
    out.append(_case(O, "identity_branch", p, lidar_points(rng, 400, r=(0.01, 0.1)), stamps_uniform(rng, p, 400)))
    p = random_path(O, rng, 5, jump=0.15)
    for s in p:                                           # |w - bw| just above 1e-7 in fp32
        s.w[:] = [float(f32(s.bw[0]) + f32(1.5e-7)), s.bw[1], s.bw[2]]
        assert F._fp32_norm_gt(np.float32(s.w[:]) - np.float32(s.bw[:]))
    out.append(_case(O, "just_above_identity", p, lidar_points(rng, 200), stamps_uniform(rng, p, 200), inconsistent=True))
    p = random_path(O, rng, 3, span=0.2, gyro=10.0)      # |w| dt up to ~1 rad over a segment
    assert max(np.linalg.norm(np.float64(s.w[:])) * (p[k + 1].time - s.time) for k, s in enumerate(p[:-1])) > 0.5
    out.append(_case(O, "large_rotation", p, lidar_points(rng, 300), stamps_uniform(rng, p, 300)))
    for name, off in (("far_2e5_-3e5_50", (2e5, -3e5, 50.0)), ("far_4.3e5", (4.3e5, 0.0, 0.0))):
        p = random_path(O, rng, 6, pos0=off)
        out.append(_case(O, name, p, lidar_points(rng, 300), stamps_uniform(rng, p, 300)))
    assert [c["name"] for c in out] == DESKEW_NAMES
    return out


def deskew_sized(O, n, seed=7):
    """one upsample-like inconsistent path and n points: for n around the block size and a handle's max_points"""
    rng = np.random.default_rng(seed + n)
    p = random_path(O, rng, 40, jump=0.15)
    return _case(O, "n%d" % n, p, lidar_points(rng, n), stamps_uniform(rng, p, n), inconsistent=True)


# ---- voxel grid ---------------------------------------------------------------------------------------------------------
def _exact_cell(x, leaf):
    return math.floor(Fraction(float(x)) / Fraction(float(f32(leaf))))


def voxel_faces(leaf, rng):
    """coordinates on leaf faces (k * leaf rounded to fp32) and one fp32 ulp either side; some of them must land in another
    cell than exact division of the fp32 coordinate by the fp32 leaf would put them"""
    k = np.arange(-40, 41)
    on = (k * float(leaf)).astype(f32)
    vals = np.concatenate([np.nextafter(on, f32(-np.inf)), on, np.nextafter(on, f32(np.inf))])
    n = 3000
    xyz = np.stack([rng.choice(vals, n), rng.choice(vals, n), rng.choice(vals, n)], axis=1).astype(f32)
    inv = f32(1) / f32(leaf)
    fp = np.floor(vals * inv).astype(np.int64)
    ex = np.array([_exact_cell(v, leaf) for v in vals])
    if float(inv) != 1 / float(f32(leaf)):                # 0.1, 0.2, 0.3: 1 / leaf is not exact in fp32
        assert (fp != ex).any(), leaf
    return xyz


def voxel_cases(seed=20261016):
    rng = np.random.default_rng(seed)
    out = []
    for leaf in (0.1, 0.2, 0.3, 0.5, 2.0):
        out.append(("faces_leaf%g" % leaf, voxel_faces(leaf, rng), leaf))
    out.append(("negative", (-rng.uniform(10, 50, (5000, 3))).astype(f32), 0.5))
    z = np.array([0.0, -0.0], f32)
    pm = np.stack([rng.choice(z, 200), rng.choice(z, 200), rng.choice(z, 200)], axis=1)
    pm = np.concatenate([pm, rng.uniform(-0.3, 0.3, (200, 3)).astype(f32)])
    assert np.signbit(pm).any() and (pm == 0).all(axis=1).sum() > 100
    out.append(("signed_zeros", pm, 0.2))
    # |x * inv| > 2^24 with a negative minimum: floor(x * inv) - min_b is rounded in fp32
    far = np.stack([rng.uniform(-3e7, 3e7, 4000), rng.uniform(0, 4.9, 4000), rng.uniform(0, 4.9, 4000)], axis=1).astype(f32)
    far[0, 0], far[1, 0] = -3e7, 3e7
    far[2:34] = np.stack([3e7 - 2.0 * np.arange(32), np.ones(32), np.ones(32)], axis=1)   # neighbouring fp32 values
    c = F.voxel_cells(far, 1.0)
    assert not c["overflow"]
    exact = np.floor(far[:, 0].astype(np.float64)) - c["minb"][0]
    assert (c["ijk"][:, 0] != exact).any()                 # the fp32 subtraction is inexact for some points
    ex_cells = {(int(e), int(j), int(k)) for e, j, k in zip(exact, c["ijk"][:, 1], c["ijk"][:, 2])}
    assert len(np.unique(c["key"])) < len(ex_cells)         # ... and merges points of distinct cells into one leaf
    out.append(("far_fsub", far, 1.0))
    # cell counts just below (2^31 - 2 = 1549411 * 1386 * 1) and just above (2^31 = 2^23 * 256 * 1) INT32_MAX, leaf 1
    for name, d in (("cells_below_int32max", (1549411, 1386, 1)), ("cells_above_int32max", (1 << 23, 256, 1))):
        pts = np.stack([rng.integers(0, d[0], 500), rng.integers(0, d[1], 500), np.zeros(500)], axis=1).astype(np.float64)
        pts[0] = [0, 0, 0]
        pts[1] = [d[0] - 1, d[1] - 1, 0]
        pts = pts.astype(f32)
        c = F.voxel_cells(pts, 1.0)
        assert c["d"] == list(d) and c["overflow"] == (name.startswith("cells_above"))
        out.append((name, pts, 1.0))
    out.append(("wrap", voxel_wrap(rng), 1.0))
    # n leaves of one point each
    g = np.stack(np.meshgrid(np.arange(20), np.arange(20), np.arange(10), indexing="ij"), -1).reshape(-1, 3)
    one = ((g * 1.5 + 0.25) * 0.5).astype(f32)
    r = F.voxelgrid(one, 0.5)
    assert (r["count"] == 1).all() and len(r["count"]) == len(one)
    out.append(("one_point_leaves", rng.permutation(one), 0.5))
    for n in (1, 255, 256, 257, 65537):
        out.append(("n%d" % n, lidar_points(rng, n, r=(1.0, 60.0)), 0.5))
    return out


def voxel_wrap(rng):
    """dx * dy * dz = 46340^2 <= INT32_MAX, but div_b = (46341, 46341, 2), so div_b[0] * div_b[1] wraps in int32 and so does
    the index of every point in the upper z layer: distinct cells share a key"""
    n = 3000
    x = np.concatenate([[0.75, 46340.25], rng.uniform(0.75, 46340.25, n)])
    y = np.concatenate([[0.75, 46340.25], rng.uniform(0.75, 46340.25, n)])
    z = np.concatenate([[0.75, 1.25], rng.choice([0.8, 1.2], n)])
    hi = np.array([[46340.25, 46340.25, 1.2], [46340.25, 46000.25, 1.2], [9265.5, 0.9, 0.8], [9265.5, 0.8, 0.8]])
    pts = np.concatenate([np.stack([x, y, z], 1), hi]).astype(f32)
    c = F.voxel_cells(pts, 1.0)
    assert not c["overflow"] and c["d"][0] * c["d"][1] * c["d"][2] <= F.INT32_MAX
    assert c["divb"][0] * c["divb"][1] > F.INT32_MAX
    exact = c["ijk"][:, 0] + c["ijk"][:, 1] * c["divb"][0] + c["ijk"][:, 2] * c["divb"][0] * c["divb"][1]
    assert len(np.unique(exact)) > len(np.unique(c["key"]))  # the wrap merges distinct cells
    return pts


def voxel_big_leaf(seed=5):
    """one leaf holding 2^24 + 3 points: (float)count is inexact"""
    n = (1 << 24) + 3
    assert int(f32(n)) != n
    rng = np.random.default_rng(seed)
    return rng.uniform(0.05, 0.45, (n, 3)).astype(f32), 0.5


# ---- temporal decimator -------------------------------------------------------------------------------------------------
def temporal_cases(seed=20261017):
    rng = np.random.default_rng(seed)
    xyz = lidar_points(rng, 5000, r=(0.5, 40.0))
    nrm = F.fp32_norm(xyz[1234])
    out = [("rate0", xyz, 0, 4.0), ("rate-3", xyz, -3, 4.0), ("rate1", xyz, 1, 4.0), ("rate>n", xyz, 5001, 0.0),
           ("rate7", xyz, 7, 4.0), ("min_dist_negative", xyz, 3, -1.0), ("min_dist_inf", xyz, 1, math.inf),
           ("min_dist_eq_norm", xyz, 1, float(nrm)), ("min_dist_eq_norm_r2", xyz, 2, float(nrm))]
    keep = F.temporal(xyz, 1, float(nrm))
    assert 1234 not in keep and 1234 in F.temporal(xyz, 1, float(np.nextafter(nrm, f32(0))))   # strict <
    return out
