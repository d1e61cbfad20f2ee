"""One row of the measurement model (IKFoM::h_share_model -> Localizator::calculate_H) in 50-digit arithmetic (mpmath): the
yardstick the fp32 / fp64 rows of H and h are measured against.

Written from the reference's text, not from the product's headers or the oracle, so that it is independent of both.  Line
numbers cite the reference:
  include/IKFoM/use-ikfom.cpp:16-31   h_share_model: the matches of State(updated_state) (Mapper::match), then calculate_H
  src/Modules/Mapper.cpp:51           the matched point is the world point X * X.I_Rt_L() * p
  src/Objects/State.cpp:51-62         State(const state_ikfom&, double): R = rot, pos, RLI = offset_R_L_I, tLI = offset_T_L_I
  src/Objects/State.cpp:64-73         I_Rt_L() = (RLI, tLI), inv() = RotTransl(R, pos).inv()
  src/Objects/RotTransl.cpp:29-48     inv() = (R^T, -R^T t), RT1 * RT2 = (R1 R2, R1 t2 + t1), RT * p = R p + t
  src/Objects/Match.cpp:21            distance = plane.dist_to_plane(point)
  src/Objects/Plane.cpp:27-29         dist_to_plane(p) = A x + B y + C z + D
  src/Modules/Localizator.cpp:36-56   p_lidar = S.I_Rt_L().inv() * S.inv() * point, p_imu = S.I_Rt_L() * p_lidar,
                                      C = R^T n, B = p_lidar x (RLI^T C), A = p_imu x C,
                                      row = [n, A, B, C] (B, C only with estimate_extrinsics), h = -distance

In real arithmetic the casts to float of State(...) disappear, and so does the round trip of :38: p_lidar is the LiDAR point
itself.  The state's two quaternions are normalised here: an fp64 quaternion is unit to ~1e-16, and the rotation the reference
means is the one of the unit quaternion (toRotationMatrix of a non-unit quaternion is not a rotation, and its derivative under
the state's [+] would not be exactly the row).

rows_fd differentiates dist(x [+] delta) with ikfom_mp.boxplus, the [+] the step's 50-digit reference (test_gpu_filter) uses, so
agreement of rows_exact and rows_fd says that calculate_H's row is the Jacobian of its own residual under that [+].
Inputs: x (26 floats, ikfom_mp's flat layout), p (3 floats, LiDAR frame), plane (A, B, C, D); all taken as exact.
"""
import functools

import mpmath
from mpmath import mp

import ikfom_mp as K

mp.dps = 50
FD_STEP = mpmath.mpf("1e-20")
FD_DPS = 80       # digits of the central differences: the roundoff (|g| 1e-80 / 1e-20) stays far below their h^2 truncation


def _unit(q):
    s = mpmath.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2 + q[3] ** 2)
    return [a / s for a in q]


def _vec3(v):
    return mp.matrix([K.mpf(a) if isinstance(a, mpmath.mpf) else mpmath.mpf(float(a)) for a in v])


@functools.lru_cache(maxsize=64)
def _transforms(x):
    """(R, pos, RLI, tLI) of the state tuple x, State.cpp:51-62 without the casts"""
    x = K.state(x)
    R = K.qrot(_unit(x[3:7]))
    RLI = K.qrot(_unit(x[7:11]))
    return R, mp.matrix(x[0:3]), RLI, mp.matrix(x[11:14])


def _world(T, p):
    """Mapper.cpp:51: X * X.I_Rt_L() * p = R (RLI p + tLI) + pos (RotTransl.cpp:36-48)"""
    R, pos, RLI, tLI = T
    return R * (RLI * p + tLI) + pos


def _dist(n, D, g):                                             # Plane.cpp:27-29
    return n[0] * g[0] + n[1] * g[1] + n[2] * g[2] + D


def _cross(a, b):
    return mp.matrix([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def world_point(x, p):
    return _world(_transforms(tuple(float(a) for a in x)), _vec3(p))


def rows_exact(x, p, plane, est):
    """calculate_H's row (12 mpf) and h = -distance of the match of LiDAR point p with `plane`, at state x"""
    R, pos, RLI, tLI = T = _transforms(tuple(float(a) for a in x))
    p = _vec3(p)
    n, D = _vec3(plane[:3]), K.mpf(float(plane[3]))
    g = _world(T, p)                                            # the matched point (Mapper.cpp:51)
    p_lidar = RLI.T * (R.T * (g - pos) - tLI)                   # I_Rt_L().inv() * inv() * point (Localizator.cpp:38)
    p_imu = RLI * p_lidar + tLI                                 # :39
    C = R.T * n                                                 # :43, :47 (conjugate().toRotationMatrix() = R^T)
    B = _cross(p_lidar, RLI.T * C)                              # :44, :48
    A = _cross(p_imu, C)                                        # :49
    row = [n[0], n[1], n[2], A[0], A[1], A[2]]                  # :51
    row += [B[0], B[1], B[2], C[0], C[1], C[2]] if est else [mpmath.mpf(0)] * 6    # :52 (H starts zero, :31)
    return row, -_dist(n, D, g)                                 # :55, Match.cpp:21


@functools.lru_cache(maxsize=64)
def _perturbed(x):
    """the transforms of x [+] (+-h e_k) for the 12 error-state coordinates pos, rot, offR, offT, at FD_DPS digits"""
    with mp.workdps(FD_DPS):
        out = []
        for k in range(12):
            pair = []
            for s in (1, -1):
                d = [mpmath.mpf(0)] * K.N
                d[k] = s * FD_STEP
                pair.append(_transforms(tuple(K.boxplus(list(x), d))))
            out.append(pair)
        return out


def rows_fd(x, p, plane, est):
    """the row as the derivative of dist(x [+] delta) at delta = 0 with the plane held fixed (central differences); columns
    6..11 are zero when `est` is off, as in calculate_H"""
    pert = _perturbed(tuple(float(a) for a in x))
    with mp.workdps(FD_DPS):
        p = _vec3(p)
        n, D = _vec3(plane[:3]), K.mpf(float(plane[3]))
        row = []
        for k in range(12 if est else 6):
            hi, lo = pert[k]
            row.append((_dist(n, D, _world(hi, p)) - _dist(n, D, _world(lo, p))) / (2 * FD_STEP))
    return row + [mpmath.mpf(0)] * (12 - len(row))
