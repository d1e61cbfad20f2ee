"""Inputs at the edges of the manifold algebra (csrc/lv_manifold.h) for the step, the IMU propagation and the primitives, each
checked through the 50-digit reference (ikfom_mp.py) to reach the branch it is built for.

Step cases are filter_cases.py dicts (x_prop, P, x_cur, HTH, HTh, nm, R, D, limits, max_iter, est, family) built on
filter_cases.base of a scene, plus "check": a function of the case and ikfom_mp.evaluate's result that asserts the branch.
Primitive rows are (op, inputs, label) for tests/gpu_shim/manifold_ops.h; ref_op() is the 50-digit value of one row."""
import math

import mpmath
import numpy as np
from mpmath import mp

import filter_cases as FC
import ikfom_mp as M

U = 2.0 ** -53
L = 98090.0 / 10000.0                   # the S2 length, as the reference's double
TAYLOR = 2.0 ** -13                     # cos_sinc_sqrt's Taylor bound, sqrt(sqrt(DBL_EPSILON)) (mtkmath.hpp:142-174)
TOL = 1e-11                             # MTK::tolerance<double>()

# op codes of tests/gpu_shim/manifold_ops.h
COS_SINC, SO3_EXP, SO3_LOG, A_MATRIX, S2_BX, S2_BOXPLUS, S2_BOXMINUS, S2_NX, S2_MX, ROT_TO_QUAT, QUAT_TO_ROT, BOXPLUS, \
    BOXMINUS = range(13)
N_IN, N_OUT = 64, 32
N_RES = {COS_SINC: 2, SO3_EXP: 4, SO3_LOG: 3, A_MATRIX: 9, S2_BX: 6, S2_BOXPLUS: 3, S2_BOXMINUS: 2, S2_NX: 6, S2_MX: 6,
         ROT_TO_QUAT: 4, QUAT_TO_ROT: 9, BOXPLUS: 26, BOXMINUS: 23}


# ---- fp64 helpers (only to build inputs) ---------------------------------------------------------------------------------
def qaxis(axis, ang):
    """the unit quaternion (x, y, z, w) of a rotation by ang about axis"""
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    return np.concatenate([math.sin(ang / 2) * a, [math.cos(ang / 2)]])


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def rot(axis, ang):
    """the rotation matrix of qaxis, in 50 digits rounded once"""
    a = [mpmath.mpf(float(v)) for v in np.asarray(axis, np.float64) / np.linalg.norm(axis)]
    return M.to_np(M.qrot(M.exp_q(a, ang)))


def perp(v):
    """a unit vector perpendicular to v"""
    v = np.asarray(v, np.float64)
    e = np.eye(3)[int(np.argmin(np.abs(v)))]
    p = np.cross(v, e)
    return p / np.linalg.norm(p)


def small_offset(seed, rot_scale=0.05):
    """an error-state step that moves every block a little (so dx_ and the J blocks are not trivial)"""
    rng = np.random.default_rng(seed)
    d = np.zeros(23)
    d[0:3] = rng.normal(0, 0.1, 3)
    d[3:9] = rng.normal(0, rot_scale, 6)
    d[9:21] = rng.normal(0, 0.02, 12)
    d[21:23] = rng.normal(0, rot_scale, 2)
    return d


# ---- 50-digit views the checks use ---------------------------------------------------------------------------------------
def mp_trace(q):
    R = M.qrot(M.state(q))
    return R[0, 0] + R[1, 1] + R[2, 2]


def mp_rel_quat(c, f=3):
    """x_prop^-1 x_cur of the SO3 block at flat index f, in 50 digits"""
    xp, xc = M.state(c["x_prop"]), M.state(c["x_cur"])
    return M.qmul(M.qconj(xp[f:f + 4]), xc[f:f + 4])


def mp_s2(c):
    """v_sin, theta of x_cur.grav [-] x_prop.grav (S2.hpp:146-148) in 50 digits"""
    v, o = M.grav(M.state(c["x_cur"])), M.grav(M.state(c["x_prop"]))
    vs = M.norm3(M.hat(v) * o)
    return vs, mpmath.atan2(vs, (v.T * o)[0])


def mp_chart(v):
    """v.x + length, the quantity S2_Bx's branch compares with tol (S2.hpp:217)"""
    return mpmath.mpf(float(v[0])) + M.S2_LEN


# ---- step families ---------------------------------------------------------------------------------------------------------
def _case(b, family, x_prop, x_cur, check, **over):
    return FC.case(b, family, x_prop=x_prop, x_cur=x_cur, check=check, **over)


def _with_rot(x, q, f=3):
    x = x.copy()
    x[f:f + 4] = q
    return x


def _signed(q, s):
    return q if (q[3] > 0) == (s > 0) else -q


def headings(O, b):
    """x_prop yawed across +-pi (world z) and rolled / pitched by 90 and 180 degrees (body x / y), each rotation stored once
    with w > 0 and once with w < 0 (x_cur the same rotation stored with the same sign, a small step away)"""
    xp0 = b["x_prop"]
    rots = [("yaw_%+.4f" % a, qmul(qaxis([0, 0, 1], a), xp0[3:7]))
            for a in (-math.pi, -math.pi / 2, math.pi / 2, 3 * math.pi / 4, math.pi - 1e-3, math.pi)]
    for name, axis in (("roll", [1, 0, 0]), ("pitch", [0, 1, 0])):
        for deg in (90, 180):
            rots.append(("%s_%d" % (name, deg), qmul(xp0[3:7], qaxis(axis, math.radians(deg)))))
    out = []
    for i, (name, q) in enumerate(rots):
        for s in (1, -1):
            xp = _with_rot(xp0, _signed(q, s))
            xc = O.boxplus(xp, small_offset(100 + i))
            xc[3:7] = _signed(xc[3:7], s)
            le0 = bool(mp_trace(xp[3:7]) <= 0)

            def check(c, r, s=s, le0=le0):
                assert (c["x_prop"][3 + 3] < 0) == (s < 0) and (c["x_cur"][3 + 3] < 0) == (s < 0)
                assert bool(mp_trace(c["x_prop"][3:7]) <= 0) == le0
            tag = "trace<=0" if le0 else "trace>0"
            out.append(_case(b, "%s_%s_w%s" % (name, tag, "+" if s > 0 else "-"), xp, xc, check))
    assert sum("trace<=0" in c["family"] for c in out) >= 8
    return out


def iterates(O, b, seed=3):
    """both SO3 blocks of x_cur 1, 2, 3, pi - 1e-3 and pi - 1e-6 rad from x_prop's, about random and axis-aligned axes; past
    pi (pi + 1e-3, 3.5 rad), where log wraps to the shorter rotation; and x_cur stored with the other sign, where the relative
    quaternion has w < 0"""
    rng = np.random.default_rng(seed)
    xp = b["x_prop"]
    out = []
    angles = [1.0, 2.0, 3.0, math.pi - 1e-3, math.pi - 1e-6]
    specs = [(a, "random", rng.normal(size=3), rng.normal(size=3), 1) for a in angles]
    specs += [(a, "axis%d" % (k % 3), np.eye(3)[k % 3], np.eye(3)[(k + 1) % 3], 1) for k, a in enumerate(angles)]
    specs += [(math.pi + 1e-3, "random", rng.normal(size=3), rng.normal(size=3), 1), (3.5, "axis2", [0, 0, 1], [1, 0, 0], 1)]
    specs += [(1.0, "random", rng.normal(size=3), rng.normal(size=3), -1), (math.pi - 1e-6, "axis0", [1, 0, 0], [0, 1, 0], -1)]
    for i, (ang, kind, a1, a2, s) in enumerate(specs):
        xc = O.boxplus(xp, small_offset(200 + i) * np.r_[np.ones(3), np.zeros(6), np.ones(14)])
        xc[3:7] = s * qmul(xp[3:7], qaxis(a1, ang))
        xc[7:11] = s * qmul(xp[7:11], qaxis(a2, ang))

        def check(c, r, ang=ang, s=s):
            for f in (3, 7):
                q = mp_rel_quat(c, f)
                wrapped = ang > math.pi
                assert (q[3] < 0) == (wrapped != (s < 0))            # the relative rotation's w: < 0 past pi or stored negated
                n = M.norm3(M.so3_log(q))
                assert abs(n - (2 * math.pi - ang if wrapped else ang)) < 1e-9
        out.append(_case(b, "iterate_%s_%.6g%s" % (kind, ang, "_neg" if s < 0 else ""), xp, xc, check))
    return out


def gravities(O, b):
    """x_cur.grav 1, 2, 3 rad from x_prop.grav; equal to it (v_sin = 0, theta = 0); at its antipode (v_sin = 0, theta = pi: the
    3.1415926 branch); v_sin 0.9 and 1.1 tol (theta ~1e-12, either side of the v_sin < tol test)"""
    xp = b["x_prop"]
    g = xp[23:26]
    base = O.boxplus(xp, small_offset(300) * np.r_[np.ones(21), np.zeros(2)])
    out = []
    for ang in (1.0, 2.0, 3.0):
        xc = base.copy()
        xc[23:26] = rot(perp(g), ang) @ g

        def check(c, r, ang=ang):
            vs, th = mp_s2(c)
            assert vs > M.TOL and abs(th - ang) < 1e-9
        out.append(_case(b, "grav_%g_rad" % ang, xp, xc, check))
    for name, gc in (("equal", g.copy()), ("antipode", -g)):
        xc = base.copy()
        xc[23:26] = gc

        def check(c, r, anti=name == "antipode"):
            vs, th = mp_s2(c)
            assert vs == 0 and (abs(th) > M.TOL) == anti
            d = M.boxminus(M.state(c["x_cur"]), M.state(c["x_prop"]))
            assert d[21:23] == ([mpmath.mpf("3.1415926"), 0] if anti else [0, 0])
        out.append(_case(b, "grav_%s" % name, xp, xc, check))
    for k in (0.9, 1.1):
        xc = base.copy()
        xc[23:26] = rot(perp(g), k * TOL / L ** 2) @ g

        def check(c, r, below=k < 1):
            vs, th = mp_s2(c)
            assert (vs < M.TOL) == below and vs > 0
        out.append(_case(b, "grav_vsin_%.1ftol" % k, xp, xc, check))
    return out


def chart_gravity(delta_ulps):
    """a gravity vector of the reference's length at S2_Bx's singular direction: exactly (-L, 0, 0) for delta_ulps None; else x
    the first fp64 value with x + L >= tol moved delta_ulps - 1 ulps up (delta_ulps > 0) or -delta_ulps ulps down (< 0), so
    that v.x + L, which fp64 computes exactly there, sits on that side of tol"""
    if delta_ulps is None:
        return np.array([-L, 0.0, 0.0])
    x = -L + TOL
    while x + L < TOL:
        x = np.nextafter(x, 0.0)
    while np.nextafter(x, -20.0) + L >= TOL:
        x = np.nextafter(x, -20.0)
    for _ in range(delta_ulps - 1 if delta_ulps > 0 else -delta_ulps):
        x = np.nextafter(x, 0.0 if delta_ulps > 0 else -20.0)
    x = float(x)
    r = math.sqrt((L - x) * (x + L))
    return np.array([x, r * 0.6, r * 0.8])


def charts(O, b):
    """x_prop.grav at S2_Bx's singular direction: exactly (-L, 0, 0) (the second branch), and with v.x + L 2 ulps above and
    below tol; x_cur.grav equal to it, or 0.1 rad away"""
    xp0 = b["x_prop"]
    out = []
    for du in (None, 2, -2):
        xp = xp0.copy()
        xp[23:26] = chart_gravity(du)
        for off in (0.0, 0.1):
            xc = O.boxplus(xp, small_offset(400) * np.r_[np.ones(21), np.zeros(2)])
            xc[23:26] = xp[23:26] if off == 0 else rot(perp(xp[23:26]), off) @ xp[23:26]
            second = du is None or du < 0

            def check(c, r, second=second):
                assert (mp_chart(c["x_prop"][23:26]) <= M.TOL) == second
            name = "exact" if du is None else "%+dulp" % du
            out.append(_case(b, "chart_%s_%s%s" % (name, "branch2" if second else "branch1", "_off0.1" if off else ""), xp, xc,
                             check))
    return out


def extrinsics(O, b):
    """offset_R_L_I 180 degrees about z and 90 degrees about x, with estimate_extrinsics on"""
    out = []
    for name, q in (("Rz180", qaxis([0, 0, 1], math.pi)), ("Rx90", qaxis([1, 0, 0], math.pi / 2))):
        xp = _with_rot(b["x_prop"], q, 7)
        xc = O.boxplus(xp, small_offset(500))

        def check(c, r, le0=name == "Rz180"):
            assert bool(mp_trace(c["x_prop"][7:11]) <= 0) == le0
        out.append(_case(b, "extrinsic_%s" % name, xp, xc, check, est=1))
    return out


def tolerances(O, b):
    """rotation offsets of norm 0.9 and 1.1 tol (A_matrix's norm < tol test on dx) in both SO3 blocks, and of norm exactly 0
    (x_cur's quaternions x_prop's: log's nv < tol and A_matrix's norm < tol guard 0 / 0 there)"""
    xp = b["x_prop"]
    out = []
    for k in (0.0, 0.9, 1.1):
        xc = O.boxplus(xp, small_offset(600) * np.r_[np.ones(3), np.zeros(6), np.ones(14)])
        xc[3:7] = qmul(xp[3:7], qaxis([0.48, -0.6, 0.64], k * TOL)) if k else xp[3:7]
        xc[7:11] = qmul(xp[7:11], qaxis([0.0, 0.6, 0.8], k * TOL)) if k else xp[7:11]

        def check(c, r, k=k):
            for e in (3, 6):                                      # dx = x_cur [-] x_prop, whose A_matrix the J block takes
                n = M.norm3(M.boxminus(c["x_cur"], c["x_prop"])[e:e + 3])
                assert (n < M.TOL) == (k < 1) and (n == 0) == (k == 0)
        out.append(_case(b, "rot_norm_%.1ftol" % k, xp, xc, check))
    return out


def step_cases(O, b):
    return headings(O, b) + iterates(O, b) + gravities(O, b) + charts(O, b) + extrinsics(O, b) + tolerances(O, b)


def heading_states(O, b):
    """the x_prop of every heading case (both signs), with non-zero biases, for the IMU propagation"""
    out = []
    for c in headings(O, b):
        x = c["x_prop"].copy()
        x[17:23] = [0.01, -0.02, 0.015, 0.05, -0.03, 0.04]
        out.append((c["family"], x))
    return out


# ---- primitive rows --------------------------------------------------------------------------------------------------------
def taylor_x2(k):
    """fp64 x2 values k ulps from 2^-13 (k < 0 below)"""
    x = TAYLOR
    for _ in range(abs(k)):
        x = np.nextafter(x, 0.0 if k < 0 else 1.0)
    return float(x)


def taylor_omega(k, h=2.0 ** -8):
    """w such that so3_exp's argument (h h) (w w) for the gyro (w, 0, 0) is the |k|-th fp64 value below 2^-13 (k < 0) or the
    (k+1)-th at or above it (k >= 0); h = 2^-8 is half of dt = 2^-7, so h h is exact"""
    w0 = math.sqrt(TAYLOR) / h
    ws, x, y = [w0], w0, w0
    for _ in range(12):
        x, y = np.nextafter(x, 0.0), np.nextafter(y, 10.0)
        ws += [float(x), float(y)]
    ws.sort()
    below = [w for w in ws if (h * h) * (w * w) < TAYLOR]
    above = [w for w in ws if (h * h) * (w * w) >= TAYLOR]
    return below[k] if k < 0 else above[k]


def primitive_rows(O, states, seed=11):
    """(op, inputs, label) rows at the edges of each function; `states`: flat states (x_prop of the heading and chart cases)"""
    rng = np.random.default_rng(seed)
    rows = []

    def add(op, inp, label):
        rows.append((op, np.asarray(inp, np.float64), label))
    for k in (-4, -2, -1, 0, 1, 2, 4):                             # the Taylor bound of cos_sinc_sqrt
        add(COS_SINC, [taylor_x2(k)], "taylor_%+d" % k)
    for x2 in np.geomspace(TAYLOR / 2, TAYLOR * 2, 64):
        add(COS_SINC, [x2], "taylor_band")
    for x2 in (0.0, 1e-30, 1e-8, 0.25, 2.0, 9.0, 9.8):
        add(COS_SINC, [x2], "cos_sinc")
    for k in (-2, -1, 0, 1, 2):                                    # so3_exp with half^2 |v|^2 at the bound, axis-aligned v
        add(SO3_EXP, [taylor_omega(k), 0, 0, 2.0 ** -8], "exp_taylor_%+d" % k)
    for ang in (1e-12, 1e-6, 0.5, 1.0, 2.0, 3.0, math.pi - 1e-6, math.pi, 3.5, 6.0):
        a = rng.normal(size=3)
        add(SO3_EXP, list(ang * a / np.linalg.norm(a)) + [0.5], "exp")
    for ang in (1.0, 2.0, 3.0, math.pi - 1e-3, math.pi - 1e-6, math.pi + 1e-3, 3.5, 5.0):
        for s in (1, -1):                                          # stored with w > 0 and w < 0
            a = rng.normal(size=3)
            add(SO3_LOG, s * qaxis(a, ang), "log_%s" % ("w+" if s * math.cos(ang / 2) > 0 else "w-"))
    for nv in (0.0, 1e-300, 0.9 * TOL, TOL, 1.1 * TOL, 1e-6):       # log's nv < tol clamp, nv = 0 included
        for s in (1, -1):
            v = np.array([0.48, -0.6, 0.64]) * nv
            add(SO3_LOG, list(v) + [s * math.sqrt(1 - nv * nv)], "log_nv")
    for nrm in (0.0, 1e-300, 0.9 * TOL, 1.1 * TOL, 1e-6, 1e-3, 1.0, 3.0, math.pi - 1e-6, 5.0):
        add(A_MATRIX, nrm * np.array([0.48, -0.6, 0.64]), "A_%g" % nrm)
    gravs = [chart_gravity(None), chart_gravity(2), chart_gravity(-2), chart_gravity(1), chart_gravity(-1)]
    gravs += [s[23:26] for s in states] + [np.array([0, 0, -L]), np.array([L, 0, 0]), np.array([0, L, 0])]
    for _ in range(8):
        g = rng.normal(size=3)
        gravs.append(g / np.linalg.norm(g) * L)
    for g in gravs:
        tag = "branch2" if g[0] + L <= TOL else "branch1"
        add(S2_BX, g, "Bx_" + tag)
        add(S2_NX, g, "Nx_" + tag)
        d = rng.normal(0, 0.3, 2)
        add(S2_MX, list(g) + list(d), "Mx_" + tag)
        add(S2_MX, list(g) + [0, 0], "Mx0_" + tag)
        add(S2_BOXPLUS, list(g) + list(d), "s2plus_" + tag)
        for ang in (1.0, 3.0):
            add(S2_BOXMINUS, list(rot(perp(g), ang) @ g) + list(g), "s2minus_" + tag)
        add(S2_BOXMINUS, list(g) + list(g), "s2minus_equal")
        add(S2_BOXMINUS, list(-g) + list(g), "s2minus_antipode")
    for axis, ang in (([0, 0, 1], math.pi), ([1, 0, 0], math.pi), ([0, 1, 0], math.pi), ([1, 1, 0], math.pi), ([1, 2, 3], 2.5),
                      ([1, -1, 1], 2 * math.pi / 3), ([3, -1, 2], 2.2), ([0, 0, 1], 0.5), ([1, 0, 0], math.pi / 2)):
        R = rot(axis, ang)
        add(ROT_TO_QUAT, R.reshape(-1), "r2q_trace%s" % ("<=0" if np.trace(R) <= 0 else ">0"))
    for q in (qaxis([1, 2, 3], 2.5), -qaxis([1, 2, 3], 2.5), np.array([0.1, -0.2, 0.3, -0.9])):
        add(QUAT_TO_ROT, q, "q2r")
    for s in states:
        for ang in (1.0, 3.0, math.pi - 1e-6, 3.5):
            d = small_offset(int(rng.integers(1 << 30)))
            a = rng.normal(size=6)
            d[3:6], d[6:9] = ang * a[:3] / np.linalg.norm(a[:3]), ang * a[3:] / np.linalg.norm(a[3:])
            add(BOXPLUS, list(s) + list(d), "boxplus")
            y = O.boxplus(s, d)
            add(BOXMINUS, list(y) + list(s), "boxminus")
        for k in (-1, 0, 1):                                       # |d_rot|^2 / 4 at the Taylor bound
            d = np.zeros(23)
            d[3] = taylor_omega(k, 0.5)
            add(BOXPLUS, list(s) + list(d), "boxplus_taylor")
    return rows


def pack(rows):
    ops = np.array([r[0] for r in rows], np.int32)
    inp = np.zeros((len(rows), N_IN))
    for i, r in enumerate(rows):
        inp[i, :len(r[1])] = r[1]
    return ops, inp


def mp_rot_to_quat(R):
    """Eigen's Quaternion(Matrix3) (Shepperd's method: trace > 0, else from the largest diagonal entry) in 50 digits"""
    R = [[mpmath.mpf(float(R[i][j])) for j in range(3)] for i in range(3)]
    q = [0, 0, 0, 0]
    t = R[0][0] + R[1][1] + R[2][2]
    if t > 0:
        t = mpmath.sqrt(t + 1)
        q[3] = t / 2
        t = mpmath.mpf(1) / 2 / t
        q[0], q[1], q[2] = (R[2][1] - R[1][2]) * t, (R[0][2] - R[2][0]) * t, (R[1][0] - R[0][1]) * t
    else:
        i = 0
        if R[1][1] > R[0][0]:
            i = 1
        if R[2][2] > R[i][i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = mpmath.sqrt(R[i][i] - R[j][j] - R[k][k] + 1)
        q[i] = t / 2
        t = mpmath.mpf(1) / 2 / t
        q[3] = (R[k][j] - R[j][k]) * t
        q[j] = (R[j][i] + R[i][j]) * t
        q[k] = (R[k][i] + R[i][k]) * t
    return q


def ref_op(op, inp):
    """the 50-digit value of one row (a list of mpf, N_RES[op] long)"""
    v = [mpmath.mpf(float(a)) for a in inp]
    if op == COS_SINC:
        x = mpmath.sqrt(v[0])
        return [mpmath.cos(x), mpmath.sin(x) / x if x != 0 else mpmath.mpf(1)]
    if op == SO3_EXP:
        return M.exp_q(v[0:3], 2 * v[3])
    if op == SO3_LOG:
        return M.so3_log(v[0:4])
    if op == A_MATRIX:
        A = M.A_matrix(v[0:3])
        return [A[i, j] for i in range(3) for j in range(3)]
    if op == S2_BX:
        B = M.s2_Bx(mp.matrix(v[0:3]))
        return [B[i, j] for i in range(3) for j in range(2)]
    if op == S2_NX:
        N = M.s2_Nx_yy(mp.matrix(v[0:3]))
        return [N[i, j] for i in range(2) for j in range(3)]
    if op == S2_MX:
        X = M.s2_Mx(mp.matrix(v[0:3]), v[3:5])
        return [X[i, j] for i in range(3) for j in range(2)]
    if op == S2_BOXPLUS:
        g = M.s2_boxplus(mp.matrix(v[0:3]), v[3:5])
        return [g[0], g[1], g[2]]
    if op == S2_BOXMINUS:
        return M.s2_boxminus(mp.matrix(v[0:3]), mp.matrix(v[3:6]))
    if op == ROT_TO_QUAT:
        return mp_rot_to_quat(np.asarray(inp[:9]).reshape(3, 3))
    if op == QUAT_TO_ROT:
        R = M.qrot(v[0:4])
        return [R[i, j] for i in range(3) for j in range(3)]
    if op == BOXPLUS:
        return M.boxplus(v[0:26], v[26:49])
    if op == BOXMINUS:
        return M.boxminus(v[0:26], v[26:52])
    raise ValueError(op)


# the blocks of a flat state (x, 26) and of an error state (d, 23): (start, end, kind)
X_BLOCKS = ((0, 3, "vect"), (3, 7, "so3"), (7, 11, "so3"), (11, 14, "vect"), (14, 17, "vect"), (17, 20, "vect"), (20, 23, "vect"),
            (23, 26, "s2"))
D_BLOCKS = ((0, 3, "vect"), (3, 6, "so3"), (6, 9, "so3"), (9, 12, "vect"), (12, 15, "vect"), (15, 18, "vect"), (18, 21, "vect"),
            (21, 23, "s2"))


def bar(op, inp, ref):
    """the bar of each output entry of one row: 4 ulps of the output's largest entry (the reference's own fp64 rounding), one
    more where the product takes S2_Bx's reciprocal (DESIGN section 2), plus A_matrix's cancellation in (1 - cos n) / n^2 at
    small n (U / n), which the reference's formula carries too.  The 23-state boxplus and boxminus are held block by block: 4
    ulps of each block's largest entry, 5 for the S2 block, and 8 for the SO3 blocks, whose Hamilton product adds 4-term sums
    (4 ulps of |q| = 1) to exp's or log's own; boxminus's SO3 and S2 blocks are angles computed from products of unit-size
    quantities, so there the ulps are of max(|block|, 1 rad)."""
    n_out = N_RES[op]
    r = np.array([abs(float(a)) for a in ref])
    if op in (BOXPLUS, BOXMINUS):
        b = np.zeros(n_out)
        for s, e, kind in (X_BLOCKS if op == BOXPLUS else D_BLOCKS):
            scale = r[s:e].max()
            if op == BOXMINUS and kind != "vect":
                scale = max(scale, 1.0)
            b[s:e] = {"vect": 4.0, "so3": 8.0, "s2": 5.0}[kind] * U * scale
        return b
    k = 5.0 if op in (S2_BX, S2_NX, S2_MX, S2_BOXPLUS, S2_BOXMINUS) else 4.0
    b = k * U * r.max()
    if op == A_MATRIX:
        n = float(np.linalg.norm(inp[:3]))
        b += 2 * U / n if n > 0 else 0.0
    return np.full(n_out, b)


# ---- checks shared by the host-build and device tests -----------------------------------------------------------------------
def check_primitive_branch(op, inp, label):
    """assert that a primitive row reaches the branch its label names (50-digit or exact fp64 quantities)"""
    if label.startswith("taylor_") and label != "taylor_band":
        assert (inp[0] < TAYLOR) == label.startswith("taylor_-")
    if label.startswith("exp_taylor_"):
        assert ((inp[3] * inp[3]) * (inp[0] * inp[0]) < TAYLOR) == label.startswith("exp_taylor_-")
    if label.startswith("log_w"):
        assert (inp[3] < 0) == label.endswith("-")
    if label.endswith("branch2") or label.endswith("branch1"):
        v = inp[3:6] if op == S2_BOXMINUS else inp[:3]             # boxminus takes the chart at o
        assert (mp_chart(v) <= M.TOL) == label.endswith("branch2")
    if label in ("s2minus_equal", "s2minus_antipode"):
        v, o = mp.matrix([mpmath.mpf(float(a)) for a in inp[0:3]]), mp.matrix([mpmath.mpf(float(a)) for a in inp[3:6]])
        assert M.norm3(M.hat(v) * o) == 0
    if label.startswith("r2q_trace"):
        assert (inp[0] + inp[4] + inp[8] <= 0) == label.endswith("<=0")


def primitive_errors(rows, out):
    """per label: the largest error / bar over the rows' entries against the 50-digit reference (each row's branch checked
    first).  A non-finite output counts as inf, so a missing 0 / 0 guard cannot pass."""
    worst = {}
    for i, (op, inp, label) in enumerate(rows):
        check_primitive_branch(op, inp, label)
        ref = ref_op(op, inp)
        got = out[i, :N_RES[op]]
        if not np.isfinite(got).all():
            worst[label] = math.inf
            continue
        err = np.array([float(abs(mpmath.mpf(float(got[j])) - ref[j])) for j in range(N_RES[op])])
        b = bar(op, inp, ref)
        ratio = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err > 0, math.inf, 0.0))
        worst[label] = max(worst.get(label, 0.0), float(ratio.max()))
    return worst


C_BAR = 8           # the step's bars: C_BAR * kappa * 2^-53, as test_gpu_filter.test_step_against_mp


def _err(a, m):
    return float(np.abs(a - m).max() / max(np.abs(m).max(), 1e-300))


def step_errors(c, r, dx, x):
    """dx_ and the new iterate (relative to max(1, |dx_no_degenerate_|)) against ikfom_mp.evaluate's result r"""
    xs = max(1.0, float(np.abs(M.to_np(r["dnd"])).max()))
    return dict(dx=_err(dx, M.to_np(r["dx"])), x=float(np.abs(x - M.to_np(r["x"])).max()) / xs)


def print_step_table(rows, title):
    print("\n%-38s %9s %9s  %-29s %-29s" % ("family", "kappa", "bar", title, "oracle vs mp (dx, x, P)"))
    for f, kappa, e, eo in rows:
        print("%-38s %9.1e %9.1e  %8.1e %8.1e %8.1e    %8.1e %8.1e %8.1e" % (f, kappa, C_BAR * kappa * U, e["dx"], e["x"], e["P"],
                                                                         eo["dx"], eo["x"], eo["P"]))


# ---- IMU propagation ---------------------------------------------------------------------------------------------------------
def imu_samples(seed, x, k, rates):
    """k samples from state x; rates: |omega| dt per sample (dt cycles through 2.5e-3, 0.02, 0.05)"""
    rng = np.random.default_rng(seed)
    dts = np.array([(2.5e-3, 0.02, 0.05)[i % 3] for i in range(k)])
    acc = -x[23:26] + rng.normal(0, 0.5, (k, 3))
    gyr = np.zeros((k, 3))
    for i in range(k):
        a = rng.normal(size=3)
        gyr[i] = rates[i % len(rates)] / dts[i] * a / np.linalg.norm(a)
    return acc, gyr, dts


def spin_run(x0, n=20000, dt=2.5e-3, rate=10.0, seed=21):
    """n samples at 1 / dt spinning at `rate` rad/s about a fixed tilted body axis, the specific force that holds the
    velocity still (R_k^T (-grav) plus 0.05 m/s^2 of noise); x0's biases are zero, so omega is the gyro"""
    rng = np.random.default_rng(seed)
    axis = np.array([0.3, -0.4, 0.866])
    axis /= np.linalg.norm(axis)
    w = rate * axis
    gyr = np.tile(w, (n, 1))
    R0 = M.to_np(M.qrot(M.state(x0[3:7])))
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    acc = np.zeros((n, 3))
    for k in range(n):
        th = k * dt * rate
        Rk = R0 @ (np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K)
        acc[k] = Rk.T @ (-x0[23:26]) + rng.normal(0, 0.05, 3)
    return acc, gyr, np.full(n, dt)


def mp_propagate_state(x, acc, gyr, dts, dps=30):
    """the state part of esekf::predict (x [+] f dt, esekfom.hpp:287 with use-ikfom.cpp:49-61) over all samples, in dps
    digits; biases and gravity as in x (constant)"""
    with mp.workdps(dps):
        x = M.state(x)
        g0 = M.grav(x)
        bg = [x[17 + i] for i in range(3)]
        ba = [x[20 + i] for i in range(3)]
        for k in range(len(dts)):
            dt = mpmath.mpf(float(dts[k]))
            R = M.qrot(x[3:7])
            a_in = R * mp.matrix([mpmath.mpf(float(acc[k, i])) - ba[i] for i in range(3)])
            om = [mpmath.mpf(float(gyr[k, i])) - bg[i] for i in range(3)]
            for i in range(3):
                x[i] += dt * x[14 + i]
                x[14 + i] += dt * (a_in[i] + g0[i])
            x[3:7] = M.qmul(x[3:7], M.exp_q(om, dt))
        return x


def _ld_hat(v):
    z = np.longdouble(0)
    return np.array([[z, -v[2], v[1]], [v[2], z, -v[0]], [-v[1], v[0], z]], dtype=np.longdouble)


def _ld_A(v):
    n2 = v @ v
    n = np.sqrt(n2)
    if n < TOL:
        return np.eye(3, dtype=np.longdouble)
    H = _ld_hat(v)
    return np.eye(3, dtype=np.longdouble) + (1 - np.cos(n)) / n2 * H + (1 - np.sin(n) / n) / n2 * H @ H


def _ld_Bx(v):
    Lq = np.longdouble(L)
    if v[0] + Lq > TOL:
        d = Lq + v[0]
        return np.array([[-v[1], -v[2]], [Lq - v[1] * v[1] / d, -v[2] * v[1] / d], [-v[2] * v[1] / d, Lq - v[2] * v[2] / d]],
                        dtype=np.longdouble) / Lq
    B = np.zeros((3, 2), dtype=np.longdouble)
    B[1, 1], B[2, 0] = -1, 1
    return B


def _ld_qrot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], dtype=np.longdouble)


def _ld_qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz], dtype=np.longdouble)


def ld_predict(x, P, acc, gyr, dts, noise):
    """esekf::predict (ikfom_mp.predict's F and G, dense) over all samples in np.longdouble (64-bit significand); x, P:
    longdouble arrays, updated and returned"""
    ld = np.longdouble
    x, P = np.array(x, dtype=ld), np.array(P, dtype=ld).reshape(23, 23)
    Qd = np.array([noise[0]] * 3 + [noise[1]] * 3 + [noise[2]] * 3 + [noise[3]] * 3, dtype=ld)
    I3 = np.eye(3, dtype=ld)
    for k in range(len(dts)):
        dt = ld(dts[k])
        q = x[3:7]
        R = _ld_qrot(q)
        g0 = x[23:26].copy()
        om = np.array(gyr[k], dtype=ld) - x[17:20]
        a_b = np.array(acc[k], dtype=ld) - x[20:23]
        a_in = R @ a_b
        B = _ld_Bx(g0)
        Mx0 = -_ld_hat(g0) @ B
        Nx = 1 / (ld(L) * ld(L)) * B.T @ _ld_hat(g0)
        A = _ld_A(-om * dt)
        F = np.eye(23, dtype=ld)
        F[0:3, 12:15] += dt * I3
        F[12:15, 3:6] += -(R @ _ld_hat(a_b)) * dt
        F[12:15, 18:21] += -R * dt
        F[12:15, 21:23] += Mx0 * dt
        F[3:6, 15:18] += -A * dt
        F[21:23, 21:23] = Nx @ Mx0
        G = np.zeros((23, 12), dtype=ld)
        G[12:15, 3:6] = -R * dt
        G[3:6, 0:3] = -A * dt
        G[15:18, 6:9] = dt * I3
        G[18:21, 9:12] = dt * I3
        P = F @ P @ F.T + (G * Qd) @ G.T
        x[0:3] += dt * x[14:17]
        x[14:17] += dt * (a_in + g0)
        th = np.sqrt(om @ om) * dt / 2
        sc = np.sin(th) / th * dt / 2 if th != 0 else dt / 2
        x[3:7] = _ld_qmul(q, np.concatenate([sc * om, [np.cos(th)]]))
    return x, P
