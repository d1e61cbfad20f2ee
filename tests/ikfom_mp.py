"""IKFoM for the LIMO-Velo state in 50-digit arithmetic (mpmath): the yardstick the fp64 filter kernels are measured against.

Written from the reference's text, not from the product's headers or the oracle, so that it is independent of both.  Line
numbers cite the reference (include/IKFoM/...): esekfom.hpp (esekf::predict, update_iterated_dyn_share_modified), mtkmath.hpp
(A_matrix, exp, log), SOn.hpp (SO3), S2.hpp (S2<double, 98090, 10000, 1>), build_manifold.hpp (state boxplus / oplus),
use-ikfom.cpp (f, df_dx, df_dw).

Flat state: 26 numbers, [0:3) pos [3:7) rot (x, y, z, w) [7:11) offset_R_L_I [11:14) offset_T_L_I [14:17) vel [17:20) bg
[20:23) ba [23:26) grav; error state: 23, pos 0 rot 3 offR 6 offT 9 vel 12 bg 15 ba 18 grav 21 (use-ikfom.hpp:12-21).
Arguments may be floats or mpf; results are mpf (states: lists, matrices: mp.matrix).  to_np() rounds to float64.
"""
import mpmath
import numpy as np
from mpmath import mp

mp.dps = 50

N = 23
TOL = mpmath.mpf("1e-11")               # MTK::tolerance<double>() (mtkmath.hpp:122)
S2_LEN = mpmath.mpf(98090.0 / 10000.0)  # S2<double, 98090, 10000, 1>: length = scalar(den) / scalar(num) (S2.hpp:104), a
                                        # double: 9.809 - 7.2e-16.  Near the chart's edge (v.x + length <= tol, S2.hpp:217) that
                                        # rounding is a relative 1e-4 of the chart, so the restatement takes the reference's double
SO3_IDX = (3, 6)
S2_IDX = 21
_Q = {3: 3, 6: 7}                       # error-state index -> flat index of the quaternion
_VECT = ((0, 0), (9, 11), (12, 14), (15, 17), (18, 20))   # (error-state index, flat index) of the vect3 blocks


def mpf(v):
    return mpmath.mpf(v) if not isinstance(v, mpmath.mpf) else v


def vec(v):
    return mp.matrix([mpf(float(a)) if not isinstance(a, mpmath.mpf) else a for a in v])


def mat(A):
    A = np.asarray(A) if not isinstance(A, mp.matrix) else A
    if isinstance(A, mp.matrix):
        return A.copy()
    M = mp.matrix(A.shape[0], A.shape[1])
    for i in range(A.shape[0]):
        for j in range(A.shape[1]):
            M[i, j] = mpf(float(A[i, j]))
    return M


def to_np(A):
    if isinstance(A, mp.matrix):
        return np.array([[float(A[i, j]) for j in range(A.cols)] for i in range(A.rows)]).squeeze() \
            if A.cols > 1 else np.array([float(A[i]) for i in range(A.rows)])
    return np.array([float(a) for a in A])


def state(x):
    return [mpf(float(a)) if not isinstance(a, mpmath.mpf) else a for a in x]


# ---- SO3 / mtkmath ------------------------------------------------------------------------------------------------------
def hat(v):                                                     # mtkmath.hpp hat()
    return mp.matrix([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


def norm3(v):
    return mpmath.sqrt(v[0] ** 2 + v[1] ** 2 + v[2] ** 2)


def A_matrix(v):                                                # mtkmath.hpp:236-247
    sq = v[0] ** 2 + v[1] ** 2 + v[2] ** 2
    nv = mpmath.sqrt(sq)
    if nv < TOL:
        return mp.eye(3)
    H = hat(v)
    return mp.eye(3) + (1 - mpmath.cos(nv)) / sq * H + (1 - mpmath.sin(nv) / nv) / sq * H * H


def exp_q(v, scale):
    """MTK::exp (mtkmath.hpp:250-256) as used by SO3::exp (SOn.hpp:283-287): quaternion (x, y, z, w) of the rotation
    v * scale; `scale` is what SO3::exp receives (it passes scale / 2 on)"""
    half = mpf(scale) / 2
    th = norm3(v) * abs(half)
    c = mpmath.cos(th)
    sinc = mpmath.sin(th) / th if th != 0 else mpf(1)
    m = sinc * half
    return [m * v[0], m * v[1], m * v[2], c]


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return [aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
            aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz]


def qconj(q):
    return [-q[0], -q[1], -q[2], q[3]]


def qrot(q):
    """Eigen::Quaternion::toRotationMatrix (unit quaternion)"""
    x, y, z, w = q
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                      [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def so3_log(q):                                                 # SOn.hpp:293-297 -> mtkmath.hpp:268-285, scale 2, +-periodic
    nv = mpmath.sqrt(q[0] ** 2 + q[1] ** 2 + q[2] ** 2)
    if nv < TOL:
        nv = TOL
    s = 2 / nv * mpmath.atan(nv / q[3])
    return [s * q[0], s * q[1], s * q[2]]


# ---- S2<double, 98090, 10000, 1> ----------------------------------------------------------------------------------------
def s2_Bx(v):                                                   # S2.hpp:217-230 (S2_typ 1)
    L = S2_LEN
    if v[0] + L > TOL:
        d = L + v[0]
        B = mp.matrix([[-v[1], -v[2]], [L - v[1] * v[1] / d, -v[2] * v[1] / d], [-v[2] * v[1] / d, L - v[2] * v[2] / d]])
        return B / L
    B = mp.matrix(3, 2)
    B[1, 1] = -1
    B[2, 0] = 1
    return B


def s2_boxplus(v, delta):                                       # S2.hpp:136-142, scale 1 -> exp(Bu, 1/2): angle |Bu|
    Bu = s2_Bx(v) * mp.matrix([delta[0], delta[1]])
    return qrot(exp_q(Bu, 1)) * v


def s2_boxminus(v, o):                                          # S2.hpp:144-167: v [-] o
    c = hat(v) * o
    v_sin = norm3(c)
    v_cos = (v.T * o)[0]
    theta = mpmath.atan2(v_sin, v_cos)
    if v_sin < TOL:
        return [mpf("3.1415926"), mpf(0)] if abs(theta) > TOL else [mpf(0), mpf(0)]
    r = theta / v_sin * s2_Bx(o).T * hat(o) * v
    return [r[0], r[1]]


def s2_Nx_yy(v):                                                # S2.hpp:259-264
    return 1 / S2_LEN ** 2 * s2_Bx(v).T * hat(v)


def s2_Mx(v, delta):
    """S2.hpp:266-280.  The rotation exp(Bu) there is taken with scale scalar(1/2), an integer division: 0, so it is the
    identity and Mx = -hat(v) A(Bu)^T Bx."""
    Bx = s2_Bx(v)
    dn = mpmath.sqrt(mpf(delta[0]) ** 2 + mpf(delta[1]) ** 2)
    if dn < TOL:
        return -hat(v) * Bx
    Bu = Bx * mp.matrix([delta[0], delta[1]])
    return -(qrot(exp_q(Bu, 0)) * hat(v) * A_matrix(Bu).T * Bx)


# ---- the state (build_manifold.hpp:192-199) -----------------------------------------------------------------------------
def grav(x):
    return mp.matrix([x[23], x[24], x[25]])


def boxplus(x, d):
    """x [+] d, field by field: vect3 +=, SO3 *= exp(d) (SOn.hpp:233-236), S2 boxplus"""
    x = state(x)
    d = [mpf(a) for a in d]
    for e, f in _VECT:
        for i in range(3):
            x[f + i] = x[f + i] + d[e + i]
    for e in SO3_IDX:
        f = _Q[e]
        x[f:f + 4] = qmul(x[f:f + 4], exp_q(d[e:e + 3], 1))
    g = s2_boxplus(grav(x), d[21:23])
    x[23:26] = [g[0], g[1], g[2]]
    return x


def boxminus(x, y):
    """x [-] y (SOn.hpp:237-239: log(y^-1 x); S2.hpp:144-167)"""
    x, y = state(x), state(y)
    d = [mpf(0)] * N
    for e, f in _VECT:
        for i in range(3):
            d[e + i] = x[f + i] - y[f + i]
    for e in SO3_IDX:
        f = _Q[e]
        d[e:e + 3] = so3_log(qmul(qconj(y[f:f + 4]), x[f:f + 4]))
    d[21:23] = s2_boxminus(grav(x), grav(y))
    return d


def _block_J(e, dx, x_now, x_prop):
    """the J block of error-state block e (esekfom.hpp:1659-1697, 1769-1815): A(dx_e)^T for SO3, Nx(x_now) Mx(x_prop, dx_e)
    for S2"""
    if e in SO3_IDX:
        return A_matrix(dx[e:e + 3]).T
    return s2_Nx_yy(grav(x_now)) * s2_Mx(grav(x_prop), dx[21:23])


def _dim(e):
    return 3 if e in SO3_IDX else 2


def _apply_rows(M, e, J, cols):
    d = _dim(e)
    B = mp.matrix(d, cols)
    for i in range(d):
        for j in range(cols):
            B[i, j] = M[e + i, j]
    B = J * B
    for i in range(d):
        for j in range(cols):
            M[e + i, j] = B[i, j]


def _apply_cols(M, e, J, rows):
    d = _dim(e)
    B = mp.matrix(rows, d)
    for i in range(rows):
        for j in range(d):
            B[i, j] = M[i, e + j]
    B = B * J.T
    for i in range(rows):
        for j in range(d):
            M[i, e + j] = B[i, j]


# ---- one evaluation of update_iterated_dyn_share_modified ---------------------------------------------------------------
def sym_eig_sorted(A6):
    """eigenpairs of the symmetric 6x6 block, ascending, each vector's largest-magnitude component positive.  Eigen's
    EigenSolver leaves the order and the signs unspecified; the product's degenerate branch uses this convention."""
    E, Q = mp.eigsy(A6)
    order = sorted(range(6), key=lambda j: E[j])
    V = mp.matrix(6, 6)
    ev = []
    for jj, j in enumerate(order):
        ev.append(E[j])
        col = [Q[k, j] for k in range(6)]
        imax = max(range(6), key=lambda k: abs(col[k]))
        sg = -1 if col[imax] < 0 else 1
        for k in range(6):
            V[k, jj] = sg * col[k]
    return ev, V


def evaluate(x_prop, P_prop, x_cur, HTH, HTh, R, D, limits, it, t, max_iter):
    """One pass of the loop body, esekfom.hpp:1647-1817, for Nm >= 23 (the else branch of :1701), in the reference's own form
    (two 23x23 inverses).  it: the loop variable i (-1 first), t: converged evaluations so far.  Returns a dict:
      dx (dx_ of :1733), dnd (dx_no_degenerate_, :1743-1744), x (the new iterate), conv (dyn_share.converge after :1762),
      t, finish (:1764), P (the exit block's covariance, or None), degenerate (some eigenvalue < D), eig (ascending),
      kappa (2-norm condition numbers of P_, of P_temp and of I + HTH P_[:12, :12] / R, the 12x12 system the
      matrix-inversion-lemma form of the gain solves instead of the two inverses)."""
    R, D = mpf(R), mpf(D)
    xp, xc = state(x_prop), state(x_cur)
    dx = boxminus(xc, xp)                                       # :1651-1652
    dx_new = mp.matrix(dx)
    P_ = mat(P_prop)                                            # :1655
    for e in SO3_IDX + (S2_IDX,):                               # :1659-1697
        J = _block_J(e, dx, xc, xp)
        d = _dim(e)
        seg = J * mp.matrix([dx_new[e + i] for i in range(d)])
        for i in range(d):
            dx_new[e + i] = seg[i]
        _apply_rows(P_, e, J, N)
        _apply_cols(P_, e, J, N)
    H = mat(HTH)
    Hh = mat(np.asarray(HTh, dtype=np.float64).reshape(12, 1)) if not isinstance(HTh, mp.matrix) else HTh
    P_temp = mp.inverse(P_ / R)                                 # :1722-1726
    for i in range(12):
        for j in range(12):
            P_temp[i, j] += H[i, j]
    P_inv = mp.inverse(P_temp)
    P12 = P_inv[:, 0:12]
    K_h = P12 * Hh                                              # :1727 (h_x^T h = HTh)
    K_x = mp.matrix(N, N)
    KxH = P12 * H                                               # :1729
    for i in range(N):
        for j in range(12):
            K_x[i, j] = KxH[i, j]
    dx_ = K_h + (K_x - mp.eye(N)) * dx_new                      # :1733
    # degeneracy, :1736-1744
    A6 = H[0:6, 0:6]
    ev, V = sym_eig_sorted(A6)
    prod = mpf(1)
    for v in ev:
        prod *= v
    if prod < mpf("1e-20"):
        V = mp.eye(6)
    sel = V.copy()
    for j in range(6):
        if ev[j] < D:
            for c in range(6):
                sel[j, c] = 0
    head = mp.inverse(V) * sel * dx_[0:6, 0]
    dnd = [dx_[i] for i in range(N)]
    for i in range(6):
        dnd[i] = head[i]
    x_new = boxplus(xc, dnd)                                    # :1747
    conv = all(abs(dx_[i]) <= mpf(limits[i]) for i in range(N))  # :1748-1756
    t = t + (1 if conv else 0)                                  # :1757
    if not t and it == max_iter - 2:                            # :1759-1762
        conv = True
    finish = t > 1 or it == max_iter - 1                        # :1764
    P_out = None
    if finish:                                                  # :1766-1817
        L_ = P_.copy()
        Kx = K_x.copy()
        dxl = [dx_[i] for i in range(N)]
        for e in SO3_IDX + (S2_IDX,):
            J = _block_J(e, dxl, x_new, xp)
            d = _dim(e)
            for i in range(N):                                  # L_ rows = J * P_ rows
                col = J * mp.matrix([P_[e + a, i] for a in range(d)])
                for a in range(d):
                    L_[e + a, i] = col[a]
            for i in range(12):
                col = J * mp.matrix([Kx[e + a, i] for a in range(d)])
                for a in range(d):
                    Kx[e + a, i] = col[a]
            _apply_cols(L_, e, J, N)
            _apply_cols(P_, e, J, N)
        P_out = L_ - Kx[:, 0:12] * P_[0:12, :]
    return dict(dx=[dx_[i] for i in range(N)], dnd=dnd, x=x_new, conv=bool(conv), t=t, finish=bool(finish), P=P_out,
                degenerate=any(v < D for v in ev), eig=ev, prod=prod,
                kappa=(cond2(P_), cond2(P_temp), cond2(mp.eye(12) + H * P_[0:12, 0:12] / R)))


def cond2(A):
    s = mp.svd_r(A, compute_uv=False)
    s = [abs(v) for v in s]
    return max(s) / min(s) if min(s) > 0 else mpmath.inf


# ---- esekf::predict (esekfom.hpp:279-384) with use-ikfom.cpp:49-90 --------------------------------------------------------
def predict(x, P, acc, gyro, dt, q_gyr, q_acc, q_bg, q_ba):
    """one IMU sample.  P: mp.matrix or array.  F and G are sparse; they are applied entry by entry."""
    x = state(x)
    P = mat(P)
    dt = mpf(dt)
    acc = [mpf(a) for a in acc]
    gyro = [mpf(a) for a in gyro]
    rot = qrot(x[3:7])
    g0 = grav(x)
    omega = [gyro[i] - x[17 + i] for i in range(3)]             # in.gyro.boxminus(omega, s.bg)
    a_b = mp.matrix([acc[i] - x[20 + i] for i in range(3)])
    a_in = rot * a_b
    f = [mpf(0)] * 24                                           # get_f, use-ikfom.cpp:49-61
    for i in range(3):
        f[i] = x[14 + i]
        f[3 + i] = omega[i]
        f[12 + i] = a_in[i] + g0[i]
    fx = {}                                                     # df_dx (24 x 23), use-ikfom.cpp:63-79
    for i in range(3):
        fx[(i, 12 + i)] = mpf(1)
        fx[(3 + i, 15 + i)] = mpf(-1)
    RH = rot * hat(a_b)
    Mx = s2_Mx(g0, [0, 0])
    for i in range(3):
        for j in range(3):
            fx[(12 + i, 3 + j)] = -RH[i, j]
            fx[(12 + i, 18 + j)] = -rot[i, j]
        for j in range(2):
            fx[(12 + i, 21 + j)] = Mx[i, j]
    fw = {}                                                     # df_dw (24 x 12), use-ikfom.cpp:82-90
    for i in range(3):
        for j in range(3):
            fw[(12 + i, 3 + j)] = -rot[i, j]
        fw[(3 + i, i)] = mpf(-1)
        fw[(15 + i, 6 + i)] = mpf(1)
        fw[(18 + i, 9 + i)] = mpf(1)
    # x_.oplus(f_, dt) (:287): vect += f dt, SO3 *= exp(f dt), S2: exp(f dt) of a zero segment
    xb = list(x)
    for i in range(3):
        x[i] += dt * f[i]
        x[14 + i] += dt * f[12 + i]
    x[3:7] = qmul(x[3:7], exp_q(f[3:6], dt))
    # F_x1 = I (:289); vect rows copied (:290-302); SO3 rows: exp(., scalar(1/2)) = I, A(-f dt) applied (:305-330)
    fxf, fwf = {}, {}
    for e, _ in _VECT:
        for (i, j), v in fx.items():
            if e <= i < e + 3:
                fxf[(i, j)] = v
        for (i, j), v in fw.items():
            if e <= i < e + 3:
                fwf[(i, j)] = v
    for e in SO3_IDX:
        A = A_matrix([-f[e + i] * dt for i in range(3)])
        for (src, dst) in ((fx, fxf), (fw, fwf)):
            cols = sorted({j for (i, j) in src if e <= i < e + 3})
            for j in cols:
                for a in range(3):
                    s = sum(A[a, b] * src.get((e + b, j), 0) for b in range(3))
                    if s != 0:
                        dst[(e + a, j)] = s
    # S2 rows (:336-371): the f segment of grav is zero, so its rows of f_x_final / f_w_final are zero and
    # F_x1's block is Nx(grav after) * I * Mx(grav before, 0)
    Fb = s2_Nx_yy(grav(x)) * s2_Mx(grav(xb), [0, 0])
    F = {(i, i): mpf(1) for i in range(N)}
    F[(21, 21)], F[(21, 22)], F[(22, 21)], F[(22, 22)] = Fb[0, 0], Fb[0, 1], Fb[1, 0], Fb[1, 1]
    for (i, j), v in fxf.items():                               # F_x1 += f_x_final dt (:380)
        F[(i, j)] = F.get((i, j), 0) + v * dt
    rows = {}
    for (i, j), v in F.items():
        rows.setdefault(i, []).append((j, v))
    FP = mp.matrix(N, N)
    for i, lst in rows.items():
        for c in range(N):
            FP[i, c] = mpmath.fsum(v * P[j, c] for j, v in lst)
    Pn = mp.matrix(N, N)
    for r in range(N):
        for i, lst in rows.items():
            Pn[r, i] = mpmath.fsum(v * FP[r, j] for j, v in lst)
    Qd = [q_gyr] * 3 + [q_acc] * 3 + [q_bg] * 3 + [q_ba] * 3
    Gr = {}
    for (i, j), v in fwf.items():
        Gr.setdefault(i, []).append((j, v * dt))
    for i, li in Gr.items():
        for k, lk in Gr.items():
            s = mpf(0)
            for j, a in li:
                for j2, b in lk:
                    if j == j2:
                        s += a * mpf(Qd[j]) * b
            Pn[i, k] += s
    return x, Pn
