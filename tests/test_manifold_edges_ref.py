"""The manifold algebra at its edges (tests/manifold_cases.py) through the oracle and the host build of the product's headers
(tests/cpu_shim), against the 50-digit IKFoM restatement (tests/ikfom_mp.py): any heading with the quaternion stored either
sign, iterates up to and past pi, gravity far from x_prop's, at its antipode and at the S2 chart's singular direction, the
Taylor bound and the 1e-11 tolerances, rot_to_quat's second branch through lv_init_state_host, and a long spinning run.
test_gpu_manifold_edges.py runs the same families on the device."""
import math

import mpmath
import numpy as np
import pytest

import filter_cases as FC
import ikfom_mp as M
import manifold_cases as MC
import shim_binding as S

U = 2.0 ** -53


@pytest.fixture(scope="module")
def bases(O, scene_xaloc, scene_kitti):
    return [FC.base(O, scene_xaloc), FC.base(O, scene_kitti)]          # kitti: estimate_extrinsics off, Q singular


@pytest.fixture(scope="module")
def rows(O, bases):
    states = [c["x_prop"] for b in bases for c in MC.headings(O, b) + MC.charts(O, b)]
    return MC.primitive_rows(O, states)


def test_primitives_against_mp(rows):
    """every lv_manifold.h function of the host build within its bar (manifold_cases.bar) of the 50-digit reference, each row
    on the branch its label names"""
    ops, inp = MC.pack(rows)
    worst = MC.primitive_errors(rows, S.manifold(ops, inp))
    print("\n" + "\n".join("%-22s %.3f" % kv for kv in sorted(worst.items())))
    assert all(v <= 1.0 for v in worst.values()), worst


def _cos_sinc_ref(x2):
    """mtkmath.hpp:142-174 in Python floats (IEEE doubles, no contraction): the branch and the series as written there"""
    if x2 >= math.sqrt(math.sqrt(2.0 ** -52)):
        x = math.sqrt(x2)
        return math.cos(x), math.sin(x) / x
    cosi, sinc, term = 1.0, 1.0, -1 / 2. * x2
    for i in range(3):
        cosi += term
        term *= (1 / 3., 1 / 5., 1 / 7.)[i]
        sinc += term
        term *= -(1 / 4., 1 / 6., 1 / 8.)[i] * x2
    return cosi, sinc


def test_cos_sinc_and_boxplus_bit_for_bit_at_the_taylor_bound(O, rows):
    """Within a few ulps both sides of cos_sinc_sqrt's bound are right, so only the bits show which side ran: the host build
    equals mtkmath.hpp's text (in Python doubles) bit for bit at 2^-13 +- 1, 2, 4 ulps and on 64 values across [2^-14, 2^-12],
    and its state boxplus equals the oracle's bit for bit there"""
    sel = [r for r in rows if r[0] == MC.COS_SINC]
    ops, inp = MC.pack(sel)
    out = S.manifold(ops, inp)
    for i, (_, x, label) in enumerate(sel):
        assert tuple(out[i, :2]) == _cos_sinc_ref(float(x[0])), (label, x[0])
    bp = [r for r in rows if r[2] == "boxplus_taylor"]
    assert len(bp) >= 3
    for _, x, _ in bp:
        assert (S.boxplus(x[:26], x[26:49]) == O.boxplus(x[:26], x[26:49])).all()
    for x2 in np.geomspace(MC.TAYLOR / 2, MC.TAYLOR * 2, 64):
        d = np.zeros(23)
        d[3:6] = math.sqrt(4 * x2) * np.array([0.48, -0.6, 0.64])
        x = bp[0][1][:26]
        assert (S.boxplus(x, d) == O.boxplus(x, d)).all(), x2


def step_kappa(r):
    """the largest condition number of ikfom_mp.evaluate's three (P_, the reference's P_temp, the 12x12 system the product
    solves); where P_ itself is singular to fp64 (cond > 2^53: at gravity's antipode the S2 J block of the reference, Nx Mx with
    A(Bu) at |Bu| = 3.1415926, has rank 1) the reference's two inverses carry no information and the 12x12 system's is used"""
    k = [float(v) for v in r["kappa"]]
    return k[2] if k[0] > 1 / U else max(k)


def _step_rows(O, bases, stepper):
    rows = []
    for b in bases:
        for c in MC.step_cases(O, b):
            it = c["max_iter"] - 1
            r = FC.mp_eval(c, it=it)
            c["check"](c, r)
            kappa = step_kappa(r)
            oprm = O.make_params(max_num_iters=c["max_iter"], estimate_extrinsics=c["est"], lidar_noise=c["R"],
                                 degeneracy_threshold=c["D"], limits=c["limits"])
            dx_o, x_o, P_now, Kx, conv_o = O.update_step(c["x_prop"], c["P"], c["x_cur"], oprm, c["HTH"], c["HTh"])
            P_o = O.update_finish(c["x_prop"], x_o, dx_o, P_now, Kx)
            eo = MC.step_errors(c, r, dx_o, x_o)
            eo["P"] = MC._err(P_o, M.to_np(r["P"]))
            e = stepper(c, r, it, oprm)
            rows.append((c["family"], kappa, e, eo))
            assert bool(conv_o) == r["conv"], c["family"]
            bar = MC.C_BAR * kappa * U
            for k in ("dx", "x", "P"):
                assert e[k] <= bar, (c["family"], k, e[k], bar)
                assert eo[k] <= bar, (c["family"], "oracle", k, eo[k], bar)
    return rows


def test_step_edges_host_build(O, bases):
    """every step family of both scenes at the last evaluation: the host build's dx_, iterate and exit-block P (and the
    oracle's) within 8 kappa 2^-53 of the 50-digit evaluation, each family on the branch it is built for"""
    def stepper(c, r, it, oprm):
        st, dx, x, P, done = S.step(c["x_prop"], c["P"], c["x_cur"], S.make_params(oprm), c["HTH"], c["HTh"], c["nm"], it, 0)
        assert st == 0 and done == 1
        e = MC.step_errors(c, r, dx, x)
        e["P"] = MC._err(P, M.to_np(r["P"]))
        return e
    MC.print_step_table(_step_rows(O, bases, stepper), "host build vs mp (dx, x, P)")


def _noise(prm):
    return (prm.covariance_gyroscope, prm.covariance_acceleration, prm.covariance_bias_gyroscope, prm.covariance_bias_acceleration)


def test_predict_from_every_heading_host_build(lv, O, bases):
    """lv_predict_host from every heading of both scenes (both signs) over 6 samples with |omega| dt of 0.5, 1.5 and 3 rad,
    and across the Taylor bound of so3_exp, against the 50-digit esekf::predict"""
    for b in bases:
        sc = b["scene"]
        prm = sc.prm
        noise = _noise(prm)
        for name, x in MC.heading_states(O, b):
            acc, gyr, dts = MC.imu_samples(len(name), x, 6, (0.5, 1.5, 3.0))
            xh, Ph, xm, Pm = x.copy(), sc.P0.copy(), x, sc.P0
            for i in range(len(dts)):
                xh, Ph = lv.predict_host(prm, xh, Ph, acc[i], gyr[i], dts[i])
                xm, Pm = M.predict(xm, Pm, acc[i], gyr[i], dts[i], *noise)
            xm, Pm = M.to_np(xm), M.to_np(Pm)
            assert np.abs(xh - xm).max() <= 64 * U * max(1.0, np.abs(xm).max()), name
            assert np.abs(Ph - Pm).max() <= 64 * U * np.abs(Pm).max(), name
    scene_xaloc = bases[0]["scene"]
    prm = scene_xaloc.prm
    noise = _noise(prm)
    x = bases[0]["x_prop"].copy()
    for k in (-2, -1, 0, 1):
        w = MC.taylor_omega(k)
        assert ((2.0 ** -8) ** 2 * (w * w) < MC.TAYLOR) == (k < 0)
        xh, Ph = lv.predict_host(prm, x, scene_xaloc.P0, -x[23:26], [w, 0, 0], 2.0 ** -7)
        xm, Pm = M.predict(x, scene_xaloc.P0, -x[23:26], [w, 0, 0], 2.0 ** -7, *noise)
        xo, Po = O.predict(x, scene_xaloc.P0, -x[23:26], [w, 0, 0], 2.0 ** -7, *noise)
        assert (xh == xo).all() and np.abs(xh - M.to_np(xm)).max() <= 8 * U * np.abs(x).max()


def test_long_spinning_run_host_build(lv, O, scene_xaloc):
    """20 000 samples at 400 Hz spinning at 10 rad/s through lv_predict_host: x against a 30-digit state-only propagation, P
    against np.longdouble, the quaternion's norm drift against the oracle's (neither renormalises, as SOn.hpp's boxplus
    does not)"""
    x0 = scene_xaloc.x_prop.copy()
    acc, gyr, dts = MC.spin_run(x0)
    prm = scene_xaloc.prm
    x, P = x0.copy(), scene_xaloc.P0.copy()
    xo, Po = x0.copy(), scene_xaloc.P0.copy()
    for i in range(len(dts)):
        x, P = lv.predict_host(prm, x, P, acc[i], gyr[i], dts[i])
        xo, Po = O.predict(xo, Po, acc[i], gyr[i], dts[i], *_noise(prm))
    assert (x == xo).all()                                         # the state, norm drift included, is the oracle's bit for bit
    check_long_run(x0, scene_xaloc.P0, acc, gyr, dts, _noise(prm), x, P, xo)


def check_long_run(x0, P0, acc, gyr, dts, noise, x, P, xo):
    """Bars from a drift of eps = 4 n 2^-53 in the quaternion (n samples, no renormalisation): the quaternion within eps, its
    direction within eps, the velocity within 2 eps |g| T and the position within eps |g| T^2 (T = n dt: a rotation off by eps
    mis-resolves the specific force by 2 eps |g|), P within eps relative.  The exact propagation keeps |q0|; the oracle's
    fp64 propagation, which like SOn.hpp's boxplus never renormalises, drifts by ~n/2 ulps, and the product's norm must follow
    that drift within 8 sqrt(n) ulps (the rounding the two orders of operations do not share), which a product that
    renormalised, or drifted twice as fast, would not.  xo: the oracle's state after the same samples."""
    n = len(dts)
    eps = 4 * n * U
    gT = float(np.linalg.norm(x0[23:26])) * float(np.sum(dts))
    xm = M.to_np(MC.mp_propagate_state(x0, acc, gyr, dts))
    _, Pl = MC.ld_predict(x0, P0, acc, gyr, dts, noise)
    Pl = Pl.astype(np.float64)
    e = dict(q=np.abs(x[3:7] - xm[3:7]).max(), dir=np.abs(x[3:7] / np.linalg.norm(x[3:7]) - xm[3:7] / np.linalg.norm(xm[3:7])).max(),
             vel=np.abs(x[14:17] - xm[14:17]).max(), pos=np.abs(x[0:3] - xm[0:3]).max(), P=np.abs(P - Pl).max() / np.abs(Pl).max())
    bars = dict(q=eps, dir=eps, vel=2 * eps * gT, pos=eps * gT * float(np.sum(dts)), P=eps)
    nq, nqo, nm = (float(np.linalg.norm(v[3:7])) - 1 for v in (x, xo, xm))
    print("\nlong run, error / bar: " + "  ".join("%s %.2e / %.1e" % (k, e[k], bars[k]) for k in e) +
          "\n|q| - 1: product %.2e, oracle %.2e, exact %.2e (|q0| - 1 = %.2e)" % (nq, nqo, nm, float(np.linalg.norm(x0[3:7])) - 1))
    for k in e:
        assert e[k] <= bars[k], (k, e[k], bars[k])
    assert abs(nq) <= eps and abs(nqo) <= eps
    walk = 8 * math.sqrt(n) * U
    assert abs(nqo) > 2 * walk, nqo                                 # the reference's drift is there to be followed
    assert abs(nq - nqo) <= walk, (nq, nqo, walk)
    assert abs(nm - (float(np.linalg.norm(x0[3:7])) - 1)) <= 2 * U
    for k in (0, 1, 2, 14, 15, 16):                               # the state moved: the run is not vacuous
        assert np.isfinite(x[k])
    assert np.abs(x[3:7] - x0[3:7]).max() > 0.1


def test_rot_to_quat_through_init_state_host(lv, O):
    """lv_init_state_host's offset_R_L_I from I_Rotation_L with trace <= 0 (rot_to_quat's second branch, each diagonal entry
    the largest once) and > 0, against Eigen's Quaternion(Matrix3) in 50 digits, and the oracle's bit for bit"""
    for R in rot_to_quat_matrices():
        q = check_init_state(lv, O, R, lambda prm: lv.init_state_host(prm))
        assert q is not None


def rot_to_quat_matrices():
    out = []
    for axis, ang in (([1, 0, 0], math.pi), ([0, 1, 0], math.pi), ([0, 0, 1], math.pi), ([1, 2, 3], 2.5), ([3, -1, 2], 2.2),
                      ([1, -1, 1], 2 * math.pi / 3 + 1e-3), ([0, 0, 1], 0.5), ([1, 0, 0], math.pi / 2)):
        out.append(np.asarray(MC.rot(axis, ang), np.float32))
    return out


def check_init_state(lv, O, R32, init):
    """R32: I_Rotation_L (float32, row-major as the YAML lists it); lv_init_state reads it column-major (quirk 10)"""
    import os
    prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"))
    for i in range(9):
        prm.I_Rotation_L[i] = float(R32.reshape(-1)[i])
    x, _ = init(prm)
    Rm = R32.astype(np.float64).T                                  # the matrix rot_to_quat receives
    trace = Rm[0, 0] + Rm[1, 1] + Rm[2, 2]
    qm = MC.mp_rot_to_quat(Rm)
    qo = O.init_state(initial_gravity=prm.initial_gravity[:], I_Rotation_L=prm.I_Rotation_L[:],
                      I_Translation_L=prm.I_Translation_L[:])[0][7:11]
    assert np.abs(x[7:11] - np.array([float(v) for v in qm])).max() <= 4 * U, (trace, x[7:11])
    assert (x[7:11] == qo).all()
    if trace <= 0:                                                 # the second branch: the largest diagonal's entry is positive
        assert x[7 + int(np.argmax(np.diag(Rm)))] > 0
    return x[7:11]
