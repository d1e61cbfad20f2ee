"""Seeded inputs for the 23-DoF step and the IMU propagation (test_gpu_filter.py), each built to reach one path, and each
checked through the 50-digit reference (ikfom_mp.py) to reach it.

A case is a dict: x_prop, P (P_prop), x_cur, HTH, HTh, nm, R, D, limits, max_iter, est (estimate_extrinsics), family."""
import numpy as np

import ikfom_mp as M

U = 2.0 ** -53


def base(O, scene):
    """the scene's normal equations at its propagated state (what the first evaluation of an update sees)"""
    om = O.Map(O.KNN_KDTREE)
    om.build(scene.map)
    st, HTH, HTh, nm = om.measure_reduced(scene.x_prop, scene.oprm, scene.sweep)
    assert st == 0 and nm > 1000
    return dict(x_prop=scene.x_prop.copy(), P=scene.P0.copy(), x_cur=scene.x_prop.copy(), HTH=HTH, HTh=HTh, nm=nm,
                R=scene.oprm.lidar_noise, D=scene.oprm.degeneracy_threshold, limits=list(scene.oprm.limits),
                max_iter=scene.oprm.max_num_iters, est=scene.oprm.estimate_extrinsics, om=om, scene=scene)


def case(b, family, **over):
    c = {k: v for k, v in b.items() if k not in ("om", "scene")}
    c.update(over)
    c["family"] = family
    return c


def aged_P(O, b, cycles, seed=0):
    """P after `cycles` oracle predict + update cycles (8 IMU samples of 2.5 ms, then one evaluation on the scene's normal
    equations, each at a random small offset): how P looks after a long run.  With estimate_extrinsics off the extrinsic block
    of P is never measured and keeps its initial size while the rest shrinks."""
    sc = b["scene"]
    prm = sc.prm
    cov = (prm.covariance_gyroscope, prm.covariance_acceleration, prm.covariance_bias_gyroscope, prm.covariance_bias_acceleration)
    rng = np.random.default_rng(seed)
    x, P = b["x_prop"].copy(), b["P"].copy()
    oprm = sc.oprm
    for _ in range(cycles):
        for _ in range(8):
            x, P = O.predict(x, P, -x[23:26] + rng.normal(0, 0.2, 3), rng.normal(0, 0.05, 3), 2.5e-3, *cov)
        x[:7] = b["x_prop"][:7]
        dx, x_new, P_now, Kx, conv = O.update_step(x, P, x, oprm, b["HTH"], b["HTh"])
        P = O.update_finish(x, x_new, dx, P_now, Kx)
        P = 0.5 * (P + P.T)
    return P


def conditioning(O, b, cycles=(16, 200, 2000)):
    out = [case(b, "P0")]
    for k in cycles:
        out.append(case(b, "P_aged_%d" % k, P=aged_P(O, b, k)))
    return out


def nm_scaled(b, nms=(23, 24, 1000, 65000, 260000, 4000000)):
    """HTH and HTh grow with the number of matches: the scene's equations rescaled to Nm rows"""
    return [case(b, "Nm_%d" % n, HTH=b["HTH"] * (n / b["nm"]), HTh=b["HTh"] * (n / b["nm"]), nm=n) for n in nms]


def far_iterate(O, b, seed=1):
    """an iterate 0.3 rad (both rotations) and 0.3 rad of gravity away from x_prop: the J blocks are far from identity"""
    rng = np.random.default_rng(seed)
    d = np.zeros(23)
    d[0:3] = rng.normal(0, 0.2, 3)
    for e in (3, 6):
        v = rng.normal(0, 1, 3)
        d[e:e + 3] = 0.3 * v / np.linalg.norm(v)
    d[21:23] = [0.3 * 0.6, -0.3 * 0.8]
    d[12:21] = rng.normal(0, 0.05, 9)
    return case(b, "iterate_0.3rad", x_cur=O.boxplus(b["x_prop"], d))


def _rot6(seed):
    q, r = np.linalg.qr(np.random.default_rng(seed).normal(size=(6, 6)))
    return q * np.sign(np.diag(r))


def with_block(b, family, ev, V=None, D=None):
    """HTH with its 6x6 pose block replaced by V diag(ev) V^T (the coupling to the extrinsic block kept, scaled down so that
    HTH stays positive definite)"""
    HTH = b["HTH"].copy()
    V = np.eye(6) if V is None else V
    HTH[0:6, 0:6] = (V * np.asarray(ev, np.float64)) @ V.T
    HTH[0:6, 0:6] = 0.5 * (HTH[0:6, 0:6] + HTH[0:6, 0:6].T)
    HTH[0:6, 6:] *= 1e-3
    HTH[6:, 0:6] *= 1e-3
    return case(b, family, HTH=HTH, D=b["D"] if D is None else D)


def degeneracy(b):
    """eigenvalues of HTH[0:6, 0:6] around the threshold D.  Each case records the decision it is built for; the step must
    take the decision the 50-digit eigenvalues of the fp64 matrix dictate."""
    D = b["D"]
    big = np.abs(b["HTH"][0:6, 0:6]).max()
    spread = [D * 40, big * 0.3, big * 0.5, big * 0.7, big * 0.9, big]
    out = []
    V = _rot6(7)
    ulp = np.spacing(big)
    for k in (-300, 300):                                       # a few hundred ulps of |HTH| below / above D
        ev = [D + k * ulp] + spread[1:]
        out.append(with_block(b, "eig_D%+d_ulp" % k, ev, V))
    out.append(with_block(b, "eig_exactly_D", [D] + spread[1:]))          # diagonal: the eigenvalue IS D
    for m in (1, 3, 6):
        ev = [D * (0.1 + 0.1 * i) for i in range(m)] + spread[m:]
        out.append(with_block(b, "eig_%d_below_D" % m, ev, V))
    # exactly planar, a threefold eigenvalue 0 < D in a rotated basis: prod < 1e-20 replaces the eigenvectors by the identity,
    # which (unlike with a diagonal block) changes dx_no_degenerate_; the masked directions are then the first three axes
    out.append(with_block(b, "eig_planar_prod_lt_1e-20", [0.0, 0.0, 0.0, D * 2, D * 3, D * 4], V))
    out.append(with_block(b, "D_zero", spread, V, D=0.0))
    return out


def check_path(c, mp_result):
    """assert, through the 50-digit eigenvalues, that a degeneracy case lands where its name says, beyond rounding"""
    ev = [float(v) for v in mp_result["eig"]]
    D = c["D"]
    f = c["family"]
    tol = 16 * U * np.abs(c["HTH"][0:6, 0:6]).max()
    if f.startswith("eig_D-"):
        assert ev[0] < D - tol, (ev[0], D)
    elif f.startswith("eig_D+"):
        assert ev[0] > D + tol, (ev[0], D)
    elif f == "eig_exactly_D":
        assert mp_result["eig"][0] == D
    elif f.startswith("eig_") and "below" in f:
        m = int(f.split("_")[1])
        assert sum(v < D for v in ev) == m
    elif f == "eig_planar_prod_lt_1e-20":
        assert mp_result["prod"] < 1e-20
    elif f == "D_zero":
        assert not mp_result["degenerate"]


def pivot_every_step(b, tries=4000):
    """S11 = P[:12, :12] / R and Q = HTH chosen so that the 12x12 Gauss-Jordan of the gain (I + Q S11, partial pivoting)
    swaps rows at each of its first 11 steps.  Found by a seeded search; the property is re-checked here."""
    for seed in range(tries):
        rng = np.random.default_rng(seed)
        A = rng.normal(size=(12, 12))
        Q = A @ A.T * 10 ** rng.uniform(2, 5)
        B = rng.normal(size=(12, 12))
        S = B @ B.T * 10 ** rng.uniform(-4, -1) * b["R"]
        M1 = np.eye(12) + Q @ (S / b["R"])
        if count_swaps(M1) == 11:
            P = b["P"].copy()
            P[0:12, 0:12] = S
            P[0:12, 12:] = 0
            P[12:, 0:12] = 0
            return case(b, "pivot_swap_every_step", HTH=Q, P=P)
    raise AssertionError("no matrix found")


def pivot_ties(b):
    """exact ties in |pivot| at the first Gauss-Jordan step: P[:12, :12] diagonal, so each entry of I + Q S11 is one product,
    and Q[1][0] = +-Q[2][0] the largest of column 0; partial pivoting must take row 1 (the lowest).  Same sign and opposite sign."""
    out = []
    P = b["P"].copy()
    P[0:12, 0:12] = np.diag(np.diag(P[0:12, 0:12]))
    P[0:12, 12:] = 0
    P[12:, 0:12] = 0
    for sign in (1.0, -1.0):
        Q = b["HTH"].copy()
        q = 4.0 * (np.abs(Q[:, 0]).max() + b["R"] / P[0, 0])
        Q[1, 0] = Q[0, 1] = q
        Q[2, 0] = Q[0, 2] = sign * q
        M1 = np.eye(12) + Q * (np.diag(P)[:12] / b["R"])[None, :]
        col = np.abs(M1[:, 0])
        assert col[1] == col[2] == col.max() and (col[[0] + list(range(3, 12))] < col[1]).all()
        out.append(case(b, "pivot_tie_%s" % ("same_sign" if sign > 0 else "opposite_sign"), HTH=Q, P=P))
    return out


def count_swaps(M1):
    M = np.array(M1, dtype=np.float64)
    n = 0
    for k in range(12):
        p = k + int(np.argmax(np.abs(M[k:, k])))
        if p != k:
            n += 1
            M[[k, p]] = M[[p, k]]
        M[k] /= M[k, k]
        for i in range(12):
            if i != k:
                M[i] -= M[i, k] * M[k]
    return n


def mp_eval(c, it=-1, t=0, max_iter=None):
    return M.evaluate(c["x_prop"], c["P"], c["x_cur"], c["HTH"], c["HTh"], c["R"], c["D"], c["limits"], it, t,
                      c["max_iter"] if max_iter is None else max_iter)
