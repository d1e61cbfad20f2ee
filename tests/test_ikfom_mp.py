"""The 50-digit IKFoM restatement (ikfom_mp.py) against the oracle and against the host build of the product's step
(tests/cpu_shim), on the three scenes.  Each fp64 implementation must sit within 8 kappa * 2^-53 of it, kappa the condition number
the reference's formulation works at; the manifold operations within a few ulps."""
import numpy as np
import pytest

import filter_cases as FC
import ikfom_mp as M
import shim_binding as S

U = 2.0 ** -53


def _err(a, m):
    return float(np.abs(a - m).max() / max(np.abs(m).max(), 1e-300))


def test_manifold_ops_match_oracle(O, scene_xaloc):
    rng = np.random.default_rng(0)
    x = scene_xaloc.x_prop
    for scale in (1e-6, 0.01, 0.3, 1.5):
        d = rng.normal(0, scale, 23)
        xo, xm = O.boxplus(x, d), M.to_np(M.boxplus(x, d))
        assert np.abs(xo - xm).max() <= 16 * U * max(1.0, np.abs(x).max())
        assert np.abs(O.boxminus(xo, x) - M.to_np(M.boxminus(xo, x))).max() <= 64 * U * max(1.0, np.abs(d).max())
        if scale < 1:                                            # beyond pi a rotation wraps: no round trip
            assert np.abs(M.to_np(M.boxminus(M.boxplus(x, d), x)) - d).max() <= 64 * U * np.abs(d).max()


@pytest.mark.parametrize("name", ["scene_xaloc", "scene_kitti", "scene_ouster"])
def test_one_evaluation_oracle_and_shim(O, request, name):
    """dx_, the iterate and the exit block's P of one evaluation at the propagated state and at a far iterate"""
    sc = request.getfixturevalue(name)
    b = FC.base(O, sc)
    for c in (FC.case(b, "scene"), FC.far_iterate(O, b)):
        it = c["max_iter"] - 1
        r = FC.mp_eval(c, it=it)
        bar = 8 * float(max(r["kappa"])) * U
        dxm, xm, Pm = M.to_np(r["dx"]), M.to_np(r["x"]), M.to_np(r["P"])
        dx, x_new, P_now, Kx, conv = O.update_step(c["x_prop"], c["P"], c["x_cur"], sc.oprm, c["HTH"], c["HTh"])
        P_o = O.update_finish(c["x_prop"], x_new, dx, P_now, Kx)
        st, dxs, xs, Ps, done = S.step(c["x_prop"], c["P"], c["x_cur"], S.make_params(sc.oprm), c["HTH"], c["HTh"], c["nm"],
                                       it, 0)
        assert st == 0 and done == 1 and bool(conv) == r["conv"]
        for got_dx, got_x, got_P in ((dx, x_new, P_o), (dxs, xs, Ps)):
            assert _err(got_dx, dxm) <= bar and np.abs(got_x - xm).max() <= bar and _err(got_P, Pm) <= bar


def test_predict_matches_oracle(O, scene_xaloc):
    sc = scene_xaloc
    prm = sc.prm
    cov = (prm.covariance_gyroscope, prm.covariance_acceleration, prm.covariance_bias_gyroscope, prm.covariance_bias_acceleration)
    rng = np.random.default_rng(3)
    x, P = sc.x_prop.copy(), sc.P0.copy()
    x[17:23] = [0.01, -0.02, 0.015, 0.05, -0.03, 0.04]
    xm, Pm = x, P
    for i in range(6):
        acc, gyr, dt = -x[23:26] + rng.normal(0, 1, 3), rng.normal(0, 2, 3), [0.0, 1e-6, 2.5e-3, 0.05, 0.05, 2.5e-3][i]
        x, P = O.predict(x, P, acc, gyr, dt, *cov)
        xm, Pm = M.predict(xm, Pm, acc, gyr, dt, *cov)
    xm, Pm = M.to_np(xm), M.to_np(Pm)
    assert np.abs(x - xm).max() <= 64 * U * max(1.0, np.abs(xm).max())
    assert np.abs(P - Pm).max() <= 64 * U * np.abs(Pm).max()


def test_degeneracy_cases_take_their_path(O, scene_xaloc):
    """the generators of the degeneracy family land where their names say, beyond rounding"""
    b = FC.base(O, scene_xaloc)
    for c in FC.degeneracy(b):
        FC.check_path(c, FC.mp_eval(c))
    assert FC.count_swaps(np.eye(12) + FC.pivot_every_step(b)["HTH"] @ (FC.pivot_every_step(b)["P"][:12, :12] / b["R"])) == 11
