"""The rows of H and h against the 50-digit calculate_H (tests/measure_mp.py), without a GPU.

rows_exact is checked against rows_fd, the derivative of the residual under the [+] of the step's 50-digit reference.  Then
the product's arithmetic built for the host (tests/cpu_shim) and the oracle are held to rows_exact entry by entry, with the
bars of tests/measure_cases.py derived from the fp32 chain.  The bit-exact comparisons of shim, oracle and device cannot see a
misreading of calculate_H that the two transcriptions share; these can.  Run with -s for the error / bar table.
"""
import math

import numpy as np
import pytest

import measure_cases as MC
import measure_mp as M
import shim_binding as S


def _shim_rows(sm, prm, x, xyz):
    got = sm.match_all(x, prm, xyz, rows=True)
    v = got["valid"] == 1
    return xyz[v], got["plane"][v], got["rows"][v]


def _check(tag, x, xyz, plane, rows, est, oracle_rows=None):
    r_row, r_h, worst = MC.row_errors(x, xyz, plane, rows, est)
    print("\n  %-32s %6d matches  row err/bar %.3g  h err/bar %.3g  worst row err %.3g m" % (tag, len(xyz), r_row.max(),
                                                                                            r_h.max(), worst))
    assert len(xyz) > 100
    assert r_row.max() <= 1.0 and r_h.max() <= 1.0, tag
    if oracle_rows is not None:
        hx, h = oracle_rows
        o_row, o_h, _ = MC.row_errors(x, xyz, plane, np.concatenate([hx, h[:, None]], axis=1), est)
        assert o_row.max() <= 1.0 and o_h.max() <= 1.0, tag + " (oracle)"
    return worst


@pytest.mark.parametrize("name", ["scene_xaloc", "scene_kitti", "scene_ouster"])
def test_rows_exact_is_the_derivative_under_boxplus(name, request):
    """calculate_H's row is d dist(x [+] delta) / d delta at 0, to 1e-25, on 2000 sampled matches of each scene, and on the
    large-extrinsic state with estimate_extrinsics on"""
    sc = request.getfixturevalue(name)
    sm = S.ShimMap(sc.map, sc.prm.voxel_size, sc.prm.MAX_DIST_PLANE)
    prm = S.make_params(sc.oprm, sc.prm.voxel_size)
    xyz, plane, _ = _shim_rows(sm, prm, sc.x_prop, sc.sweep)
    sel = np.random.default_rng(7).choice(len(xyz), 2000, replace=False)
    gap = MC.fd_gap(sc.x_prop, xyz[sel], plane[sel], True)
    print("\n  %s: |rows_exact - rows_fd| <= %.2g" % (name, gap))
    assert gap <= 1e-25


def test_rows_exact_matches_the_definition_on_one_point():
    """a hand-checkable case: identity state, p = (1, 2, 3), plane z = 5: dist = 3 - 5, row = [n, p x n, p x n, n]"""
    x = [0.0] * 26
    x[6] = x[10] = 1.0
    row, h = M.rows_exact(x, [1.0, 2.0, 3.0], [0.0, 0.0, 1.0, -5.0], True)
    assert [float(v) for v in row] == [0, 0, 1, 2, -1, 0, 2, -1, 0, 0, 0, 1] and float(h) == 2.0
    row_off, _ = M.rows_exact(x, [1.0, 2.0, 3.0], [0.0, 0.0, 1.0, -5.0], False)
    assert [float(v) for v in row_off[6:]] == [0] * 6


@pytest.mark.parametrize("name", ["scene_xaloc", "scene_kitti", "scene_ouster"])
def test_shim_and_oracle_rows_against_mp(O, name, request):
    """every matched point of the scene: the shim's rows and the oracle's within C_ROW u32 s of rows_exact, h within
    C_H u32 (s + |D|)"""
    sc = request.getfixturevalue(name)
    sm = S.ShimMap(sc.map, sc.prm.voxel_size, sc.prm.MAX_DIST_PLANE)
    prm = S.make_params(sc.oprm, sc.prm.voxel_size)
    xyz, plane, rows = _shim_rows(sm, prm, sc.x_prop, sc.sweep)
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.map)
    st, hx, h = om.measure(sc.x_prop, sc.oprm, sc.sweep)
    assert st == 0 and hx.shape[0] == len(xyz)
    _check(name, sc.x_prop, xyz, plane, rows, bool(sc.prm.estimate_extrinsics), (hx, h))


def test_large_extrinsic_rows_against_mp(O, scene_xaloc):
    """offset_R_L_I 30 degrees from the configured one, offset_T_L_I (0.5, -0.3, 1.2), estimate_extrinsics on: the order of
    world_to_lidar's factors, R^T against R_LI^T and the operands of B all show here"""
    sc = scene_xaloc
    x, sweep = MC.large_extrinsic(O, sc)
    sm = S.ShimMap(sc.map, sc.prm.voxel_size, sc.prm.MAX_DIST_PLANE)
    oprm = O.make_params(estimate_extrinsics=True)
    xyz, plane, rows = _shim_rows(sm, S.make_params(oprm, sc.prm.voxel_size), x, sweep)
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.map)
    st, hx, h = om.measure(x, oprm, sweep)
    assert st == 0 and hx.shape[0] == len(xyz) and len(xyz) > 0.8 * len(sweep)
    _check("xaloc, large extrinsic", x, xyz, plane, rows, True, (hx, h))
    sel = np.random.default_rng(8).choice(len(xyz), 2000, replace=False)
    assert MC.fd_gap(x, xyz[sel], plane[sel], True) <= 1e-25


@pytest.fixture(scope="module")
def far(lv):
    return MC.far_scenes(lv)


@pytest.mark.parametrize("k", [0, 1])
def test_far_rows_against_mp(O, far, k):
    """the sweep-built scene at (2e5, -3e5, 50) and (4.3e5, 0, 0): the world point's ulp is 1.6-3 cm, and the rotational
    columns lose that much lever arm; the bar, which grows with s, covers it"""
    sc = far[k]
    oprm = O.make_params()
    sm = sc.shim_map(S, 0.4)
    xyz, plane, rows = _shim_rows(sm, S.make_params(oprm, 0.4), sc.x, sc.queries)
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.build)
    st, hx, h = om.measure(sc.x, oprm, sc.queries)
    assert st == 0 and hx.shape[0] == len(xyz)
    worst = _check(sc.name, sc.x, xyz, plane, rows, True, (hx, h))
    assert worst > 1e-3          # the lost lever arm is real, and the bar is what admits it
    sel = np.random.default_rng(9).choice(len(xyz), min(500, len(xyz)), replace=False)
    assert MC.fd_gap(sc.x, xyz[sel], plane[sel], True) <= 1e-25


def test_exact_gram_helper():
    """gram_diffs' exact sums against Fractions, on rows spanning 1e-9 .. 1e5 with values one ulp and 1e-12 off the exact
    Gram; an entry with a zero bar must be exactly zero"""
    from fractions import Fraction
    rng = np.random.default_rng(3)
    rows = rng.normal(0, 1, (300, 13)) * 10.0 ** rng.integers(-9, 6, (300, 13))
    rows[:, 11] = 0.0
    exact = [[sum(Fraction(a) * Fraction(b) for a, b in zip(rows[:, i], rows[:, j])) for j in range(13)] for i in range(12)]
    got = np.array([[float(exact[i][j]) for j in range(13)] for i in range(12)])
    got[3, 5] = np.nextafter(got[3, 5], math.inf)
    got[7, 12] *= 1 - 1e-12
    diff, mag = MC.gram_diffs(rows, got[:, :12], got[:, 12])
    for i in range(12):
        for j in range(i, 13):
            assert diff[i, j] == float(abs(Fraction(got[i, j]) - exact[i][j]))
            assert mag[i, j] == float(sum(abs(Fraction(a) * Fraction(b)) for a, b in zip(rows[:, i], rows[:, j])))
    r = MC.gram_errors(rows, got[:, :12], got[:, 12], 1.0)
    assert r[7, 12] > 1.0 and r[11, 11] == 0.0
    got[11, 11] = 1e-300
    assert MC.gram_errors(rows, got[:, :12], got[:, 12], 1.0)[11, 11] == math.inf
