"""The match stage on constructed neighbour sets (tests/match_cases.py), host build against the oracle and float64.

For every family, origin, variant and voxel size the host build of the product's search, neighbour order and fit
(tests/cpu_shim) must equal the oracle bit for bit, neighbour ids in slot order included, and the ids must come in the
product's order: ascending (distance, x, y, z, id).  The fit of the full-rank sets is held against float64 least squares,
the two gates are put exactly on their thresholds and one ulp either side, and the equal-x family is shown to reach the
bucket positions where the lane count of the level-0 search would order a tied pair differently."""
import collections

import numpy as np
import pytest

import match_cases as M
import shim_binding as S

EPS32 = float(np.finfo(np.float32).eps)
VOXELS = (0.2, 0.4, 0.6)
SETS = [(o, w) for o in M.ORIGINS for w in (False, True)]
FULL_RANK = ("tie", "equal_x", "rank2", "equal_norms")


def identity(O):
    x, _ = O.init_state()
    x[0:3] = 0
    x[3:7] = [0, 0, 0, 1]
    x[7:11] = [0, 0, 0, 1]
    x[11:14] = 0
    return x


def same_bits(a, b):
    """equal, NaN equal to NaN (the host and the device do not produce the same NaN payload)"""
    a, b = np.asarray(a), np.asarray(b)
    return (a == b) | (np.isnan(a) & np.isnan(b))


def check_against_oracle(got, ref, cases, gate):
    """got: a product build's match_all; ref: the oracle's.  Returns the mask of queries with five neighbours in the gate."""
    inside = np.isfinite(got["nn_sqd"][:, 4])
    assert not (ref["nn_sqd"][~inside, 4].astype(np.float64) < gate).any()
    assert (got["nn_sqd"][inside] == ref["nn_sqd"][inside]).all()
    assert (got["nn_idx"][inside] == ref["nn_idx"][inside]).all()
    assert (got["valid"] == ref["valid"]).all()
    assert same_bits(got["plane"], ref["plane"]).all() and same_bits(got["dist"], ref["dist"]).all()
    ids = M.point_ids(cases)
    for i in np.nonzero(inside)[0]:
        want, d = M.expected_order(cases[i], ids[i])
        assert (got["nn_idx"][i] == want).all(), (cases[i].family, got["nn_idx"][i], want)
        assert (got["nn_sqd"][i] == d).all()
    return inside


@pytest.fixture(scope="module")
def data(O):
    out = {}
    for o, w in SETS:
        pts, qs, cases = M.build(o, w)
        om = O.Map(O.KNN_KDTREE)
        om.build(pts)
        out[(o, w)] = (pts, qs, cases, om)
    return out


@pytest.mark.parametrize("voxel", VOXELS)
@pytest.mark.parametrize("origin,wide", SETS)
def test_host_build_equals_oracle_in_slot_order(O, data, origin, wide, voxel):
    pts, qs, cases, om = data[(origin, wide)]
    x = identity(O)
    oprm = O.make_params()
    sm = S.ShimMap(pts, voxel, 2.0, capacity=16 * len(pts))
    got = sm.match_all(x, S.make_params(oprm, voxel), qs)
    ref = om.match_all(x, oprm, qs)
    assert (got["g"] == qs).all()                                  # identity state: the world point is the query
    inside = check_against_oracle(got, ref, cases, oprm.max_dist_plane ** 2)
    level, _ = sm.query_stats(x, qs)
    fam = collections.Counter(c.family for c in cases)
    at0 = collections.Counter(c.family for c, lv0 in zip(cases, level == 0) if lv0)
    print("\n%s %s voxel %.1f: %d sets, %d with five in the gate, %d accepted; settled at level 0 per family: %s"
          % (origin, "wide" if wide else "compact", voxel, len(cases), int(inside.sum()), int(got["valid"].sum()),
             {f: "%d/%d" % (at0[f], n) for f, n in sorted(fam.items())}))
    if wide:                                                       # the fifth beyond every certified radius: the ring search
        assert not any(lv0 for c, lv0 in zip(cases, level == 0) if c.family in ("tie", "equal_x", "duplicate"))
    elif origin == "origin":
        assert (level == 0).mean() > 0.9


def nan_map(O):
    """the compact origin map with five copies of the origin added: (points, queries, index of the NaN query, oracle map)"""
    pts, qs, cases = M.build("origin", False)
    c = M.nan_case()
    pts, qs = np.concatenate([pts, c.points]), np.concatenate([qs, c.query[None]])
    om = O.Map(O.KNN_KDTREE)
    om.build(pts)
    return pts, qs, len(qs) - 1, om


def test_nan_plane_of_five_coincident_points_is_accepted(O):
    """five copies of the origin: the back substitution divides by a zero pivot and |NaN| > threshold is false, so the plane
    is accepted with NaN coefficients, as in the reference (Utils.cpp:47-62 with Eigen 3.3).  The update that takes it in
    ends as the oracle's does: the same status, the same x bit for bit (NaN where the NaN row reached it), the same P"""
    pts, qs, i, om = nan_map(O)
    x = identity(O)
    _, P0 = O.init_state()
    oprm = O.make_params()
    ref = om.match_all(x, oprm, qs)
    assert ref["valid"][i] == 1 and np.isnan(ref["plane"][i]).all() and np.isnan(ref["dist"][i])
    abcd, ok = S.plane_fit(pts[-5:], 0.05)
    assert ok and np.isnan(abcd).all()
    sm = S.ShimMap(pts, 0.4, 2.0, capacity=16 * len(pts))
    got = sm.match_all(x, S.make_params(oprm, 0.4), qs)
    assert got["valid"][i] == 1 and np.isnan(got["plane"][i]).all()
    st, x1, P1, logs = sm.update(x, P0, S.make_params(oprm, 0.4), qs)
    st_o, x_o, P_o, logs_o = om.update_iterated(x, P0, oprm, qs)
    assert st == st_o == 2 and np.isnan(x1).any() and same_bits(x1, x_o).all()
    assert (P1 == P0).all() and (P_o == P0).all()
    assert len(logs) == len(logs_o) >= 1 and np.isnan(logs[0]["HTH"]).all()


@pytest.mark.parametrize("voxel", VOXELS)
def test_equal_x_pairs_reach_lane_dependent_orders(O, data, voxel):
    """the equal-x family puts tied pairs at halo-bucket positions that a 4-lane and an 8-lane scan would order differently
    (lowest lane first, then earlier position): without the full tie order the plane would depend on the lane count"""
    n_pairs, split = 0, 0
    for origin in M.ORIGINS:
        pts, qs, cases, om = data[(origin, False)]
        sm = S.ShimMap(pts, voxel, 2.0, capacity=16 * len(pts))
        dump = sm.dump()
        ids = M.point_ids(cases)
        for c, cid in zip(cases, ids):
            for a, b in c.ties:
                pa, pb = M.halo_positions(dump, c.query, sm.k, cid[[a, b]])
                if pa < 0 or pb < 0:
                    continue
                n_pairs += 1
                split += M.lane_order(pa, pb, 4) != M.lane_order(pa, pb, 8)
    print("\nvoxel %.1f: %d equal-x pairs in their query's bucket, %d ordered differently by 4 and 8 lanes" % (voxel, n_pairs, split))
    assert n_pairs > 0 and split > 0


def _fit_bar(pts, abcd):
    A = pts.astype(np.float64)
    sol, _, rank, sv = np.linalg.lstsq(A, -np.ones(5), rcond=None)
    norm = np.linalg.norm(sol)
    exact = np.concatenate([sol / norm, [1.0 / norm]])
    cond = sv[0] / sv[-1]
    err = np.abs(abcd.astype(np.float64) - exact)
    return err[:3].max() / (EPS32 * cond), err[3] / (EPS32 * cond * max(1.0, abs(exact[3]))), exact


@pytest.mark.parametrize("origin,wide", SETS)
def test_full_rank_fits_against_float64(data, origin, wide):
    """within test_plane_fit_exact's bar of float64 lstsq, and the accept bit follows the exact residuals outside the
    fp32 uncertainty; every one of the 120 row orders of a set meets the same bar"""
    pts, qs, cases, om = data[(origin, wide)]
    worst, distinct = 0.0, []
    for c in cases:
        if c.family not in FULL_RANK:
            continue
        abcd, ok = S.plane_fit(c.points, 0.05)
        u_coef, u_d, exact = _fit_bar(c.points, abcd)
        assert u_coef <= 64 and u_d <= 64, (c.family, u_coef, u_d)
        res = np.abs(c.points.astype(np.float64) @ exact[:3] + exact[3])
        unc = 32 * EPS32 * (np.abs(c.points).max() + 1.0)
        if abs(0.05 - res.max()) > 2 * unc:
            assert ok == (res.max() <= 0.05), c.family
        worst = max(worst, u_coef)
        if c.family in ("tie", "equal_x") and len(distinct) < 4:
            planes = set()
            for p in M.permutations5():
                a2, _ = S.plane_fit(c.points[list(p)], 0.05)
                assert max(_fit_bar(c.points, a2)[:2]) <= 64
                planes.add(a2.tobytes())
            distinct.append(len(planes))
    print("\n%s %s: coefficients within %.1f x cond x ulp32; distinct planes over the 120 row orders of four sets: %s"
          % (origin, "wide" if wide else "compact", worst, distinct))


def test_rank_deficient_fits(O, data):
    """Eigen's basic solution: an exactly zero column is never a pivot and its component is exactly 0; the host build and
    the oracle agree bit for bit on every rank-deficient set (checked in slot order above), here on the fit alone"""
    pts, qs, cases, om = data[("origin", False)]
    by = {c.family: c for c in cases}
    abcd, _ = S.plane_fit(by["zero_column"].points, 0.05)
    assert abcd[0] == 0.0 and np.isfinite(abcd).all()
    for fam in ("origin_plane", "origin_line", "origin_line_ulp", "equal_norms", "collinear", "collinear_ulp", "duplicate"):
        abcd, ok = S.plane_fit(by[fam].points, 0.05)
        assert np.isfinite(abcd).all() or fam == "origin_line", (fam, abcd)


def _gate_cases(O):
    """sets whose fifth neighbour is at squared distance (9 / 64)^2 m^2 exactly (9^2 = 1 + 16 + 64 = 16 + 16 + 49 ...)"""
    u = 2.0 ** -6
    rng = np.random.default_rng(11)
    fifth = M.sphere(81)
    cases = []
    for slot in range(12):
        q = M._lattice_query("origin", slot)
        near = M._fill(rng, set(), 4, 16, 64)
        v = near + [fifth[rng.integers(len(fifth))]]
        cases.append(M.Case("gate", q, q + np.asarray(v, np.float64) * u))
    return cases


def _run_both(O, cases, oprm, voxel=0.4):
    pts = np.concatenate([c.points for c in cases])
    qs = np.stack([c.query for c in cases])
    om = O.Map(O.KNN_KDTREE)
    om.build(pts)
    sm = S.ShimMap(pts, voxel, 2.0, capacity=16 * len(pts))
    x = identity(O)
    got, ref = sm.match_all(x, S.make_params(oprm, voxel), qs), om.match_all(x, oprm, qs)
    check_against_oracle(got, ref, cases, oprm.max_dist_plane ** 2)
    return got


def test_max_dist_plane_at_its_threshold(O):
    """Plane.cpp:40: sq_dists.back() < MAX_DIST_PLANE^2, in double.  MAX_DIST_PLANE = 9/64 squares to the fifth distance
    exactly: rejected; one ulp above: accepted (when the fit is); one ulp below: rejected"""
    cases = _gate_cases(O)
    d5 = np.float32((9 / 64) ** 2)
    assert all(M.sq_dist32(c.query, c.points).max() == d5 for c in cases)
    m = 9 / 64
    assert m * m == float(d5)
    planes = {}
    for mdp, expect in ((m, False), (np.nextafter(m, np.inf), True), (np.nextafter(m, -np.inf), False)):
        oprm = O.make_params(max_dist_plane=mdp, planes_threshold=1.0)
        assert (float(d5) < mdp * mdp) == expect
        got = _run_both(O, cases, oprm)
        assert (got["valid"] == expect).all(), (mdp, got["valid"])
        planes[expect] = got
    assert planes[True]["valid"].all()


def own_residuals(cases):
    """each set's largest fp32 |residual| under its own fit, rows in neighbour order, unfused (Utils.cpp:60-61)"""
    res = []
    for c, ids in zip(cases, M.point_ids(cases)):
        p = c.points[M.expected_order(c, ids)[0] - ids[0]].astype(np.float32)
        a = S.plane_fit(p, 1.0)[0]
        r = ((a[0] * p[:, 0] + a[1] * p[:, 1]) + a[2] * p[:, 2]) + a[3]
        res.append(np.abs(r).max())
    return np.array(res, np.float32)


def test_planes_threshold_at_the_fits_own_residual(O):
    """Utils.cpp:62: a set is rejected when some |residual| > PLANES_THRESHOLD.  With the threshold equal to a set's own
    largest fp32 |residual| every set whose largest residual is <= it is accepted, one ulp below it that set is not"""
    cases = _gate_cases(O)
    res = own_residuals(cases)
    for i in (int(np.argmin(res)), int(np.argmax(res)), len(cases) // 2):
        for thr in (res[i], np.nextafter(res[i], np.float32(np.inf)), np.nextafter(res[i], np.float32(-np.inf))):
            oprm = O.make_params(planes_threshold=float(thr))
            got = _run_both(O, cases, oprm)
            assert (got["valid"].astype(bool) == (res <= thr)).all(), (i, thr)


def near_tie_window(sqd6):
    """queries whose 5th and 6th nearest raw squared distances lie within PointType_CMP's 1e-10 (the comparator's window)"""
    return np.abs(sqd6[:, 5] - sqd6[:, 4]) < 1e-10


def test_near_ties_inside_the_comparators_window(O):
    """The product's search is the exact 5-NN in raw fp32 distance; its order within 1e-10 is (x, y, z, id).  The reference's
    heap admits a candidate only below top().dist, where top() is the maximum under PointType_CMP, so inside the 1e-10 window
    it can keep c and drop b (near_tie_cases).  Every query where the heap's five differ from the exact five must lie in
    that window (5th and 6th raw distances within 1e-10); they are counted, for the oracle's heap and for the reference
    ikd-Tree (oracle/_ref) where it is built."""
    cases = M.near_tie_cases()
    pts = np.concatenate([c.points for c in cases])
    qs = np.stack([c.query for c in cases])
    x, oprm = identity(O), O.make_params()
    sm = S.ShimMap(pts, 0.4, 2.0, capacity=16 * len(pts))
    got = sm.match_all(x, S.make_params(oprm, 0.4), qs)
    exact = np.sort(M.sq_dist32(qs[:, None, :], np.stack([c.points for c in cases])), 1)
    assert (np.sort(got["nn_sqd"], 1) == exact[:, :5]).all()                 # the exact five, by raw distance
    window = near_tie_window(exact)
    assert window.all()
    maps = [("oracle heap", O.Map(O.KNN_KDTREE))] + ([("reference ikd-Tree", O.Map(O.KNN_REF_IKDTREE))] if O.ref_available() else [])
    for name, om in maps:
        om.build(pts)
        ref = om.match_all(x, oprm, qs)
        differ = (np.sort(ref["nn_sqd"], 1) != exact[:, :5]).any(1)
        assert not (differ & ~window).any()
        same = ~differ
        if name == "oracle heap":                                              # same five: the same order and the same plane
            assert (got["nn_idx"][same] == ref["nn_idx"][same]).all()
        assert (got["valid"][same] == ref["valid"][same]).all() and same_bits(got["plane"][same], ref["plane"][same]).all()
        print("\n%s: %d of %d near-tie queries hold a different fifth neighbour than the exact 5-NN, all inside the "
              "comparator's window" % (name, int(differ.sum()), len(qs)))
    if not O.ref_available():
        pytest.skip("oracle/_ref not built: the reference ikd-Tree's count is not taken")
