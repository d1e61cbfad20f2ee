"""The device match stage on the constructed neighbour sets of tests/match_cases.py.

For every family, origin and variant, at voxel 0.2 / 0.4 / 0.6, with 4 or 8 lanes per level-0 query or the per-launch policy,
and with neighbour reuse on or off, lv_match_all, lv_measure_reduced, one lv_correct and lv_last_neighbours must give the same
bits in every setting (the reference has no voxel size and no lanes), and lv_match_all must equal the oracle bit for bit,
neighbour ids in slot order included, in the product's (distance, x, y, z, id) order.  The equal-x pairs sit at bucket
positions that 4 and 8 lanes order differently (test_match_cases), so a tie order that stopped at x fails here.  The gates
are put at their thresholds on the device, the NaN plane's update is held against the oracle's, and the fit kernel's per-set
arithmetic runs on 1e5 adversarial sets against the host build."""
import numpy as np
import pytest

import gpu_shim_binding as GS
import match_cases as M
import shim_binding as S
from test_match_cases import SETS, VOXELS, _gate_cases, check_against_oracle, identity, nan_map, own_residuals, same_bits

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200, method="thread")]

SETTINGS = [(v, g, r) for v in VOXELS for g in (4, 8, None) for r in (True, False)]


def _localizer(lv, monkeypatch, pts, voxel=0.4, group=None, reuse=True, **over):
    for k in ("LV_SEARCH_GROUP", "LV_NO_REUSE"):
        monkeypatch.delenv(k, raising=False)
    if group is not None:
        monkeypatch.setenv("LV_SEARCH_GROUP", str(group))
    if not reuse:
        monkeypatch.setenv("LV_NO_REUSE", "1")
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 16, max_points=4096, **over)
    prm.voxel_size = voxel
    loc = lv.Localizer(prm)
    loc.map_build(pts)
    return loc, prm


def _run(lv, monkeypatch, pts, qs, x, voxel, group, reuse):
    loc, prm = _localizer(lv, monkeypatch, pts, voxel, group, reuse)
    got = loc.match_all(x, qs)
    red = loc.measure_reduced(x, qs)
    _, P0 = lv.init_state_host(prm)
    loc.set_state(x, P0)
    cor = loc.correct(qs)
    last = loc.last_neighbours(len(qs))
    loc.close()
    return dict(match=got, reduced=red, correct=cor, last=last, P0=P0)


@pytest.mark.parametrize("origin,wide", SETS)
def test_every_setting_gives_the_oracles_bits(lv, O, monkeypatch, origin, wide):
    pts, qs, cases = M.build(origin, wide)
    x = identity(O)
    oprm = O.make_params()
    om = O.Map(O.KNN_KDTREE)
    om.build(pts)
    base = None
    for voxel, group, reuse in SETTINGS:
        out = _run(lv, monkeypatch, pts, qs, x, voxel, group, reuse)
        if base is None:
            base = out
        a, b = out["match"], base["match"]
        where = (voxel, group, reuse)
        assert (a["nn_idx"] == b["nn_idx"]).all() and (a["nn_sqd"] == b["nn_sqd"]).all(), where
        assert (a["valid"] == b["valid"]).all() and same_bits(a["plane"], b["plane"]).all(), where
        assert same_bits(a["dist"], b["dist"]).all(), where
        ra, rb = out["reduced"], base["reduced"]
        assert ra[0] == rb[0] and ra[3] == rb[3] and (ra[1] == rb[1]).all() and (ra[2] == rb[2]).all(), where
        ca, cb = out["correct"], base["correct"]
        assert ca[0] == cb[0] and (ca[1] == cb[1]).all() and (ca[2] == cb[2]).all(), where
        assert len(ca[3]) == len(cb[3]) and all(la["n_matches"] == lb["n_matches"] for la, lb in zip(ca[3], cb[3])), where
        # lv_last_neighbours reports the search's slots, before the fit orders them: the same map points, tie order aside
        assert (np.sort(out["last"], 1) == np.sort(base["last"], 1)).all(), where
        check_against_oracle(a, om.match_all(x, oprm, qs), cases, oprm.max_dist_plane ** 2)
    st_o, HTH_o, HTh_o, nm_o = om.measure_reduced(x, oprm, qs)
    st, HTH, HTh, nm = base["reduced"]
    assert st == st_o and nm == nm_o
    assert np.abs(HTH - HTH_o).max() <= 1e-12 * max(np.abs(HTH_o).max(), 1e-300)
    st_c, x_c, P_c, logs = base["correct"]
    st_u, x_u, P_u, logs_u = om.update_iterated(x, base["P0"], oprm, qs)
    assert st_c == st_u and len(logs) == len(logs_u) and np.abs(x_c - x_u).max() < 1e-9
    print("\n%s %s: %d sets, %d accepted, correct status %d after %d evaluations, identical over %d settings"
          % (origin, "wide" if wide else "compact", len(cases), int(base["match"]["valid"].sum()), st_c, len(logs),
             len(SETTINGS)))


def test_nan_plane_reaches_the_device_update_as_in_the_reference(lv, O, monkeypatch):
    """five copies of the origin give an accepted NaN plane (Utils.cpp:47-62); its row makes the normal equations NaN, and
    lv_correct ends as the oracle's update does: the same status, NaN in x where the oracle has it, P as it was"""
    pts, qs, i, om = nan_map(O)
    x = identity(O)
    oprm = O.make_params()
    out = _run(lv, monkeypatch, pts, qs, x, 0.4, None, True)
    assert out["match"]["valid"][i] == 1 and np.isnan(out["match"]["plane"][i]).all()
    assert np.isnan(out["reduced"][1]).all()
    st_c, x_c, P_c, logs = out["correct"]
    st_o, x_o, P_o, logs_o = om.update_iterated(x, out["P0"], oprm, qs)
    assert st_c == st_o == lv.TOO_FEW_MATCHES and len(logs) == len(logs_o)
    assert (np.isnan(x_c) == np.isnan(x_o)).all() and np.isnan(x_c).any()
    assert same_bits(x_c[~np.isnan(x_o)], x_o[~np.isnan(x_o)]).all() or np.abs(x_c - x_o)[~np.isnan(x_o)].max() < 1e-9
    assert (P_c == out["P0"]).all() and (P_o == out["P0"]).all()


def test_gates_at_their_thresholds_on_the_device(lv, O, monkeypatch):
    """MAX_DIST_PLANE squaring exactly to the fifth distance, and one ulp either side; PLANES_THRESHOLD at a set's own largest
    residual and one ulp either side: the device gives the oracle's accept bits (test_match_cases spells out which)"""
    cases = _gate_cases(O)
    pts = np.concatenate([c.points for c in cases])
    qs = np.stack([c.query for c in cases])
    x = identity(O)
    m = 9 / 64
    runs = [dict(max_dist_plane=v, planes_threshold=1.0) for v in (m, np.nextafter(m, np.inf), np.nextafter(m, -np.inf))]
    res = own_residuals(cases)
    for t in (res.min(), res.max()):
        runs += [dict(planes_threshold=float(v)) for v in (t, np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(-np.inf)))]
    for r in runs:
        oprm = O.make_params(**r)
        om = O.Map(O.KNN_KDTREE)
        om.build(pts)
        over = {"MAX_DIST_PLANE": r["max_dist_plane"]} if "max_dist_plane" in r else {}
        loc, prm = _localizer(lv, monkeypatch, pts, PLANES_THRESHOLD=r["planes_threshold"], **over)
        got = loc.match_all(x, qs)
        loc.close()
        check_against_oracle(got, om.match_all(x, oprm, qs), cases, oprm.max_dist_plane ** 2)
        if "max_dist_plane" in r:
            assert (got["valid"] == (float(np.float32(m * m)) < r["max_dist_plane"] ** 2)).all()
        else:
            assert (got["valid"].astype(bool) == (res <= np.float32(r["planes_threshold"]))).all()


def test_fit_arithmetic_on_adversarial_sets_equals_the_host_build():
    """the shipped canonical_neighbour_order, plane_fit, plane_dist and jacobian_row on 1e5 sets (near-collinear 1..64 ulps off,
    tied pivots, equidistant and duplicate rows, rows permuted), one device thread per set, against the host build"""
    q, g, ids = M.adversarial_sets()
    x = np.zeros(26)
    x[3:7] = [0.1, -0.2, 0.3, 0.9273618495495704]
    x[7:11] = [0, 0, 0, 1]
    x[:3] = [1.5, -2.0, 0.25]
    dev = S.fit_sets(q, g, ids, x, 0.05, True, L=GS.lib())
    host = S.fit_sets(q, g, ids, x, 0.05, True)
    assert (dev["ids"] == host["ids"]).all() and (dev["ok"] == host["ok"]).all()
    assert same_bits(dev["plane"], host["plane"]).all() and same_bits(dev["dist"], host["dist"]).all()
    assert same_bits(dev["rows"], host["rows"]).all()
    assert (np.sort(dev["ids"], 1) == np.sort(ids, 1)).all()
    print("\n%d adversarial sets: %d accepted, %d NaN planes; device = host build bit for bit"
          % (len(q), int(host["ok"].sum()), int(np.isnan(host["plane"]).any(1).sum())))
