"""The measurement path over a sweep of voxel sizes x all eight bench sweeps, under a timeout (VERDICT r1 item 1).

Round 1 left a hang open: lv_search_kernel<4> (4 lanes per query) never finished on bench sweeps 5 and 7 at
voxel_size 0.35 (deterministic in isolation; the 1- and 8-lane instantiations of the same source were fine).  The per-query
kernel exists with 4 and 8 lanes (lv_search_kernel<4> is the default for launches of 40 000 queries or more; both run on
the maps of test_gpu_geometry.py), and this test pins both, LV_SEARCH_GROUP=4 and =8: every voxel size the grid can take
(k = 1, 2, 3 downsample cells per edge; 0.3, 0.35 and 0.5 round to a neighbour), every bench sweep, bit-exact against the
oracle.
A kernel that does not terminate fails the test through pytest-timeout (thread method: the process is ended)."""
import numpy as np
import pytest

import bench

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

VOXELS = [0.2, 0.3, 0.35, 0.4, 0.5, 0.6]


@pytest.fixture(scope="module")
def scene(lv, O):
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=8, prm=prm)
    om = O.Map(O.KNN_REF_IKDTREE if O.ref_available() else O.KNN_KDTREE)
    om.build(mp)
    oprm = bench.oracle_params(O, prm)
    ref = []
    for k in range(8):
        st, HTH, HTh, nm = om.measure_reduced(x_props[k], oprm, sweeps[k])
        full = om.match_all(x_props[k], oprm, sweeps[k]) if k in (5, 7) else None
        ref.append((HTH, HTh, nm, full))
    return dict(prm=prm, map=mp, sweeps=sweeps, x_props=x_props, ref=ref)


@pytest.mark.parametrize("group", [4, 8])
@pytest.mark.parametrize("voxel", VOXELS)
def test_every_voxel_size_every_sweep(lv, scene, monkeypatch, voxel, group):
    monkeypatch.setenv("LV_SEARCH_GROUP", str(group))              # read at every direct launch and when a graph is built
    prm = bench.config_params(lv, "cfg1")
    prm.voxel_size = voxel
    loc = lv.Localizer(prm)
    loc.map_build(scene["map"])
    loc.map_status()
    for k in range(8):
        HTH, HTh, nm, full = scene["ref"][k]
        st, gH, gh, gn = loc.measure_reduced(scene["x_props"][k], scene["sweeps"][k])
        assert st == 0 and gn == nm, (voxel, k, gn, nm)
        assert np.abs(gH - HTH).max() <= 1e-12 * np.abs(HTH).max()
        assert np.abs(gh - HTh).max() <= 1e-12 * np.abs(HTh).max() + 1e-15
        if full is not None:                                        # the two sweeps that hung: per point, bit for bit
            got = loc.match_all(scene["x_props"][k], scene["sweeps"][k])
            inside = np.isfinite(got["nn_sqd"][:, 4])
            assert (got["nn_sqd"][inside] == full["nn_sqd"][inside]).all()
            assert (got["valid"] == full["valid"]).all() and (got["plane"] == full["plane"]).all()
    # whole updates too (graph replay, reuse kernel, ring search)
    x0, P0 = lv.init_state_host(prm)
    for k in (5, 7):
        loc.set_state(scene["x_props"][k], P0)
        st, x, P, logs = loc.correct(scene["sweeps"][k])
        assert st == 0 and logs[0]["n_matches"] == scene["ref"][k][2]
    loc.close()


def test_scattered_map_reports_capacity_instead_of_hanging(lv):
    """ADVICE r1 (high): isolated random points need 27 slots each; a table that runs out must flag LV_ERR_CAPACITY,
    never spin.  The same cloud fits once max_map_points is raised."""
    rng = np.random.default_rng(5)
    pts = rng.uniform(-300, 300, (200_000, 3)).astype(np.float32)
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=200_000, max_points=4096)
    loc = lv.Localizer(prm)
    loc.map_build(pts)                                              # 5.4 M slots wanted, 1 M available
    with pytest.raises(RuntimeError, match="LV_ERR_CAPACITY"):
        loc.map_status()
    loc.close()
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=4_000_000, max_points=4096)
    loc = lv.Localizer(prm)
    loc.map_build(pts)
    loc.map_status()
    assert loc.map_size() == len(pts)
    x = np.zeros(26); x[6] = 1; x[10] = 1; x[23] = 9.809
    st, HTH, HTh, nm = loc.measure_reduced(x, pts[:4096] + np.float32(0.01))
    assert st == 0 and nm == 0                                      # nothing has five neighbours within 2 m
    loc.close()
