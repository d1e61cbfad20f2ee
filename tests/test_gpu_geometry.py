"""The search and the map update on the maps of tests/geometry.py, on every shape of the level-0 search kernel, and the
device tick started from an empty map.

Each scene is built for a path the dense surface map never takes (a map grown from raw sweeps, sparse and blind queries,
a cavity with more occupied voxels around it than the ring search lists, a 3 200-point halo bucket, tiny maps, coordinates
far from the origin); test_cpu_shim proves the share of queries on that path.  Here every K1 shape — LV_SEARCH_GROUP 4 and
8 (read at every direct launch) and the unpinned per-launch policy — must give the oracle's answers: no
query with five neighbours inside the gate missed, squared distances bit-exact, accept bit / plane / distance bit-exact
except for queries whose 5th and 6th neighbours are exactly equidistant at different coordinates, normal equations to
1e-12.  On the scenes with enough matches a whole update must not depend on reuse, graph replay or PDL, and must pass
check_every_evaluation.  A kernel that does not terminate fails through pytest-timeout."""
import numpy as np
import pytest

import bench
import geometry as geo
from test_gpu_configs import _check_points
from test_gpu_fullsize import check_every_evaluation

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200, method="thread")]

SHAPES = (4, 8, None)                                        # LV_SEARCH_GROUP; None: search_group()'s policy
UPDATE_SCENES = ("sweep_built", "blind", "cluster")          # enough matches for a whole update


@pytest.fixture(scope="module")
def scenes(lv, O):
    out = {}
    for sc in geo.all_scenes(lv):
        om = sc.oracle_map(O, O.KNN_REF_IKDTREE if O.ref_available() else O.KNN_KDTREE)
        out[sc.name] = (sc, om)
    return out


def _cases():
    out = []
    for sc_name, voxels in [("sweep_built", (0.2, 0.4, 0.6)), ("sparse", (0.2, 0.4, 0.6)), ("blind", (0.2, 0.4, 0.6)),
                            ("cavity", (0.4,)), ("cluster", (0.4,)), ("tiny1", (0.4,)), ("tiny4", (0.4,)),
                            ("tiny5", (0.2, 0.4, 0.6)), ("tiny6", (0.2, 0.4, 0.6))]:
        out += [(sc_name, v) for v in voxels]
    for o in geo.FAR_OFFSETS:
        for kind in ("sweep_built", "sparse"):
            out += [("%s@%g,%g,%g" % ((kind,) + o), v) for v in (0.2, 0.4, 0.6)]
    return out


@pytest.mark.parametrize("name,voxel", _cases())
def test_every_search_shape_matches_the_oracle(lv, O, scenes, monkeypatch, name, voxel):
    sc, om = scenes[name]
    oprm = O.make_params()
    ref_set = set(map(tuple, om.points().tolist())) if sc.adds else None
    st_o, HTH_o, HTh_o, nm_o = om.measure_reduced(sc.x, oprm, sc.queries)
    loc = sc.localizer(lv, sc.params(lv, voxel))
    if sc.adds:                                                     # the map the rule grew: the oracle's, up to voxel-face ulps
        got_set = set(map(tuple, loc.map_points().tolist()))
        assert len(got_set ^ ref_set) <= 1e-4 * len(ref_set), (len(got_set ^ ref_set), len(ref_set))
    else:
        assert loc.map_size() == len(sc.build)
    for group in SHAPES:
        if group is None:
            monkeypatch.delenv("LV_SEARCH_GROUP", raising=False)
        else:
            monkeypatch.setenv("LV_SEARCH_GROUP", str(group))
        got = _check_points(loc, om, oprm, sc.x, sc.queries, max_ties=None if name == "cluster" else 4,
                            points=np.concatenate([sc.build] + sc.adds), oracle_ids=not sc.adds)
        st, HTH, HTh, nm = loc.measure_reduced(sc.x, sc.queries)
        assert st == st_o
        if got["ties"] == 0:
            assert nm == nm_o, (group, nm, nm_o)
            assert np.abs(HTH - HTH_o).max() <= 1e-12 * max(np.abs(HTH_o).max(), 1e-300)
            assert np.abs(HTh - HTh_o).max() <= 1e-12 * max(np.abs(HTh_o).max(), 1e-300) + 1e-15
        else:
            assert abs(nm - nm_o) <= got["ties"]
    loc.close()


@pytest.mark.parametrize("name", UPDATE_SCENES)
def test_update_on_the_scene_needs_no_switch_and_matches_the_oracle(lv, O, scenes, monkeypatch, name):
    """the update with reuse, graph replay and PDL on equals the all-off run bit for bit, on every K1 shape, and every
    evaluation matches the oracle at the GPU's own iterate"""
    sc, om = scenes[name]
    oprm = O.make_params()
    prm = sc.params(lv, 0.4)
    x0, P0 = lv.init_state_host(prm)

    def run(env):
        for k in ("LV_NO_REUSE", "LV_NO_GRAPH", "LV_NO_PDL", "LV_SEARCH_GROUP"):
            monkeypatch.delenv(k, raising=False)
        for k in env:
            monkeypatch.setenv(*(k.split("=") if "=" in k else (k, "1")))
        loc = sc.localizer(lv, sc.params(lv, 0.4))                   # the switches are read by lv_create
        loc.set_state(sc.x, P0)
        out = loc.correct(sc.queries)
        return loc, out

    loc, base = run(["LV_NO_REUSE", "LV_NO_GRAPH", "LV_NO_PDL"])
    st, x, P, logs = base
    assert st == 0 and logs[0]["n_matches"] > 1000
    check_every_evaluation(O, om, oprm, sc.x, P0, sc.queries, logs, loc)
    loc.close()
    for env in ([], ["LV_SEARCH_GROUP=4"], ["LV_SEARCH_GROUP=8"]):
        loc, (st1, x1, P1, l1) = run(env)
        loc.close()
        assert st1 == 0 and len(l1) == len(logs), env
        assert (x1 == x).all() and (P1 == P).all(), env
        for a, b in zip(logs, l1):
            assert a["n_matches"] == b["n_matches"]
            assert (a["HTH"] == b["HTH"]).all() and (a["HTh"] == b["HTh"]).all() and (a["dx"] == b["dx"]).all()


@pytest.mark.parametrize("via", ["host", "device"])
def test_tick_from_an_empty_map(lv, O, via):
    """main.cpp:84-102 from the first sweep on: correct (on an empty map it returns LV_EMPTY_MAP, Localizator.cpp:24, and keeps
    the sweep), then map_add_last_sweep (the first one builds the map un-downsampled at the current state, Mapper.cpp:26; the
    later ones apply the 0.2 m rule).  Sixteen ticks over the eight bench sweeps, visited twice: the second visit re-observes
    the same places (points already held, cells with several old points).  The oracle runs the same chain."""
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=8, prm=prm)
    x0, P0 = lv.init_state_host(prm)
    oprm = bench.oracle_params(O, prm)
    loc = lv.Localizer(prm)
    om = O.Map(O.KNN_KDTREE)
    oms = [om] + ([O.Map(O.KNN_REF_IKDTREE)] if O.ref_available() else [])
    probe = O.Map(O.KNN_KDTREE)                     # any non-empty map: match_all's world points on tick 0
    probe.build(np.zeros((1, 3), np.float32))
    # the first sweep defines the map frame: it is placed at its true pose.  (From a perturbed prior, a map made of one sweep
    # is off by up to 0.4 m at range and the next update's normal equations are too ill-conditioned for the 1e-9 step bar.)
    x, P = truths[0].copy(), P0.copy()
    for t in range(16):
        k = t % 8
        sweep = sweeps[k]
        if t > 0:                                   # re-anchor on this sweep's prior (the sweeps are cast at the true poses)
            x, _ = loc.get_state()
            x[:7] = x_props[k][:7]
            # with no IMU propagation between the ticks the covariance would only shrink, and the normal equations of a
            # collapsed prior are too ill-conditioned for the 1e-9 step bar: it restarts from the initial one
            P = P0.copy()
        loc.set_state(x, P)
        x_prior, P_prior = x.copy(), P.copy()
        d = None
        if via == "host":
            st, x, P, logs = loc.correct(sweep, time=0.1 * t)
        else:
            d = loc.upload(sweep)
            st = loc.correct_device(d, len(sweep), time=0.1 * t)
            if st == 0:
                st, logs = loc.last_logs()
            x, P = loc.get_state()
        st_o, x_o, P_o, logs_o = om.update_iterated(x_prior, P_prior, oprm, sweep)
        if t == 0:
            assert st == st_o == lv.EMPTY_MAP and loc.map_size() == 0
            x, P = loc.get_state()
            assert (x == x_prior).all() and (P == P_prior).all()         # no update: the state is left as it was
            g = probe.match_all(x_prior, oprm, sweep)["g"]
        else:
            assert st == st_o == 0 and len(logs) == len(logs_o)
            # at the GPU's iterates, against an oracle over the GPU's own map (the two maps may differ by voxel-face ulp
            # cases, checked below)
            same = O.Map(O.KNN_KDTREE)
            same.build(loc.map_points())
            check_every_evaluation(O, same, oprm, x_prior, P_prior, sweep, logs, loc)
            assert loc.L.lv_last_time_updated(loc.h) == pytest.approx(0.1 * t)
            loc.set_state(x, P)                     # inspection calls move the device state
            g = om.match_all(x, oprm, sweep)["g"]
        loc.map_add_last_sweep(downsample=True)
        for o in oms:
            o.add(g, downsample=True)
        loc.map_status()
        if d is not None:
            loc.device_free(d)
        got = set(map(tuple, loc.map_points().tolist()))
        assert len(got) == loc.map_size()
        if t == 0:
            assert loc.map_size() == len(sweep)     # built, not downsampled
        for o in oms:
            ref = set(map(tuple, o.points().tolist()))
            assert len(got ^ ref) <= 1e-4 * len(ref), (t, len(got ^ ref), len(ref))
        if t == 9:                                  # the grown map serves queries like a kd-tree over its own points
            ok = O.Map(O.KNN_KDTREE)
            ok.build(loc.map_points())
            _check_points(loc, ok, oprm, x_props[(t + 1) % 8], sweeps[(t + 1) % 8])
            loc.set_state(x, P)
    loc.close()
