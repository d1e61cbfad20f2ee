"""Map growth on the device (lv_map_reserve, lv_map_set_growth, lv_map_info).

A growth re-hashes the voxel and block tables into larger ones and copies the arena's used prefix, on the handle's stream;
content, ids, insertion order and arena indices are kept.  So a handle that starts small and grows must give, tick by tick,
exactly what a handle born at the final capacity gives: the same status, bit-identical logs, x and P, the same neighbours
and the same map.  That holds with the update graph and neighbour reuse on or off (a growth drops the
cached update graphs: they embed the old table and arena pointers).

Peak device memory: the scattered-cloud test needs a 4 M-point capacity (27 table slots per isolated point), about 6.5 GB
per handle, and runs its two handles one after the other; every other test stays under 1 GB.
"""
import numpy as np
import pytest

import bench
from test_gpu_configs import _check_points

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1200, method="thread")]

N_TICKS = 60
RINGS, AZIMUTHS = 8, 256               # 2048-point sweeps: 27 n = 55 296 slots per add keeps the steps small


@pytest.fixture(scope="module")
def road(lv, O):
    """60 sweeps along the road at 5 m spacing (new ground every tick), their predicted states, the first one's truth"""
    prm = bench.config_params(lv, "cfg1", max_points=RINGS * AZIMUTHS)
    world = lv.SynthWorld(bench.SEED + 1, 100_000)
    rng = np.random.default_rng(7)
    sweeps, x_props, truths = [], [], []
    for i in range(N_TICKS):
        truth = world.pose(15.0 + 5.0 * i, prm)
        sweeps.append(world.sweep(truth, rings=RINGS, azimuths=AZIMUTHS, seed=300 + i))
        d = np.zeros(23)
        d[0:3] = rng.uniform(-0.05, 0.05, 3)
        d[3:6] = rng.uniform(-0.5, 0.5, 3) * np.pi / 180.0
        x_props.append(O.boxplus(truth, d))
        truths.append(truth)
    return dict(world=world, sweeps=sweeps, x_props=x_props, truths=truths)


def _params(lv, cap):
    return bench.config_params(lv, "cfg1", max_points=RINGS * AZIMUTHS, max_map_points=cap)


def _stream(lv, road, prm, grow_limit=0, checkpoints=(9, 19, 29)):
    """the device tick (lv_correct_device + lv_map_add_last_sweep) over the road from an empty map"""
    loc = lv.Localizer(prm)
    if grow_limit:
        loc.map_set_growth(grow_limit)
    x0, P0 = lv.init_state_host(prm)
    d_sweeps = [loc.upload(s) for s in road["sweeps"]]
    out, caps = [], []
    for t in range(N_TICKS):
        n = len(road["sweeps"][t])
        loc.set_state(road["truths"][0] if t == 0 else road["x_props"][t], P0)
        st = loc.correct_device(d_sweeps[t], n, time=0.1 * t)
        rec = dict(st=st)
        if st == lv.OK:
            rec["st"], rec["logs"] = loc.last_logs()
            rec["x"], rec["P"] = loc.get_state()
            rec["nn"] = loc.last_neighbours(n)
        loc.map_add_last_sweep(downsample=True)
        if t in checkpoints:
            rec["points"] = loc.map_points()
        caps.append(loc.map_info()["capacity_points"])
        out.append(rec)
    loc.map_status()
    info = loc.map_info()
    final = loc.map_points()
    for d in d_sweeps:
        loc.device_free(d)
    loc.close()
    return out, info, final, caps


def _same_run(a, b):
    for t, (ra, rb) in enumerate(zip(a, b)):
        assert ra["st"] == rb["st"], t
        assert ra.keys() == rb.keys(), t
        if "logs" in ra:
            assert len(ra["logs"]) == len(rb["logs"]), t
            for la, lb in zip(ra["logs"], rb["logs"]):
                for k in la:
                    assert np.array_equal(la[k], lb[k]), (t, k)
            assert np.array_equal(ra["x"], rb["x"]) and np.array_equal(ra["P"], rb["P"]), t
            assert np.array_equal(ra["nn"], rb["nn"]), t
        if "points" in ra:
            assert np.array_equal(ra["points"], rb["points"]), t


def test_growth_during_the_device_tick(lv, road, monkeypatch):
    """a handle born at 8192 points with growth on grows at least three times while it streams; a handle born at the final
    capacity must agree tick by tick, with and without graph replay and reuse"""
    base = None
    for env in ([], ["LV_NO_GRAPH"], ["LV_NO_REUSE"]):
        for k in ("LV_NO_GRAPH", "LV_NO_REUSE"):
            monkeypatch.delenv(k, raising=False)
        for k in env:
            monkeypatch.setenv(k, "1")
        grown, info, final, caps = _stream(lv, road, _params(lv, 8192), grow_limit=1 << 22)
        assert info["growths"] >= 3, info
        assert info["error_flags"] == 0
        # growths between two ticks that replay the same update graph (one sweep size: one capacity bucket)
        assert sum(1 for t in range(2, N_TICKS) if caps[t] != caps[t - 1]) >= 1, caps
        assert sum(1 for r in grown if r["st"] == lv.OK) >= N_TICKS // 2
        big, binfo, bfinal, _ = _stream(lv, road, _params(lv, info["capacity_points"]))
        assert binfo["growths"] == 0 and binfo["capacity_points"] == info["capacity_points"]
        _same_run(grown, big)
        assert np.array_equal(final, bfinal) and len(final) == info["points"] == binfo["points"]
        if base is None:
            base = grown
        else:
            _same_run(grown, base)


def test_scattered_cloud_grows_instead_of_failing(lv):
    """the 200 000 scattered points that need a 4 M-point handle (27 slots per isolated point): added in 4096-point batches
    to a 200 000-point handle with growth on, the map ends up as the 4 M-point handle's"""
    rng = np.random.default_rng(5)
    pts = rng.uniform(-300, 300, (200_000, 3)).astype(np.float32)
    x = np.zeros(26); x[6] = 1; x[10] = 1; x[23] = 9.809
    q = pts[:4096] + np.float32(0.01)

    def run(cap, grow):
        loc = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=cap, max_points=4096))
        if grow:
            loc.map_set_growth(1 << 24)
        for i in range(0, len(pts), 4096):
            loc.map_add(pts[i:i + 4096], downsample=True)
        assert loc.L.lv_map_status(loc.h) == lv.OK, lv.lib().lv_last_error()
        out = loc.map_size(), loc.map_points(), loc.measure_reduced(x, q), loc.map_info()
        loc.close()
        return out

    n, p, (st, HTH, HTh, nm), info = run(200_000, True)
    assert n == len(pts) and info["growths"] >= 1 and info["capacity_points"] <= 4_000_000, info
    n_b, p_b, (st_b, HTH_b, HTh_b, nm_b), _ = run(4_000_000, False)
    assert n_b == n and np.array_equal(p, p_b)
    assert st == st_b == 0 and nm == nm_b and np.array_equal(HTH, HTH_b) and np.array_equal(HTh, HTh_b)


def test_build_larger_than_capacity(lv, O, scene_xaloc):
    sc = scene_xaloc
    m = len(sc.map)
    grown = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=m // 4, max_points=1 << 16))
    with pytest.raises(RuntimeError, match="LV_ERR_CAPACITY"):
        grown.map_build(sc.map)                                       # growth off: as without growth
    grown.map_set_growth(1 << 20)
    grown.map_build(sc.map)
    grown.map_status()
    born = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=grown.map_info()["capacity_points"],
                                            max_points=1 << 16))
    born.map_build(sc.map)
    assert grown.map_size() == born.map_size() == m
    assert np.array_equal(grown.map_points(), born.map_points())
    a, b = grown.measure_reduced(sc.x_prop, sc.sweep), born.measure_reduced(sc.x_prop, sc.sweep)
    assert a[0] == b[0] == 0 and a[3] == b[3] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    ra, rb = grown.correct(sc.sweep), born.correct(sc.sweep)
    assert ra[0] == rb[0] == 0 and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2])
    grown.close()
    born.close()


def test_growth_limit(lv, O, scene_xaloc):
    """past lv_map_set_growth's limit a call that cannot be staged is refused with LV_ERR_CAPACITY and a message naming the
    limit; the map built before it is untouched and still answers like the oracle"""
    sc = scene_xaloc
    m = len(sc.map)
    loc = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 16, max_points=1 << 16))
    loc.map_set_growth(1 << 17)
    loc.map_build(sc.map)
    info = loc.map_info()
    assert info["capacity_points"] == 1 << 17 and info["growths"] == 1
    extra = np.concatenate([sc.map, sc.map])[: (1 << 17) + 1] + np.float32(0.05)
    st = loc.L.lv_map_add(loc.h, lv._f(np.ascontiguousarray(extra)), len(extra), 1)
    assert st == lv.ERR_CAPACITY
    msg = lv.lib().lv_last_error().decode()
    assert "growth limit" in msg and str(1 << 17) in msg, msg
    assert loc.L.lv_map_status(loc.h) == lv.OK
    assert loc.map_size() == m and loc.map_info()["capacity_points"] == 1 << 17
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.map)
    _check_points(loc, om, sc.oprm, sc.x_prop, sc.sweep)
    loc.close()


def test_reserve_mid_sequence_equals_a_handle_born_there(lv, O, scene_xaloc):
    sc = scene_xaloc
    world = sc.world
    xs = [world.pose(8.0 + 1.5 * i, sc.prm) for i in range(6)]
    sweeps = [world.sweep(x, rings=32, azimuths=256, seed=400 + i) for i, x in enumerate(xs)]
    x0, P0 = lv.init_state_host(sc.prm)

    def run(cap, reserve_at=None):
        loc = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=cap, max_points=1 << 16))
        loc.map_build(sc.map[:60_000])
        out = []
        for i, (x, s) in enumerate(zip(xs, sweeps)):
            if i == reserve_at:
                loc.map_reserve(1 << 19)
                before = loc.map_info()
                loc.map_reserve(1 << 18)                          # below the capacity: nothing happens
                assert loc.map_info() == before
            loc.set_state(sc.x_prop if i == 0 else x, P0)
            st, xo, P, logs = loc.correct(s)
            loc.map_add(bench.world_points(s, xo), downsample=True)
            out.append((st, xo, P, logs, loc.last_neighbours(len(s))))
        out.append(loc.map_points())
        info = loc.map_info()
        loc.close()
        return out, info

    a, ia = run(1 << 17, reserve_at=3)
    b, ib = run(1 << 19)
    assert ia["growths"] == 1 and ia["capacity_points"] == ib["capacity_points"] == 1 << 19
    assert ia["voxel_slots"] == ib["voxel_slots"] and ia["arena_entries"] == ib["arena_entries"]
    for ra, rb in zip(a[:-1], b[:-1]):
        assert ra[0] == rb[0] == 0
        assert np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2]) and np.array_equal(ra[4], rb[4])
        for la, lb in zip(ra[3], rb[3]):
            assert all(np.array_equal(la[k], lb[k]) for k in la)
    assert np.array_equal(a[-1], b[-1])


def test_map_info_and_ceilings(lv, scene_xaloc):
    sc = scene_xaloc
    loc = lv.Localizer(lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 16, max_points=1 << 16))
    info = loc.map_info()
    assert info["capacity_points"] == 1 << 16 and info["voxel_slots"] == 1 << 18 and info["growths"] == 0
    assert info["points"] == 0 and info["arena_top"] == 16 and info["growth_limit"] == 0
    assert info["arena_entries"] == 96 * (1 << 16) + (4 << 20)
    assert info["bytes"] > 16 * info["arena_entries"] + 32 * info["voxel_slots"]
    loc.map_set_growth(1 << 20)
    loc.map_build(sc.map[:30_000])
    caps, n_changes = [loc.map_info()["capacity_points"]], 0
    for i in range(1, 8):
        loc.map_add(sc.map[30_000 * i // 2:30_000 * i // 2 + 30_000] + np.float32(0.03 * i), downsample=True)
        c = loc.map_info()["capacity_points"]
        n_changes += c != caps[-1]
        caps.append(c)
    info = loc.map_info()
    n_changes += caps[0] != 1 << 16
    assert info["growths"] == n_changes and info["growth_limit"] == 1 << 20
    assert info["points"] == loc.map_size() and info["error_flags"] == 0
    assert 0 < info["slots_used"] <= info["voxel_slots"] // 2 and 0 < info["blocks_used"] <= info["block_slots"] // 2
    assert 16 < info["arena_top"] <= info["arena_entries"]
    # past the hard ceilings: refused, the map untouched, the ceiling named
    assert loc.L.lv_map_reserve(loc.h, (1 << 24) + 1) == lv.ERR_CAPACITY
    assert "2^26" in lv.lib().lv_last_error().decode()
    assert loc.map_info() == info
    loc.close()
