"""lv_prelocalize and PCD maps on the GPU: device scores bit for bit against the host build (tests/cpu_shim/preloc.cpp), the winner
under the tie rule, the base candidate against lv_match_all, the strided subset, growth, the empty map, the effect on the filter;
finding the start pose from metres and tens of degrees off; and a sequence saved to PCD and resumed in a second handle."""
import math
import os

import numpy as np
import pytest

import preloc_ref as R

pytestmark = pytest.mark.gpu

FAR = np.array([2e5, -3e5, 50.0])
WINDOW = dict(radius=1.2, step=0.4, yaw_range=0.25, yaw_step=0.0625)
PI32 = float(np.float32(math.pi))


def xaloc(lv, **over):
    over.setdefault("max_map_points", 1 << 20)
    over.setdefault("max_points", 1 << 15)
    return lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), **over)


def offset_state(x, a, b, theta):
    """x moved by a u + b v and turned by theta about the gravity axis (the search's own axes)"""
    g, u, v = R.axes(x)
    y = R.rotate_state(x, g, theta)
    y[0:3] = np.asarray(x[0:3]) + a * np.array(u) + b * np.array(v)
    return y


@pytest.fixture(scope="module")
def scene(lv):
    prm = xaloc(lv)
    world = lv.SynthWorld(20261016, 400000)
    mp = world.map()
    truth = world.pose(40.0, prm)
    sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=5)
    base = offset_state(truth, 0.5, -0.3, math.radians(8.0))
    return prm, mp, sweep, base


def run_device(lv, prm, mp, sweep, base, scores=True, reserve=None, **window):
    loc = lv.Localizer(prm)
    try:
        loc.map_build(mp)
        if reserve:
            loc.map_reserve(reserve)
        loc.init_state()
        _, P0 = loc.get_state()
        loc.set_state(base, P0)
        d = loc.upload(np.ascontiguousarray(sweep, np.float32))
        loc.profile(reset=True)
        st, out = loc.prelocalize(d, len(sweep), scores=scores, **window)
        launches = loc.profile()["total_launches"]
        x, P = loc.get_state()
        loc.device_free(d)
        return st, out, x, P, P0, launches
    finally:
        loc.close()


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
@pytest.mark.parametrize("max_points,n_points", [(512, None), (4096, 300), (4096, None)], ids=["strided", "all", "strided4096"])
def test_scores_equal_host_build(lv, scene, far, max_points, n_points):
    prm, mp, sweep, base = scene
    if n_points:
        sweep = sweep[:n_points]
    if far:
        mp = (mp.astype(np.float64) + FAR).astype(np.float32)
        base = base.copy()
        base[0:3] += FAR
    win = dict(WINDOW, max_points=max_points)
    st, out, x, P, P0, launches = run_device(lv, prm, mp, sweep, base, **win)
    assert st == lv.OK and launches == 1
    hs, hbest, _, _ = R.host_scores(base, sweep, mp, prm.map_downsample_size, prm.voxel_size, **win)
    I, K = R.grid(**WINDOW)
    W = 2 * I + 1
    assert out["scores"].reshape(-1).tobytes() == hs.tobytes()
    assert out["index"] == hbest == R.winner(hs, I, K)
    k, q = divmod(hbest, W * W)
    assert (out["k"], out["i"], out["j"]) == (k - K, q // W - I, q % W - I)
    assert out["score"] == hs[hbest] and out["points"] == min(len(sweep), max_points) and out["candidates"] == len(hs)
    xh = R.host_candidate(base, WINDOW["step"], WINDOW["yaw_step"], out["k"], out["i"], out["j"])
    assert out["x"].tobytes() == xh.tobytes()
    assert x.tobytes() == xh.tobytes() and P.tobytes() == P0.tobytes()     # lv_set_state(out->x, NULL)


def test_base_candidate_equals_match_all(lv, scene):
    prm, mp, sweep, base = scene
    S = 1000
    st, out, x, P, P0, _ = run_device(lv, prm, mp, sweep, base, radius=0.0, step=0.4, yaw_range=0.0, yaw_step=0.1, max_points=S)
    assert st == lv.OK and out["candidates"] == 1 and (out["k"], out["i"], out["j"]) == (0, 0, 0)
    assert x.tobytes() == np.asarray(base).tobytes()
    loc = lv.Localizer(prm)
    try:
        loc.map_build(mp)
        sub = sweep[R.subset(len(sweep), S)]
        g = loc.match_all(base, sub)["g"]
    finally:
        loc.close()
    k = R.voxel_k(prm.map_downsample_size, prm.voxel_size)
    occ = R.occupancy(mp, prm.map_downsample_size, k)
    want = int((np.isin(R.keys(R.voxels(g, prm.map_downsample_size, k)), occ) & R.stored(g)).sum())
    assert out["score"] == want


def test_growth_gives_the_same_scores(lv, scene):
    prm, mp, sweep, base = scene
    small = xaloc(lv, max_map_points=1 << 19)
    a = run_device(lv, small, mp, sweep, base, **WINDOW, max_points=2048)
    b = run_device(lv, small, mp, sweep, base, reserve=1 << 22, **WINDOW, max_points=2048)
    assert a[0] == b[0] == lv.OK
    assert a[1]["scores"].tobytes() == b[1]["scores"].tobytes() and a[1]["x"].tobytes() == b[1]["x"].tobytes()


def test_empty_map(lv, scene):
    prm, mp, sweep, base = scene
    loc = lv.Localizer(prm)
    try:
        loc.init_state()
        x0, P0 = loc.get_state()
        d = loc.upload(np.ascontiguousarray(sweep, np.float32))
        st, _ = loc.prelocalize(d, len(sweep), max_points=512, **WINDOW)
        assert st == lv.EMPTY_MAP
        x, P = loc.get_state()
        assert x.tobytes() == x0.tobytes() and P.tobytes() == P0.tobytes()
        # an async first build that the gate left without points: the map is still empty
        d_n = loc.upload(np.array([5], np.int64))
        assert loc.correct_device_async(d, d_n, len(sweep), 100, 1.0) == lv.EMPTY_MAP
        loc.map_add_last_sweep()
        st, _ = loc.prelocalize(d, len(sweep), max_points=512, **WINDOW)
        assert st == lv.EMPTY_MAP
        x, P = loc.get_state()
        assert x.tobytes() == x0.tobytes() and P.tobytes() == P0.tobytes()
        loc.device_free(d)
        loc.device_free(d_n)
    finally:
        loc.close()


# ---- finding the start pose ------------------------------------------------------------------------------------------------------
REC = dict(radius=5.0, step=0.4, yaw_range=PI32, yaw_step=math.radians(2.0), max_points=2048)


def pose_err(O, x, truth):
    d = O.boxminus(x, truth)
    return float(np.linalg.norm(d[0:3])), float(np.degrees(np.linalg.norm(d[3:6])))


@pytest.mark.parametrize("extrinsic", [False, True], ids=["xaloc", "extrinsic"])
def test_finds_the_start_pose(lv, O, extrinsic):
    prm = xaloc(lv)
    if extrinsic:                                   # 30 degrees about z and an offset along every axis
        c, s = math.cos(math.radians(30)), math.sin(math.radians(30))
        for i, v in enumerate((0.5, -0.3, 1.2)):
            prm.I_Translation_L[i] = v
        for i, v in enumerate((c, -s, 0.0, s, c, 0.0, 0.0, 0.0, 1.0)):
            prm.I_Rotation_L[i] = v
    world = lv.SynthWorld(20261017, 1000000)
    mp = world.map()
    rng = np.random.default_rng(2026)
    loc = lv.Localizer(prm)
    report = []
    try:
        loc.map_build(mp)
        loc.init_state()
        _, P0 = loc.get_state()
        truths = (60.0, 140.0) if not extrinsic else (100.0,)
        for s_road in truths:
            truth = world.pose(s_road, prm)
            sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=int(s_road))
            d = loc.upload(np.ascontiguousarray(sweep, np.float32))
            for case in range(8 if not extrinsic else 3):
                a, b = rng.uniform(-4, 4, 2)
                th = rng.uniform(-150, 150) * math.pi / 180
                start = offset_state(truth, a, b, th)
                # lv_correct alone from the same error (recorded, not asserted)
                loc.set_state(start, P0)
                st0, xc, _, _ = loc.correct(sweep, 1.0)
                alone = pose_err(O, xc, truth)
                loc.set_state(start, P0)
                st, out = loc.prelocalize(d, len(sweep), scores=True, **REC)
                assert st == lv.OK
                # the winner within 2 grid steps and 2 yaw steps of the truth (the offsets that undo the start error)
                assert abs(out["k"] * REC["yaw_step"] + th) <= 2 * REC["yaw_step"] + 1e-9, (case, out["k"], th)
                assert abs(out["i"] * 0.4 + a) <= 0.8 + 1e-6 and abs(out["j"] * 0.4 + b) <= 0.8 + 1e-6, (case, out["i"], out["j"], a, b)
                # the margin over the best candidate more than 1 m or 10 degrees from the winner
                I, K = R.grid(**{k: REC[k] for k in ("radius", "step", "yaw_range", "yaw_step")})
                sc = out["scores"]
                kk, ii, jj = np.meshgrid(np.arange(-K, K + 1), np.arange(-I, I + 1), np.arange(-I, I + 1), indexing="ij")
                far = (np.hypot(ii - out["i"], jj - out["j"]) * 0.4 > 1.0) | (np.abs(kk - out["k"]) * 2.0 > 10.0)
                margin = out["score"] - int(sc[far].max())
                n_corr = 0
                for n_corr in range(1, 4):
                    st, x, _, _ = loc.correct(sweep, 1.0 + n_corr)
                    e = pose_err(O, x, truth)
                    if e[0] < 0.05 and e[1] < 0.5:
                        break
                report.append((s_road, case, round(a, 2), round(b, 2), round(math.degrees(th), 1), out["k"], out["i"], out["j"],
                               out["score"], margin, n_corr, e, alone))
                assert e[0] < 0.05 and e[1] < 0.5, report[-1]
            loc.device_free(d)
    finally:
        loc.close()
        for r in report:
            print("PRELOC", r)


# ---- a saved map, a resumed sequence -----------------------------------------------------------------------------------------------
def tick_states(world, prm, t0, n):
    return [world.pose(20.0 + 1.5 * t, prm) for t in range(t0, t0 + n)]


def test_saved_map_resumed_sequence(lv, O, tmp_path):
    prm = xaloc(lv)
    world = lv.SynthWorld(20261018, 400000)
    truths = tick_states(world, prm, 0, 21)
    sweeps = [world.sweep(x, rings=32, azimuths=256, seed=100 + t) for t, x in enumerate(truths)]
    A = lv.Localizer(prm)
    B = lv.Localizer(prm)
    try:
        A.init_state()
        x, P = A.get_state()
        A.set_state(truths[0], P)

        def tick(loc, t):
            x, P = loc.get_state()
            step = O.boxminus(truths[t], truths[t - 1]) if t > 0 else np.zeros(23)
            loc.set_state(O.boxplus(x, step), P)        # the prediction: the true motion since the last tick
            st, x, P, logs = loc.correct(sweeps[t], float(t))
            loc.map_add_last_sweep()
            return st, logs

        for t in range(10):
            tick(A, t)
        mp = A.map_points()
        path = tmp_path / "map.pcd"
        lv.pcd_write(path, mp)
        xs, Ps = A.get_state()
        loaded = lv.pcd_read(path)
        assert loaded.tobytes() == mp.tobytes()
        B.map_build(loaded)
        B.set_state(xs, Ps)
        assert B.map_points().tobytes() == mp.tobytes()
        for t in range(10, 20):
            sa, la = tick(A, t)
            sb, lb = tick(B, t)
            xa, Pa = A.get_state()
            xb, Pb = B.get_state()
            assert sa == sb and xa.tobytes() == xb.tobytes() and Pa.tobytes() == Pb.tobytes(), t
            assert len(la) == len(lb) and all(a["HTH"].tobytes() == b["HTH"].tobytes() and a["dx"].tobytes() == b["dx"].tobytes()
                                              and a["n_matches"] == b["n_matches"] for a, b in zip(la, lb)), t
            assert A.map_points().tobytes() == B.map_points().tobytes(), t
            assert len(la) > 0, t                   # the update ran
        # how far the resumed sequence is from the truth (recorded, not asserted: the sweeps are mostly ground, and what is
        # checked here is that the resumed handle computes what the original one does)
        print("RESUMED", t, pose_err(O, A.get_state()[0], truths[19]))
    finally:
        A.close()
        B.close()
