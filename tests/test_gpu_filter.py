"""The 23-DoF algebra of the update (lv_ieskf_step_kernel) and of the IMU propagation (lv_predict_kernel) on the GPU, against the
50-digit IKFoM restatement of tests/ikfom_mp.py, on inputs built to reach the paths whole updates on easy scenes never reach:
ill-conditioned P, singular Q, every pivot a row swap, eigenvalues of HTH at the degeneracy threshold, every loop-control entry
state, Nm at the 23 boundary, IMU batches across the staging-buffer size.  The step and predict kernels are the shipped ones,
launched through tests/gpu_shim (filter_cases.py builds the inputs)."""
import numpy as np
import pytest

import bench
import filter_cases as FC
import ikfom_mp as M

pytestmark = pytest.mark.gpu


# ---- staging buffers of the asynchronous entry points -----------------------------------------------------------------
@pytest.fixture(scope="module")
def cfg1(lv, O):
    """the benchmark's update size: a 65 536-point sweep against a 1 M-point map"""
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=bench.MAP_POINTS + 4 * 65536, max_points=65536)
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=1, prm=prm)
    x0, P0 = lv.init_state_host(prm)
    return dict(prm=prm, map=mp, sweep=sweeps[0], x_prop=x_props[0], P0=P0)


QUEUED = 4          # updates queued ahead of the calls under test: ~1 ms of GPU work at cfg1 size


def _imu(rng, k, x):
    acc = -x[23:26] + rng.normal(0, 0.5, (k, 3))
    gyr = rng.normal(0, 0.3, (k, 3))
    dt = np.full(k, 2.5e-3)
    return acc, gyr, dt


def test_propagate_after_queued_update_uses_its_own_samples(lv, cfg1):
    """lv_correct_device queues whole updates and returns; two lv_propagate_device calls follow at once.  Each call stages its
    samples in one pinned buffer and queues the copy behind the update: the second call must not refill that buffer before
    the first call's copy has run, or the first launch integrates the second call's samples."""
    prm = cfg1["prm"]
    loc = lv.Localizer(prm)
    loc.map_build(cfg1["map"])
    d_sweep = loc.upload(cfg1["sweep"])
    n = len(cfg1["sweep"])
    rng = np.random.default_rng(5)
    A = _imu(rng, 512, cfg1["x_prop"])
    B = _imu(rng, 300, cfg1["x_prop"])
    loc.set_state(cfg1["x_prop"], cfg1["P0"])
    for _ in range(QUEUED):                                        # the updates on their own, synchronously
        st, x_u, P_u, logs = loc.correct(cfg1["sweep"])
        assert st == 0
    loc.set_state(cfg1["x_prop"], cfg1["P0"])
    for _ in range(QUEUED):
        loc.correct_device(d_sweep, n)
    loc.propagate_device(*A)
    loc.propagate_device(*B)
    x, P = loc.get_state()
    xr, Pr = x_u, P_u
    for acc, gyr, dt in (A, B):
        for i in range(len(dt)):
            xr, Pr = lv.predict_host(prm, xr, Pr, acc[i], gyr[i], dt[i])
    assert np.abs(x - xr).max() <= 1e-12 * max(1.0, np.abs(xr).max()), np.abs(x - xr).max()
    assert np.abs(P - Pr).max() <= 1e-12 * np.abs(Pr).max(), np.abs(P - Pr).max()
    loc.device_free(d_sweep)
    loc.close()


def test_state_upload_after_queued_update_is_not_overwritten(lv, O, cfg1):
    """The host state reaches the device through the pinned mirror of the update's control block.  lv_correct_device
    uploads a new state behind a queued update; a later lv_set_state + lv_propagate_device uploads again.  The second upload
    must not refill the mirror before the first copy has run: the second update has to start from its own state."""
    prm = cfg1["prm"]
    loc = lv.Localizer(prm)
    loc.map_build(cfg1["map"])
    d_sweep = loc.upload(cfg1["sweep"])
    n = len(cfg1["sweep"])
    x1 = cfg1["x_prop"]
    d = np.zeros(23)
    d[0:3] = [0.3, -0.2, 0.1]
    x2 = O.boxplus(x1, d)
    loc.set_state(x1, cfg1["P0"])
    st, _, _, logs_ref = loc.correct(cfg1["sweep"])                # the update from x1 on its own
    assert st == 0
    loc.set_state(x2, cfg1["P0"])
    for _ in range(QUEUED):
        loc.correct_device(d_sweep, n)                             # updates from x2 (queued)
    loc.set_state(x1, cfg1["P0"])
    loc.correct_device(d_sweep, n)                                 # update B from x1: its upload queues behind A
    loc.set_state(x2, cfg1["P0"])
    A = _imu(np.random.default_rng(6), 4, x2)
    loc.propagate_device(*A)                                       # uploads x2 while B's upload may still be queued
    st, logs = loc.last_logs()
    assert st == 0 and len(logs) == len(logs_ref)
    for a, b in zip(logs, logs_ref):
        assert a["n_matches"] == b["n_matches"]
        assert np.abs(a["HTH"] - b["HTH"]).max() <= 1e-12 * np.abs(b["HTH"]).max()
        assert np.abs(a["dx"] - b["dx"]).max() <= 1e-12
    x, P = loc.get_state()
    xr, Pr = x2, cfg1["P0"]
    for i in range(4):
        xr, Pr = lv.predict_host(prm, xr, Pr, A[0][i], A[1][i], A[2][i])
    assert np.abs(x - xr).max() <= 1e-12 * max(1.0, np.abs(xr).max())
    loc.device_free(d_sweep)
    loc.close()


# ---- the step kernel on its own, against the 50-digit reference -------------------------------------------------------------
import gpu_shim_binding as GS  # noqa: E402

U = 2.0 ** -53
C_BAR = 8           # the fixed constant of the step's bars: C_BAR * kappa * 2^-53


def _err(a, m):
    return float(np.abs(a - m).max() / max(np.abs(m).max(), 1e-300))


@pytest.fixture(scope="module")
def step_cases(lv, O, scene_xaloc, scene_kitti):
    out = []
    for sc in (scene_xaloc, scene_kitti):                    # kitti: estimate_extrinsics off, Q singular
        b = FC.base(O, sc)
        out += FC.conditioning(O, b) + FC.nm_scaled(b) + [FC.far_iterate(O, b)] + FC.degeneracy(b) + [FC.pivot_every_step(b)]
        out += FC.pivot_ties(b)
    return out


def test_packed_partials_round_trip(step_cases):
    """the harness's packing of HTH / HTh / Nm into one partials row is the fit kernel's: launch_reduce_partials gives it back"""
    c = step_cases[0]
    r = GS.step(c["x_prop"], c["P"], c["x_cur"], c["HTH"], c["HTh"], c["nm"], c["R"], c["D"], c["limits"], c["max_iter"])
    assert (r["reduced"][:144].reshape(12, 12) == c["HTH"]).all()
    assert (r["reduced"][144:156] == c["HTh"]).all() and r["reduced"][156] == c["nm"]


def test_step_against_mp(O, step_cases):
    """every case family, at the last evaluation (so the exit block runs): dx_, the new iterate (relative to the larger of 1
    and the step) and P within
    8 kappa * 2^-53 of the 50-digit reference (kappa: the largest 2-norm condition number of P_, of the matrix the reference
    inverts and of the 12x12 system the device solves), the flags equal to its decisions.  The oracle's error (the
    reference's two-inverse form in fp64) is printed beside the device's (pytest -s): neither form is uniformly the more
    accurate, see DESIGN.md section 2."""
    rows = []
    for c in step_cases:
        it = c["max_iter"] - 1
        r = FC.mp_eval(c, it=it)
        FC.check_path(c, r)
        g = GS.step(c["x_prop"], c["P"], c["x_cur"], c["HTH"], c["HTh"], c["nm"], c["R"], c["D"], c["limits"], c["max_iter"],
                    c["est"], it=it, t=0, n_evals=c["max_iter"])
        oprm = O.make_params(max_num_iters=c["max_iter"], estimate_extrinsics=c["est"], lidar_noise=c["R"],
                             degeneracy_threshold=c["D"], limits=c["limits"])
        dx_o, x_o, P_now, Kx, conv_o = O.update_step(c["x_prop"], c["P"], c["x_cur"], oprm, c["HTH"], c["HTh"])
        P_o = O.update_finish(c["x_prop"], x_o, dx_o, P_now, Kx)
        dxm, xm, Pm = M.to_np(r["dx"]), M.to_np(r["x"]), M.to_np(r["P"])
        kappa = float(max(r["kappa"]))
        bar = C_BAR * kappa * U
        # the iterate's error follows the step it took: relative to max(1, |dx_no_degenerate_|)
        xs = max(1.0, float(np.abs(M.to_np(r["dnd"])).max()))
        e = dict(dx=_err(g["dx"], dxm), x=float(np.abs(g["x"] - xm).max()) / xs, P=_err(g["P"], Pm))
        eo = dict(dx=_err(dx_o, dxm), x=float(np.abs(x_o - xm).max()) / xs, P=_err(P_o, Pm))
        rows.append((c["family"], kappa, e, eo))
        assert g["status"] == 0 and g["done"] == 1
        assert g["degenerate"] == int(r["degenerate"]), c["family"]
        assert g["converged"] == int(r["conv"]), c["family"]
        for k in ("dx", "x", "P"):
            assert e[k] <= bar, (c["family"], k, e[k], bar)
    print("\n%-28s %9s  %-29s %-29s" % ("family", "kappa", "device vs mp (dx, x, P)", "oracle vs mp (dx, x, P)"))
    for f, kappa, e, eo in rows:
        print("%-28s %9.1e  %8.1e %8.1e %8.1e    %8.1e %8.1e %8.1e" % (f, kappa, e["dx"], e["x"], e["P"], eo["dx"], eo["x"], eo["P"]))


@pytest.mark.parametrize("max_iter", [0, 1, 2, 3, 7])
def test_loop_control_entry_states(step_cases, max_iter):
    """every (MAX_NUM_ITERS, iter, t, converged) entry state of one evaluation: the converged flag, t, iter, whether the
    update finishes (esekfom.hpp:1757-1764) as the reference decides them"""
    c = step_cases[0]
    for conv_case in (True, False):
        limits = [1e3] * 23 if conv_case else [1e-12] * 23
        cc = dict(c, limits=limits, max_iter=max_iter)
        for it in range(-1, max_iter):
            for t in range(0, 3):
                r = FC.mp_eval(cc, it=it, t=t)
                g = GS.step(cc["x_prop"], cc["P"], cc["x_cur"], cc["HTH"], cc["HTh"], cc["nm"], cc["R"], cc["D"], limits,
                            max_iter, it=it, t=t, n_evals=it + 1)
                key = (max_iter, it, t, conv_case)
                assert g["converged"] == int(r["conv"]), key
                assert g["t"] == r["t"] and g["iter"] == it + 1 and g["n_evals"] == it + 2, key
                assert g["done"] == int(r["finish"]), key
                if r["finish"]:
                    assert _err(g["P"], M.to_np(r["P"])) <= C_BAR * float(max(r["kappa"])) * U, key


def test_too_few_matches_leaves_the_iterate(step_cases):
    c = step_cases[0]
    for nm, st in ((22, 2), (23, 0)):
        g = GS.step(c["x_prop"], c["P"], c["x_cur"], c["HTH"], c["HTh"], nm, c["R"], c["D"], c["limits"], c["max_iter"])
        assert g["status"] == st
        if st:
            assert g["done"] == 1 and (g["x"] == c["x_cur"]).all()


# ---- IMU propagation ----------------------------------------------------------------------------------------------------------
def _imu_case(rng, k, x, dt, w_scale, gyro_zero=False):
    acc = -x[23:26] + rng.normal(0, 0.5, (k, 3))
    gyr = np.zeros((k, 3)) if gyro_zero else rng.normal(0, 1, (k, 3)) * w_scale
    return acc, gyr, np.full(k, dt)


@pytest.mark.parametrize("dt,w", [(0.0, 1.0), (1e-6, 1.0), (2.5e-3, 1.0), (0.05, 1.0), (0.05, 35.0), (2.5e-3, 0.0)])
def test_predict_against_mp(lv, O, scene_xaloc, dt, w):
    """one launch of the predict kernel over 8 samples against the 50-digit esekf::predict; |omega| dt reaches ~3 rad at
    dt = 0.05, w = 35; w = 0 is a gyro of exactly zero; the biases are not zero"""
    sc = scene_xaloc
    prm = sc.prm
    noise = (prm.covariance_gyroscope, prm.covariance_acceleration, prm.covariance_bias_gyroscope, prm.covariance_bias_acceleration)
    x = sc.x_prop.copy()
    x[17:23] = [0.01, -0.02, 0.015, 0.05, -0.03, 0.04]
    rng = np.random.default_rng(int(1e6 * dt) + int(w))
    acc, gyr, dts = _imu_case(rng, 8, x, dt, w, gyro_zero=(w == 0.0))
    xg, Pg = GS.predict(x, sc.P0, acc, gyr, dts, noise)
    xm, Pm = x, sc.P0
    for i in range(8):
        xm, Pm = M.predict(xm, Pm, acc[i], gyr[i], dts[i], *noise)
    xm, Pm = M.to_np(xm), M.to_np(Pm)
    # 8 samples of a well-conditioned 23x23 product: tens of ulps
    assert np.abs(xg - xm).max() <= 64 * U * max(1.0, np.abs(xm).max()), np.abs(xg - xm).max()
    assert np.abs(Pg - Pm).max() <= 64 * U * np.abs(Pm).max(), np.abs(Pg - Pm).max() / np.abs(Pm).max()


@pytest.mark.parametrize("k", [1, 511, 512, 513, 1100, 2000])
def test_propagate_batches_are_one_launch(lv, scene_xaloc, k):
    """lv_propagate_device stages its samples in batches of 512: the result must be bit-identical to ONE launch over all k"""
    sc = scene_xaloc
    prm = sc.prm
    noise = (prm.covariance_gyroscope, prm.covariance_acceleration, prm.covariance_bias_gyroscope, prm.covariance_bias_acceleration)
    acc, gyr, dts = _imu_case(np.random.default_rng(k), k, sc.x_prop, 2.5e-3, 0.5)
    loc = lv.Localizer(prm)
    loc.set_state(sc.x_prop, sc.P0)
    loc.propagate_device(acc, gyr, dts)
    x, P = loc.get_state()
    loc.close()
    xg, Pg = GS.predict(sc.x_prop, sc.P0, acc, gyr, dts, noise)
    assert (x == xg).all() and (P == Pg).all()


# ---- loop control and the Nm boundary through lv_correct ---------------------------------------------------------------------
from test_gpu_fullsize import check_every_evaluation  # noqa: E402

SWITCHES = ("LV_NO_GRAPH", "LV_NO_REUSE")


def _evals_by_loop_rule(logs, max_iter):
    """the number of evaluations esekfom.hpp:1634-1764 runs given the `converged` flags it logged (forced convergence at
    i = max - 2 does not count toward t)"""
    t = 0
    for k, lg in enumerate(logs):
        i = k - 1
        forced = not t and i == max_iter - 2
        if lg["converged"] and not forced:
            t += 1
        if t > 1 or i == max_iter - 1:
            return k + 1
    return None


@pytest.mark.parametrize("max_iter", [1, 2, 7])
def test_update_loop_through_lv_correct(lv, O, scene_xaloc, monkeypatch, max_iter):
    """whole updates with MAX_NUM_ITERS 1, 2 and 7 (up to 8 evaluations: the deepest update graph, the log at its capacity,
    the reuse kernel on evaluations 4..7), LIMITS 1e-9 (never converges), the YAML's and 1e3 (converges at once), with the
    update graph and neighbour reuse each on and off: the number of evaluations follows the loop rule from the logged
    `converged` flags, every evaluation matches the oracle at the GPU's own iterate (check_every_evaluation, which also
    checks the flags and the final P), and the four switch settings agree bit for bit"""
    sc = scene_xaloc
    for limit in (1e-9, None, 1e3):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=1 << 19, max_points=1 << 16,
                                  MAX_NUM_ITERS=max_iter)
        if limit is not None:
            for i in range(23):
                prm.LIMITS[i] = limit
        oprm = O.make_params(max_num_iters=max_iter, estimate_extrinsics=prm.estimate_extrinsics,
                             max_dist_plane=prm.MAX_DIST_PLANE, planes_threshold=prm.PLANES_THRESHOLD,
                             lidar_noise=prm.LiDAR_noise, degeneracy_threshold=prm.degeneracy_threshold, limits=list(prm.LIMITS))
        om = O.Map(O.KNN_KDTREE)
        om.build(sc.map)
        runs = []
        for no_graph in (False, True):
            for no_reuse in (False, True):
                for k, on in zip(SWITCHES, (no_graph, no_reuse)):
                    if on:
                        monkeypatch.setenv(k, "1")
                    else:
                        monkeypatch.delenv(k, raising=False)
                loc = lv.Localizer(prm)
                loc.map_build(sc.map)
                loc.set_state(sc.x_prop, sc.P0)
                st, x, P, logs = loc.correct(sc.sweep)
                assert st == 0
                n = _evals_by_loop_rule(logs, max_iter)
                assert n == len(logs), (limit, no_graph, no_reuse, n, len(logs))
                if limit == 1e-9:
                    assert len(logs) == max_iter + 1 and not any(lg["converged"] for lg in logs[:max(max_iter - 1, 0)])
                if limit == 1e3:
                    assert len(logs) == min(2, max_iter + 1) and all(lg["converged"] for lg in logs)
                check_every_evaluation(O, om, oprm, sc.x_prop, sc.P0, sc.sweep, logs, loc, P_gpu=P)
                runs.append((x, P, logs))
                loc.close()
        for x, P, logs in runs[1:]:
            assert (x == runs[0][0]).all() and (P == runs[0][1]).all() and len(logs) == len(runs[0][2])
            for a, b in zip(logs, runs[0][2]):
                assert a["n_matches"] == b["n_matches"] and (a["dx"] == b["dx"]).all() and a["converged"] == b["converged"]
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)


@pytest.mark.parametrize("K", [22, 23, 24])
def test_nm_boundary_through_lv_correct(lv, O, scene_xaloc, K):
    """sweep subsets with exactly K matches at the propagated state (K matched points chosen with the oracle's valid bits, plus
    60 points without a plane): 22 stops with LV_TOO_FEW_MATCHES and leaves the state as it was, 23 and 24 run the whole
    update, checked evaluation by evaluation"""
    sc = scene_xaloc
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.map)
    valid = om.match_all(sc.x_prop, sc.oprm, sc.sweep)["valid"].astype(bool)
    rng = np.random.default_rng(0)
    idx = np.sort(np.concatenate([rng.choice(np.nonzero(valid)[0], K, replace=False),
                                  rng.choice(np.nonzero(~valid)[0], 60, replace=False)]))
    sub = sc.sweep[idx]
    assert om.measure_reduced(sc.x_prop, sc.oprm, sub)[3] == K
    loc = lv.Localizer(sc.prm)
    loc.map_build(sc.map)
    loc.set_state(sc.x_prop, sc.P0)
    st, x, P, logs = loc.correct(sub)
    if K == 22:
        assert st == lv.TOO_FEW_MATCHES
        x_after, P_after = loc.get_state()
        assert (x_after == sc.x_prop).all() and (P_after == sc.P0).all()
    else:
        assert st == 0 and logs[0]["n_matches"] == K
        check_every_evaluation(O, om, sc.oprm, sc.x_prop, sc.P0, sub, logs, loc, P_gpu=P)
    loc.close()
