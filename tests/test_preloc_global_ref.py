"""The host build of lv_prelocalize_global (csrc/lv_preloc_bound.h, tests/cpu_shim/preloc.cpp) against the numpy
restatement of tests/preloc_bound_ref.py and the brute force of lv_prelocalize's host build: the cell bound is at least every exact
score in the cell and equals it on single candidates, the pruned search returns the brute force's winner under the tie rule,
and on a whole-map window the bound prunes most of the candidates.  No GPU."""
import math

import numpy as np
import pytest

import preloc_bound_ref as B
import preloc_ref as R
from test_preloc_ref import FAR, make_scene

PI32 = float(np.float32(math.pi))
YAW = math.radians(2.0)


def random_cells(rng, I, K, l, n):
    """n random cells of level l, the clipped last row and column of cells included"""
    W = 2 * I + 1
    C = (W + (1 << l) - 1) >> l
    ci, cj = rng.integers(0, C, n), rng.integers(0, C, n)
    ci[: n // 4] = C - 1                      # a quarter on the clipped edge
    cj[n // 8: n // 4 + n // 8] = C - 1
    return np.stack([rng.integers(0, 2 * K + 1, n), np.full(n, l), ci, cj], axis=1)


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
def test_bound_is_at_least_every_score(lv, far):
    prm, mp, sweep, base = make_scene(lv, None, far)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    I, K, S = 50, 90, 512
    sc = B.Scene(base, sweep, mp, ds, vs, 0.4, YAW, I, K, S)
    rng = np.random.default_rng(7 + far)
    for l in range(0, 7):
        cells = random_cells(rng, I, K, l, 400)
        hb = B.host_bounds(base, sweep, mp, ds, vs, 0.4, YAW, I, K, S, cells)
        rb = np.array([sc.bound(tuple(c)) for c in cells])
        assert (hb >= rb).all(), (l, np.nonzero(hb < rb)[0][:5])
        if l <= 1:                             # boxes of at most 2 x 2 x 2 blocks: the block masks answer exactly
            assert (hb == rb).all(), l
        # every candidate of the cell scored by the restatement: the fewer the larger the cells
        n_exact = {0: 400, 1: 100, 2: 30, 3: 12, 4: 4, 5: 2, 6: 1}[l]
        ex = np.array([sc.exact_max(tuple(c)) for c in cells[:n_exact]])
        assert (rb[:n_exact] >= ex).all(), (l, np.nonzero(rb[:n_exact] < ex)[0][:5])
        if l == 0:                             # one candidate: the box is one voxel, the bound is the score
            assert (hb == ex).all() and (rb == ex).all()


def test_single_candidate_bound_is_the_brute_force_score(lv):
    prm, mp, sweep, base = make_scene(lv, None, False)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    win = dict(radius=1.2, step=0.4, yaw_range=0.25, yaw_step=0.0625)
    I, K = R.grid(**win)
    W = 2 * I + 1
    scores, _, _, _ = R.host_scores(base, sweep, mp, ds, vs, max_points=2048, **win)
    idx = np.arange(len(scores))
    cells = np.stack([idx // (W * W), np.zeros_like(idx), (idx % (W * W)) // W, idx % W], axis=1)
    hb = B.host_bounds(base, sweep, mp, ds, vs, win["step"], win["yaw_step"], I, K, 2048, cells)
    assert hb.tobytes() == scores.tobytes()


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
@pytest.mark.parametrize("win,max_points", [
    (dict(radius=1.2, step=0.4, yaw_range=0.25, yaw_step=0.0625), 512),
    (dict(radius=6.0, step=0.4, yaw_range=PI32, yaw_step=math.radians(6.0)), 2048),
    (dict(radius=3.0, step=0.3, yaw_range=1.0, yaw_step=0.1), 300),
], ids=["small", "all-headings", "odd"])
def test_search_equals_brute_force(lv, far, win, max_points):
    prm, mp, sweep, base = make_scene(lv, None, far)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    I, K = R.grid(**win)
    scores, best, _, _ = R.host_scores(base, sweep, mp, ds, vs, max_points=max_points, **win)
    assert best == R.winner(scores, I, K)
    idx, score, st = B.host_search(base, sweep, mp, ds, vs, max_points=max_points, **win)
    assert (idx, score) == (best, int(scores[best]))
    assert st["candidates"] == len(scores) and 0 < st["candidates_scored"] <= len(scores)
    S = min(len(sweep), max_points)
    assert st["probes"] == S * (st["cells_bounded"] + st["candidates_scored"])
    # the exhaustive mode scores every candidate through the same exact path and bounds nothing
    idx0, score0, st0 = B.host_search(base, sweep, mp, ds, vs, max_points=max_points, prune=False, **win)
    assert (idx0, score0) == (best, int(scores[best]))
    assert st0["candidates_scored"] == len(scores) and st0["cells_bounded"] == 0


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
def test_search_equals_brute_force_with_tilted_gravity(lv, far):
    """gravity 12 degrees off the world z axis (a pitched IMU mount): the offsets leave the xy plane, the voxel boxes grow
    tall in z, and the pruned search still returns the brute force's winner"""
    prm, mp, sweep, base = make_scene(lv, None, far)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    base = base.copy()
    c, s_ = math.cos(math.radians(12.0)), math.sin(math.radians(12.0))
    g = np.asarray(base[23:26])
    base[23:26] = [g[0], c * g[1] - s_ * g[2], s_ * g[1] + c * g[2]]
    win = dict(radius=4.0, step=0.4, yaw_range=PI32, yaw_step=math.radians(12.0))
    I, K = R.grid(**win)
    scores, best, _, _ = R.host_scores(base, sweep, mp, ds, vs, max_points=1024, **win)
    assert best == R.winner(scores, I, K)
    idx, score, st = B.host_search(base, sweep, mp, ds, vs, max_points=1024, **win)
    assert (idx, score) == (best, int(scores[best]))
    assert st["candidates_scored"] <= len(scores)


# ---- pruning on a whole-map window ---------------------------------------------------------------------------------------------
# Measured with this build on the 100 k-point SynthWorld below (DESIGN.md §5e): candidates_scored / candidates = PRUNED_SHARE
# or less.  The counts depend on the inputs only, so this holds on every machine.
PRUNED_SHARE = 0.001


def test_whole_map_window_prunes(lv):
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml")
    world = lv.SynthWorld(20261019, 100000)
    mp = world.map()
    truth = world.pose(30.0, prm)
    sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=9)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    # the start: the map's centre, the truth's attitude turned by 100 degrees; the window covers every occupied voxel
    lo, hi, _ = B.host_extent(mp, ds, vs)
    k = R.voxel_k(ds, vs)
    face = lambda b: float(np.float32(float((int(b) - R.BIAS) * k)) * np.float32(ds))
    wlo = np.array([face(b) for b in lo])
    whi = np.array([face(b + 1) for b in hi])
    g, u, v = R.axes(truth)
    start = R.rotate_state(truth, g, math.radians(100.0))
    start[0:2] = 0.5 * (wlo[0:2] + whi[0:2])
    corners = np.array([[x, y, z] for x in (wlo[0], whi[0]) for y in (wlo[1], whi[1]) for z in (wlo[2], whi[2])])
    radius = float(np.max(np.abs(np.concatenate([(corners - start[0:3]) @ np.array(u), (corners - start[0:3]) @ np.array(v)]))))
    win = dict(radius=radius, step=0.4, yaw_range=PI32, yaw_step=YAW)
    idx, score, st = B.host_search(start, sweep, mp, ds, vs, max_points=1024, **win)
    share = st["candidates_scored"] / st["candidates"]
    print("WHOLE-MAP", win, st, "share %.5f" % share, "score", score)
    assert st["candidates"] == lv.preloc_count(**win) > 1 << 21
    assert share <= PRUNED_SHARE, st
    # the winner is the truth within a grid step and a yaw step or two
    I, K = R.grid(**win)
    W = 2 * I + 1
    kk, q = divmod(idx, W * W)
    x = R.candidate(start, win["step"], win["yaw_step"], kk - K, q // W - I, q % W - I)
    assert np.linalg.norm(x[0:2] - truth[0:2]) < 0.8 and abs((kk - K) * win["yaw_step"] + math.radians(100.0)) <= 2 * win["yaw_step"]
