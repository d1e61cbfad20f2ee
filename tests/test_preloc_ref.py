"""The host build of lv_prelocalize's arithmetic (csrc/lv_preloc.h, tests/cpu_shim/preloc.cpp) against the numpy restatement of
tests/preloc_ref.py: heading frames and offsets bit for bit, every candidate's score, the winner under the tie rule and the
winner's state.  A score may differ only by points that lie within an ulp of a cell face (listed when any occur).  No GPU."""
import math

import numpy as np
import pytest

import preloc_ref as R
import shim_binding

FAR = np.array([2e5, -3e5, 50.0])


def make_scene(lv, O, far, n_points=None):
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml")
    world = lv.SynthWorld(20261016, 400000)
    mp = world.map()
    truth = world.pose(40.0, prm)
    # beams up to 15 degrees: enough of them hit walls, which is what tells the candidates apart (the ground scores alike)
    sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=5)
    if n_points:
        sweep = sweep[:n_points]
    # the base: 0.5 m and 0.3 m off along the search axes, 8 degrees off in heading
    g, u, v = R.axes(truth)
    base = R.candidate(truth, 1.0, 1.0, 0, 0, 0)
    base = R.rotate_state(base, g, math.radians(8.0))
    base[0:3] += 0.5 * np.array(u) - 0.3 * np.array(v)
    if far:
        mp = (mp.astype(np.float64) + FAR).astype(np.float32)
        base[0:3] += FAR
    return prm, mp, sweep, base


WINDOW = dict(radius=1.2, step=0.4, yaw_range=0.25, yaw_step=0.0625)


@pytest.mark.parametrize("far", [False, True], ids=["near", "far"])
@pytest.mark.parametrize("max_points,n_points", [(512, None), (4096, 300)], ids=["strided", "all"])
def test_host_build_equals_restatement(lv, O, far, max_points, n_points):
    prm, mp, sweep, base = make_scene(lv, O, far, n_points)
    ds, vs = prm.map_downsample_size, prm.voxel_size
    I, K = R.grid(**WINDOW)
    W = 2 * I + 1
    scores, best, frames, offs = R.host_scores(base, sweep, mp, ds, vs, max_points=max_points, **WINDOW)
    ref, hit, w = R.score_all(base, sweep, mp, ds, vs, max_points=max_points, **WINDOW)
    S = min(len(sweep), max_points)
    assert hit.shape == (len(scores), S)
    # frames and offsets bit for bit
    g, u, v = R.axes(base)
    for k in range(-K, K + 1):
        Rm, t = R.lidar_to_world(R.rotate_state(base, g, float(k) * float(np.float32(WINDOW["yaw_step"]))))
        assert frames[k + K, :9].tobytes() == Rm.reshape(9).tobytes(), k
        assert frames[k + K, 9:].tobytes() == t.tobytes(), k
    o_ref = np.array([[R.offset64(u, v, i * float(np.float32(0.4)), j * float(np.float32(0.4))) for j in range(-I, I + 1)]
                      for i in range(-I, I + 1)]).reshape(-1, 3).astype(np.float32)
    assert offs.tobytes() == o_ref.tobytes()
    # every score; a difference only where scored points sit within an ulp of a cell face
    diff = np.nonzero(scores != ref)[0]
    face = R.at_face(w, ds)
    flagged = [(int(c), int(scores[c]), int(ref[c]), int(face[c].sum())) for c in diff]
    for c, a, b, nf in flagged:
        assert abs(a - b) <= nf, (c, a, b, nf)
    assert len(diff) == 0, flagged          # none on these scenes: the restatement is exact
    assert ref.max() > 0.5 * S              # the window holds the truth: most points land in the map
    assert best == R.winner(scores, I, K)
    k, q = divmod(best, W * W)
    ci, cj = divmod(q, W)
    xh = R.host_candidate(base, WINDOW["step"], WINDOW["yaw_step"], k - K, ci - I, cj - I)
    xr = R.candidate(base, WINDOW["step"], WINDOW["yaw_step"], k - K, ci - I, cj - I)
    assert xh.tobytes() == xr.tobytes()
    # the winner undoes the offset to within a grid step: -8 degrees is about -2 heading steps; -0.5 u + 0.3 v, plus what the
    # heading moves the LiDAR (1.25 m ahead of the IMU) and the heading's residual, about (-1, 1) position steps
    assert abs(k - K + 2) <= 1 and abs(ci - I + 1) <= 1 and abs(cj - I - 1) <= 1, (k - K, ci - I, cj - I)


def test_base_candidate_is_the_base_state(lv, O):
    prm, mp, sweep, base = make_scene(lv, O, False)
    assert R.host_candidate(base, 0.4, 0.05, 0, 0, 0).tobytes() == np.asarray(base, np.float64).tobytes()


def test_axes(lv, O):
    x = np.zeros(26)
    x[23:26] = [0.3, -0.2, -9.8]
    g, u, v = R.axes(x)
    out = np.zeros(9)
    shim_binding.lib().shim_preloc_axes(x.ctypes.data_as(R.C.POINTER(R.C.c_double)), out.ctypes.data_as(R.C.POINTER(R.C.c_double)))
    assert out.tobytes() == np.array(g + u + v).tobytes()
    assert abs(np.dot(g, u)) < 1e-15 and abs(np.dot(u, v)) < 1e-15 and abs(np.linalg.norm(v) - 1) < 1e-15
    x[23:26] = [-9.8, 0.1, 0.0]                     # |g_x| > 0.9: u starts from the y axis
    g, u, v = R.axes(x)
    assert abs(u[1]) > 0.99 and np.allclose(np.cross(g, u), v, atol=1e-15)
