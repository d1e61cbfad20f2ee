"""The measurement stage on the device held to the mathematics: rows of H and h against the 50-digit calculate_H, and the
tensor-core fold of HTH / HTh / Nm against the exact Gram of the rows it folds, entry by entry.

Rows: lv_measure against rows_exact / rows_fd (tests/measure_mp.py) with the bars of tests/measure_cases.py, and bit for bit
against the host build of the same arithmetic.  Fold: sweeps with exactly one accepted point must give HTH = r r^T,
HTh = r h and Nm = 1 exactly (one product plus exact zeros, wherever the point sits: every lane of a tile, first and last
block of a group, the short last group, the tiles past the 528-block grid); every other sweep must meet gamma(n) u64
sum_k |H_ki H_kj| entry by entry, gamma from the summation tree (measure_cases.fold_gamma).  Run with -s for the tables.
"""
import os

import numpy as np
import pytest

import measure_cases as MC
import shim_binding as S

pytestmark = pytest.mark.gpu

TILE = 128                      # points per tile (kMeasureThreads); the grid holds at most 528 blocks in groups of 32
N_BIG = 1 << 18
SIZES = [1, 127, 128, 129, 4095, 4096, 4097, 67584, 67585, 135169, 262144]
MASKS = ["all", "none", "every 4th lane", "one warp", "alternate tiles", "last tile"]


class Big:
    """a handle with room for 2^18-point sweeps on the xaloc map; the accepted points of the xaloc sweep (the pool) and their
    rows; filler points 500 m off the map, which nothing accepts"""

    def __init__(self, lv, sc):
        self.sc = sc
        self.x = sc.x_prop
        prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=1 << 19, max_points=N_BIG)
        self.loc = lv.Localizer(prm)
        self.loc.map_build(sc.map)
        got = self.loc.match_all(self.x, sc.sweep)
        self.pool = np.ascontiguousarray(sc.sweep[got["valid"] == 1])
        st, hx, h = self.loc.measure(self.x, self.pool)
        assert st == 0 and len(h) == len(self.pool) > 4096
        self.rows = np.concatenate([hx, h[:, None]], axis=1)
        self.filler = np.resize(sc.sweep + np.float32([0, 0, 500.0]), (N_BIG, 3))
        assert self.loc.measure_reduced(self.x, self.filler)[3] == 0

    def sweep(self, n, idx, which=None):
        """n slots of filler with pool points at idx (pool point `which[k]`, default k mod pool); returns the sweep and the
        rows the accepted points must have, in input order"""
        idx = np.asarray(idx, np.int64)
        k = np.arange(len(idx)) % len(self.pool) if which is None else np.asarray(which)
        xyz = self.filler[:n].copy()
        xyz[idx] = self.pool[k]
        return xyz, self.rows[k]


@pytest.fixture(scope="module")
def big(lv, scene_xaloc):
    b = Big(lv, scene_xaloc)
    yield b
    b.loc.close()


def _rows(loc, x, xyz):
    st, hx, h = loc.measure(x, xyz)
    assert st == 0
    return np.concatenate([hx, h[:, None]], axis=1)


# ---- rows on the device -----------------------------------------------------------------------------------------------------
def _device_rows_against_mp(loc, x, xyz, sm, sprm, est, tag):
    got = loc.match_all(x, xyz)
    v = got["valid"] == 1
    rows = _rows(loc, x, xyz)
    ref = sm.match_all(x, sprm, xyz, rows=True)
    assert (ref["valid"] == got["valid"]).all()
    # the device's rows are the host build's, bit for bit, wherever both fitted the same plane; the planes differ only where
    # the 5th and 6th neighbours are exactly equidistant at different coordinates (DESIGN.md §2), at most 4 queries a scene
    same = (got["plane"][v] == ref["plane"][v]).all(1)
    assert (~same).sum() <= 4 and (rows[same] == ref["rows"][v][same]).all()
    pts, plane = xyz[v], got["plane"][v]
    r_row, r_h, worst = MC.row_errors(x, pts, plane, rows, est)
    sel = np.random.default_rng(11).choice(len(pts), min(500, len(pts)), replace=False)
    gap = MC.fd_gap(x, pts[sel], plane[sel], est)
    print("\n  %-32s %6d matches (%d tied)  row err/bar %.3g  h err/bar %.3g  worst row err %.3g m  |exact - fd| %.2g"
          % (tag, len(pts), (~same).sum(), r_row.max(), r_h.max(), worst, gap))
    assert len(pts) > 100 and r_row.max() <= 1.0 and r_h.max() <= 1.0 and gap <= 1e-25
    return worst


@pytest.mark.parametrize("name", ["scene_xaloc", "scene_kitti", "scene_ouster", "large extrinsic"])
def test_device_rows_against_mp(lv, O, name, request):
    sc = request.getfixturevalue("scene_xaloc" if name == "large extrinsic" else name)
    x, xyz, est = sc.x_prop, sc.sweep, bool(sc.prm.estimate_extrinsics)
    if name == "large extrinsic":
        x, xyz = MC.large_extrinsic(O, sc)
        assert est
    loc = lv.Localizer(sc.prm)
    loc.map_build(sc.map)
    sm = S.ShimMap(sc.map, sc.prm.voxel_size, sc.prm.MAX_DIST_PLANE)
    _device_rows_against_mp(loc, x, xyz, sm, S.make_params(sc.oprm, sc.prm.voxel_size), est, name)
    loc.close()


@pytest.fixture(scope="module")
def far(lv):
    return MC.far_scenes(lv)


@pytest.mark.parametrize("k", [0, 1])
def test_far_device_rows_against_mp(lv, O, far, k):
    sc = far[k]
    prm = sc.params(lv, 0.4)
    loc = sc.localizer(lv, prm)
    worst = _device_rows_against_mp(loc, sc.x, sc.queries, sc.shim_map(S, 0.4), S.make_params(O.make_params(), 0.4),
                                    bool(prm.estimate_extrinsics), sc.name)
    assert worst > 1e-3
    loc.close()


# ---- one accepted point: exact --------------------------------------------------------------------------------------------
def _single(big, n, i, which=0):
    xyz, r = big.sweep(n, [i], [which])
    st, HTH, HTh, nm = big.loc.measure_reduced(big.x, xyz)
    row, h = r[0, :12], r[0, 12]
    ok = st == 0 and nm == 1 and bool((HTH == np.outer(row, row)).all()) and bool((HTh == row * h).all())
    return ok or (n, i, nm)


def test_single_match_at_every_lane(big):
    bad = [_single(big, TILE, lane, lane) for lane in range(TILE)]
    assert all(b is True for b in bad), [b for b in bad if b is not True]


@pytest.mark.parametrize("n,i", [
    (4096, 5), (4096, 31 * TILE + 100),                         # first and last block of a full group (one group)
    (8192, 32 * TILE + 3), (8192, 63 * TILE + 127),             # the same in the second group
    (4097, 4096),                                               # a group of one block
    (67584, 0), (67584, 511 * TILE + 64),                       # 528 blocks: groups 0 and 15
    (67584, 512 * TILE + 9), (67584, 527 * TILE + 127),         # first and last block of the short last group (16 blocks)
    (67585, 67584), (67712, 528 * TILE + 77),                   # tile 528: block 0's second tile
    (135169, 528 * TILE + 40), (135169, 1055 * TILE + 3),       # second tiles of blocks 0 and 527
    (135169, 135168), (N_BIG, N_BIG - 1),                       # block 0's third tile, block 463's fourth
])
def test_single_match_across_blocks_groups_and_tiles(big, n, i):
    assert _single(big, n, i, i % len(big.pool)) is True


# ---- the fold against the exact Gram --------------------------------------------------------------------------------------
def _mask(name, n):
    i = np.arange(n)
    lane, tile = i % TILE, i // TILE
    return {"all": np.ones(n, bool), "none": np.zeros(n, bool), "every 4th lane": lane % 4 == 0, "one warp": lane // 32 == 2,
            "alternate tiles": tile % 2 == 0, "last tile": tile == tile[-1]}[name]


def _fold_ratio(loc, x, xyz, n_expect, rows_expect=None):
    rows = _rows(loc, x, xyz)
    if rows_expect is not None:
        assert (rows == rows_expect).all()
    st, HTH, HTh, nm = loc.measure_reduced(x, xyz)
    assert st == 0 and nm == len(rows) == n_expect
    assert (HTH == HTH.T).all()
    return MC.gram_errors(rows, HTH, HTh, MC.fold_gamma(len(xyz))), HTH, HTh


@pytest.mark.parametrize("n", SIZES)
def test_fold_against_exact_gram(big, n):
    line = []
    for name in MASKS:
        m = _mask(name, n)
        xyz, rows = big.sweep(n, np.flatnonzero(m))
        r, _, _ = _fold_ratio(big.loc, big.x, xyz, int(m.sum()), rows)
        line.append("%s %.3g" % (name, r.max()))
        assert r.max() <= 1.0, (n, name, np.unravel_index(r.argmax(), r.shape))
    print("\n  n %6d  gamma %3.0f  worst err/bar: %s" % (n, MC.fold_gamma(n), ", ".join(line)))


def _mixed_range_scene(O, x):
    """a map of two planes seen from the LiDAR at 0.5 m and at 100 m: the near plane 0.3 m from the sensor (its points at range
    0.5 on a circle of radius 0.4) under a 0.03 m grid, the far one 60 m away (range 100 on a circle of radius 80) with a 0.05 m
    patch around each query; 64 queries of each, alternating lane by lane"""
    rng = np.random.default_rng(12)
    R, RL = O.quat_to_rot(x[3:7]), O.quat_to_rot(x[7:11])

    def basis(nrm):
        e1 = np.cross(nrm, [0.3, 0.5, 0.8])
        e1 /= np.linalg.norm(e1)
        return e1, np.cross(nrm, e1)

    def unit(v):
        return v / np.linalg.norm(v)

    n1, n2 = unit(rng.normal(size=3)), unit(rng.normal(size=3))
    (a1, a2), (b1, b2) = basis(n1), basis(n2)
    t = rng.uniform(0, 2 * np.pi, 64)
    near = 0.3 * n1 + 0.4 * (np.cos(t)[:, None] * a1 + np.sin(t)[:, None] * a2)
    t = rng.uniform(0, 2 * np.pi, 64)
    far = 60.0 * n2 + 80.0 * (np.cos(t)[:, None] * b1 + np.sin(t)[:, None] * b2)
    u = np.arange(-0.6, 0.6, 0.03)
    grid = 0.3 * n1 + u[:, None, None] * a1 + u[None, :, None] * a2
    v = np.arange(-0.2, 0.21, 0.05)
    patch = far[:, None, None, :] + v[None, :, None, None] * b1 + v[None, None, :, None] * b2
    lidar_map = np.concatenate([grid.reshape(-1, 3), patch.reshape(-1, 3)])
    world = (lidar_map @ RL.T + x[11:14]) @ R.T + x[0:3]
    q = np.empty((TILE, 3))
    q[0::2], q[1::2] = near, far
    return world.astype(np.float32), q.astype(np.float32)


def test_fold_mixes_near_and_far_points_in_one_tile(lv, O, scene_xaloc):
    sc = scene_xaloc
    world, q = _mixed_range_scene(O, sc.x_prop)
    prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=1 << 16, max_points=4096)
    loc = lv.Localizer(prm)
    loc.map_build(world)
    xyz = np.tile(q, (4, 1))
    got = loc.match_all(sc.x_prop, xyz)
    rng_m = np.linalg.norm(xyz.astype(np.float64), axis=1)
    near, far = (got["valid"] == 1) & (rng_m < 1), (got["valid"] == 1) & (rng_m > 50)
    assert near.sum() >= 0.9 * 256 and far.sum() >= 0.9 * 256
    r, _, _ = _fold_ratio(loc, sc.x_prop, xyz, int(got["valid"].sum()))
    print("\n  0.5 m and 100 m points, 4 tiles: worst err/bar %.3g" % r.max())
    assert r.max() <= 1.0
    loc.close()


def test_fold_without_extrinsics_is_exactly_zero_there(lv, scene_kitti):
    """kitti, estimate_extrinsics off: rows and columns 6..11 of HTH and entries 6..11 of HTh are exactly zero"""
    sc = scene_kitti
    assert not sc.prm.estimate_extrinsics
    loc = lv.Localizer(sc.prm)
    loc.map_build(sc.map)
    r, HTH, HTh = _fold_ratio(loc, sc.x_prop, sc.sweep, int(loc.match_all(sc.x_prop, sc.sweep)["valid"].sum()))
    assert (HTH[6:, :] == 0).all() and (HTH[:, 6:] == 0).all() and (HTh[6:] == 0).all()
    assert (HTH[:6, :6] != 0).all()
    print("\n  kitti, extrinsics off: worst err/bar %.3g" % r.max())
    assert r.max() <= 1.0
    loc.close()


# ---- the fold inside an update ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 135169])
def test_first_evaluation_of_an_update_against_exact_gram(big, n):
    """lv_correct's first evaluation measures at x_prop with a fresh search, reduces in the step kernel and replays the update
    graph: its logged normal equations meet the entry-wise bar against the exact Gram of lv_measure(x_prop)'s rows"""
    xyz = big.sc.sweep if n == 0 else big.sweep(n, np.arange(n))[0]
    rows = _rows(big.loc, big.x, xyz)
    big.loc.set_state(big.x, big.sc.P0)
    st, _, _, logs = big.loc.correct(xyz)
    assert st == 0 and logs[0]["n_matches"] == len(rows)
    r = MC.gram_errors(rows, logs[0]["HTH"], logs[0]["HTh"], MC.fold_gamma(len(xyz)))
    print("\n  lv_correct, n %d: first evaluation worst err/bar %.3g" % (len(xyz), r.max()))
    assert r.max() <= 1.0 and (logs[0]["HTH"] == logs[0]["HTH"].T).all()


@pytest.mark.parametrize("count", [129, 4097])
def test_device_count_far_below_the_launch_bound(lv, big, count):
    """lv_correct_device_async sizes its grid from n_max = 2^18 (528 blocks, 17 groups) while the device count is 129 or 4097:
    blocks past the count's tiles write zeros, zero group rows add +0 and each group row keeps its warp in the reduction, so
    every evaluation equals lv_correct on the same points bit for bit"""
    loc = big.loc
    xyz = big.sweep(N_BIG, np.arange(N_BIG))[0]
    d_xyz, d_n = loc.upload(xyz), loc.upload(np.array([count], np.int64))
    try:
        loc.set_state(big.x, big.sc.P0)
        assert loc.correct_device_async(d_xyz, d_n, N_BIG, 1, 1.0) == lv.OK
        st, logs = loc.last_logs()
        x_a, P_a = loc.get_state()
    finally:
        loc.device_free(d_xyz)
        loc.device_free(d_n)
    loc.set_state(big.x, big.sc.P0)
    st2, x_b, P_b, logs2 = loc.correct(xyz[:count])
    assert st == st2 == 0 and len(logs) == len(logs2) and logs[0]["n_matches"] == count
    for a, b in zip(logs, logs2):
        assert a["n_matches"] == b["n_matches"]
        assert (a["HTH"] == b["HTH"]).all() and (a["HTh"] == b["HTh"]).all()
    assert (x_a == x_b).all() and (P_a == P_b).all()
