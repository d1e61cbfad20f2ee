"""The map update against its numpy restatement (tests/map_ref.py), voxel by voxel, and the restatement against the oracle and
the reference's own ikd-Tree — no GPU needed.

The host build (tests/cpu_shim) runs the product's per-item functions of lv_voxel_map.h serially.  After every add its whole
layout must equal the restatement's exactly: own extents (coordinate bits, ids, order), halo buckets, the slot set, block masks
and counters, and pass the layout checker.  Against the ikd-Tree (point by point, box tests over the whole tree) the
restatement may differ only in `flagged` cells, where a point's index cell and the boxes holding it disagree; there is no
count bar."""
import numpy as np
import pytest

import bench
import geometry as geo
import map_ref as R
import shim_binding as S

VOXEL_K = {0.2: 1, 0.4: 2, 0.6: 3}


def _world(sweep, x, O):
    RW = O.quat_to_rot(x[3:7])
    RL = O.quat_to_rot(x[7:11])
    return ((sweep.astype(np.float64) @ RL.T + x[11:14]) @ RW.T + x[0:3]).astype(np.float32)


def _same_layout(sm, ref, what):
    d = sm.dump()
    bad = R.check_layout(d)
    assert not bad, (what, bad)
    diff = ref.layout().diff(d.layout())
    assert not diff, (what, diff)
    assert int(d.counters[R.CTR_ERROR]) == 0, what
    return d


def run_sequence(build, adds, voxel, capacity=0, downsample=True):
    """the host build and the restatement through the same sequence, compared after every add"""
    sm = S.ShimMap(build, voxel, 2.0, capacity=capacity)
    ref = R.MapRef(VOXEL_K[voxel])
    ref.add(build, downsample=False)
    assert ref.clamped == 0
    _same_layout(sm, ref, "build")
    for i, a in enumerate(adds):
        sm.add(a, downsample=downsample)
        ref.add(a, downsample=downsample)
        assert ref.clamped == 0
        _same_layout(sm, ref, "add %d" % i)
    return sm, ref


def xaloc_sweeps(sc, O):
    rng = np.random.default_rng(3)
    out = []
    for k in range(3):
        x = sc.truth.copy()
        x[0:3] += [1.5 * k, 0.2 * k, 0.0]
        out.append(_world(sc.sweep, x, O) + rng.normal(0, 0.01, (len(sc.sweep), 3)).astype(np.float32))
    return out


@pytest.mark.parametrize("voxel", [0.2, 0.4, 0.6])
def test_host_build_equals_restatement_on_three_sweeps(O, scene_xaloc, voxel):
    """the xaloc map, then three sweeps streamed in with the 0.2 m rule (test_cpu_shim's sequence)"""
    sm, ref = run_sequence(scene_xaloc.map, xaloc_sweeps(scene_xaloc, O), voxel)
    assert ref.size() > len(scene_xaloc.map)
    assert "cached" in ref.merge_paths


def _restated_scenes():
    return [("sweep_built", v) for v in (0.2, 0.4, 0.6)] + [("sparse", v) for v in (0.2, 0.4, 0.6)] + \
           [("blind", 0.4), ("cavity", 0.4), ("cluster", 0.4)] + [("tiny%d" % n, v) for n in (1, 6) for v in (0.2, 0.6)]


@pytest.fixture(scope="module")
def geo_scenes(lv):
    return {sc.name: sc for sc in geo.all_scenes(lv)}


@pytest.mark.parametrize("name,voxel", _restated_scenes())
def test_host_build_equals_restatement_on_geometry_scenes(geo_scenes, name, voxel):
    sc = geo_scenes[name]
    sm, ref = run_sequence(sc.build, sc.adds, voxel, capacity=sc.capacity)
    if name in ("sweep_built", "cluster") and voxel >= 0.4:
        # map_merge_run caches own cells while a voxel's points plus one per group fit kCellCache = 48: both paths run here
        assert ref.merge_paths == {"cached", "uncached"}, ref.merge_paths


@pytest.mark.parametrize("name", ["sweep_built@200000,-300000,50", "sparse@430000,0,0"])
@pytest.mark.parametrize("voxel", [0.2, 0.6])
def test_layout_holds_at_clamped_keys(geo_scenes, name, voxel):
    """far scenes whose voxel coordinates clamp: outside the restatement, but every structural invariant holds, halo buckets
    included (where shim_map_check gives up), after a downsampled add on top"""
    sc = geo_scenes[name]
    assert geo.clamps(sc.build, voxel).any() or voxel == 0.6
    sm = S.ShimMap(sc.build, voxel, 2.0, capacity=sc.capacity)
    assert not R.check_layout(sm.dump())
    rng = np.random.default_rng(7)
    add = sc.build[rng.integers(0, len(sc.build), 5000)] + rng.normal(0, 0.1, (5000, 3)).astype(np.float32)
    sm.add(add, downsample=True)
    d = sm.dump()
    assert not R.check_layout(d) and int(d.counters[R.CTR_ERROR]) == 0


# ---- the restatement against the oracle and the reference ikd-Tree -------------------------------------------------------
def _set(xyz):
    return set(map(tuple, np.asarray(xyz, np.float32).tolist()))


def _unexplained(ref, other_xyz):
    """points of the symmetric difference whose index cell is not flagged"""
    got = _set(ref.points()[0])
    diff = got ^ _set(other_xyz)
    if not diff:
        return 0, []
    pts = np.array(sorted(diff), np.float32)
    cellset = ref.flagged_set()
    c = R.cells(pts)
    bad = [tuple(p) for p, q in zip(pts.tolist(), map(tuple, c.tolist())) if q not in cellset]
    return len(diff), bad


def _backends(O):
    return [O.KNN_KDTREE] + ([O.KNN_REF_IKDTREE] if O.ref_available() else [])


OFFSETS = [(0.0, 0.0, 0.0), (1e4, 0.0, 0.0), (6e4, -6e4, 0.0), (2e5, 1.5e5, 50.0)]


@pytest.fixture(scope="module")
def bench_sweeps(lv):
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=4, prm=prm)
    return sweeps, truths


@pytest.mark.parametrize("offset", OFFSETS)
def test_restatement_against_the_ikd_tree(O, bench_sweeps, offset):
    """a raw sweep as the map and three sweeps added with the rule, moved by `offset`: the host build equals the restatement,
    and every point the restatement and the ikd-Tree disagree on lies in a flagged cell.  The last offset is still inside the key range at voxel 0.4."""
    sweeps, truths = bench_sweeps
    off = np.asarray(offset, np.float64)
    pts = []
    for k in range(4):
        x = truths[k].copy()
        x[0:3] += off
        pts.append(bench.world_points(sweeps[k], x))
    sm, ref = run_sequence(pts[0], pts[1:], 0.4)        # the host build equals the restatement here too, after every add
    frac = len(ref.flagged) / len(ref.cells_seen)
    print("offset %s: %d flagged cells of %d touched (%.2e)" % (offset, len(ref.flagged), len(ref.cells_seen), frac))
    if not off.any():
        assert frac < 1e-3                     # the exemption is not vacuous near the origin
    oracle = None
    for be in _backends(O):
        om = O.Map(be)
        om.build(pts[0])
        for a in pts[1:]:
            om.add(a, downsample=True)
        got = om.points()
        n, bad = _unexplained(ref, got)
        print("  backend %d: %d points differ, %d unexplained" % (be, n, len(bad)))
        if oracle is None:
            oracle = _set(got)                 # the oracle (KNN_KDTREE): Add_Points point by point, deterministic
            assert not bad, (be, n, bad[:5])
        else:
            # at the far offset some runs of the ikd-Tree keep two points of one unflagged cell that the oracle and other runs
            # of the tree do not (DESIGN.md §2; the cause is not established).  There, and only there, at most four such points
            # are let through, each one where this run of the tree differs from the oracle too
            own = _set(got) ^ oracle
            if offset != OFFSETS[-1]:
                assert not bad, (be, n, bad[:5])
            assert len(bad) <= 4 and all(p in own for p in bad), (be, n, [p for p in bad if p not in own][:5])
    if off.any() and offset[0] >= 6e4:
        assert len(ref.flagged) > 0


def across_in_voxel(k, rng, n=200):
    """pairs for one add, away from the rest of the family: A on a face fl(c ds) inside a voxel (c % k != 0) that divides back
    to c - 1, so A wins the empty cell c - 1 and then lies in the box of cell c, a later group of the same voxel; B at the
    centre of cell c, closer to it, must then replace A (empty for k = 1, where every face is a voxel face)"""
    c = np.arange(-4000, 4000, dtype=np.int64)
    across = c[(R.cells(R.cell_lo(c)[:, None])[:, 0] == c - 1) & (c % k != 0)]
    if len(across) == 0:
        return np.zeros((0, 3), np.float32)
    pick = rng.choice(across, n)
    axis = rng.integers(0, 3, n)
    a = (np.floor(rng.uniform(25, 45, (n, 3))) * 0.2 + 0.1).astype(np.float32)     # cell centres on the other axes
    a[np.arange(n), axis] = R.cell_lo(pick)
    b = a.copy()
    b[np.arange(n), axis] = R.cell_lo(pick) + np.float32(0.1)
    return np.concatenate([a, b])


def face_family(k, seed=0):
    """points at +-1 ulp of cell faces and voxel faces, old points whose box is across a voxel face, exact duplicates and
    near copies 1e-7 away; returns (build, [adds])"""
    rng = np.random.default_rng(seed)
    ds = R.DS
    # faces fl(c ds) whose value divides back to c - 1: the point there is indexed in cell c - 1 but lies in box c
    c = np.arange(-4000, 4000, dtype=np.int64)
    lo = R.cell_lo(c)
    across = c[R.cells(lo[:, None])[:, 0] == c - 1]
    vface = across[across % k == 0]
    pick = rng.choice(vface, 200, replace=len(vface) < 200)
    base = rng.uniform(-3, 3, (len(pick), 3)).astype(np.float32)
    axis = rng.integers(0, 3, len(pick))
    old = base.copy()
    old[np.arange(len(pick)), axis] = R.cell_lo(pick)                 # an ulp outside its voxel by the box test
    # new points near the centre of the box those old points lie in
    near = old.copy()
    near[np.arange(len(pick)), axis] = R.cell_lo(pick) + np.float32(0.1)
    # +-1 ulp around faces of every kind
    faces = rng.choice(c, 400)
    fx = rng.uniform(-3, 3, (800, 3)).astype(np.float32)
    ax2 = rng.integers(0, 3, 800)
    f = np.concatenate([R.cell_lo(faces)] * 2)
    fx[np.arange(800), ax2] = np.concatenate([np.nextafter(f[:400], np.float32(np.inf)), np.nextafter(f[400:], np.float32(-np.inf))])
    surface = rng.uniform(-3, 3, (3000, 3)).astype(np.float32)
    build = np.concatenate([old, surface, fx[:400]])
    adds = [np.concatenate([near, fx[400:], surface[:300], (surface[300:600] + np.float32(1e-7)).astype(np.float32),
                            surface[600:700], surface[600:700], across_in_voxel(k, rng)]),
            np.concatenate([old[::-1], fx[:400] + np.float32(1e-7), near[::2]])]
    return build, adds


@pytest.mark.parametrize("voxel", [0.2, 0.4, 0.6])
def test_face_family(O, voxel):
    """the restatement equals the host build on the face family, and differs from the ikd-Tree there — only in flagged cells"""
    build, adds = face_family(VOXEL_K[voxel])
    sm, ref = run_sequence(build, adds, voxel)
    total = 0
    for be in _backends(O):
        om = O.Map(be)
        om.build(build)
        for a in adds:
            om.add(a, downsample=True)
        n, bad = _unexplained(ref, om.points())
        assert not bad, (be, n, bad[:5])
        total += n
    assert total > 0                          # the family does reach the cases where the two rules part
    assert len(ref.flagged) > 0


@pytest.mark.parametrize("voxel", [0.4, 0.6])
def test_winner_across_a_face_inside_its_voxel(O, voxel):
    """A = fl(c * 0.2) divides back to c - 1 (at voxel 0.4, c = -21: A = -4.2000003): A is indexed in cell c - 1 but lies in
    the box of cell c, and both cells are in one voxel.  B at the centre of cell c is added with A.  A wins cell c - 1, then is
    an old point of cell c, and B replaces it: the map keeps {B} as the ikd-Tree does, on the cached path of map_merge_run as
    on the uncached one."""
    k = VOXEL_K[voxel]
    c = np.arange(-40, 40, dtype=np.int64)
    c = c[(R.cells(R.cell_lo(c)[:, None])[:, 0] == c - 1) & (c % k != 0)]
    c = int(c[np.argmin(np.abs(c + 21))])
    a = np.float32([R.cell_lo(np.int64(c)), 0.05, 0.05])
    assert R.cells(a[None])[0, 0] == c - 1 and R.box_cell(a[None])[0, 0] == c
    b = a.copy()
    b[0] = a[0] + np.float32(0.1)
    for fill in (0, 60):                                               # 60 more points in the voxel: the uncached path
        pad = np.float32([[R.cell_lo(np.int64(c)) + np.float32(0.1), 0.2 * (k - 1) + 0.1, 0.05]] * fill).reshape(-1, 3)
        build = np.concatenate([np.float32([[3.0, 3.0, 3.0]]), pad]).astype(np.float32)
        sm, ref = run_sequence(build, [np.float32([a, b])], voxel)
        assert ref.merge_paths == {"uncached" if fill else "cached"}
        got = _set(ref.points()[0])
        assert tuple(b.tolist()) in got and tuple(a.tolist()) not in got
        for be in _backends(O):
            om = O.Map(be)
            om.build(build)
            om.add(np.float32([a, b]), downsample=True)
            assert _set(om.points()) == got, be


def test_restatement_rules_by_hand():
    """tie rules and ids on hand-made cells (k = 2, one voxel)"""
    ref = R.MapRef(2)
    a = np.float32([0.05, 0.05, 0.05])                                 # cell (0, 0, 0), centre 0.1f
    ref.add(np.float32([a, [0.3, 0.3, 0.3]]), downsample=False)         # cells (0,0,0) and (1,1,1) of voxel (0,0,0)
    assert ref.next_id == 2 and ref.size() == 2
    # the very point the cell holds, new: it wins the tie, but it is the same point, so nothing changes
    ref.add(np.float32([a]))
    assert ref.size() == 2 and len(ref.touched) == 0 and ref.next_id == 3
    # two new points at exactly the same, smaller distance to the centre: the later one replaces the old point
    h = np.float32(2.0 ** -10)
    c = np.float32(0.1)
    ref.add(np.float32([[c + h, c, c], [c - h, c, c], [np.nan, 0, 0], [1e9, 0, 0]]))
    xyz, ids = ref.points()
    assert ids.tolist() == [1, 4] and (xyz[1] == np.float32([c - h, c, c])).all()
    assert ref.next_id == 7                                            # ids count the unstored NaN and 1e9 points too
    assert len(ref.touched) == 1
