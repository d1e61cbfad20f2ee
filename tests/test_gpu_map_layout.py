"""The device map update (lv_map.cu: keys -> sort -> merge -> dilate -> halo, map_grow, map_clear) checked after every add, three
ways: the layout checker of tests/map_ref.py, the numpy restatement exactly, and the host build (tests/cpu_shim) exactly.

The layout is fixed per voxel by the sequence of adds whatever the thread order: own extents (coordinate bits, ids, order),
halo buckets, the slot set, block masks, the counters and arena_top.  So the warp form of the halo regeneration, concurrent
voxel_insert CAS, the dirty-flag dedup of map_dilate_item, bump allocation of relocated extents, block_mark races and the
growth re-hash are all compared with something exact.  Touched and dirty lists are compared as sets of voxel keys."""
import numpy as np
import pytest

import bench
import geometry as geo
import gpu_shim_binding as GS
import map_ref as R
import shim_binding as S

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]

VOXEL_K = {0.2: 1, 0.4: 2, 0.6: 3}


class Trio:
    """the device map, the host build and the restatement through the same adds"""

    def __init__(self, voxel, cap, max_points, host_cap=0, restate=True):
        self.g = GS.GsMap(cap, max_points, voxel)
        self.h = S.ShimMap(np.zeros((0, 3), np.float32), voxel, 2.0, capacity=host_cap)
        self.r = R.MapRef(VOXEL_K[voxel]) if restate else None
        self.n = 0

    def add(self, xyz, downsample=True):
        self.g.add(xyz, downsample)
        self.h.add(xyz, downsample)
        if self.r is not None:
            self.r.add(xyz, downsample)
            assert self.r.clamped == 0
        self.n += 1
        return self.check("add %d" % self.n)

    def check(self, what):
        return check_all(self.g, self.h, self.r, what)


def check_all(g, h, r, what, lists=True):
    """lists=False: not right after an add (a growth leaves the counters of the last add's lists but not the lists)"""
    gd = g.dump()
    if not lists:
        gd.touched = gd.dirty = np.zeros(0, np.uint32)
    bad = R.check_layout(gd, halo=r is None)          # with a restatement its buckets are compared with the device's below
    assert not bad, (what, bad)
    gl = gd.layout()
    assert int(gd.counters[R.CTR_ERROR]) == 0, what
    if r is not None:
        diff = r.layout().diff(gl, lists)
        assert not diff, (what, "restatement", diff)
    if h is not None:
        hd = h.dump()
        diff = hd.layout().diff(gl, lists)
        assert not diff, (what, "host build", diff)
        assert gd.counters[R.CTR_ARENA_TOP] == hd.counters[R.CTR_ARENA_TOP], what
    return gd


@pytest.fixture(scope="module")
def geo_scenes(lv):
    return {sc.name: sc for sc in geo.all_scenes(lv)}


def _scene_cases():
    out = [("sweep_built", v) for v in (0.2, 0.4, 0.6)] + [("sparse", v) for v in (0.2, 0.4, 0.6)]
    out += [("blind", 0.2), ("cavity", 0.4), ("cluster", 0.4), ("tiny1", 0.2), ("tiny6", 0.6)]
    return out


@pytest.mark.parametrize("name,voxel", _scene_cases())
def test_geometry_scenes(geo_scenes, name, voxel):
    """the scenes of tests/geometry.py: cluster's 3 200-point bucket and relocated extents, sweep_built's own extents beyond
    kCellCache, sparse's isolated voxels"""
    sc = geo_scenes[name]
    mp = max(len(sc.build), max((len(a) for a in sc.adds), default=0))
    t = Trio(voxel, max(1 << 16, sc.capacity), mp, host_cap=sc.capacity)
    t.add(sc.build, downsample=False)
    for a in sc.adds:
        t.add(a)
    if name == "cluster":
        # the add keeps one point of one of the cluster's eight cells: the bucket drops from 3 200 points to ~2 800
        assert "uncached" in t.r.merge_paths and t.r.layout().halo_counts.max() > 2560


@pytest.mark.parametrize("voxel", [0.2, 0.4, 0.6])
def test_face_family(voxel):
    """points at +-1 ulp of cell and voxel faces, old points an ulp outside their voxel, duplicates, 1e-7 copies, and new
    winners on a face inside their voxel that lie in the box of a later cell of the same add (test_map_ref.face_family)"""
    from test_map_ref import face_family
    build, adds = face_family(VOXEL_K[voxel])
    t = Trio(voxel, 1 << 16, 8192)
    t.add(build, downsample=False)
    for a in adds:
        t.add(a)


def test_bench_sequence_from_an_empty_map(lv):
    """the map side of test_tick_from_an_empty_map: the eight bench sweeps at their true poses, visited twice; the first builds
    the map, the others add with the rule (re-observed places: cells with old points, the same point again)"""
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=8, prm=prm)
    t = Trio(0.4, 1 << 19, prm.max_points, host_cap=1 << 18)
    for i in range(16):
        t.add(bench.world_points(sweeps[i % 8], truths[i % 8]), downsample=i > 0)
    assert t.r.merge_paths == {"cached", "uncached"}


def test_scattered_map_at_high_table_load():
    """1 500 isolated points in 65 536 slots (27 slots each: load 0.62): probe chains of 50-80 slots under concurrent CAS.
    (At load 0.7 some key of such a map already needs more than kMaxProbes = 128 probes, and the add reports a full table.)"""
    rng = np.random.default_rng(21)
    pts = rng.uniform(-150, 150, (1500, 3)).astype(np.float32)
    t = Trio(0.2, 1 << 14, 2048, host_cap=1 << 14)
    assert t.g.dims()[0][0] == 1 << 16
    t.add(pts[:750], downsample=False)
    gd = t.add(pts[750:])
    assert int(gd.counters[R.CTR_SLOTS_USED]) > 0.6 * (1 << 16)


def test_non_finite_and_huge_points():
    """NaN, +-inf and 1e9 coordinates are not stored but still take ids"""
    rng = np.random.default_rng(22)
    base = rng.uniform(-5, 5, (3000, 3)).astype(np.float32)
    t = Trio(0.4, 1 << 16, 4096)
    t.add(base, downsample=False)
    bad = base[:400].copy()
    bad[0:100, 0] = np.nan
    bad[100:200, 1] = np.inf
    bad[200:300, 2] = -np.inf
    bad[300:400, 0] = np.float32(1e9)
    mixed = np.concatenate([bad, base[400:800] + np.float32(0.03)])[rng.permutation(800)]
    t.add(mixed)
    t.add(bad, downsample=False)
    assert t.r.next_id == 3000 + 800 + 400


def test_device_count_adds():
    """MapAddCount: a count below min_points adds nothing (ids unchanged), a count above the bound is clamped to it, and
    build_if_empty builds an empty map without the rule"""
    rng = np.random.default_rng(23)
    a = rng.uniform(-4, 4, (3000, 3)).astype(np.float32)
    b = (a[:2000] + rng.normal(0, 0.05, (2000, 3))).astype(np.float32)
    g = GS.GsMap(1 << 16, 4096, 0.4)
    r = R.MapRef(2)
    h = S.ShimMap(np.zeros((0, 3), np.float32), 0.4, 2.0)
    # build_if_empty on an empty map, device count 2500 of 3000: builds from the first 2500 points
    g.add(a, downsample=True, count=2500, min_points=10, build_if_empty=True)
    r.add(a, downsample=True, count=2500, min_points=10, build_if_empty=True)
    h.add(a[:2500], downsample=False)
    check_all(g, h, r, "build_if_empty")
    # below min_points: nothing, not even ids
    g.add(b, count=5, min_points=10, build_if_empty=True)
    r.add(b, count=5, min_points=10, build_if_empty=True)
    assert r.next_id == 2500
    check_all(g, None, r, "below min_points")
    # above the bound: clamped to the 2000 points handed in; the map is not empty, so the rule applies
    g.add(b, count=10 ** 6, min_points=10, build_if_empty=True)
    r.add(b, count=10 ** 6, min_points=10, build_if_empty=True)
    h.add(b, downsample=True)
    check_all(g, h, r, "clamped count")
    assert r.next_id == 4500
    g.close()


def test_growth_mid_sequence_equals_the_map_born_big(lv):
    """map_grow between adds (voxel_rehash_item, block_rehash_item, the arena copy): the map then takes more adds and ends
    equal to a map allocated at the larger capacity from the start, apart from slot positions, arena_top included"""
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=4, prm=prm)
    pts = [bench.world_points(sweeps[i], truths[i]) for i in range(4)]
    small = GS.GsMap(1 << 17, 1 << 16, 0.4)
    big = GS.GsMap(1 << 20, 1 << 16, 0.4)
    r = R.MapRef(2)
    for i, p in enumerate(pts):
        if i == 2:
            small.grow(1 << 20)
            assert small.dims()[0][0] == big.dims()[0][0]
            check_all(small, None, r, "after growth", lists=False)
        for m in (small, big):
            m.add(p, downsample=i > 0)
        r.add(p, downsample=i > 0)
        ds, db = check_all(small, None, r, "small %d" % i), check_all(big, None, r, "big %d" % i)
        assert not ds.layout().diff(db.layout()) and ds.counters[R.CTR_ARENA_TOP] == db.counters[R.CTR_ARENA_TOP]
    small.close()
    big.close()


def test_clear_then_rebuild():
    rng = np.random.default_rng(24)
    a = rng.uniform(-6, 6, (4000, 3)).astype(np.float32)
    b = rng.uniform(-6, 6, (3000, 3)).astype(np.float32)
    t = Trio(0.6, 1 << 16, 4096)
    t.add(a, downsample=False)
    t.add(b)
    t.g.clear()
    h2 = S.ShimMap(np.zeros((0, 3), np.float32), 0.6, 2.0)
    r2 = R.MapRef(3)
    for m in (t.g, h2, r2):
        m.add(b, downsample=False)
    check_all(t.g, h2, r2, "rebuilt")
    for m in (t.g, h2, r2):
        m.add(a)
    check_all(t.g, h2, r2, "after the rebuild")


@pytest.mark.parametrize("name", ["sweep_built@200000,-300000,50", "sparse@430000,0,0"])
@pytest.mark.parametrize("voxel", [0.2, 0.6])
def test_far_scenes_with_clamped_keys(geo_scenes, name, voxel):
    """beyond the key range: no restatement, but the structure holds and the device equals the host build"""
    sc = geo_scenes[name]
    t = Trio(voxel, max(1 << 16, sc.capacity), len(sc.build), host_cap=sc.capacity, restate=False)
    t.add(sc.build, downsample=False)
    rng = np.random.default_rng(25)
    t.add(sc.build[rng.integers(0, len(sc.build), 5000)] + rng.normal(0, 0.1, (5000, 3)).astype(np.float32))


def test_c_abi_map_equals_the_restatement(lv, O, scene_xaloc):
    """lv_map_build, lv_map_add and lv_map_add_last_sweep: lv_map_points (id order) and lv_map_info's points, slots and blocks
    equal the restatement's exactly"""
    sc = scene_xaloc
    om = O.Map(O.KNN_KDTREE)
    om.build(sc.map)
    loc = lv.Localizer(sc.prm)
    r = R.MapRef(VOXEL_K[round(float(sc.prm.voxel_size), 1)])

    def same(what):
        info = loc.map_info()
        lay = r.layout()
        xyz, _ = r.points()
        assert (info["points"], info["slots_used"], info["blocks_used"]) == (lay.points, lay.slots_used, lay.blocks_used), what
        assert info["error_flags"] == 0
        got = loc.map_points()
        assert got.shape == xyz.shape and (got.view(np.uint32) == xyz.view(np.uint32)).all(), what

    loc.map_build(sc.map)
    r.add(sc.map, downsample=False)
    same("lv_map_build")
    rng = np.random.default_rng(26)
    near = (sc.map[:20000] + rng.normal(0, 0.02, (20000, 3))).astype(np.float32)
    loc.map_add(near, downsample=True)
    r.add(near)
    same("lv_map_add")
    x = sc.x_prop.copy()
    for k in range(2):
        loc.set_state(x, sc.P0)
        st, xa, Pa, _ = loc.correct(sc.sweep)
        assert st == 0
        g = om.match_all(xa, sc.oprm, sc.sweep)["g"]          # the fp32 world points lv_map_add_last_sweep merges
        loc.map_add_last_sweep(downsample=True)
        r.add(g)
        same("lv_map_add_last_sweep %d" % k)
        x = xa.copy()
        x[0] += 0.3
    loc.close()
