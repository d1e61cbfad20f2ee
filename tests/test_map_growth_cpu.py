"""Map growth on the host build of the product's per-item code (tests/cpu_shim's shim_map_grow) — no GPU needed.

A growth re-hashes every slot of the voxel and block tables into larger ones (voxel_rehash_item / block_rehash_item of
lv_voxel_map.h, the functions lv_map.cu's rehash kernel runs) and copies the arena's used prefix, so every arena index
stays valid.  On every scene of tests/geometry.py the map is grown at least three times between its build and adds; after
each growth it must be the never-grown map: the same structure (shim_map_check), the same points in id order, the same
slot and block counts, and the same search, plane fit and Jacobian rows, bit for bit.  Sweeps added after a growth must
give the map a handle born at the larger capacity builds.
"""
import ctypes as C

import numpy as np
import pytest

import geometry as geo
import shim_binding as S

K_SLOTS_USED, K_BLOCKS_USED, K_ARENA_TOP = 5, 7, 0    # lv_voxel_map.h kCtr*


def grow(sm, cap):
    S.lib().shim_map_grow(C.c_void_p(sm.h), int(cap))


def counter(sm, k):
    return int(S.lib().shim_map_counter(C.c_void_p(sm.h), k))


@pytest.fixture(scope="module")
def geo_scenes(lv):
    return {sc.name: sc for sc in geo.all_scenes(lv)}


NAMES = ["sweep_built", "sparse", "blind", "cavity", "cluster", "tiny1", "tiny4", "tiny5", "tiny6"]
NAMES += ["%s@%g,%g,%g" % ((kind,) + o) for o in geo.FAR_OFFSETS for kind in ("sweep_built", "sparse")]


def _same_map(a, b, sc, voxel):
    """a (grown) holds exactly what b (never grown) holds"""
    clamped = geo.clamps(sc.build, voxel).any()
    assert a.check() == b.check()
    assert a.check() == 0 or clamped                               # clamped keys break check()'s own neighbour walk
    assert a.error() == b.error() == 0
    assert a.size() == b.size()
    assert (a.points() == b.points()).all()                        # id order
    for k in (K_SLOTS_USED, K_BLOCKS_USED, K_ARENA_TOP):
        assert counter(a, k) == counter(b, k), k


def _same_answers(a, b, sc, voxel, O):
    prm = S.make_params(O.make_params(), voxel)
    ga, gb = a.match_all(sc.x, prm, sc.queries), b.match_all(sc.x, prm, sc.queries)
    for key in ("valid", "nn_idx", "nn_sqd", "plane", "dist", "g", "rows"):
        assert np.array_equal(ga[key], gb[key]), key


@pytest.mark.parametrize("name", NAMES)
def test_growth_between_adds_keeps_the_map(O, geo_scenes, name):
    sc = geo_scenes[name]
    voxel = 0.4
    ref = S.ShimMap(sc.build, voxel, geo.GATE, capacity=sc.capacity)             # never grown
    sm = S.ShimMap(sc.build, voxel, geo.GATE, capacity=sc.capacity // 8)
    growths = 0
    # at least three growths: two after the build, one after every add (and a third after the build when there is no add);
    # the capacity rises geometrically from 1/8 of the scene's to the scene's
    steps = [None, None] + list(sc.adds) + ([None] if not sc.adds else [])
    for i, step in enumerate(steps):
        if step is not None:
            ref.add(step, downsample=True)
            sm.add(step, downsample=True)
        grow(sm, int(sc.capacity / 8 * 8 ** ((i + 1) / len(steps))))
        growths += 1
        _same_map(sm, ref, sc, voxel)
        _same_answers(sm, ref, sc, voxel, O)
    assert growths >= 3


@pytest.mark.parametrize("name", ["sweep_built", "cluster"])
def test_adds_after_a_growth_equal_a_map_born_big(O, geo_scenes, name):
    sc = geo_scenes[name]
    voxel = 0.4
    big = S.ShimMap(sc.build, voxel, geo.GATE, capacity=sc.capacity)
    sm = S.ShimMap(sc.build, voxel, geo.GATE, capacity=sc.capacity // 8)
    grow(sm, sc.capacity // 4)
    grow(sm, sc.capacity)
    for a in sc.adds:
        big.add(a, downsample=True)
        sm.add(a, downsample=True)
    _same_map(sm, big, sc, voxel)
    _same_answers(sm, big, sc, voxel, O)


def test_growth_of_an_empty_map_and_a_scattered_cloud(O):
    """an empty map grows to an empty map; a scattered cloud (27 slots per point) keeps every slot through two growths"""
    sm = S.ShimMap(np.zeros((0, 3), np.float32), 0.4, geo.GATE, capacity=1000)
    grow(sm, 4000)
    assert sm.size() == 0 and counter(sm, K_SLOTS_USED) == 0 and sm.error() == 0
    rng = np.random.default_rng(5)
    pts = rng.uniform(-300, 300, (20_000, 3)).astype(np.float32)
    ref = S.ShimMap(pts[:10_000], 0.4, geo.GATE, capacity=16 * 20_000)
    sm = S.ShimMap(pts[:10_000], 0.4, geo.GATE, capacity=2 * 20_000)
    grow(sm, 8 * 20_000)
    ref.add(pts[10_000:], downsample=True)
    sm.add(pts[10_000:], downsample=True)
    grow(sm, 16 * 20_000)
    assert counter(sm, K_SLOTS_USED) > 27 * 19_000
    assert sm.check() == ref.check() == 0
    assert (sm.points() == ref.points()).all()
    for k in (K_SLOTS_USED, K_BLOCKS_USED, K_ARENA_TOP):
        assert counter(sm, k) == counter(ref, k)
