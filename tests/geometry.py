"""Seeded map geometries for the search paths the dense surface map of conftest.Scene never reaches.

On a SynthWorld surface map with queries on its surfaces nearly every query is settled by level 0 in its home voxel's
halo bucket.  Each scene here is built for one other path of the search (lv_voxel_search.h, lv_measure.cu) or of the map
update (lv_voxel_map.h):

  sweep_built   raw first sweep as the map (built without the 0.2 m rule, as Mapper.cpp:26 does), three more sweeps added
                at their true poses with the rule, queries = a later sweep at its predicted state: very dense voxels near the
                sensor (own extents above kCellCache, uncached map_merge_run), sparse rings at range (K1b)
  sparse        uniform points, mean spacing 0.5 m: most queries uncertified at level 0, ring search with a finite bound
  blind         surfaces, queries 0.9-1.9 m off them: no level-0 slot but five points inside the gate (the blind path)
  cavity        every 0.4 m voxel of a volume occupied except an empty sphere of radius 1.3 m, queries near its centre: blind,
                with more than kRingCands (1024) occupied voxels in the r = 5 cube
  cluster       one 0.4 m voxel holding 3200 points, repeated map points, then a downsampled add into both: a 3200-point
                halo bucket through the per-query scan, cells with several old points
  tiny          maps of 1, 4, 5 and 6 points: fewer than five neighbours
  far           sweep_built and sparse moved to (2e5, -3e5, 50) and (4.3e5, 0, 0): fp32 ulps of 0.016-0.03 m, and voxel
                coordinates past the 21-bit key range, where voxel_of_cell clamps

A scene is its map (`build`, then `adds`, each merged with the 0.2 m rule), its queries (LiDAR frame), the state to measure
them at and the voxel sizes it is meant for.  Identity-pose scenes give their queries in the world frame.
"""
import numpy as np

import bench

GATE = 2.0                      # MAX_DIST_PLANE of xaloc.yaml
FAR_OFFSETS = ((2e5, -3e5, 50.0), (4.3e5, 0.0, 0.0))
KEY_BIAS, KEY_MAX = 1 << 20, 0x1FFFFF


class GeoScene:
    def __init__(self, name, build, queries, x, voxels, adds=(), path="", scattered=False):
        self.name = name
        self.build = np.ascontiguousarray(build, np.float32)
        self.adds = [np.ascontiguousarray(a, np.float32) for a in adds]
        self.queries = np.ascontiguousarray(queries, np.float32)
        self.x = np.array(x, np.float64)
        self.voxels = tuple(voxels)
        self.path = path
        # map points the tables are sized for: isolated points (scattered maps) take 27 table slots each
        self.capacity = (16 if scattered else 4) * self.n_map_input()

    def n_map_input(self):
        return len(self.build) + sum(len(a) for a in self.adds)

    def oracle_map(self, O, backend=None):
        om = O.Map(O.KNN_KDTREE if backend is None else backend)
        om.build(self.build)
        for a in self.adds:
            om.add(a, downsample=True)
        return om

    def shim_map(self, S, voxel):
        sm = S.ShimMap(self.build, voxel, GATE, capacity=self.capacity)
        for a in self.adds:
            sm.add(a, downsample=True)
        return sm

    def localizer(self, lv, prm):
        loc = lv.Localizer(prm)
        loc.map_build(self.build)
        for a in self.adds:
            loc.map_add(a, downsample=True)
        loc.map_status()
        return loc

    def params(self, lv, voxel):
        prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_map_points=max(1 << 16, self.capacity),
                                  max_points=max(4096, len(self.queries), max((len(a) for a in self.adds), default=0)))
        prm.voxel_size = voxel
        return prm


def identity_state(lv):
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml")
    x, P = lv.init_state_host(prm)
    x[0:3] = 0
    x[3:7] = [0, 0, 0, 1]
    x[7:11] = [0, 0, 0, 1]
    x[11:14] = 0
    return x, P


def _shift(x, offset):
    x = np.array(x, np.float64).copy()
    x[0:3] += offset
    return x


def sweep_built(lv, offset=(0.0, 0.0, 0.0)):
    prm = bench.config_params(lv, "cfg1")
    world, mp, sweeps, x_props, truths = bench.make_scene(lv, 0, n_sweeps=5, prm=prm)
    off = np.asarray(offset, np.float64)
    build = bench.world_points(sweeps[0], _shift(truths[0], off))
    adds = [bench.world_points(sweeps[k], _shift(truths[k], off)) for k in (1, 2, 3)]
    name = "sweep_built" if not off.any() else "sweep_built@%g,%g,%g" % tuple(offset)
    if off.any():
        # far from the origin the 0.2 m rule of the map update does not reproduce the reference's box test (DESIGN.md §2):
        # these scenes test the search, so all four sweeps go in un-downsampled
        build, adds = np.concatenate([build] + adds), []
    return GeoScene(name, build, sweeps[4][::2], _shift(x_props[4], off), (0.2, 0.4, 0.6), adds,
                    "uncached merge, relocations, K1b at range")


def sparse(lv, offset=(0.0, 0.0, 0.0)):
    rng = np.random.default_rng(101)
    lo, hi = np.array([-15.0, -15.0, -4.0]), np.array([15.0, 15.0, 4.0])
    n = int(np.prod(hi - lo) / 0.5 ** 3)
    off = np.asarray(offset, np.float64)
    pts = (rng.uniform(lo, hi, (n, 3)) + off).astype(np.float32)
    q = (rng.uniform(lo + 2.5, hi - 2.5, (6000, 3)) + off).astype(np.float32)
    x, _ = identity_state(lv)
    name = "sparse" if not off.any() else "sparse@%g,%g,%g" % tuple(offset)
    return GeoScene(name, pts, q, x, (0.2, 0.4, 0.6), (), "uncertified at level 0, finite ring bound", scattered=True)


def blind(lv):
    world = lv.SynthWorld(20260924, 100000)
    prm = lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml")
    truth = world.pose(8.0, prm)
    g = bench.world_points(world.sweep(truth, rings=32, azimuths=256, seed=20260931), truth)
    rng = np.random.default_rng(102)
    d = rng.normal(0, 1, (len(g), 3))
    d *= (rng.uniform(0.9, 1.9, len(g)) / np.linalg.norm(d, axis=1))[:, None]
    x, _ = identity_state(lv)
    return GeoScene("blind", world.map(), (g + d).astype(np.float32), x, (0.2, 0.4, 0.6), (), "no level-0 slot")


CAVITY_CENTRE = np.array([0.2, 0.2, 0.2])            # the centre of a 0.4 m voxel
CAVITY_RADIUS = 1.3


def cavity(lv):
    rng = np.random.default_rng(103)
    ax = np.arange(-4.0, 4.4, 0.2)
    grid = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3) + 0.1    # two points per axis and 0.4 m voxel
    grid += rng.uniform(-0.04, 0.04, grid.shape)
    keep = np.linalg.norm(grid - CAVITY_CENTRE, axis=1) > CAVITY_RADIUS
    d = rng.normal(0, 1, (3000, 3))
    d *= (rng.uniform(0, 0.18, 3000) / np.linalg.norm(d, axis=1))[:, None]
    x, _ = identity_state(lv)
    return GeoScene("cavity", grid[keep], CAVITY_CENTRE + d, x, (0.4,), (), "blind, n_list > kRingCands")


CLUSTER_VOXEL = np.array([5.2, 1.2, -0.4])            # low corner of the 0.4 m voxel holding the cluster


def cluster(lv):
    rng = np.random.default_rng(104)
    world = lv.SynthWorld(20260925, 40000)
    base = world.map()
    blob = CLUSTER_VOXEL + rng.uniform(0.01, 0.39, (3200, 3))
    dup = np.repeat(base[:1500], 3, axis=0)
    build = np.concatenate([base, blob.astype(np.float32), dup])
    # the add: a few points into ONE of the cluster's eight 0.2 m cells (the rule keeps one point of that cell; the other seven
    # keep the bucket above the staging budget), exact copies and near copies of repeated points, and fresh surface points
    cell = CLUSTER_VOXEL + 0.2 + rng.uniform(0.01, 0.19, (8, 3))
    near = base[1500:2500] + rng.normal(0, 0.002, (1000, 3))
    add = np.concatenate([cell, base[:400], base[:200] + 1e-7, near, base[3000:6000] + rng.normal(0, 0.05, (3000, 3))])
    q = np.concatenate([CLUSTER_VOXEL + 0.2 + rng.normal(0, 0.25, (2500, 3)),
                        base[rng.integers(0, 2500, 2500)] + rng.normal(0, 0.05, (2500, 3)),
                        base[rng.integers(0, len(base), 2000)] + rng.normal(0, 0.1, (2000, 3))])
    x, _ = identity_state(lv)
    return GeoScene("cluster", build, q, x, (0.4,), [add.astype(np.float32)], "3200-point bucket, n_old > 1")


def tiny(lv, n):
    rng = np.random.default_rng(105 + n)
    pts = np.float32([3.0, -2.0, 1.0]) + rng.normal(0, 0.3, (n, 3))
    pts[:, 2] = 1.0 + 0.01 * rng.normal(0, 1, n)                # nearly a plane, so five points can fit one
    q = pts[rng.integers(0, n, 400)] + rng.normal(0, 0.3, (400, 3))
    x, _ = identity_state(lv)
    return GeoScene("tiny%d" % n, pts, q, x, (0.2, 0.4, 0.6), (), "fewer than five neighbours")


def all_scenes(lv):
    out = [sweep_built(lv), sparse(lv), blind(lv), cavity(lv), cluster(lv)]
    out += [tiny(lv, n) for n in (1, 4, 5, 6)]
    out += [sweep_built(lv, o) for o in FAR_OFFSETS] + [sparse(lv, o) for o in FAR_OFFSETS]
    return out


def clamps(points, voxel):
    """True where a point's voxel coordinate falls outside the 21-bit key range (voxel_of_cell clamps it)"""
    k = max(1, int(np.floor(voxel / 0.2 + 0.5)))
    c = np.floor(np.floor(points.astype(np.float32) / np.float32(0.2)) / k) + KEY_BIAS
    return ((c < 0) | (c > KEY_MAX)).any(1)


def max_voxel_count(points, voxel):
    k = max(1, int(np.floor(voxel / 0.2 + 0.5)))
    c = np.floor(np.floor(points.astype(np.float32) / np.float32(0.2)) / k).astype(np.int64)
    _, cnt = np.unique(c, axis=0, return_counts=True)
    return int(cnt.max())


def cube_occupancy(points, centre, voxel, r):
    """occupied voxels in the (2r+1)^3 cube around the voxel of `centre`"""
    v = np.floor(points / voxel).astype(np.int64)
    h = np.floor(np.asarray(centre) / voxel).astype(np.int64)
    inside = (np.abs(v - h) <= r).all(1)
    return len(np.unique(v[inside], axis=0))
