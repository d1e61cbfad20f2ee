"""lv_process_cloud_device — Accumulator::process (msg2points -> temporal_downsample -> sort_points) on the message bytes in
HBM — against the composition of the host functions, bit for bit on every output: lv_pointcloud2_to_points_checked on the
same bytes, the decimation rule on the raw message index (frontend_ref.temporal), lv_time_sort_indices on the kept times,
then the gathers.  Then the chain bag -> lv_process_cloud_device -> lv_compensate_device -> lv_voxelgrid_downsample_device ->
lv_correct_device against the same chain on host buffers."""
import ctypes as C

import numpy as np
import pytest

import bagwriter as W
import frontend_ref as F
from test_bag_reader import OUSTER as BAG_OUSTER, VELO as BAG_VELO, BagMessage, PC2View
from test_wire_format import make_cloud

pytestmark = pytest.mark.gpu

LIDARS = ["velodyne", "hesai", "ouster", "custom"]
STAMP_US = 1_695_000_000_350_000
FRT = 0.1


def u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


def u64(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def prm(lv):
    return lv.default_params(max_points=1 << 16, max_map_points=1 << 16)


@pytest.fixture(scope="module")
def loc(lv, prm):
    h = lv.Localizer(prm)
    yield h
    h.close()


def host_checked(lv, lidar, pts, stamp_us, sb, ob, frt, data_bytes=None):
    """lv_pointcloud2_to_points_checked on the array's bytes"""
    L = lv.lib()
    pts = np.ascontiguousarray(pts)
    n = len(pts)
    xyz, t = np.zeros((n, 3), np.float32), np.zeros(n, np.float64)
    inten, rng = np.zeros(n, np.float32), np.zeros(n, np.float32)
    fp, dp = C.POINTER(C.c_float), C.POINTER(C.c_double)
    lay = lv.cloud_layout(lidar, pts.dtype)
    L.lv_pointcloud2_to_points_checked.argtypes = None        # test_bag_reader declares them with its own layout struct
    st = L.lv_pointcloud2_to_points_checked(lv.LIDAR_TYPES[lidar], C.byref(lay), pts.ctypes.data_as(C.POINTER(C.c_uint8)),
                                            C.c_int64(pts.nbytes if data_bytes is None else data_bytes), C.c_int64(n),
                                            C.c_uint64(stamp_us), int(sb), int(ob), C.c_double(frt), xyz.ctypes.data_as(fp),
                                            t.ctypes.data_as(dp), inten.ctypes.data_as(fp), rng.ctypes.data_as(fp))
    assert st == lv.OK
    return xyz, t, inten, rng


def host_process(lv, lidar, pts, stamp_us, sb, ob, frt, rate, md):
    """the composition lv_process_cloud_device must equal"""
    xyz, t, inten, rng = host_checked(lv, lidar, pts, stamp_us, sb, ob, frt)
    keep = F.temporal(xyz, rate, md)
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rng[order], order.astype(np.int32)


def assert_same(got, ref, what=""):
    names = ("xyz", "time", "intensity", "range", "idx")
    for name, a, b in zip(names, got, ref):
        assert a.shape == b.shape, (what, name, a.shape, b.shape)
        if name == "time":
            assert (u64(a) == u64(b)).all(), (what, name)
        else:
            assert (u32(a) == u32(b)).all(), (what, name)


def device_process(lv, loc, lidar, pts, stamp_us, sb, ob, frt, rate, md, shift=0):
    """the message's bytes at base + shift of a device buffer (the alignment a bag hands out is arbitrary)"""
    pts = np.ascontiguousarray(pts)
    n, nb = len(pts), pts.nbytes
    d_msg = loc.device_alloc(nb + 16)
    outs = [loc.device_alloc(max(k * n, 1)) for k in (12, 8, 4, 4, 4)]
    try:
        lv._check(loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg + shift), pts.ctypes.data_as(C.c_void_p), nb))
        m = loc.process_cloud_device(lidar, lv.cloud_layout(lidar, pts.dtype), d_msg + shift, nb, n, stamp_us, sb, ob, frt, rate, md,
                                     *outs)
        host = (np.empty((m, 3), np.float32), np.empty(m), np.empty(m, np.float32), np.empty(m, np.float32), np.empty(m, np.int32))
        return tuple(loc.download(d, a) for d, a in zip(outs, host))
    finally:
        for d in [d_msg] + outs:
            loc.device_free(d)


# ---- every LiDAR type x time semantics x rate x min_dist ---------------------------------------------------------------
@pytest.mark.parametrize("lidar", LIDARS)
@pytest.mark.parametrize("sb,ob", [(False, True), (True, True), (False, False), (True, False)])
@pytest.mark.parametrize("rate", [0, 1, 4, 7])
@pytest.mark.parametrize("md", [0.0, 3.0])
def test_process_cloud_equals_host_composition(lv, loc, lidar, sb, ob, rate, md):
    rng = np.random.default_rng(17)
    pts = make_cloud(lidar, 3001, rng)
    near = rng.choice(len(pts), 400, replace=False)               # some points inside min_dist
    for k in "xyz":
        pts[k][near] *= np.float32(0.02)
    pts = pts[rng.permutation(len(pts))]                          # times out of message order: the sort has work
    got = loc.process_cloud(lidar, pts, STAMP_US, sb, ob, FRT, rate, md)
    ref = host_process(lv, lidar, pts, STAMP_US, sb, ob, FRT, rate, md)
    assert len(ref[0]) > 0
    assert_same(got, ref, (lidar, sb, ob, rate, md))
    assert (np.diff(got[1]) >= 0).all()


# ---- edge families, on the unaligned layouts and at base + 0 / 1 / 2 -------------------------------------------------------
def edge_clouds(lidar, rate):
    rng = np.random.default_rng(23)
    out = {}
    for n in sorted({0, 1, max(rate - 1, 0), 255, 256, 257}):
        out["n%d" % n] = make_cloud(lidar, n, rng)
    c = make_cloud(lidar, 700, rng)
    for k in "xyz":
        c[k] *= np.float32(1e-3)
    out["all_within_min_dist"] = c
    c = make_cloud(lidar, 700, rng)
    out["reversed"] = c[::-1].copy()
    c = make_cloud(lidar, 900, rng)
    for k, v in (("x", np.nan), ("y", np.nan), ("z", np.nan)):
        c[k][rng.choice(900, 50, replace=False)] = v
    out["nan_xyz"] = c
    c = make_cloud(lidar, 600, rng)
    tf = {"velodyne": "time", "ouster": "t"}.get(lidar, "timestamp")
    if lidar == "ouster":
        # a whole column shares one t (128 rings), the message shuffled so that stability is visible; and t around 1e9 ns,
        # where nanosec2sec carries into the seconds
        c = make_cloud(lidar, 128 * 16, rng)
        c["t"] = np.repeat(np.arange(16, dtype=np.uint32) * 1_000_000, 128)
        out["column_ties"] = c[rng.permutation(len(c))]
        c = make_cloud(lidar, 600, rng)
        c["t"] = (999_999_700 + rng.integers(0, 600, 600)).astype(np.uint32)
        c["t"][[0, -1]] = (999_999_000, 1_000_000_300)
        out["t_near_1e9ns"] = c
    else:
        z = np.where(rng.random(600) < 0.5, -0.0, 0.0)
        c[tf][:] = z
        c[tf][[0, -1]] = 0.0
        out["signed_zero"] = c
        c = make_cloud(lidar, 600, rng)
        mid = rng.choice(np.arange(1, 599), 60, replace=False)
        c[tf][mid[:30]] = np.inf
        c[tf][mid[30:]] = -np.inf
        out["inf"] = c
        c = make_cloud(lidar, 600, rng)
        c[tf][:] = c[tf][rng.integers(0, 20, 600)]               # heavy ties without a column structure
        out["ties"] = c[rng.permutation(600)]
    return out


STAMPS = [STAMP_US, (2**31 + 5) * 1_000_000 + 999_999, (2**32 + 7) * 1_000_000 + 1, 999_999]   # int truncation of the seconds


@pytest.mark.parametrize("lidar", LIDARS)
@pytest.mark.parametrize("rate,md", [(1, 0.0), (4, 3.0), (7, 3.0)])
@pytest.mark.parametrize("shift", [0, 1, 2])
def test_process_cloud_edge_families(lv, loc, lidar, rate, md, shift):
    for name, pts in edge_clouds(lidar, rate).items():
        for k, stamp in enumerate(STAMPS):
            sb, ob = k % 2 == 0, k < 2
            got = device_process(lv, loc, lidar, pts, stamp, sb, ob, FRT, rate, md, shift)
            ref = host_process(lv, lidar, pts, stamp, sb, ob, FRT, rate, md)
            assert_same(got, ref, (lidar, name, stamp, rate, md, shift))
        if name == "all_within_min_dist" and md > 0:
            assert len(got[0]) == 0
        if name == "nan_xyz":                                     # dropped by min_dist < |p|, not an error
            assert len(got[0]) > 0 and not np.isnan(got[0]).any()


# ---- sizes and the handle's scratch ----------------------------------------------------------------------------------------
def sized_cloud(lidar, rings, cols, seed):
    rng = np.random.default_rng(seed)
    c = make_cloud(lidar, rings * cols, rng)
    if lidar == "ouster":
        c["t"] = np.repeat(np.arange(cols, dtype=np.uint32) * (100_000_000 // cols), rings)
    else:
        c["time"] = np.repeat(np.linspace(0, 0.1, cols, dtype=np.float32), rings)
    return c


def test_process_cloud_sizes_reuse_the_scratch(lv, prm):
    clouds = [("ouster", sized_cloud("ouster", 128, 2048, 1)),        # cfg3 shape
              ("velodyne", sized_cloud("velodyne", 64, 1024, 2)),     # cfg1 shape
              ("velodyne", sized_cloud("velodyne", 128, 16384, 3))]   # 2^21 points
    loc = lv.Localizer(prm)
    for lidar, pts in clouds:
        got = loc.process_cloud(lidar, pts, STAMP_US, False, True, FRT, 4, 3.0)
        fresh = lv.Localizer(prm)
        assert_same(got, fresh.process_cloud(lidar, pts, STAMP_US, False, True, FRT, 4, 3.0), ("fresh", len(pts)))
        fresh.close()
        assert_same(got, host_process(lv, lidar, pts, STAMP_US, False, True, FRT, 4, 3.0), ("host", len(pts)))
    prof = loc.profile()
    assert prof["total_launches"] == 6 * len(clouds)
    loc.close()


# ---- refusals -----------------------------------------------------------------------------------------------------------------
def raw_call(lv, loc, lidar, lay, d_data, data_bytes, n, outs, rate=4, md=3.0):
    m = C.c_int64(-1)
    st = loc.L.lv_process_cloud_device(loc.h, lv.LIDAR_TYPES[lidar], C.byref(lay), C.c_void_p(d_data), data_bytes, n, STAMP_US, 1, 1,
                                       FRT, rate, md, *[C.c_void_p(o) for o in outs], C.byref(m))
    return st, m.value


def test_process_cloud_refusals_leave_the_handle_usable(lv, prm):
    rng = np.random.default_rng(31)
    good = make_cloud("velodyne", 1000, rng)
    ref = host_process(lv, "velodyne", good, STAMP_US, True, True, FRT, 4, 3.0)
    bad_t = good.copy()
    bad_t["time"][3] = np.nan                                     # index 3: kept by rate 4
    dropped_nan = good.copy()
    dropped_nan["time"][4] = np.nan                                # index 4: decimated away, never sorted
    assert 3 in F.temporal(host_checked(lv, "velodyne", good, STAMP_US, True, True, FRT)[0], 4, 3.0)
    loc = lv.Localizer(prm)
    n, nb = len(good), good.nbytes
    d_msg = loc.device_alloc(2 * nb + 64)
    outs = [loc.device_alloc(k * n) for k in (12, 8, 4, 4, 4)]
    lay = lv.cloud_layout("velodyne", good.dtype)

    def check_next_call():
        st, m = raw_call(lv, loc, "velodyne", lay, d_msg, nb, n, outs)
        assert st == lv.OK and m == len(ref[0])
        got = tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref))
        assert_same(got, ref, "after a refusal")

    lv._check(loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg), bad_t.ctypes.data_as(C.c_void_p), nb))
    st, m = raw_call(lv, loc, "velodyne", lay, d_msg, nb, n, outs)
    assert st == lv.ERR_ARG and b"timestamp" in loc.L.lv_last_error() and m == 0
    lv._check(loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg), good.ctypes.data_as(C.c_void_p), nb))
    check_next_call()
    bad_lay = lv.CloudLayout.from_buffer_copy(lay)
    bad_lay.off_time = lay.point_step - 2
    assert raw_call(lv, loc, "velodyne", bad_lay, d_msg, nb, n, outs)[0] == lv.ERR_ARG
    check_next_call()
    assert raw_call(lv, loc, "velodyne", lay, d_msg, nb - 1, n, outs)[0] == lv.ERR_ARG
    check_next_call()
    for k, o in enumerate(outs):                                  # any output inside the message bytes
        over = list(outs)
        over[k] = d_msg + nb - 4
        st, _ = raw_call(lv, loc, "velodyne", lay, d_msg, nb, n, over)
        assert st == lv.ERR_ARG and b"overlaps" in loc.L.lv_last_error(), k
        check_next_call()
    # a NaN time that the decimator drops is never sorted: no error, and the host composition is defined
    assert_same(device_process(lv, loc, "velodyne", dropped_nan, STAMP_US, True, True, FRT, 4, 3.0),
                host_process(lv, "velodyne", dropped_nan, STAMP_US, True, True, FRT, 4, 3.0), "dropped NaN")
    for d in [d_msg] + outs:
        loc.device_free(d)
    loc.close()


# ---- the chain from the bag to the update -------------------------------------------------------------------------------------
def test_bag_to_update_chain_equals_host_chain(lv, scene_xaloc, tmp_path):
    """skewed Velodyne and Ouster sweeps of the synthetic scene in a bag: lv_bag_parse_pointcloud2 -> lv_process_cloud_device ->
    lv_compensate_device -> lv_voxelgrid_downsample_device -> lv_correct_device equals _checked -> host decimation / sort ->
    lv_compensate -> lv_voxelgrid_downsample -> lv_correct bit for bit: state, covariance and every log"""
    sc = scene_xaloc
    rng = np.random.default_rng(9)
    t1, t2 = 10.0, 10.1
    st_t = np.linspace(t1 - 0.012, t2 - 0.004, 4)
    imu_t = np.arange(st_t[0] + 0.5e-3, t2 + 4e-3, 2.5e-3)
    imu_a = (np.array([0.3, -0.2, 9.8]) + rng.normal(0, 0.05, (len(imu_t), 3))).astype(np.float32)
    imu_w = (np.array([0.0, 0.0, 0.5]) + rng.normal(0, 0.01, (len(imu_t), 3))).astype(np.float32)
    states = []
    for ts in st_t:
        x = sc.world.pose(8.0 + 15.0 * (ts - t1), sc.prm).copy()
        x[14:17] = [15.0, 0.0, 0.0]
        j = int(np.searchsorted(imu_t, ts))
        states.append(lv.state_from_ikfom(sc.prm, x, ts, imu_a[j], imu_w[j]))
    path = lv.compensator_upsample(states, imu_a, imu_w, imu_t)
    X2 = lv.compensator_get_t2(path, t2)
    # the synthetic sweep fires azimuth-major; the messages carry it ring-major, so time order != message order
    rings, cols = 32, 256
    xyz = sc.sweep.reshape(cols, rings, 3).transpose(1, 0, 2).reshape(-1, 3)
    col = np.tile(np.arange(cols), rings)
    velo = np.zeros(len(xyz), BAG_VELO)
    ous = np.zeros(len(xyz), BAG_OUSTER)
    for p in (velo, ous):
        p["x"], p["y"], p["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    velo["time"] = (col * (0.099 / (cols - 1))).astype(np.float32)
    ous["t"] = (col * (99_000_000 // (cols - 1))).astype(np.uint32)
    ous["reflectivity"] = rng.integers(0, 60000, len(ous))
    ous["range"] = (np.linalg.norm(xyz, axis=1) * 1000).astype(np.uint32)
    bag = str(tmp_path / "chain.bag")
    W.write_bag(bag, {1: ("/velodyne_points", "sensor_msgs/PointCloud2"), 2: ("/os_cloud_node/points", "sensor_msgs/PointCloud2")},
                [(1, 10, 0, W.pointcloud2(velo, 10, 0)), (2, 10, 0, W.pointcloud2(ous, 10, 0))])
    L = lv.lib()
    L.lv_bag_next.argtypes = [C.c_void_p, C.POINTER(BagMessage)]
    L.lv_bag_parse_pointcloud2.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.POINTER(PC2View)]
    handle = C.c_void_p()
    assert L.lv_bag_open(bag.encode(), C.byref(handle)) == lv.OK
    msgs, m = [], BagMessage()
    while L.lv_bag_next(handle, C.byref(m)) == 1:
        v = PC2View()
        lidar = "velodyne" if m.topic == b"/velodyne_points" else "ouster"
        assert L.lv_bag_parse_pointcloud2(C.cast(m.data, C.c_void_p), m.size, lv.LIDAR_TYPES[lidar], C.byref(v)) == lv.OK
        msgs.append((lidar, v, np.ctypeslib.as_array(v.data, shape=(v.data_bytes,)).copy(), C.cast(v.data, C.c_void_p).value % 8))
    L.lv_bag_close.argtypes = [C.c_void_p]
    L.lv_bag_close(handle)
    assert [g[0] for g in msgs] == ["velodyne", "ouster"]
    rate, md, leaf = 2, 3.0, 0.5
    loc = lv.Localizer(sc.prm)
    loc.map_build(sc.map)
    for lidar, v, raw, shift in msgs:
        n = v.n_points
        stamp_us = v.stamp_sec * 1_000_000 + v.stamp_nsec // 1000
        pts = raw.view(BAG_VELO if lidar == "velodyne" else BAG_OUSTER)
        # host chain
        hx, ht, _, _, _ = host_process(lv, lidar, pts, stamp_us, True, True, FRT, rate, md)
        assert ht[0] >= t1 and ht[-1] < t2
        q = loc.compensate(path, X2, hx, ht)
        assert 0.5 < np.linalg.norm(q - hx, axis=1).max() < 5.0           # the sweep really was skewed
        ds = loc.voxelgrid_downsample(q, leaf)
        loc.set_state(sc.x_prop, sc.P0)
        st, x, P, logs = loc.correct(ds)
        assert st == lv.OK and len(logs) > 0
        # device chain, the message bytes at the alignment the bag handed out
        d_msg = loc.device_alloc(v.data_bytes + 16)
        d_xyz, d_t, d_ds = loc.device_alloc(12 * n), loc.device_alloc(8 * n), loc.device_alloc(12 * n)
        lv._check(L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg + shift), raw.ctypes.data_as(C.c_void_p), v.data_bytes))
        k = loc.process_cloud_device(lidar, lv.CloudLayout.from_buffer_copy(v.layout), d_msg + shift, v.data_bytes, n, stamp_us, True, True, FRT, rate, md, d_xyz, d_t)
        assert k == len(hx)
        loc.compensate_device(path, X2, d_xyz, d_t, k, d_xyz)
        mm = loc.voxelgrid_downsample_device(d_xyz, k, leaf, d_ds)
        loc.set_state(sc.x_prop, sc.P0)
        assert loc.correct_device(d_ds, mm) == lv.OK
        st2, logs2 = loc.last_logs()
        x2, P2 = loc.get_state()
        assert (u32(loc.download(d_ds, np.empty((mm, 3), np.float32))) == u32(ds)).all()
        assert (u32(loc.download(d_xyz, np.empty((k, 3), np.float32))) == u32(q)).all()
        assert (u64(loc.download(d_t, np.empty(k))) == u64(ht)).all()
        assert st2 == st and (x2 == x).all() and (P2 == P).all() and len(logs2) == len(logs)
        for a, b in zip(logs, logs2):
            assert all(np.array_equal(a[key], b[key]) for key in a)
        for d in (d_msg, d_xyz, d_t, d_ds):
            loc.device_free(d)
    loc.close()
