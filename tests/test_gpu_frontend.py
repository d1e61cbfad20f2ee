"""The front end of a tick on the GPU (deskew, voxel grid, temporal decimator) against the independent restatements of
frontend_ref, on the edge-case families of frontend_cases, and the three stages feeding the update.

Deskew bar.  The kernel and the oracle run the same unfused fp32 operations in the same order; only sinf / cosf differ
(CUDA documents at most 2 ulp for each, glibc stays within 1).  So |sin| and 1 - cos differ by at most 3 ulp <= 3 u32 each,
one more u32 for the cast of 1 - cos, and E = I + s K + c K^2 (|K| = |K^2| = 1) by at most 7 u32 in norm; R E carries that to
the world point and the orthogonal back transform keeps it: 7 u32 |p + tLI|.  Every later rounding acts on values that
already differ and can land one ulp apart (2 u32 M): 3-term dot plus add in X * I_Rt_L, in the world point and in the back
transform, a dozen in all.  That bounds k by about 7 + 24 = 31.  Measured, (e_gpu - e_oracle) / (u32 M) stays at or below 2.2 on every
family (DESIGN.md 5b), so the test holds the kernel to k = 8, a quarter of the bound.  Where no sinf / cosf is evaluated
(|w - bw| <= 1e-7, the identity branch of SO3Math::Exp) the kernel must equal the oracle bit for bit."""
import ctypes as C

import numpy as np
import pytest
import torch

import frontend_cases as FC
import frontend_ref as F
from test_gpu_fullsize import check_every_evaluation

pytestmark = pytest.mark.gpu

K = FC.K
MAX_POINTS = 1 << 16


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def dev(a):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


@pytest.fixture(scope="module")
def prm(lv):
    return lv.params_from_yaml(lv.CONFIG_DIR + "/xaloc.yaml", max_points=MAX_POINTS, max_map_points=1 << 16)


@pytest.fixture(scope="module")
def deskew(O):
    out = {}
    for c in FC.deskew_cases(O):
        c["exact"] = F.compensate(c["path"], c["Xt2"], c["xyz"], c["t"])
        c["oracle"] = O.compensate(c["path"], c["Xt2"], c["xyz"], c["t"])
        out[c["name"]] = c
    return out


def lv_path(lv, c):
    return [lv.State32.from_buffer_copy(s) for s in c["path"]], lv.State32.from_buffer_copy(c["Xt2"])


def compensate_status(lv, loc, path, X2, xyz, t):
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    t = np.ascontiguousarray(t, np.float64)
    out = np.zeros_like(xyz)
    arr = (lv.State32 * len(path))(*path)
    st = loc.L.lv_compensate(loc.h, arr, len(path), C.byref(X2), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                             t.ctypes.data_as(C.POINTER(C.c_double)), C.c_int64(len(t)), out.ctypes.data_as(C.POINTER(C.c_float)))
    return st, out


def compensate_all_ways(lv, loc, c):
    """host entry, device entry out of place, device entry in place: all three must give the same bits"""
    path, X2 = lv_path(lv, c)
    host = loc.compensate(path, X2, c["xyz"], c["t"])
    n = len(c["t"])
    d_xyz, d_t, d_out = dev(c["xyz"]), dev(c["t"]), torch.empty((n, 3), dtype=torch.float32, device="cuda")
    loc.compensate_device(path, X2, d_xyz.data_ptr(), d_t.data_ptr(), n, d_out.data_ptr())
    out_of_place = d_out.cpu().numpy()
    assert (bits(d_xyz.cpu().numpy()) == bits(c["xyz"])).all()          # the input is untouched
    loc.compensate_device(path, X2, d_xyz.data_ptr(), d_t.data_ptr(), n, d_xyz.data_ptr())
    in_place = d_xyz.cpu().numpy()
    assert (bits(host) == bits(out_of_place)).all() and (bits(host) == bits(in_place)).all()
    return host


def check_bar(got, qo, exact, name):
    q, _, M = exact
    e_gpu, e_o = np.abs(got - q).max(axis=1), np.abs(qo - q).max(axis=1)
    ratio = (e_gpu - e_o) / (F.U32 * M)
    print("deskew %-22s e_gpu/(uM) max %.2f  e_oracle/(uM) max %.2f  (e_gpu-e_oracle)/(uM) max %.2f  e_gpu max %.2e m"
          % (name, (e_gpu / (F.U32 * M)).max(), (e_o / (F.U32 * M)).max(), ratio.max(), e_gpu.max()))
    assert (e_gpu <= e_o + K * F.U32 * M).all(), (name, ratio.max())


@pytest.mark.parametrize("name", FC.DESKEW_NAMES)
def test_deskew_families_against_50_digits(lv, prm, deskew, name):
    c = deskew[name]
    loc = lv.Localizer(prm)
    got = compensate_all_ways(lv, loc, c)
    loc.close()
    check_bar(got, c["oracle"], c["exact"], name)
    if name == "identity_branch":                     # no transcendental evaluated: same operations, same bits
        assert (bits(got) == bits(c["oracle"])).all()
    if c["inconsistent"]:
        # the bar is below a thousandth of the distance to a neighbouring segment's result (frontend_cases proves it for
        # every point), so a point deskewed from the wrong segment fails here
        FC.deskew_separation(c, c["exact"])


@pytest.mark.parametrize("n", [1, 255, 256, 257, MAX_POINTS])
def test_deskew_sizes(lv, O, prm, n):
    c = FC.deskew_sized(O, n)
    loc = lv.Localizer(prm)
    got = compensate_all_ways(lv, loc, c)
    loc.close()
    qo = O.compensate(c["path"], c["Xt2"], c["xyz"], c["t"])
    rng = np.random.default_rng(n)
    sub = np.unique(np.concatenate([np.arange(min(n, 4)), np.arange(250, 262), np.arange(n - 4, n),
                                    rng.integers(0, n, 100)]))
    sub = sub[(sub >= 0) & (sub < n)]
    ex = F.compensate(c["path"], c["Xt2"], c["xyz"][sub], c["t"][sub])
    check_bar(got[sub], qo[sub], ex, c["name"])
    FC.deskew_separation(dict(c, xyz=c["xyz"][sub], t=c["t"][sub], seg=c["seg"][sub]), ex)
    # every other point: next to the oracle (whose own bar the CPU suite checks) within twice the bar
    M = np.abs(c["xyz"]).max(axis=1) + max(np.abs(np.float64(s.pos[:])).max() for s in c["path"]) + 1.0
    assert (np.abs(got - qo).max(axis=1) <= 2 * K * F.U32 * M).all()


def test_deskew_refusals_leave_the_handle_usable(lv, O, prm, deskew):
    rng = np.random.default_rng(11)
    loc = lv.Localizer(prm)
    long_path = [lv.State32.from_buffer_copy(s) for s in FC.random_path(O, rng, 257)]
    st, _ = compensate_status(lv, loc, long_path, long_path[-1], np.ones((4, 3), np.float32),
                              np.linspace(long_path[0].time, long_path[-1].time, 4))
    assert st == lv.ERR_CAPACITY
    c = deskew["ns256"]
    path, X2 = lv_path(lv, c)
    t = c["t"].copy()
    for bad in ("after", "before", "order", "nan"):
        tb = t.copy()
        if bad == "after":
            tb[-1] = np.nextafter(path[-1].time, np.inf)
        elif bad == "before":
            tb[0] = np.nextafter(path[0].time, -np.inf)
        elif bad == "order":
            tb[100], tb[101] = tb[101], tb[100]
            assert tb[100] > tb[101]
        else:
            tb[37] = np.nan
        st, _ = compensate_status(lv, loc, path, X2, c["xyz"], tb)
        assert st == lv.ERR_ARG, bad
        assert b"timestamp" in loc.L.lv_last_error()
        # the next valid call on the same handle, with a shorter path: the bad flag and the staged path are reset
        short = deskew["ns3"]
        p3, X3 = lv_path(lv, short)
        st, got = compensate_status(lv, loc, p3, X3, short["xyz"], short["t"])
        assert st == lv.OK
        check_bar(got, short["oracle"], short["exact"], "ns3 after " + bad)
        fresh = lv.Localizer(prm)
        assert (bits(fresh.compensate(p3, X3, short["xyz"], short["t"])) == bits(got)).all()
        fresh.close()
    loc.close()


# ---- voxel grid ---------------------------------------------------------------------------------------------------------
def voxel_both_entries(loc, xyz, leaf):
    host = loc.voxelgrid_downsample(xyz, leaf)
    n = len(xyz)
    d_in, d_out = dev(xyz), torch.full((n, 3), np.nan, dtype=torch.float32, device="cuda")
    m = loc.voxelgrid_downsample_device(d_in.data_ptr(), n, leaf, d_out.data_ptr())
    device = d_out[:m].cpu().numpy()
    assert (bits(host) == bits(device)).all()
    return host


def check_voxel(got, xyz, leaf, name):
    r = F.voxelgrid(xyz, leaf, exact=True)
    if r["overflow"]:                                 # PCL warns and hands the input on
        assert (bits(got) == bits(xyz)).all(), name
        return
    assert got.shape == r["out"].shape, (name, got.shape, r["out"].shape)
    assert (bits(got) == bits(r["out"])).all(), name
    assert r["count"].sum() == len(xyz)
    tol = r["count"][:, None] * F.U32 * np.abs(xyz).max()
    assert (np.abs(r["out"].astype(np.float64) - r["mean"]) <= tol).all()


@pytest.mark.parametrize("name", [c[0] for c in FC.voxel_cases()])
def test_voxelgrid_families_bit_exact(lv, prm, name):
    xyz, leaf = {c[0]: c[1:] for c in FC.voxel_cases()}[name]
    loc = lv.Localizer(prm)
    check_voxel(voxel_both_entries(loc, xyz, leaf), xyz, leaf, name)
    loc.close()


def test_voxelgrid_one_leaf_past_2_24_points(lv, prm):
    xyz, leaf = FC.voxel_big_leaf()
    loc = lv.Localizer(prm)
    got = voxel_both_entries(loc, xyz, leaf)
    loc.close()
    check_voxel(got, xyz, leaf, "big_leaf")
    assert got.shape == (1, 3)


def test_voxelgrid_scratch_reuse_across_sizes(lv, prm):
    rng = np.random.default_rng(3)
    clouds = [FC.lidar_points(rng, n, r=(1.0, 80.0)) for n in (1000000, 10, 300000, 1)]
    loc = lv.Localizer(prm)
    for xyz in clouds:
        got = voxel_both_entries(loc, xyz, 0.5)
        fresh = lv.Localizer(prm)
        assert (bits(fresh.voxelgrid_downsample(xyz, 0.5)) == bits(got)).all()
        fresh.close()
        check_voxel(got, xyz, 0.5, "reuse n=%d" % len(xyz))
    loc.close()


def test_voxelgrid_device_refuses_overlap(lv, prm):
    rng = np.random.default_rng(4)
    xyz = FC.lidar_points(rng, 1000)
    loc = lv.Localizer(prm)
    buf = dev(np.concatenate([xyz, xyz]))
    m = C.c_int64(0)
    for off in (0, 3 * 999, -3 * 999):
        base = buf.data_ptr() + 4 * 3 * 1000 * (off < 0)
        st = loc.L.lv_voxelgrid_downsample_device(loc.h, C.c_void_p(base), C.c_int64(1000), C.c_float(0.5),
                                                  C.c_void_p(base + 4 * off), C.byref(m))
        assert st == lv.ERR_ARG and b"overlaps" in loc.L.lv_last_error(), off
    # adjacent ranges are fine
    assert loc.voxelgrid_downsample_device(buf.data_ptr(), 1000, 0.5, buf.data_ptr() + 12 * 1000) > 0
    loc.close()


# ---- temporal decimator -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c[0] for c in FC.temporal_cases()])
def test_temporal_families_bit_exact(lv, prm, name):
    xyz, rate, md = {c[0]: c[1:] for c in FC.temporal_cases()}[name]
    loc = lv.Localizer(prm)
    got, gi = loc.temporal_downsample(xyz, rate, md)
    loc.close()
    ri = F.temporal(xyz, rate, md)
    assert (gi == ri).all() and (bits(got) == bits(xyz[ri])).all()


# ---- the front end feeding the update -----------------------------------------------------------------------------------
def test_deskew_downsample_update_chain(lv, O, scene_xaloc):
    """a skewed sweep (15 m/s, 0.5 rad/s yaw over 0.1 s): lv_compensate_device -> lv_voxelgrid_downsample_device ->
    lv_correct_device equals the host-buffer chain bit for bit, and the update passes check_every_evaluation on the GPU's own
    downsampled points"""
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
    xyz, t = sc.sweep, np.linspace(t1, t2, len(sc.sweep))
    n, leaf = len(xyz), 0.5
    loc = lv.Localizer(sc.prm)
    loc.map_build(sc.map)
    # host buffers
    q = loc.compensate(path, X2, xyz, t)
    assert 0.5 < np.linalg.norm(q - xyz, axis=1).max() < 5.0              # the sweep really was skewed
    ds = loc.voxelgrid_downsample(q, leaf)
    loc.set_state(sc.x_prop, sc.P0)
    st, x, P, logs = loc.correct(ds)
    assert st == lv.OK and len(logs) > 0
    # device buffers end to end
    d_xyz, d_t = dev(xyz), dev(t)
    d_ds = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    loc.compensate_device(path, X2, d_xyz.data_ptr(), d_t.data_ptr(), n, d_xyz.data_ptr())
    m = loc.voxelgrid_downsample_device(d_xyz.data_ptr(), n, leaf, d_ds.data_ptr())
    loc.set_state(sc.x_prop, sc.P0)
    assert loc.correct_device(d_ds.data_ptr(), m) == lv.OK
    st2, logs2 = loc.last_logs()
    x2, P2 = loc.get_state()
    ds2 = d_ds[:m].cpu().numpy()
    assert (bits(ds2) == bits(ds)).all() and (bits(d_xyz.cpu().numpy()) == bits(q)).all()
    assert st2 == st and (x2 == x).all() and (P2 == P).all() and len(logs2) == len(logs)
    for a, b in zip(logs, logs2):
        assert all(np.array_equal(a[k], b[k]) for k in a)
    om = O.Map(O.KNN_REF_IKDTREE if O.ref_available() else O.KNN_KDTREE)
    om.build(sc.map)
    check_every_evaluation(O, om, sc.oprm, sc.x_prop, sc.P0, ds2, logs2, loc, P_gpu=P2)
    loc.close()
