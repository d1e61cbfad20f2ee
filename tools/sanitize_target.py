"""What compute-sanitizer runs (tools/gpu_sanitize.sh): every kernel of the path once or twice on a small scene, checked against
the oracle so that a sanitizer-induced slowdown cannot hide a wrong result.  Both search paths, the map update, the device tick,
the message front end."""
import os
import sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as G
lv = G.load_package(); O = G.load_oracle()
VARIANTS = (None, "4", "8")                    # every shape of the level-0 search (None: the per-launch policy)
if os.environ.get("LV_SANITIZE_QUICK"):
    VARIANTS = ("4",)
for group in VARIANTS:
    os.environ.pop("LV_SEARCH_GROUP", None)
    if group:
        os.environ["LV_SEARCH_GROUP"] = group
    prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=1 << 17, max_points=1 << 13)
    world = lv.SynthWorld(20260924, 40000)
    truth = world.pose(10.0, prm)
    sweep = world.sweep(truth, rings=16, azimuths=256, seed=1)
    far = sweep[:512] + np.float32([0.0, 0.0, 0.9])                 # queries off the surfaces: ring search, blind queries
    sweep = np.ascontiguousarray(np.concatenate([sweep, far]))
    loc = lv.Localizer(prm)
    loc.map_build(world.map())
    loc.init_state()
    x0, P0 = loc.get_state()
    d = np.zeros(23); d[0:3] = [0.04, -0.03, 0.02]; d[3:6] = [0.004, -0.003, 0.005]
    x_prop = O.boxplus(truth, d)
    om = O.Map(O.KNN_KDTREE); om.build(world.map())
    oprm = O.make_params(max_num_iters=prm.MAX_NUM_ITERS, estimate_extrinsics=prm.estimate_extrinsics, max_dist_plane=prm.MAX_DIST_PLANE,
                         planes_threshold=prm.PLANES_THRESHOLD, lidar_noise=prm.LiDAR_noise, degeneracy_threshold=prm.degeneracy_threshold)
    got, ref = loc.match_all(x_prop, sweep), om.match_all(x_prop, oprm, sweep)
    inside = np.isfinite(got["nn_sqd"][:, 4])
    assert (got["nn_sqd"][inside] == ref["nn_sqd"][inside]).all() and (got["valid"] == ref["valid"]).all() and (got["plane"] == ref["plane"]).all()
    for k in range(2):
        loc.set_state(x_prop, P0)
        st, x, P, logs = loc.correct(sweep)
        st_o, x_o, P_o, logs_o = om.update_iterated(x_prop, P0, oprm, sweep)
        assert st == st_o == 0 and len(logs) == len(logs_o) and np.abs(x - x_o).max() < 1e-7
        assert loc.last_neighbours(len(sweep)).shape == (len(sweep), 5)
        loc.map_add_last_sweep(True)
        om.add(om.match_all(x, oprm, sweep)["g"], downsample=True)
        loc.map_status()
        assert abs(loc.map_size() - len(om.points())) <= 2
        loc.propagate_device(np.tile([0.0, 0.0, 9.8], (4, 1)), np.zeros((4, 3)), np.full(4, 1e-3))
    loc.close()
    print("sanitize target: search group %s ok" % (group or "default"), flush=True)

# the message front end (lv_process_cloud_device): velodyne / ouster bytes at an odd device address, against the host composition
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import test_gpu_cloud_frontend as T
from test_wire_format import make_cloud
loc = lv.Localizer(lv.default_params(max_points=1 << 13, max_map_points=1 << 13))
rng = np.random.default_rng(3)
for lidar in ("velodyne", "ouster"):
    pts = make_cloud(lidar, 3000, rng)[rng.permutation(3000)]
    T.assert_same(T.device_process(lv, loc, lidar, pts, T.STAMP_US, False, True, 0.1, 4, 3.0, shift=1),
                  T.host_process(lv, lidar, pts, T.STAMP_US, False, True, 0.1, 4, 3.0), lidar)
loc.close()
print("sanitize target: process cloud ok", flush=True)

# the LiDAR buffer (lv_lidar_*): a ring that wraps, ties at t2, a late message, clears, against the restatement
import lidar_buffer_ref as R
from test_gpu_lidar_buffer import DeviceBuffer, same_window, velodyne_message
loc = lv.Localizer(lv.default_params(max_points=1 << 13, max_map_points=1 << 13))
dev, ref = DeviceBuffer(loc, 2000, n_max=4096), R.LidarBuffer()
for j in range(8):
    xyz, t = velodyne_message(rng, 1.0 + 0.01 * j - (0.03 if j == 5 else 0.0), 8)
    if ref.size() + len(t) > 2000:
        ref.clear(1.0 + 0.01 * j - 0.02)
        loc.lidar_clear_async(1.0 + 0.01 * j - 0.02)
    dev.push(xyz, t)
    ref.push_message(xyz, t)
    same_window(lv, dev, ref, float(t[0]), float(t[-1]), j)
assert loc.async_status() == (lv.OK, "")
dev.close()
loc.close()
print("sanitize target: lidar buffer ok", flush=True)

# full points: the buffer's lane kernels, the full voxel grid (and its pass-through) and the stamp, against the restatement
import full_points_ref as P
from test_gpu_full_points import FullBuffer, same_window as same_full_window
loc = lv.Localizer(lv.default_params(max_points=1 << 13, max_map_points=1 << 13))
dev, ref = FullBuffer(loc, 2000, n_max=4096), P.LidarBufferFull()
for j in range(8):
    xyz, t = velodyne_message(rng, 1.0 + 0.01 * j - (0.03 if j == 5 else 0.0), 8)
    inten, rg = (None, None) if j == 2 else (rng.uniform(0, 255, len(t)).astype(np.float32), rng.uniform(0, 90, len(t)).astype(np.float32))
    if ref.size() + len(t) > 2000:
        ref.clear(1.0 + 0.01 * j - 0.02)
        loc.lidar_clear_async(1.0 + 0.01 * j - 0.02)
    dev.push(xyz, t, inten, rg)
    ref.push_message(xyz, t, inten, rg)
    same_full_window(dev, ref, float(t[0]), float(t[-1]), j)
loc.lidar_reserve(2500)
same_full_window(dev, ref, -np.inf, np.inf, "reserve")
for pts, leaf in ((sweep[:3000], 0.5), (np.array([[0, 0, 0], [8388607, 255, 0], [8388608, 0, 0]], np.float32), 1.0)):
    n = len(pts)
    t, inten, rg = rng.uniform(0, 20, n), rng.uniform(0, 255, n).astype(np.float32), rng.uniform(0, 90, n).astype(np.float32)
    got, want = loc.voxelgrid_downsample_full(pts, t, inten, leaf), P.voxelgrid_full(pts, t, inten, leaf)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
d_t, d_n, d_s = loc.upload(np.sort(rng.uniform(1.7e9, 1.7e9 + 0.1, 3000))), loc.upload(np.array([3000], np.int64)), loc.device_alloc(8)
loc.cloud_stamp_async(d_t, d_n, 3000, d_s)
assert loc.async_status() == (lv.OK, "")
dev.close()
for d in (d_t, d_n, d_s):
    loc.device_free(d)
loc.close()
print("sanitize target: full points ok", flush=True)

# the Velodyne packet front end (lv_process_velodyne_device, both forms): packets at an odd device address, a bad block flag, a
# dual-return packet and a stamp that does not convert (the deferred flag), against the restatement
import ctypes as C
import velodyne_cases as VC
loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 13))
cal = lv.velodyne_calibration()
outs = [loc.device_alloc(k * 384 * 20) for k in (12, 8, 4, 4, 4)]
d_msg, d_n = loc.device_alloc(1214 * 20 + 8), loc.device_alloc(8)
for name, pk in (("scan", VC.packets(rng, 20)), ("flags", VC.edge_packets(rng)["bad_flags"]), ("dual", VC.dual_packets(rng))):
    ref = VC.process(pk, cal, 2, 0.5)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg + 1), raw.ctypes.data_as(C.c_void_p), raw.nbytes) == 0
    loc.process_velodyne_device_async(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, outs[0], outs[1], d_n, *outs[2:])
    m = int(loc.download(d_n, np.zeros(1, np.int64))[0])
    got = [loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref)]
    assert m == len(ref[0]) and all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, ref)), name
    assert loc.async_status()[0] == (lv.ERR_ARG if name == "dual" else lv.OK), name
    if name != "dual":
        assert loc.process_velodyne_device(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, *outs) == len(ref[0])
for d in outs + [d_msg, d_n]:
    loc.device_free(d)
loc.close()
print("sanitize target: process velodyne ok", flush=True)

# the Ouster packet front end (lv_process_ouster_device, both forms): packets at an odd device address, across the frame wrap, with
# invalid columns, ids >= W, ranges of 0 and garbage in the range words' upper bits, against the restatement
import ouster_cases as OC
loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 13))
cal = OC.calibration(lv, 1024, 32, OC.ORIGIN_MM, rng)
outs = [loc.device_alloc(k * 16 * 32 * 12) for k in (12, 8, 4, 4, 4)]
d_msg, d_n = loc.device_alloc(OC.packet_bytes(32) * 12 + 8), loc.device_alloc(8)
for name, pk in (("frame", OC.packets(rng, 12, 1024, 32, m0=1000)), ("sparse", OC.packets(rng, 5, 1024, 32, invalid=0.3, bad_m=0.3))):
    ref = OC.process(pk, cal, 2, 0.5)
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg + 1), raw.ctypes.data_as(C.c_void_p), raw.nbytes) == 0
    loc.process_ouster_device_async(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, outs[0], outs[1], d_n, *outs[2:])
    m = int(loc.download(d_n, np.zeros(1, np.int64))[0])
    got = [loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref)]
    assert m == len(ref[0]) and all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, ref)), name
    assert loc.async_status()[0] == lv.OK, name
    assert loc.process_ouster_device(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, *outs) == len(ref[0])
for d in outs + [d_msg, d_n]:
    loc.device_free(d)
loc.close()
print("sanitize target: process ouster ok", flush=True)

# the Ouster UDP profiles of firmware 2.2+ (lv_process_ouster_packets_device, both forms): packets at an odd device address, across
# the frame wrap, with random packet headers and footers, flag bits above the range masks and a second return, against the restatement
import ouster_profile_cases as OP
loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 13))
outs = [loc.device_alloc(k * 16 * 32 * 12) for k in (12, 8, 4, 4, 4)]
d_msg, d_n = loc.device_alloc(OP.profile_packet_bytes(OP.DUAL, 32) * 12 + 8), loc.device_alloc(8)
for profile in OP.NEW_PROFILES:
    for name, pk in (("frame", OP.profile_packets(rng, 12, 1024, 32, profile, m0=1000)),
                     ("sparse", OP.profile_packets(rng, 5, 1024, 32, profile, invalid=0.3, bad_m=0.3))):
        ref = OP.profile_process(pk, cal, profile, 2, 0.5)
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        assert loc.L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg + 1), raw.ctypes.data_as(C.c_void_p), raw.nbytes) == 0
        loc.process_ouster_device_async(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, outs[0], outs[1], d_n, *outs[2:], profile=profile)
        m = int(loc.download(d_n, np.zeros(1, np.int64))[0])
        got = [loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref)]
        assert m == len(ref[0]) and all(np.array_equal(a.view(np.uint8), b.view(np.uint8)) for a, b in zip(got, ref)), (profile, name)
        assert loc.async_status()[0] == lv.OK, (profile, name)
        assert loc.process_ouster_device(d_msg + 1, raw.nbytes, len(pk), cal, 2, 0.5, *outs, profile=profile) == len(ref[0])
for d in outs + [d_msg, d_n]:
    loc.device_free(d)
loc.close()
print("sanitize target: process ouster profiles ok", flush=True)
