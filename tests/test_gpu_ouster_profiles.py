"""lv_process_ouster_packets_device(_async) on the lidar UDP profiles of Ouster firmware 2.2+ (and LEGACY through the same entry
point) against the host chain, bit for bit: lv_ouster_packets_to_points, lv_temporal_downsample on its output,
lv_time_sort_indices, then the gathers, and the NumPy restatement of tests/ouster_profile_cases.py.  Then 9 launches for every profile,
refusals that leave the handle usable, and a packet-only RNG19 stream through the windowed device tick, pushed and merged, against
the chain that decodes on the host."""
import ctypes as C

import numpy as np
import pytest

import frontend_ref as F
import ouster_cases as OC
import ouster_profile_cases as OP
from test_gpu_async_tick import Bufs, get_count, put_count
from test_gpu_full_points import same_full
from test_gpu_lidar_buffer import MD, RATE, bits
from test_gpu_ouster import OusterChain, os1_frames
from test_gpu_world_clouds import upload

pytestmark = pytest.mark.gpu
f32 = np.float32
PROFILES = (OP.LEGACY,) + OP.NEW_PROFILES


@pytest.fixture(scope="module")
def loc(lv):
    h = lv.Localizer(lv.default_params(max_points=1 << 18, max_map_points=1 << 16))
    yield h
    h.close()


def host_chain(lv, loc, pk, cal, profile, rate, md):
    """lv_ouster_packets_to_points -> lv_temporal_downsample (device, on the point list) -> lv_time_sort_indices"""
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal, profile)
    _, keep = loc.temporal_downsample(xyz, rate, md) if len(xyz) else (None, np.zeros(0, np.int32))
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


def same(got, ref, what, fields=5):
    for name, a, b in list(zip(("xyz", "time", "intensity", "range", "idx"), got, ref))[:fields]:
        assert a.shape == b.shape and bits(a) == bits(b), (what, name, a.shape, b.shape)


def device_run(loc, d_msg, shift, pk, cal, profile, rate, md, outs, d_n=None, optional=True):
    """the packets at d_msg + shift; the synchronous form, or the async one with its count at d_n"""
    raw = np.frombuffer(pk.tobytes(), np.uint8)
    if len(raw):
        upload(loc, d_msg + shift, raw)
    o = outs if optional else outs[:2] + [None] * 3
    if d_n is None:
        m = loc.process_ouster_device(d_msg + shift, len(raw), len(pk), cal, rate, md, *o, profile=profile)
    else:
        put_count(loc, d_n, -5)
        loc.process_ouster_device_async(d_msg + shift, len(raw), len(pk), cal, rate, md, o[0], o[1], d_n, *o[2:], profile=profile)
        m = get_count(loc, d_n)
    host = (np.empty((m, 3), f32), np.empty(m), np.empty(m, f32), np.empty(m, f32), np.empty(m, np.int32))
    return tuple(loc.download(d, a) for d, a in zip(outs, host))


@pytest.mark.parametrize("H,Wc", [(16, 512), (64, 1024), (128, 2048)])
@pytest.mark.parametrize("profile", PROFILES)
def test_profiles_equal_the_host_chain(lv, loc, profile, H, Wc):
    rng = np.random.default_rng(200 + 4 * H + profile)
    n_packets = 24
    pk = OP.profile_packets(rng, n_packets, Wc, H, profile, m0=Wc - 100, ts0=1_712_345_678 * 10**9 + 999_990_000,
                            invalid=0.05, bad_m=0.05)                 # frame wrap and ns -> s carry
    cal = OC.calibration(lv, Wc, H, OC.ORIGIN_MM, rng)
    n = 16 * H * n_packets
    b = Bufs(loc)
    d_msg = b(pk.nbytes + 16)
    outs = [b(k * n) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    for rate in (1, 3, 8):
        for md in (0.0, 0.9, 3.0):
            ref = host_chain(lv, loc, pk, cal, profile, rate, md)
            same(ref, OP.profile_process(pk, cal, profile, rate, md), ("restatement", rate, md))
            assert len(ref[0]) > 0.5 * n / rate
            for shift in range(4):
                for asyn in (False, True):
                    got = device_run(loc, d_msg, shift, pk, cal, profile, rate, md, outs, d_n if asyn else None)
                    same(got, ref, (rate, md, shift, asyn))
            got = device_run(loc, d_msg, 1, pk, cal, profile, rate, md, outs, d_n, optional=False)
            same(got, ref, (rate, md, "xyz and time only"), 2)
    assert loc.async_status() == (lv.OK, "")
    b.free()


def test_nine_launches_for_every_profile(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 15, max_map_points=1 << 12))
    rng = np.random.default_rng(5)
    cal = OC.calibration(lv, 512, 32)
    b = Bufs(loc)
    d_msg = b(OP.profile_packet_bytes(OP.DUAL, 32) * 4 + 8)
    outs = [b(k * 16 * 32 * 4) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    for profile in PROFILES:
        pk = OP.profile_packets(rng, 4, 512, 32, profile)
        ref = OP.profile_process(pk, cal, profile, 4, 3.0)
        for asyn in (False, True):
            loc.profile()                                              # reset the counters
            same(device_run(loc, d_msg, 0, pk, cal, profile, 4, 3.0, outs, d_n if asyn else None), ref, (profile, asyn))
            assert loc.profile()["total_launches"] == 9, (profile, asyn)
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


def test_refusals_leave_the_handle_usable(lv):
    loc = lv.Localizer(lv.default_params(max_points=1 << 14, max_map_points=1 << 12))
    rng = np.random.default_rng(13)
    cal = OC.calibration(lv, 1024, 16)
    b = Bufs(loc)
    outs = [b(k * 2560) for k in (12, 8, 4, 4, 4)]
    d_n = b(8)
    L = loc.L
    m = C.c_int64(-1)
    for profile in PROFILES:
        pk = OP.profile_packets(rng, 10, 1024, 16, profile)
        raw = np.frombuffer(pk.tobytes(), np.uint8)
        d_msg = b.upload(raw)
        ref = OP.profile_process(pk, cal, profile, 4, 3.0)
        loc.profile()
        for nb, prof in ((len(raw) - 1, profile), (len(raw), -1), (len(raw), 4), (len(raw), 1 << 20)):
            assert L.lv_process_ouster_packets_device(loc.h, d_msg, nb, 10, C.byref(cal), prof, 4, 3.0, *outs, C.byref(m)) == lv.ERR_ARG
            assert m.value == 0
            put_count(loc, d_n, 123)
            assert L.lv_process_ouster_packets_device_async(loc.h, d_msg, nb, 10, C.byref(cal), prof, 4, 3.0, *outs, d_n) == lv.ERR_ARG
            assert get_count(loc, d_n) == 123                          # the count was not written
        assert loc.profile()["total_launches"] == 0
        assert loc.process_ouster_device(d_msg, len(raw), 10, cal, 4, 3.0, *outs, profile=profile) == len(ref[0])
        same(tuple(loc.download(d, np.empty_like(a)) for d, a in zip(outs, ref)), ref, ("after the refusals", profile))
    assert loc.async_status() == (lv.OK, "")
    b.free()
    loc.close()


# ---- a packet-only RNG19 stream through the windowed device tick --------------------------------------------------------------------
class ProfileChain(OusterChain):
    """OusterChain on packets of `profile`: on the device lv_process_ouster_packets_device_async, then the full push or (merge) the
    full merge of the primary LiDAR; otherwise lv_ouster_packets_to_points, the decimator on the rank and lv_time_sort_indices pushed
    onto the restated deque"""

    def __init__(self, lv, sc, cal, msgs, delta, device, profile, merge=False):
        super().__init__(lv, sc, cal, msgs, delta, device)
        self.profile, self.merge = profile, merge
        if device and merge:
            self.loc.lidar_reserve_merge(2 * self.nm // RATE)

    def receive(self, g):
        if not self.device:
            xyz, t, inten, rg, _ = self.lv.ouster_to_points(g["raw"], self.cal, self.profile)
            keep = F.temporal(xyz, RATE, MD)
            order = keep[self.lv.time_sort_indices(t[keep])]
            self.ref.push_message(xyz[order], t[order], inten[order], rg[order])
            return t[order]
        upload(self.loc, self.d_msg, g["raw"])
        self.loc.process_ouster_device_async(self.d_msg, len(g["raw"]), g["n_packets"], self.cal, RATE, MD, self.d_p[0], self.d_p[1],
                                             self.d_k, self.d_p[2], self.d_p[3], profile=self.profile)
        if self.merge:
            self.loc.lidar_merge_full_async(*self.d_p, self.d_k, g["n"])
        else:
            self.loc.lidar_push_full_async(*self.d_p, self.d_k, g["n"])
        return None


@pytest.mark.parametrize("merge", [False, True])
def test_rng19_stream_through_the_device_tick_equals_the_host_chain(lv, scene_xaloc, merge):
    sc = scene_xaloc
    rng = np.random.default_rng(54)
    cal = OC.calibration(lv, 1024, 64, OC.ORIGIN_MM, rng)
    msgs = os1_frames(lv, sc, cal)
    for g in msgs:                                                     # the same frames as RNG19_RFL8_SIG16_NIR16 packets
        g["pk"] = OP.encode_profile(g["pk"], OP.RNG19, rng)
        g["raw"] = np.frombuffer(g["pk"].tobytes(), np.uint8).copy()
    host = ProfileChain(lv, sc, cal, msgs, 0.02, False, OP.RNG19)
    dev = ProfileChain(lv, sc, cal, msgs, 0.02, True, OP.RNG19, merge)
    seen = dict(ticks=0, gated=0, updates=0)
    latest = -np.inf
    for i, g in enumerate(msgs):
        latest = max(latest, float(host.receive(g).max()))
        dev.receive(g)
        for _ in range(14):
            a, b = host.tick(latest), dev.tick(latest)
            assert a == b and host.t2 == dev.t2, (i, a, b)
            if a == "fov":
                break
            seen["ticks"] += 1
            rh, rd = host.result(), dev.result()
            assert bits(rh[2]) == bits(rd[2]) and bits(rh[3]) == bits(rd[3]) and rh[4] == rd[4], (i, host.t2)
            assert bits(host.loc.map_points()) == bits(dev.loc.map_points()), (i, host.t2)
            if a == "gated":
                seen["gated"] += 1
                continue
            assert rh[0] == rd[0] and len(rh[1]) == len(rd[1]) and all(
                all(np.array_equal(p[k], q[k], equal_nan=True) for k in p) for p, q in zip(rh[1], rd[1])), (i, host.t2)
            seen["updates"] += rh[0] == lv.OK
            for key in ("ds", "full"):
                same_full(dev.published[key], host.published[key], (i, host.t2, key))
            assert dev.published["stamps"] == host.published["stamps"]
    assert dev.loc.async_status() == (lv.OK, "")
    assert seen["ticks"] >= 15 and seen["gated"] >= 1 and seen["updates"] >= 5, seen
    assert host.imu_stamps == dev.imu_stamps
    host.close()
    dev.close()
