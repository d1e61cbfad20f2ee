"""The Livox front end without a GPU.

lv_bag_parse_livox on bags written by tests/bagwriter.py: several CustomMsg messages among IMU messages, an empty message, frame_id
lengths that put the records at every address mod 4; it refuses truncations, bytes after the records and a point_num that is not the
record count.  lv_livox_to_points (the host build of lv_wire.h's decoder) then lv_time_sort_indices equal the NumPy restatement of
tests/livox_cases.py bit for bit: times at the ns -> s boundary, a time base at its limit (one past it is refused), every tag mask
bit, NaN and sub-min_dist points (decimated on the rank by frontend_ref.temporal), equal offset times.  Every argument refusal of
lv_process_livox_device(_async) happens before any device call (the device pointers below are never dereferenced)."""
import ctypes as C

import numpy as np
import pytest

import bagwriter as W
import livox_cases as LC
from test_bag_reader import BagMessage

BASE = 1 << 40                       # a device address that is never touched


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype.itemsize == 8 else np.uint32).tobytes()


def same(got, ref, what):
    assert len(got) == len(ref) == 5, what
    for name, a, b in zip(("xyz", "time", "intensity", "range", "idx"), got, ref):
        assert a.shape == b.shape and bits(a) == bits(b), (what, name)


# ---- the bag reader ---------------------------------------------------------------------------------------------------------------
def read_bag(lv, path):
    L = lv.lib()
    L.lv_bag_next.argtypes = [C.c_void_p, C.POINTER(BagMessage)]
    L.lv_bag_close.argtypes = [C.c_void_p]
    bag = C.c_void_p()
    assert L.lv_bag_open(path.encode(), C.byref(bag)) == lv.OK
    out, m = [], BagMessage()
    while L.lv_bag_next(bag, C.byref(m)) == 1:
        v = lv.LivoxView()
        st = L.lv_bag_parse_livox(C.cast(m.data, C.c_void_p), m.size, C.byref(v)) if m.type == b"livox_ros_driver/CustomMsg" else None
        recs = np.frombuffer(C.string_at(v.data, v.data_bytes), LC.RECORD).copy() if st == lv.OK and v.n_points else None
        out.append((m.type.decode(), st, v, recs, (v.data or 0) % 4))
    L.lv_bag_close(bag)
    return out


def test_bag_parse_livox_round_trip(lv, tmp_path):
    rng = np.random.default_rng(5)
    sets = [LC.records(rng, n) for n in (1000, 0, 17, 333, 64)]
    frames = ["livox_frame", "", "a", "ab", "abc"]
    msgs, conns = [], {0: ("/livox/imu", "sensor_msgs/Imu"), 1: ("/livox/lidar", "livox_ros_driver/CustomMsg")}
    for k, (recs, frame) in enumerate(zip(sets, frames)):
        msgs.append((0, 100, k, W.imu(100, k, (0, 0, 0, 1), (0.1, 0.2, 0.3), (0.0, 0.1, 9.8))))
        msgs.append((1, 100, 1000 + k, LC.custom_msg(recs, 1_700_000_000 * 10**9 + k, 100, 50_000 * k, frame, k, lidar_id=k + 1)))
    path = str(tmp_path / "livox.bag")
    W.write_bag(path, conns, msgs)
    got = read_bag(lv, path)
    assert [g[0] for g in got] == ["sensor_msgs/Imu", "livox_ros_driver/CustomMsg"] * len(sets)
    lidar = [g for g in got if g[1] is not None]
    for k, (g, recs) in enumerate(zip(lidar, sets)):
        _, st, v, got_recs, _ = g
        assert st == lv.OK
        assert (v.stamp_sec, v.stamp_nsec, v.timebase, v.point_num, v.lidar_id) == (100, 50_000 * k, 1_700_000_000 * 10**9 + k, len(recs), k + 1)
        assert v.n_points == len(recs) and v.data_bytes == 19 * len(recs)
        if len(recs):
            assert got_recs.tobytes() == recs.tobytes()
    # the Python helper reads the same
    v, recs = lv.bag_parse_livox(msgs[1][3])
    assert v.n_points == len(sets[0]) and recs.tobytes() == sets[0].tobytes()
    # the same message with frame_id lengths 0 .. 3 puts its records at every address mod 4
    seen = set()
    for k in range(4):
        path = str(tmp_path / ("align%d.bag" % k))
        W.write_bag(path, {1: conns[1]}, [(1, 100, 0, LC.custom_msg(sets[2], 77, frame="f" * k))])
        (_, st, v, got_recs, mod4), = read_bag(lv, path)
        assert st == lv.OK and v.timebase == 77 and got_recs.tobytes() == sets[2].tobytes()
        seen.add(mod4)
    assert seen == {0, 1, 2, 3}


def test_bag_parse_livox_refusals(lv):
    L = lv.lib()
    rng = np.random.default_rng(6)
    recs = LC.records(rng, 10)
    good = LC.custom_msg(recs, 5 * 10**9)
    v = lv.LivoxView()
    assert L.lv_bag_parse_livox(good, len(good), C.byref(v)) == lv.OK and v.n_points == 10
    for cut in (1, 5, 19, len(good) - 4 - 190, len(good) - 1):          # truncated anywhere
        assert L.lv_bag_parse_livox(good, len(good) - cut, C.byref(v)) == lv.ERR_ARG, cut
    assert L.lv_bag_parse_livox(good + b"\x00", len(good) + 1, C.byref(v)) == lv.ERR_ARG             # trailing byte
    for pn in (9, 11, 0):
        bad = LC.custom_msg(recs, 5 * 10**9, point_num=pn)
        assert L.lv_bag_parse_livox(bad, len(bad), C.byref(v)) == lv.ERR_ARG, pn
    empty = LC.custom_msg(recs[:0], 5 * 10**9)
    assert L.lv_bag_parse_livox(empty, len(empty), C.byref(v)) == lv.OK and v.n_points == 0 and v.data_bytes == 0
    assert L.lv_bag_parse_livox(None, len(good), C.byref(v)) == lv.ERR_ARG
    assert L.lv_bag_parse_livox(good, len(good), None) == lv.ERR_ARG


# ---- the host decoder against the restatement ------------------------------------------------------------------------------------
def host_chain(lv, recs, timebase, mask, rate, md):
    """lv_livox_to_points -> the decimator on the rank (frontend_ref.temporal) -> lv_time_sort_indices"""
    import frontend_ref as F
    xyz, t, inten, rg, idx = lv.livox_to_points(recs, timebase, mask)
    keep = F.temporal(xyz, rate, md)
    order = keep[lv.time_sort_indices(t[keep])] if len(keep) else keep
    return xyz[order], t[order], inten[order], rg[order], idx[order]


@pytest.mark.parametrize("mask", sorted(set(LC.MASKS) | {1 << b for b in range(8)}))
def test_livox_to_points_equals_the_restatement(lv, mask):
    rng = np.random.default_rng(7 + mask)
    for name, (recs, tb) in list(LC.edge_records(rng).items()) + [("random", (LC.records(rng, 5000), 1_712_345_678 * 10**9 + 987_654_321))]:
        ref = LC.to_points(recs, tb, mask)
        same(lv.livox_to_points(recs, tb, mask), ref, (name, mask))
        assert (ref[4] == np.nonzero((recs["tag"] & mask) == 0)[0]).all()
        for rate in range(1, 9):
            for md in (0.0, 3.0):
                same(host_chain(lv, recs, tb, mask, rate, md), LC.process(recs, tb, mask, rate, md), (name, mask, rate, md))


def test_livox_time_rule_at_the_edges(lv):
    r = np.zeros(6, LC.RECORD)
    r["x"] = 10.0
    r["offset_time"] = [0, 1, 999_999_999, 1_000_000_000, 0xFFFFFFFF, 999_999_998]
    tb = 1_700_000_000 * 10**9 + 1
    xyz, t, *_ = lv.livox_to_points(r, tb, 0)
    total = [tb + int(o) for o in r["offset_time"]]
    want = [float(np.float64(s // 10**9) + np.float64(s % 10**9) * 1e-9) for s in total]
    assert t.tolist() == want
    assert t[2] == 1_700_000_001.0 and t[3] == 1_700_000_001.0 + 1e-9         # the carry into the seconds
    _, t, *_ = lv.livox_to_points(r, LC.TIMEBASE_MAX, 0)                        # the largest sum: 2^64 - 1 ns
    assert t[4] == np.float64((2**64 - 1) // 10**9) + np.float64((2**64 - 1) % 10**9) * 1e-9
    with pytest.raises(RuntimeError):
        lv.livox_to_points(r, LC.TIMEBASE_MAX + 1, 0)


def test_livox_to_points_refusals(lv):
    L = lv.lib()
    recs = LC.records(np.random.default_rng(8), 10)
    raw = np.frombuffer(recs.tobytes(), np.uint8)
    out = [np.empty(30, np.float32), np.empty(10), np.empty(10, np.float32), np.empty(10, np.float32), np.empty(10, np.int32)]
    ptr = [a.ctypes.data_as(C.c_void_p) for a in out]
    m = C.c_int64(7)

    def call(data=raw.ctypes.data_as(C.c_void_p), nb=190, n=10, tb=0, outs=ptr, n_out=True):
        m.value = 7
        st = L.lv_livox_to_points(data, nb, n, C.c_uint64(tb), 0, *outs, C.byref(m) if n_out else None)
        return st, m.value
    assert call() == (lv.OK, 10)
    assert call(outs=ptr[:2] + [None] * 3) == (lv.OK, 10)                # intensity, range and idx are optional
    for kw in (dict(data=None), dict(nb=189), dict(n=-1), dict(n=1 << 31, nb=19 << 31), dict(tb=LC.TIMEBASE_MAX + 1),
               dict(outs=[None] + ptr[1:]), dict(outs=ptr[:1] + [None] + ptr[2:])):
        assert call(**kw) == (lv.ERR_ARG, 0), kw
    assert call(n_out=False)[0] == lv.ERR_ARG


# ---- the device calls' argument checks (before any device work) --------------------------------------------------------------------
N = 100


@pytest.fixture
def dcall(lv):
    L = lv.lib()

    def run(h=None, data=BASE, data_bytes=19 * N, n=N, tb=10**18, outs=None, n_out=True, asynch=False):
        outs = outs if outs is not None else [BASE + (1 << 30) + k * (1 << 24) for k in range(5)]
        if asynch:
            st = L.lv_process_livox_device_async(h, data, data_bytes, n, tb, 0x20, 4, 3.0, *outs, BASE + (1 << 35) if n_out else None)
        else:
            m = C.c_int64(7)
            st = L.lv_process_livox_device(h, data, data_bytes, n, tb, 0x20, 4, 3.0, *outs, C.byref(m) if n_out else None)
            if n_out:
                assert m.value == 0
        return st, L.lv_last_error()
    return run


@pytest.mark.parametrize("asynch", [False, True])
def test_process_livox_refusals_before_device_work(lv, dcall, asynch):
    assert dcall(asynch=asynch) == (lv.ERR_ARG, b"process livox: null handle")
    for kw in (dict(data=None), dict(n_out=False)):
        st, msg = dcall(asynch=asynch, **kw)
        assert st == lv.ERR_ARG and b"null data" in msg, kw
    for k in (0, 1):
        outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
        outs[k] = None
        st, msg = dcall(asynch=asynch, outs=outs)
        assert st == lv.ERR_ARG and b"null data" in msg, k
    outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
    outs[2:] = [None] * 3
    assert dcall(asynch=asynch, outs=outs) == (lv.ERR_ARG, b"process livox: null handle")
    for n in (-1, 0x80000000):
        st, msg = dcall(asynch=asynch, n=n, data_bytes=1 << 45)
        assert st == lv.ERR_ARG and b"int32" in msg, n
    st, msg = dcall(asynch=asynch, data_bytes=19 * N - 1)
    assert st == lv.ERR_ARG and b"too short" in msg
    st, msg = dcall(asynch=asynch, tb=LC.TIMEBASE_MAX + 1)
    assert st == lv.ERR_ARG and b"timebase" in msg
    assert dcall(asynch=asynch, tb=LC.TIMEBASE_MAX)[1] == b"process livox: null handle"
    nb = 19 * N
    for k, size in enumerate((12, 8, 4, 4, 4)):
        for start in (BASE + nb - 1, BASE - size * N + 1, BASE):
            outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
            outs[k] = start
            st, msg = dcall(asynch=asynch, outs=outs)
            assert st == lv.ERR_ARG and b"overlaps" in msg, (k, start)
        for start in (BASE + nb, BASE - size * N):                   # adjacent ranges are fine
            outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
            outs[k] = start
            assert dcall(asynch=asynch, outs=outs) == (lv.ERR_ARG, b"process livox: null handle"), (k, start)
