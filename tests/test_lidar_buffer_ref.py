"""The LiDAR buffer without a GPU.

1. tests/lidar_buffer_ref.py (the literal restatement of Buffer / Accumulator::get) on cases worked by hand from the reference's
   text: include/Headers/Utils.hpp:9-23 (binary_search), include/Headers/Accumulator.hpp:61-74 (get), src/Objects/Buffer.cpp:26-28,
   66-70 (push, clear).  content is written newest first, as the deque holds it.
2. The host build of the device buffer's index arithmetic (csrc/lv_lidar_buffer.h through tests/cpu_shim/lidar_ring.cpp, a ring
   without lanes) equals the restatement on 10^4 seeded random push / get / clear sequences: small rings that wrap many times,
   full rings, late and overlapping messages, ties, NaN point times and windows above n_max.
"""
import ctypes as C
import math

import numpy as np
import pytest

import lidar_buffer_ref as R
import shim_binding as S


def buf_with(content):
    """a buffer whose content (newest first) is `content`: pushed oldest first"""
    b = R.LidarBuffer()
    t = np.array(content[::-1], np.float64)
    b.push_message(np.arange(3 * len(t), dtype=np.float32).reshape(-1, 3), t)
    assert list(b.times()) == [float(v) for v in content] or any(math.isnan(v) for v in content)
    return b


def get_times(b, t1, t2):
    return list(b.get(t1, t2)[1])


# ---- hand-worked cases ---------------------------------------------------------------------------------------------------------
def test_three_ties_at_t2_return_two():
    b = buf_with([5, 4, 3, 3, 3, 2, 1])
    # low 0 high 6: mid 3 (3 < 3 no: low 4), mid 5 (2 < 3: high 4), mid 4 (3 < 3 no: low 5); --high = 3
    assert R.binary_search(b.content, 3.0) == (3, [3, 5, 4])
    assert get_times(b, 2.5, 3.0) == [3, 3]               # content[4], content[3]; content[2] (also 3) is before the start
    assert get_times(b, 0.0, 3.0) == [1, 2, 3, 3]
    xyz, t = b.get(0.0, 3.0)                              # oldest inserted first: content[6] .. content[3]
    assert (xyz[:, 0] == np.float32([0, 3, 6, 9])).all()


def test_one_tie_at_t2():
    b = buf_with([5, 4, 3, 2, 1])
    assert R.binary_search(b.content, 3.0) == (1, [2, 3])   # mid 2 (low 3), mid 3 (2 < 3: high 2); --high = 1
    assert get_times(b, 0.0, 3.0) == [1, 2, 3]


def test_two_ties_at_t2():
    b = buf_with([5, 4, 3, 3, 2, 1])
    assert R.binary_search(b.content, 3.0) == (2, [2, 4, 3])
    assert get_times(b, 0.0, 3.0) == [1, 2, 3, 3]


def test_many_ties_at_t2_return_two_and_the_next_window_takes_the_rest():
    b = buf_with([7.0] * 3 + [6.0] * 64 + [5.0] * 64)
    assert get_times(b, 5.0, 6.0) == [5.0] * 64 + [6.0] * 2
    assert get_times(b, 6.0, 7.0) == [6.0] * 64 + [7.0] * 2   # t1 inclusive


def test_t1_on_a_point_time_is_inclusive():
    b = buf_with([5, 4, 3, 2, 1])
    assert R.binary_search(b.content, 4.0) == (0, [2, 0, 1])
    assert get_times(b, 2.0, 4.0) == [2, 3, 4]


def test_empty_buffer():
    b = R.LidarBuffer()
    assert R.binary_search(b.content, 1.0) == (0, [])
    xyz, t = b.get(0.0, 1.0)
    assert xyz.shape == (0, 3) and t.shape == (0,)
    b.clear(1.0)
    assert b.size() == 0


def test_all_times_below_t2():
    b = buf_with([5, 4, 3])
    assert R.binary_search(b.content, 10.0) == (0, [1, 0])
    assert get_times(b, 0.0, 10.0) == [3, 4, 5]
    assert get_times(b, 4.0, 10.0) == [4, 5]


def test_all_times_above_t2():
    b = buf_with([5, 4, 3])
    assert R.binary_search(b.content, 1.0) == (1, [1, 2])
    assert get_times(b, 0.0, 1.0) == []


def test_a_late_message_leaves_content_unsorted_and_the_probes_decide():
    b = R.LidarBuffer()
    b.push_message(np.zeros((3, 3)), [1.0, 2.0, 3.0])
    b.push_message(np.ones((2, 3)), [0.5, 0.6])            # arrives late: content = [0.6, 0.5, 3, 2, 1]
    assert list(b.times()) == [0.6, 0.5, 3.0, 2.0, 1.0]
    # t2 = 2.5: mid 2 (3 < 2.5 no: low 3), mid 3 (2 < 2.5: high 2); --high = 1, the walk starts at content[1] = 0.5
    assert R.binary_search(b.content, 2.5) == (1, [2, 3])
    assert get_times(b, 0.55, 2.5) == []                    # 0.5 < t1 breaks at once: 1 and 2 are not reached
    assert get_times(b, 0.0, 2.5) == [1.0, 2.0, 0.5]        # 3 is skipped, 0.6 (content[0]) is never visited
    # t2 = 0.7: mids 2, 3, 4 all read times >= 0.7 (low 5, --high = 3): the walk starts at content[3] = 2, so the late points
    # never come out although both lie in the window
    assert R.binary_search(b.content, 0.7) == (3, [2, 3, 4])
    assert get_times(b, 0.0, 0.7) == []


def test_clear_at_a_point_time_is_inclusive_and_past_the_newest_empties():
    b = buf_with([5, 4, 3, 2, 1])
    b.clear(2.0)
    assert list(b.times()) == [5, 4, 3]
    b.clear(0.5)
    assert list(b.times()) == [5, 4, 3]
    b.clear(10.0)
    assert b.size() == 0


def test_clear_stops_at_the_first_newer_point_in_insertion_order():
    b = R.LidarBuffer()
    b.push_message(np.zeros((3, 3)), [1.0, 2.0, 3.0])
    b.push_message(np.zeros((2, 3)), [0.5, 0.6])
    b.clear(2.5)
    assert list(b.times()) == [0.6, 0.5, 3.0]
    b = R.LidarBuffer()
    b.push_message(np.zeros((3, 3)), [1.0, float("nan"), 3.0])
    b.clear(5.0)                                            # 5 >= NaN is false: the NaN point stops the clear
    assert b.size() == 2 and math.isnan(b.times()[1])


# ---- the host build of csrc/lv_lidar_buffer.h: a ring without lanes, pushed and read with NULL lanes ---------------------------
def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def random_message(rng, clock):
    """n points, mostly ascending with ties (a firing column shares one time); sometimes late, overlapping or with a NaN"""
    n = int(rng.integers(0, 13))
    kind = rng.random()
    start = clock + (rng.uniform(-3.0, -0.5) if kind < 0.15 else rng.uniform(-0.6, 0.0) if kind < 0.3 else 0.0)
    cols = np.sort(rng.integers(0, 6, n)) * 0.25                     # quarter steps: exact ties, exact t1 / t2 hits
    t = start + cols
    if n and rng.random() < 0.03:
        t[rng.integers(0, n)] = np.nan
    xyz = rng.normal(0, 10, (n, 3)).astype(np.float32)
    return xyz, t, max(clock, start + 1.5)


def pick_time(rng, ref, clock):
    """a point time of the buffer (often: ties and exact bounds), a neighbouring quarter step, or anything"""
    ts = [v for v in ref.times() if not math.isnan(v)]
    r = rng.random()
    if ts and r < 0.6:
        return float(ts[int(rng.integers(0, len(ts)))]) + float(rng.choice([0.0, 0.0, 0.25, -0.25]))
    if r < 0.7:
        return float(rng.choice([-1e300, 1e300, -math.inf, math.inf]))
    return float(rng.uniform(clock - 6.0, clock + 1.0))


def test_host_build_equals_the_restatement():
    L = S.lib()
    rng = np.random.default_rng(20261015)
    checked = dict(gets=0, nonempty=0, unsorted=0, full=0, over=0, wrapped=0, cleared=0)
    for seq in range(10_000):
        cap = int(rng.integers(1, 40))
        ring = L.shim_lidar_create(cap, 0)
        ref = R.LidarBuffer()
        clock, pushed = 0.0, 0
        for _ in range(int(rng.integers(1, 14))):
            op = rng.random()
            if op < 0.45:
                xyz, t, clock = random_message(rng, clock)
                ok = L.shim_lidar_push(ring, _fp(xyz), _dp(t), None, None, len(t))
                fits = ref.size() + len(t) <= cap
                assert ok == int(fits), seq
                if fits:
                    ref.push_message(xyz, t)
                    pushed += len(t)
                else:
                    checked["full"] += 1
            elif op < 0.85:
                t1, t2 = pick_time(rng, ref, clock), pick_time(rng, ref, clock)
                if rng.random() < 0.5 and t1 > t2:
                    t1, t2 = t2, t1
                n_max = int(rng.integers(1, cap + 2))
                out_xyz, out_t = np.full((cap, 3), np.nan, np.float32), np.full(cap, np.nan)
                m = L.shim_lidar_get(ring, t1, t2, _fp(out_xyz), _dp(out_t), None, None, n_max)
                rx, rt = ref.get(t1, t2)
                assert m == len(rt), (seq, t1, t2)
                if m > n_max:
                    checked["over"] += 1
                else:
                    assert bits(out_xyz[:m]) == bits(rx) and bits(out_t[:m]) == bits(rt), (seq, t1, t2)
                checked["gets"] += 1
                checked["nonempty"] += m > 0
                ts = ref.times()
                checked["unsorted"] += bool((np.diff(ts[~np.isnan(ts)]) > 0).any())
            else:
                t = pick_time(rng, ref, clock)
                before = ref.size()
                L.shim_lidar_clear(ring, t)
                ref.clear(t)
                checked["cleared"] += ref.size() < before
            assert L.shim_lidar_size(ring) == ref.size(), seq
            got = np.zeros(max(ref.size(), 1))
            L.shim_lidar_content(ring, _dp(got))
            assert bits(got[:ref.size()]) == bits(ref.times()), seq
        checked["wrapped"] += pushed > cap
        L.shim_lidar_destroy(ring)
    for k, v in checked.items():
        assert v >= 300, checked


@pytest.mark.parametrize("nan_at", [0, 2, 4])
def test_nan_point_times_follow_the_comparisons(nan_at):
    L = S.lib()
    t = np.array([1.0, 2.0, 3.0, 4.0, 5.0])
    t[nan_at] = np.nan
    xyz = np.arange(15, dtype=np.float32).reshape(5, 3)
    ring = L.shim_lidar_create(8, 0)
    ref = R.LidarBuffer()
    assert L.shim_lidar_push(ring, _fp(xyz), _dp(t), None, None, 5) == 1
    ref.push_message(xyz, t)
    for t1, t2 in [(0.0, 10.0), (2.0, 4.0), (3.0, 3.0), (0.0, 1.0)]:
        ox, ot = np.zeros((5, 3), np.float32), np.zeros(5)
        m = L.shim_lidar_get(ring, t1, t2, _fp(ox), _dp(ot), None, None, 5)
        rx, rt = ref.get(t1, t2)
        assert m == len(rt) and bits(ox[:m]) == bits(rx) and bits(ot[:m]) == bits(rt), (t1, t2)
    L.shim_lidar_clear(ring, 10.0)
    ref.clear(10.0)
    assert L.shim_lidar_size(ring) == ref.size() == 5 - nan_at
    L.shim_lidar_destroy(ring)
