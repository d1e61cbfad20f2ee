"""The time-ordered merge of the LiDAR buffer without a GPU.

1. tests/lidar_merge_ref.py (the restatement): on time-ordered buffers and messages the merge is a stable sort of the
   concatenation with the buffered points first on equal times; messages that do not reach back into the buffer are the push; an
   unsorted message or buffer is appended and reported; the refusals leave the buffer unchanged; rt_apply rounds every step in fp32.
2. The host build of csrc/lv_lidar_buffer.h's merge (tests/cpu_shim/lidar_ring.cpp: the walk, the order rule, the mode, the merge
   path of every diagonal, the transform) equals the restatement bit for bit over seeded random sequences of merges, pushes and
   clears on small rings that wrap, with and without lanes and transforms: ties across sensors, empty messages, empty T_tail,
   overlaps at and just above the reserve, full rings, NaN times and unsorted batches.
"""
import ctypes as C

import numpy as np
import pytest

import full_points_ref as FP
import lidar_buffer_ref as R
import lidar_merge_ref as M
import shim_binding as S

f32 = np.float32
MODES = ["write", "append", "full", "overlap"]                 # kLidarMerge* in lv_lidar_buffer.h


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def stable_sorted(points):
    return sorted(points, key=lambda p: p[0])


def msg(rng, start, n, step=0.25, cols=6):
    """n time-sorted points on a quarter-step grid (ties inside and across messages)"""
    t = start + np.sort(rng.integers(0, cols, n)) * step
    return rng.normal(0, 10, (n, 3)).astype(f32), t


# ---- the restatement ------------------------------------------------------------------------------------------------------------
def test_sorted_merges_are_a_stable_sort_with_buffered_points_first():
    rng = np.random.default_rng(1)
    for case in range(300):
        buf = M.MergeBuffer()
        for k in range(int(rng.integers(1, 6))):
            xyz, t = msg(rng, float(rng.integers(0, 8)) * 0.25, int(rng.integers(0, 9)))
            before = list(reversed(buf.content))
            pts = M.message(xyz, t, None)
            assert buf.merge_message(xyz, t) == "write"
            assert list(reversed(buf.content)) == stable_sorted(before + pts), (case, k)


def test_ties_keep_the_buffered_point_first():
    buf = M.MergeBuffer()
    buf.merge_message(np.zeros((3, 3), f32), [1.0, 2.0, 2.0])
    assert buf.merge_message(np.ones((2, 3), f32), [2.0, 3.0]) == "write"
    assert [(p[0], p[1]) for p in reversed(buf.content)] == [(1.0, 0.0), (2.0, 0.0), (2.0, 0.0), (2.0, 1.0), (3.0, 1.0)]
    assert buf.merge_message(np.full((1, 3), 2, f32), [1.0]) == "write"     # lands after the buffered 1.0, before the 2.0s
    assert [(p[0], p[1]) for p in reversed(buf.content)][:3] == [(1.0, 0.0), (1.0, 2.0), (2.0, 0.0)]


def test_messages_that_do_not_reach_back_are_the_push():
    rng = np.random.default_rng(2)
    merged, pushed = M.MergeBuffer(), R.LidarBuffer()
    clock = 0.0
    for _ in range(40):
        xyz, t = msg(rng, clock, int(rng.integers(0, 9)))
        assert merged.merge_message(xyz, t) == "write"
        pushed.push_message(xyz, t)
        clock = float(t[-1]) if len(t) else clock              # the next one starts at or after the newest: equal times too
    assert list(merged.content) == list(pushed.content)


def test_unsorted_messages_and_buffers_are_appended_and_reported():
    buf = M.MergeBuffer()
    buf.merge_message(np.zeros((3, 3), f32), [1.0, 2.0, 3.0])
    for t in ([2.5, 2.4], [2.5, np.nan], [np.nan]):
        ref = R.LidarBuffer()
        ref.content = buf.content.copy()
        assert buf.merge_message(np.ones((len(t), 3), f32), t) == "append"
        ref.push_message(np.ones((len(t), 3), f32), t)
        assert list(map(repr, buf.content)) == list(map(repr, ref.content))
    buf = M.MergeBuffer()
    buf.push_message(np.zeros((3, 3), f32), [1.0, 3.0, 2.0])   # a push left T_tail unsorted
    assert buf.merge_message(np.ones((1, 3), f32), [1.5]) == "append"
    buf = M.MergeBuffer()
    buf.push_message(np.zeros((3, 3), f32), [3.0, 1.0, 2.0])   # unsorted below the split only: merged
    assert buf.merge_message(np.ones((1, 3), f32), [1.5]) == "write"
    assert list(buf.times()[::-1]) == [3.0, 1.0, 1.5, 2.0]


def test_refusals_leave_the_buffer_unchanged():
    buf = M.MergeBuffer(cap=6, reserve=2)
    buf.merge_message(np.zeros((4, 3), f32), [1.0, 2.0, 3.0, 4.0])
    before = list(buf.content)
    assert buf.merge_message(np.ones((1, 3), f32), [1.5]) == "overlap"      # T_tail = 2, 3, 4
    assert buf.merge_message(np.ones((3, 3), f32), [5.0, 6.0, 7.0]) == "full"
    assert buf.merge_message(np.ones((3, 3), f32), [2.0, 1.0, 7.0]) == "full"   # fullness before order
    assert list(buf.content) == before
    assert buf.merge_message(np.ones((2, 3), f32), [2.5, 9.0]) == "write"  # T_tail = 3, 4: exactly the reserve
    assert list(buf.times()[::-1]) == [1.0, 2.0, 2.5, 3.0, 4.0, 9.0]
    assert buf.merge_message(np.zeros((0, 3), f32), []) == "write" and buf.size() == 6   # empty: nothing, even on a full ring


def test_rt_apply_rounds_each_step_in_fp32():
    T = np.array([0.5, 0.25, 3.0, 1.0, 0.0, 0.0, 0.0, 1e-8, 1.0, 1.0, 2.0, 3.0], f32)
    p = np.array([[1e8, 1.0, -1.0]], f32)
    g = M.rt_apply(T, p)
    x = f32(f32(f32(f32(0.5) * f32(1e8)) + f32(0.25)) + f32(-3.0)) + f32(1.0)
    assert g[0, 0] == x and g[0, 1] == f32(1e8) + f32(2.0)
    assert g.dtype == f32
    z = M.rt_apply(np.array([1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0], f32), np.array([[-0.0, 1.0, 2.0]], f32))
    assert bits(z[:, 0]) != bits(np.array([-0.0], f32))                   # why a NULL T must not be an identity multiply


# ---- the host build of csrc/lv_lidar_buffer.h -----------------------------------------------------------------------------------
def _fp(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return np.ascontiguousarray(a).ctypes.data_as(C.POINTER(C.c_double))


def shim_content(L, ring, n):
    xyz, t, i, r = np.zeros((max(n, 1), 3), f32), np.zeros(max(n, 1)), np.zeros(max(n, 1), f32), np.zeros(max(n, 1), f32)
    L.shim_lidar_content_full(ring, _fp(xyz), _dp(t), _fp(i), _fp(r))
    return t[:n], xyz[:n], i[:n], r[:n]


def ref_content(ref, lanes):
    t, rest = M.content_arrays(ref, 5 if lanes else 3)
    xyz = rest[:, :3]
    if lanes:
        return t, xyz, rest[:, 3].copy(), rest[:, 4].copy()
    return t, xyz, np.zeros(len(t), f32), np.zeros(len(t), f32)


def sensor_message(rng, clock, sensors):
    """a message of one of `sensors` sensors: its span overlaps what the others delivered, on a grid of shared times"""
    n = int(rng.choice([0, 1, 2, 5, 9, 14]))
    kind = rng.random()
    back = rng.choice([0.0, 0.25, 0.5, 1.0, 2.0, 4.0]) if kind < 0.8 else rng.uniform(0, 3)
    start = clock - back
    t = start + np.sort(rng.integers(0, 8, n)) * 0.25
    if n and rng.random() < 0.05:
        t[rng.integers(0, n)] = np.nan                         # a NaN time
    elif n > 1 and rng.random() < 0.05:
        t = t[::-1].copy()                                     # a batch that was not time-sorted
    xyz = rng.normal(0, 10, (n, 3)).astype(f32)
    xyz[rng.random((n, 3)) < 0.02] = -0.0
    return xyz, t, max(clock, start + 2.0), int(rng.integers(0, sensors))


@pytest.mark.parametrize("lanes", [False, True])
def test_host_build_equals_the_restatement(lanes):
    L = S.lib()
    rng = np.random.default_rng(20261018 + lanes)
    seen = {k: 0 for k in MODES + ["ties", "empty_b", "empty_tail", "at_reserve", "wrapped", "transform", "push", "cleared"]}
    for seq in range(2500):
        cap = int(rng.integers(1, 48))
        reserve = int(rng.integers(1, 12))
        sensors = int(rng.integers(2, 4))
        Ts = [None] + [M.random_extrinsic(rng) for _ in range(sensors - 1)]
        ring = L.shim_lidar_create(cap, int(lanes))
        ref = M.MergeBufferFull(cap, reserve) if lanes else M.MergeBuffer(cap, reserve)
        clock, pushed = 0.0, 0
        for _ in range(int(rng.integers(1, 16))):
            op = rng.random()
            xyz, t, clock, k = sensor_message(rng, clock, sensors)
            T = Ts[k]
            if op < 0.75:
                inten = rng.uniform(0, 255, len(t)).astype(f32) if lanes and rng.random() < 0.7 else None
                rng_lane = rng.uniform(0, 80, len(t)).astype(f32) if inten is not None else None
                L_ = list(reversed(ref.content))
                b0 = t[0] if len(t) else np.nan
                split = M.split_of(L_, b0) if len(t) else len(L_)
                mode = MODES[L.shim_lidar_merge(ring, _fp(xyz), _dp(t), _fp(inten), _fp(rng_lane), len(t), _fp(T), reserve)]
                if lanes:
                    want = ref.merge_message(xyz, t, T, inten, rng_lane)
                else:
                    want = ref.merge_message(xyz, t, T)
                assert mode == want, (seq, mode, want)
                seen[mode] += 1
                seen["empty_b"] += len(t) == 0
                seen["empty_tail"] += mode == "write" and len(t) > 0 and split == len(L_) and len(L_) > 0
                seen["at_reserve"] += mode == "write" and len(L_) - split == reserve
                seen["transform"] += mode == "write" and T is not None and len(t) > 0
                seen["ties"] += mode == "write" and len(t) > 0 and bool(np.isin(t, [p[0] for p in L_[split:]]).any())
                if mode in ("write", "append"):
                    pushed += len(t)
            elif op < 0.85:
                fits = ref.size() + len(t) <= cap
                assert L.shim_lidar_push(ring, _fp(xyz), _dp(t), None, None, len(t)) == int(fits)
                if fits:
                    ref.push_message(xyz, t)
                    pushed += len(t)
                    seen["push"] += 1
            else:
                tc = float(rng.uniform(clock - 6, clock))
                before = ref.size()
                L.shim_lidar_clear(ring, tc)
                ref.clear(tc)
                seen["cleared"] += ref.size() < before
            n = ref.size()
            assert L.shim_lidar_size(ring) == n, seq
            got, want = shim_content(L, ring, n), ref_content(ref, lanes)
            for a, b, name in zip(got, want, ("time", "xyz", "intensity", "range")):
                assert bits(a) == bits(b), (seq, name)
        seen["wrapped"] += pushed > cap
        L.shim_lidar_destroy(ring)
    assert all(v >= 30 for v in seen.values()), seen


def test_host_build_windows_after_merges_equal_the_restatement():
    """the windows of a merged buffer: the reference's get on time-ordered content"""
    L = S.lib()
    rng = np.random.default_rng(5)
    ring = L.shim_lidar_create(200, 0)
    ref = M.MergeBuffer(200, 64)
    clock = 0.0
    for step in range(60):
        xyz, t, clock, _ = sensor_message(rng, clock, 3)
        if ref.size() + len(t) > 200:
            ref.clear(clock - 2.0)
            L.shim_lidar_clear(ring, clock - 2.0)
        L.shim_lidar_merge(ring, _fp(xyz), _dp(t), None, None, len(t), None, 64)
        ref.merge_message(xyz, t)
        t1 = float(rng.uniform(clock - 4, clock))
        t2 = t1 + float(rng.choice([0.0, 0.25, 0.5, 1.0]))
        ox, ot = np.zeros((200, 3), f32), np.zeros(200)
        m = L.shim_lidar_get(ring, t1, t2, _fp(ox), _dp(ot), None, None, 200)
        rx, rt = ref.get(t1, t2)
        assert m == len(rt) and bits(ox[:m]) == bits(rx) and bits(ot[:m]) == bits(rt), step
    L.shim_lidar_destroy(ring)
