"""Full points without a GPU.

1. tests/full_points_ref.py (the restatement of what the reference does to intensity, range and time between the message and the
   publishers) on hand-worked cases: the intensity sum of a leaf in the leaf's order (fp32, from +0), the range as the fp32 norm of
   the centroid, time 0, PCL's overflow pass-through of every attribute, the buffer's lanes, and the header stamp (rounding at .5 us,
   an empty cloud, a 1.7e9 s epoch).
2. The host build of the device buffer's index arithmetic with attribute lanes (csrc/lv_lidar_buffer.h through
   tests/cpu_shim/lidar_ring.cpp) equals the restatement on seeded random push / get / clear / reserve sequences: full and plain pushes,
   rings that gain lanes with points already live, re-reserves, wraps, ties and windows above n_max.
"""
import ctypes as C
import math

import numpy as np
import pytest

import frontend_ref as F
import full_points_ref as P
import lidar_buffer_ref as R
import shim_binding as S

f32 = np.float32


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


# ---- the voxel grid of full points -----------------------------------------------------------------------------------------------
def test_intensity_is_the_fp32_running_sum_in_leaf_order():
    # one leaf (leaf 1, all points in [0, 1)^3): 1e8 + 1 - 1e8 in fp32 is 0 in this order, 1 in another
    xyz = np.array([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [0.3, 0.3, 0.3]], f32)
    inten = np.array([1e8, 1.0, -1e8], f32)
    out, t, i, r = P.voxelgrid_full(xyz, np.array([5.0, 6.0, 7.0]), inten, 1.0)
    assert len(out) == 1
    s = (f32(0) + f32(1e8)) + f32(1.0)
    assert s == f32(1e8)                                               # the 1 is absorbed
    assert i[0] == (s + f32(-1e8)) / f32(3) == 0.0
    p = P.voxelgrid_full(xyz[::-1], np.zeros(3), inten[::-1], 1.0)[2]
    assert p[0] == ((f32(-1e8) + f32(1.0)) + f32(1e8)) / f32(3) == 0.0
    q = P.voxelgrid_full(xyz[[0, 2, 1]], np.zeros(3), inten[[0, 2, 1]], 1.0)[2]
    assert q[0] == f32(1.0) / f32(3)                                   # 1e8 - 1e8 first, then + 1: the order decides
    # two leaves, ascending cell index; input order inside a leaf
    xyz = np.array([[1.5, 0.2, 0.2], [0.5, 0.2, 0.2], [1.25, 0.3, 0.3], [0.25, 0.4, 0.4]], f32)
    inten = np.array([10.0, 3.0, 20.0, 4.0], f32)
    out, t, i, r = P.voxelgrid_full(xyz, np.arange(4.0), inten, 1.0)
    assert i.tolist() == [3.5, 15.0]
    assert bits(out) == bits(F.voxelgrid(xyz, 1.0)["out"])


def test_range_is_the_fp32_norm_of_the_centroid_and_time_is_zero():
    xyz = np.array([[3.0, 4.0, 0.0], [3.0, 4.0, 12.0]], f32)
    out, t, i, r = P.voxelgrid_full(xyz, np.array([1.7e9, 1.7e9 + 1]), np.zeros(2, f32), 100.0)
    assert out.tolist() == [[3.0, 4.0, 6.0]]
    assert r[0] == f32(math.sqrt(61.0)) and r.dtype == f32              # the centroid's norm, not a mean of the points' ranges (9)
    assert t.tolist() == [0.0] and t.dtype == np.float64
    # the fp32 steps: sqrt((x x + y y) + z z), each rounded, as the decoder computes |p|
    c = np.array([[0.1, 0.2, 0.3]], f32)
    x, y, z = c[0]
    assert P.norm32(c)[0] == np.sqrt(f32(f32(x * x) + f32(y * y)) + f32(z * z))


def test_overflow_passes_xyz_time_and_intensity_through_and_range_is_each_points_norm():
    # Compensator.cpp:161 builds every output point with Point(p), the passed-through ones too: set_attributes sets range = |p|
    xyz = np.array([[0, 0, 0], [(1 << 23) - 1, 255, 0], [3, 4, 12], [1 << 23, 0, 0]], f32)  # 2^23 x 256 x 1 cells > INT32_MAX
    assert F.voxel_cells(xyz, 1.0)["overflow"]
    t = np.array([1.0, 2.0, 3.0, 4.0])
    inten = np.array([7, 8, 9, 10], f32)
    out = P.voxelgrid_full(xyz, t, inten, 1.0)
    assert bits(out[0]) == bits(xyz) and bits(out[1]) == bits(t) and bits(out[2]) == bits(inten)
    assert out[3].dtype == f32 and out[3][0] == 0.0 and out[3][2] == 13.0 and out[3][3] == f32(1 << 23)
    assert bits(out[3]) == bits(P.norm32(xyz))
    assert P.stamp_us(out[1]) == 4000000                                # the passed-through times give the stamp


def test_empty_cloud():
    out = P.voxelgrid_full(np.zeros((0, 3), f32), np.zeros(0), np.zeros(0, f32), 0.5)
    assert [len(a) for a in out] == [0, 0, 0, 0]


# ---- the header stamp --------------------------------------------------------------------------------------------------------------
def test_stamp_rounds_half_away_from_zero():
    # 1/128 s = 7812.5 us exactly: std::round gives 7813 (Python's round would give 7812)
    assert 0.0078125 * 1e6 == 7812.5
    assert P.sec2microsec(0.0078125) == 7813 and round(7812.5) == 7812
    assert P.sec2microsec(3 * 0.0078125) == 23438
    # just below .5: the product is below 7812.5, so it rounds down
    t = np.nextafter(0.0078125, 0.0)
    assert t * 1e6 < 7812.5 and P.sec2microsec(t) == 7812
    assert P.sec2microsec(0.0) == 0 and P.sec2microsec(1.0) == 1000000


def test_stamp_of_an_empty_cloud_and_of_a_downsampled_one_is_zero():
    assert P.stamp_us(np.zeros(0)) == 0
    assert P.stamp_us(np.zeros(17)) == 0                                # every time of a voxel-grid output is 0


def test_stamp_at_a_unix_epoch_is_the_maximum():
    base = 1.7e9
    t = np.array([base + 0.0078125, base, base + 0.0234375, base + 0.001])
    assert all(float(v) * 1e6 == float(v * 1e6) for v in t)
    assert t[0] * 1e6 == 1700000000007812.5                             # exact: below 2^51 the spacing is 1/4
    assert P.stamp_us(t) == 1700000000023438                            # the max, not the last point (Publishers.hpp:56 is overwritten by fill)
    assert P.stamp_us(t[:2]) == 1700000000007813
    assert P.stamp_us(t[::-1]) == P.stamp_us(t)


# ---- the buffer's lanes ------------------------------------------------------------------------------------------------------------
def test_buffer_carries_the_lanes_with_the_window():
    b = P.LidarBufferFull()
    b.push_message(np.arange(9, dtype=f32).reshape(3, 3), [1.0, 2.0, 3.0], [10, 20, 30], [1.5, 2.5, 3.5])
    b.push_message(np.zeros((2, 3), f32), [3.0, 3.0])                  # no attributes: 0, 0
    xyz, t, i, r = b.get(0.0, 3.0)
    # content = [3, 3, 3(30), 2, 1]: the walk starts one before the last of the ties at t2 (two of three are returned)
    assert t.tolist() == [1.0, 2.0, 3.0, 3.0]
    assert i.tolist() == [10.0, 20.0, 30.0, 0.0] and r.tolist() == [1.5, 2.5, 3.5, 0.0]
    ref = R.LidarBuffer()
    ref.push_message(np.arange(9, dtype=f32).reshape(3, 3), [1.0, 2.0, 3.0])
    ref.push_message(np.zeros((2, 3), f32), [3.0, 3.0])
    rx, rt = ref.get(0.0, 3.0)
    assert bits(rx) == bits(xyz) and bits(rt) == bits(t)               # the same window as the xyz-only buffer
    b.clear(2.0)
    assert b.size() == 3


# ---- the host build of csrc/lv_lidar_buffer.h with lanes ---------------------------------------------------------------------------
def _fp(a):
    return None if a is None else a.ctypes.data_as(C.POINTER(C.c_float))


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_host_build_with_lanes_equals_the_restatement():
    from test_lidar_buffer_ref import pick_time, random_message
    L = S.lib()
    rng = np.random.default_rng(20261016)
    seen = dict(gets=0, nonempty=0, plain=0, full=0, gained=0, resized=0, over=0, refused=0, wrapped=0)
    for seq in range(3000):
        cap = int(rng.integers(1, 40))
        lanes = bool(rng.random() < 0.7)
        ring = L.shim_lidar_create(cap, int(lanes))
        ref = P.LidarBufferFull()
        clock, pushed = 0.0, 0
        for _ in range(int(rng.integers(1, 14))):
            op = rng.random()
            if op < 0.4:
                xyz, t, clock = random_message(rng, clock)
                n = len(t)
                full = lanes and rng.random() < 0.75
                inten = rng.uniform(0, 255, n).astype(f32) if full else None
                rg = rng.uniform(0, 100, n).astype(f32) if full else None
                ok = L.shim_lidar_push(ring, _fp(xyz), _dp(t), _fp(inten), _fp(rg), n)
                fits = ref.size() + n <= cap
                assert ok == int(fits), seq
                if fits:
                    ref.push_message(xyz, t, inten, rg)
                    pushed += n
                    seen["full" if full else "plain"] += 1
            elif op < 0.55:
                new_cap = int(rng.integers(1, 45))
                add = bool(rng.random() < 0.5)
                ok = L.shim_lidar_reserve(ring, new_cap, int(add))
                assert ok == int(ref.size() <= new_cap), seq
                if ok:
                    seen["gained"] += add and not lanes and ref.size() > 0
                    seen["resized"] += 1
                    cap, lanes = new_cap, lanes or add
                else:
                    seen["refused"] += 1
            elif op < 0.85 and lanes:
                t1, t2 = pick_time(rng, ref, clock), pick_time(rng, ref, clock)
                if rng.random() < 0.5 and t1 > t2:
                    t1, t2 = t2, t1
                n_max = int(rng.integers(1, cap + 2))
                ox, ot = np.full((cap, 3), np.nan, f32), np.full(cap, np.nan)
                oi, orr = np.full(cap, np.nan, f32), np.full(cap, np.nan, f32)
                m = L.shim_lidar_get(ring, t1, t2, _fp(ox), _dp(ot), _fp(oi), _fp(orr), n_max)
                rx, rt, ri, rr = ref.get(t1, t2)
                assert m == len(rt), (seq, t1, t2)
                if m > n_max:
                    seen["over"] += 1
                else:
                    assert bits(ox[:m]) == bits(rx) and bits(ot[:m]) == bits(rt), (seq, t1, t2)
                    assert bits(oi[:m]) == bits(ri) and bits(orr[:m]) == bits(rr), (seq, t1, t2)
                seen["gets"] += 1
                seen["nonempty"] += m > 0
            else:
                t = pick_time(rng, ref, clock)
                L.shim_lidar_clear(ring, t)
                ref.clear(t)
            assert L.shim_lidar_size(ring) == ref.size(), seq
        seen["wrapped"] += pushed > cap
        L.shim_lidar_destroy(ring)
    for k, v in seen.items():
        assert v >= 100, seen
