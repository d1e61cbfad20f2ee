"""The merge calls of the LiDAR buffer without a GPU: every argument refusal of lv_lidar_reserve_merge,
lv_lidar_merge_device_async and lv_lidar_merge_full_device_async happens on the host before any device call, so null pointers,
n_max outside [1, 2^31 - 1], an overlap reserve outside [1, 2^30], a non-finite transform entry and input ranges that overlap each
other are LV_ERR_ARG with a message naming the problem even with a null handle (the device pointers below are never
dereferenced).  A merge before lv_lidar_reserve / lv_lidar_reserve_merge and a full merge on a buffer without lanes need a handle:
tests/test_gpu_lidar_merge.py covers them."""
import ctypes as C

import numpy as np
import pytest

from test_async_tick_args import BASE, CNT, err

N = 1000
XYZ = BASE + (1 << 38)                                       # 2^35 bytes apart: n_max = 2^31 - 1 points fit between them
TIME, INT, RNG = XYZ + (1 << 35), XYZ + (2 << 35), XYZ + (3 << 35)


@pytest.fixture
def L(lv):
    return lv.lib()


def T12(*over):
    T = (C.c_float * 12)(1, 0, 0, 0, 1, 0, 0, 0, 1, 0.5, -0.25, 2.0)
    for k, v in over:
        T[k] = v
    return T


def test_reserve_merge_checks(lv, L):
    for overlap in (1, 1 << 30):
        assert L.lv_lidar_reserve_merge(None, overlap) == lv.ERR_ARG and err(L) == b"lidar reserve merge: null handle"
    for overlap in (0, -1, (1 << 30) + 1):
        assert L.lv_lidar_reserve_merge(None, overlap) == lv.ERR_ARG and b"overlap outside [1, 2^30]" in err(L), overlap


@pytest.mark.parametrize("full", [False, True])
def test_merge_checks(lv, L, full):
    what = b"lidar merge full" if full else b"lidar merge"

    def run(h=None, xyz=XYZ, t=TIME, i=INT, r=RNG, d_n=CNT, n_max=N, T=None):
        if full:
            return L.lv_lidar_merge_full_device_async(h, xyz, t, i, r, d_n, n_max, T)
        return L.lv_lidar_merge_device_async(h, xyz, t, d_n, n_max, T)

    assert run() == lv.ERR_ARG and err(L) == what + b": null handle"
    assert run(T=T12()) == lv.ERR_ARG and err(L) == what + b": null handle"
    assert run(n_max=0x7fffffff) == lv.ERR_ARG and err(L) == what + b": null handle"
    nulls = [dict(xyz=None), dict(t=None), dict(d_n=None)] + ([dict(i=None), dict(r=None)] if full else [])
    for kw in nulls:
        assert run(**kw) == lv.ERR_ARG and b"null xyz, time" in err(L) and err(L).startswith(what + b":"), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for k in (0, 4, 8, 9, 11):
        for v in (float("nan"), float("inf"), -float("inf")):
            assert run(T=T12((k, v))) == lv.ERR_ARG and b"transform entry is not finite" in err(L), (k, v)
    assert run(T=T12((9, 3.0e38))) == lv.ERR_ARG and err(L) == what + b": null handle"          # large but finite
    # input ranges that overlap each other: the count inside the times, the times over the points' end, lanes over each other
    overlapping = [dict(d_n=TIME + 8 * N - 8), dict(t=XYZ + 12 * N - 8), dict(d_n=XYZ)]
    if full:
        overlapping += [dict(r=INT + 4 * N - 4), dict(i=TIME + 8), dict(d_n=RNG + 4)]
    for kw in overlapping:
        assert run(**kw) == lv.ERR_ARG and b"input ranges overlap" in err(L), kw
    for kw in (dict(t=XYZ + 12 * N), dict(d_n=TIME + 8 * N)):                                    # adjacent ranges
        assert run(**kw) == lv.ERR_ARG and err(L) == what + b": null handle", kw


def test_plain_push_keeps_its_checks(lv, L):
    """the push does not gain the merge's input-overlap check: its behaviour is unchanged"""
    assert L.lv_lidar_push_device_async(None, XYZ, TIME, TIME, N) == lv.ERR_ARG and err(L) == b"lidar push: null handle"


def test_python_binding_passes_twelve_floats(lv):
    T = lv._transform12(np.arange(12, dtype=np.float32))
    assert list(T) == list(range(12)) and lv._transform12(None) is None
