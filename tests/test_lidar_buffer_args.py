"""The LiDAR buffer's calls without a GPU: every argument refusal of lv_lidar_reserve, lv_lidar_push_device_async,
lv_lidar_get_points_device(_async), lv_lidar_clear_async and lv_lidar_info happens on the host before any device call, so null
pointers, n_max outside [1, 2^31 - 1], a capacity outside [1, 2^30], NaN time arguments and output ranges that overlap each other
are LV_ERR_ARG with a message naming the problem even with a null handle (the device pointers below are never dereferenced).
A push, get or clear before lv_lidar_reserve needs a handle: tests/test_gpu_lidar_buffer.py covers it."""
import ctypes as C

import pytest

from test_async_tick_args import BASE, CNT, OUT, err

N = 1000
NAN = float("nan")


@pytest.fixture
def L(lv):
    return lv.lib()


def test_reserve_checks(lv, L):
    assert L.lv_lidar_reserve(None, 1000) == lv.ERR_ARG and err(L) == b"lidar reserve: null handle"
    assert L.lv_lidar_reserve(None, 1 << 30) == lv.ERR_ARG and err(L) == b"lidar reserve: null handle"
    for cap in (0, -1, (1 << 30) + 1):
        assert L.lv_lidar_reserve(None, cap) == lv.ERR_ARG and b"capacity outside" in err(L), cap


def test_push_checks(lv, L):
    def run(h=None, xyz=BASE, t=BASE + (1 << 30), d_n=CNT, n_max=N):
        return L.lv_lidar_push_device_async(h, xyz, t, d_n, n_max)

    assert run() == lv.ERR_ARG and err(L) == b"lidar push: null handle"
    assert run(n_max=0x7fffffff) == lv.ERR_ARG and err(L) == b"lidar push: null handle"
    for kw in (dict(xyz=None), dict(t=None), dict(d_n=None)):
        assert run(**kw) == lv.ERR_ARG and b"null xyz, time or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max


@pytest.mark.parametrize("sync", [False, True])
def test_get_points_checks(lv, L, sync):
    n_host = C.c_int64(-5)

    def run(h=None, t1=1.0, t2=2.0, xyz=OUT, t=OUT + (1 << 30), n_max=N, n_out=CNT):
        if sync:
            return L.lv_lidar_get_points_device(h, t1, t2, xyz, t, n_max, C.byref(n_host) if n_out else None)
        return L.lv_lidar_get_points_device_async(h, t1, t2, xyz, t, n_max, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"lidar get points: null handle"
    assert run(t1=-float("inf"), t2=float("inf")) == lv.ERR_ARG and err(L) == b"lidar get points: null handle"
    assert run(t1=3.0, t2=2.0) == lv.ERR_ARG and err(L) == b"lidar get points: null handle"    # an empty window is no error
    for kw in (dict(xyz=None), dict(t=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null xyz, time or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for kw in (dict(t1=NAN), dict(t2=NAN), dict(t1=NAN, t2=NAN)):
        assert run(**kw) == lv.ERR_ARG and b"NaN" in err(L), kw
    for t in (OUT, OUT + 12 * N - 8, OUT - 8 * N + 8):
        assert run(t=t) == lv.ERR_ARG and b"output ranges overlap" in err(L), hex(t)
    for t in (OUT + 12 * N, OUT - 8 * N):                                                      # adjacent ranges
        assert run(t=t) == lv.ERR_ARG and err(L) == b"lidar get points: null handle", hex(t)
    if not sync:
        for n_out in (OUT + 8, OUT + (1 << 30) + 8 * N - 8):
            assert run(n_out=n_out) == lv.ERR_ARG and b"output ranges overlap" in err(L), hex(n_out)
        assert run(n_out=OUT + 12 * N) == lv.ERR_ARG and err(L) == b"lidar get points: null handle"
    else:
        assert n_host.value == 0                                                               # reset before any check


def test_clear_checks(lv, L):
    assert L.lv_lidar_clear_async(None, 1.0) == lv.ERR_ARG and err(L) == b"lidar clear: null handle"
    assert L.lv_lidar_clear_async(None, float("inf")) == lv.ERR_ARG and err(L) == b"lidar clear: null handle"
    assert L.lv_lidar_clear_async(None, NAN) == lv.ERR_ARG and b"NaN" in err(L)


def test_info_checks(lv, L):
    info = lv.LidarInfo()
    assert L.lv_lidar_info(None, C.byref(info)) == lv.ERR_ARG and b"null handle" in err(L)
    assert L.lv_lidar_info(None, None) == lv.ERR_ARG
