"""The stream-ordered tick calls without a GPU: every argument refusal of lv_process_cloud_device_async,
lv_compensate_device_async, lv_voxelgrid_downsample_device_async and lv_correct_device_async happens on the host before any
device call, so null pointers, a bound n_max outside [1, 2^31 - 1], a negative min_points and output ranges that overlap an
input are LV_ERR_ARG with a message naming the problem even with a null handle (the device pointers below are never
dereferenced).  The bound against the handle's max_points needs a handle: tests/test_gpu_async_tick.py covers it."""
import ctypes as C

import pytest

BASE = 1 << 40                       # a device address that is never touched
OUT = BASE + (1 << 34)
CNT = BASE + (1 << 36)               # device counts
N = 1000


@pytest.fixture
def L(lv):
    return lv.lib()


def err(L):
    return L.lv_last_error()


def test_process_cloud_async_checks(lv, L):
    lay = lv.CloudLayout(32, 0, 4, 8, 16, 22, 0)

    def run(h=None, layout=lay, data=BASE, data_bytes=N * 32, n=N, xyz=OUT, time=OUT + (1 << 24), n_out=CNT):
        return L.lv_process_cloud_device_async(h, 0, C.byref(layout) if layout is not None else None, data, data_bytes, n, 0, 1, 1,
                                               0.1, 4, 3.0, xyz, time, None, None, None, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"process cloud: null handle"
    for kw in (dict(layout=None), dict(data=None), dict(xyz=None), dict(time=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null layout" in err(L), kw
    for n in (-1, 0x80000000):
        assert run(n=n, data_bytes=1 << 45) == lv.ERR_ARG and b"int32" in err(L), n
    assert run(xyz=BASE + 12) == lv.ERR_ARG and b"overlaps" in err(L)
    assert run(data_bytes=N * 32 - 1) == lv.ERR_ARG and b"too short" in err(L)


def test_compensate_async_checks(lv, L):
    path = (lv.State32 * 4)()
    for i in range(4):
        path[i].time = 0.1 * i
    x2 = lv.State32()

    def run(h=None, p=path, ns=4, xt2=x2, xyz=BASE, t=BASE + (1 << 30), d_n=CNT, n_max=N, out=OUT):
        return L.lv_compensate_device_async(h, p, ns, C.byref(xt2) if xt2 is not None else None, xyz, t, d_n, n_max, out)

    assert run() == lv.ERR_ARG and err(L) == b"compensate async: null handle"
    assert run(out=BASE) == lv.ERR_ARG and err(L) == b"compensate async: null handle"      # in place is fine
    for kw in (dict(p=None), dict(xt2=None), dict(xyz=None), dict(t=None), dict(d_n=None), dict(out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null" in err(L) and b"handle" not in err(L), kw
    for n_max in (0, -5, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    assert run(ns=1) == lv.ERR_ARG and b"two states" in err(L)
    for out in (BASE + 4, BASE - 12 * N + 4, BASE + (1 << 30) + 8 * N - 4, BASE + (1 << 30) - 12 * N + 4):
        assert run(out=out) == lv.ERR_ARG and b"overlaps" in err(L), hex(out)
    for out in (BASE + 12 * N, BASE - 12 * N, BASE + (1 << 30) + 8 * N):                    # adjacent ranges
        assert run(out=out) == lv.ERR_ARG and err(L) == b"compensate async: null handle", hex(out)


def test_voxelgrid_async_checks(lv, L):
    def run(h=None, xyz=BASE, d_n=CNT, n_max=N, leaf=0.5, out=OUT, n_out=CNT + 8):
        return L.lv_voxelgrid_downsample_device_async(h, xyz, d_n, n_max, C.c_float(leaf), out, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"voxel grid async: null handle"
    for kw in (dict(xyz=None), dict(d_n=None), dict(out=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null input" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for leaf in (0.0, -1.0, float("nan")):
        assert run(leaf=leaf) == lv.ERR_ARG and b"leaf" in err(L), leaf
    for out in (BASE, BASE + 12 * N - 4, BASE - 12 * N + 4):
        assert run(out=out) == lv.ERR_ARG and b"overlaps" in err(L), hex(out)
    for out in (BASE + 12 * N, BASE - 12 * N):
        assert run(out=out) == lv.ERR_ARG and err(L) == b"voxel grid async: null handle", hex(out)


def test_correct_async_checks(lv, L):
    def run(h=None, xyz=BASE, d_n=CNT, n_max=N, min_points=20):
        return L.lv_correct_device_async(h, xyz, d_n, n_max, min_points, 1.0)

    assert run() == lv.ERR_ARG and err(L) == b"correct async: null handle"
    assert run(min_points=0) == lv.ERR_ARG and err(L) == b"correct async: null handle"
    for kw in (dict(xyz=None), dict(d_n=None)):
        assert run(**kw) == lv.ERR_ARG and b"null sweep or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    assert run(min_points=-1) == lv.ERR_ARG and b"min_points" in err(L)


def test_async_status_null_handle(lv, L):
    assert L.lv_async_status(None) == lv.ERR_ARG
