"""The full-point calls without a GPU: every argument refusal of lv_lidar_reserve_full, lv_lidar_push_full_device_async,
lv_lidar_get_points_full_device_async, lv_voxelgrid_downsample_full(_device_async) and lv_cloud_stamp_device_async happens on the
host before any device call, so null pointers, n_max outside [1, 2^31 - 1], NaN times and ranges that overlap are LV_ERR_ARG with a
message naming the problem even with a null handle (the device pointers below are never dereferenced).  Full calls on a ring without
lanes, and overlaps with the ring, need a handle: tests/test_gpu_full_points.py covers them."""
import ctypes as C

import pytest

from test_async_tick_args import BASE, CNT, OUT, err

N = 1000
NAN = float("nan")
T_IN, I_IN, R_IN = BASE + (1 << 30), BASE + (2 << 30), BASE + (3 << 30)
T_OUT, I_OUT, R_OUT = OUT + (1 << 30), OUT + (2 << 30), OUT + (3 << 30)


@pytest.fixture
def L(lv):
    return lv.lib()


def test_reserve_full_checks(lv, L):
    assert L.lv_lidar_reserve_full(None, 1000) == lv.ERR_ARG and err(L) == b"lidar reserve full: null handle"
    assert L.lv_lidar_reserve_full(None, 1 << 30) == lv.ERR_ARG and err(L) == b"lidar reserve full: null handle"
    for cap in (0, -1, (1 << 30) + 1):
        assert L.lv_lidar_reserve_full(None, cap) == lv.ERR_ARG and b"capacity outside" in err(L), cap


def test_push_full_checks(lv, L):
    def run(h=None, xyz=BASE, t=T_IN, i=I_IN, r=R_IN, d_n=CNT, n_max=N):
        return L.lv_lidar_push_full_device_async(h, xyz, t, i, r, d_n, n_max)

    assert run() == lv.ERR_ARG and err(L) == b"lidar push full: null handle"
    assert run(n_max=0x7fffffff) == lv.ERR_ARG and err(L) == b"lidar push full: null handle"
    for kw in (dict(xyz=None), dict(t=None), dict(i=None), dict(r=None), dict(d_n=None)):
        assert run(**kw) == lv.ERR_ARG and b"null xyz, time, intensity, range or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max


def test_get_full_checks(lv, L):
    def run(h=None, t1=1.0, t2=2.0, xyz=OUT, t=T_OUT, i=I_OUT, r=R_OUT, n_max=N, n_out=CNT):
        return L.lv_lidar_get_points_full_device_async(h, t1, t2, xyz, t, i, r, n_max, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"lidar get points full: null handle"
    assert run(t1=3.0, t2=2.0) == lv.ERR_ARG and err(L) == b"lidar get points full: null handle"
    for kw in (dict(i=None), dict(r=None)):
        assert run(**kw) == lv.ERR_ARG and b"null intensity or range" in err(L), kw
    for kw in (dict(xyz=None), dict(t=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null xyz, time or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for kw in (dict(t1=NAN), dict(t2=NAN)):
        assert run(**kw) == lv.ERR_ARG and b"NaN" in err(L), kw
    for kw in (dict(i=OUT + 12 * N - 4), dict(r=T_OUT + 8 * N - 4), dict(i=R_OUT - 4 * N + 4), dict(r=I_OUT),
               dict(n_out=I_OUT + 4 * N - 4), dict(n_out=R_OUT), dict(i=CNT - 4 * N + 4)):
        assert run(**kw) == lv.ERR_ARG and b"output ranges overlap" in err(L), kw
    for kw in (dict(i=OUT + 12 * N), dict(r=I_OUT + 4 * N), dict(n_out=R_OUT + 4 * N), dict(i=CNT + 8)):    # adjacent
        assert run(**kw) == lv.ERR_ARG and err(L) == b"lidar get points full: null handle", kw


def test_voxelgrid_full_async_checks(lv, L):
    def run(h=None, xyz=BASE, t=T_IN, i=I_IN, d_n=CNT, n_max=N, leaf=0.5, out=OUT, to=T_OUT, io=I_OUT, ro=R_OUT, n_out=CNT + 8):
        return L.lv_voxelgrid_downsample_full_device_async(h, xyz, t, i, d_n, n_max, leaf, out, to, io, ro, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"voxel grid full: null handle"
    assert run(to=None, io=None, ro=None) == lv.ERR_ARG and err(L) == b"voxel grid full: null handle"   # every lane output is optional
    for kw in (dict(xyz=None), dict(t=None), dict(i=None), dict(d_n=None), dict(out=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"voxel grid full: null" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for leaf in (0.0, -1.0, NAN):
        assert run(leaf=leaf) == lv.ERR_ARG and b"leaf size" in err(L), leaf
    # an output over an input, or over another output; inputs may share bytes (they are only read)
    for kw in (dict(out=BASE + 12), dict(to=T_IN + 8), dict(io=I_IN - 4 * N + 4), dict(ro=I_IN + 4), dict(ro=BASE + 12 * N - 4),
               dict(io=OUT + 12 * N - 4), dict(ro=T_OUT + 4), dict(to=R_OUT - 8 * N + 4), dict(n_out=CNT), dict(n_out=OUT + 8),
               dict(n_out=R_OUT + 4 * N - 8), dict(io=CNT + 4 - 4 * N), dict(ro=CNT + 8 - 4 * N + 4)):
        assert run(**kw) == lv.ERR_ARG and b"overlaps" in err(L), kw
    for kw in (dict(out=BASE + 12 * N), dict(io=I_IN + 4 * N), dict(ro=OUT + 12 * N), dict(n_out=CNT + 8), dict(t=BASE, i=BASE)):
        assert run(**kw) == lv.ERR_ARG and err(L) == b"voxel grid full: null handle", kw


def test_voxelgrid_full_host_checks(lv, L):
    import numpy as np
    xyz, t, i = np.zeros((4, 3), np.float32), np.zeros(4), np.zeros(4, np.float32)
    o = (np.zeros((4, 3), np.float32), np.zeros(4), np.zeros(4, np.float32), np.zeros(4, np.float32))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    n_out = C.c_int64(-5)

    def run(h=None, ins=(xyz, t, i), n=4, leaf=0.5, outs=o, n_out=C.byref(n_out)):
        return L.lv_voxelgrid_downsample_full(h, *(None if a is None else p(a) for a in ins), n, leaf,
                                              *(None if a is None else p(a) for a in outs), n_out)

    assert run() == lv.ERR_ARG and err(L) == b"voxel grid full: null handle" and n_out.value == 0
    assert run(outs=(o[0], None, None, None)) == lv.ERR_ARG and err(L) == b"voxel grid full: null handle"
    for k in range(3):
        ins = tuple(None if j == k else a for j, a in enumerate((xyz, t, i)))
        assert run(ins=ins) == lv.ERR_ARG and b"null" in err(L), k
    assert run(outs=(None,) + o[1:]) == lv.ERR_ARG and b"null" in err(L)
    assert run(n_out=None) == lv.ERR_ARG and b"null" in err(L)
    for n in (-1, 0x80000000):
        assert run(n=n) == lv.ERR_ARG and b"n outside" in err(L), n
    assert run(leaf=0.0) == lv.ERR_ARG and b"leaf size" in err(L)


def test_stamp_checks(lv, L):
    def run(h=None, t=T_IN, d_n=CNT, n_max=N, stamp=OUT):
        return L.lv_cloud_stamp_device_async(h, t, d_n, n_max, stamp)

    assert run() == lv.ERR_ARG and err(L) == b"cloud stamp: null handle"
    for kw in (dict(t=None), dict(d_n=None), dict(stamp=None)):
        assert run(**kw) == lv.ERR_ARG and b"null time, count or stamp" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for kw in (dict(stamp=T_IN + 8 * N - 8), dict(stamp=T_IN), dict(stamp=CNT + 4), dict(stamp=CNT - 4)):
        assert run(**kw) == lv.ERR_ARG and b"overlaps" in err(L), kw
    for kw in (dict(stamp=T_IN + 8 * N), dict(stamp=CNT + 8), dict(stamp=CNT - 8), dict(d_n=T_IN)):   # adjacent, or two inputs
        assert run(**kw) == lv.ERR_ARG and err(L) == b"cloud stamp: null handle", kw
