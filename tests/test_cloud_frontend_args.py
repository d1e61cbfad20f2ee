"""lv_process_cloud_device without a GPU: every argument check runs on the host before any device call, so a null handle,
null buffers, a bad layout, a point count outside the int32 index range and an output overlapping the message bytes are
LV_ERR_ARG with a message naming the problem (the device pointers below are never dereferenced)."""
import ctypes as C

import pytest

BASE = 1 << 40                       # a device address that is never touched
N, STEP = 100, 32


@pytest.fixture
def call(lv):
    L = lv.lib()
    lay = lv.CloudLayout(STEP, 0, 4, 8, 16, 22, 0)        # velodyne, time at byte 22

    def run(h=None, layout=lay, data=BASE, data_bytes=N * STEP, n=N, outs=None, n_out=True, lidar=0):
        outs = outs if outs is not None else [BASE + (1 << 30) + k * (1 << 24) for k in range(5)]
        m = C.c_int64(7)
        st = L.lv_process_cloud_device(h, lidar, C.byref(layout) if layout is not None else None, data, data_bytes, n, 0, 1, 1, 0.1, 4,
                                       3.0, *outs, C.byref(m) if n_out else None)
        if n_out:
            assert m.value == 0
        return st, L.lv_last_error()
    return run


def test_null_handle_and_null_buffers(lv, call):
    assert call() == (lv.ERR_ARG, b"process cloud: null handle")
    for kw in (dict(layout=None), dict(data=None), dict(n_out=False)):
        st, msg = call(**kw)
        assert st == lv.ERR_ARG and b"null layout" in msg, kw
    for k in (0, 1):                                     # xyz, time
        outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
        outs[k] = None
        st, msg = call(outs=outs)
        assert st == lv.ERR_ARG and b"null layout" in msg, k
    outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
    outs[2:] = [None] * 3                                # intensity, range, idx are optional: past every check
    assert call(outs=outs) == (lv.ERR_ARG, b"process cloud: null handle")


def test_point_count_range(lv, call):
    for n in (-1, 0x80000000):
        st, msg = call(n=n, data_bytes=1 << 45)
        assert st == lv.ERR_ARG and b"int32" in msg, n
    assert call(n=0, data_bytes=0)[1] == b"process cloud: null handle"


def test_bad_layout(lv, call):
    cases = [(dict(off_time=STEP - 2), b"outside point_step"), (dict(off_x=-1), b"outside point_step"),
             (dict(point_step=0), b"point_step"), (dict(), b"too short")]
    for over, what in cases:
        lay = lv.CloudLayout(STEP, 0, 4, 8, 16, 22, 0)
        for k, v in over.items():
            setattr(lay, k, v)
        st, msg = call(layout=lay, data_bytes=N * STEP - (0 if over else 1))
        assert st == lv.ERR_ARG and what in msg, over
    st, msg = call(lidar=9)
    assert st == lv.ERR_ARG and b"LiDAR type" in msg
    # the ouster also reads its range field (4 bytes)
    st, msg = call(lidar=2, layout=lv.CloudLayout(STEP, 0, 4, 8, 12, 16, STEP - 3))
    assert st == lv.ERR_ARG and b"outside point_step" in msg


def test_overlapping_outputs(lv, call):
    nb = N * STEP
    for k, size in enumerate((12, 8, 4, 4, 4)):
        for start in (BASE + nb - 1, BASE - size * N + 1, BASE):
            outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
            outs[k] = start
            st, msg = call(outs=outs)
            assert st == lv.ERR_ARG and b"overlaps" in msg, (k, start)
        for start in (BASE + nb, BASE - size * N):       # adjacent ranges are fine
            outs = [BASE + (1 << 30) + j * (1 << 24) for j in range(5)]
            outs[k] = start
            assert call(outs=outs) == (lv.ERR_ARG, b"process cloud: null handle"), (k, start)
