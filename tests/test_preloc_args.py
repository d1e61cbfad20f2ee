"""lv_prelocalize's argument refusals and lv_preloc_count without a GPU: every refusal happens on the host before any device
work, so it is LV_ERR_ARG with a message naming the problem even with a null handle (the device pointer below is never
dereferenced)."""
import ctypes as C
import math

import numpy as np
import pytest

from test_async_tick_args import BASE, err

NAN, INF = float("nan"), float("inf")
PI32 = float(np.float32(math.pi))


@pytest.fixture
def L(lv):
    return lv.lib()


def params(lv, radius=2.0, step=0.4, yaw_range=0.5, yaw_step=0.05, max_points=2048):
    return lv.PrelocParams(radius, step, yaw_range, yaw_step, max_points, 0)


def formula(radius, step, yaw_range, yaw_step):
    f = lambda v: float(np.float32(v))
    I = math.floor(f(radius) / f(step) + 1e-9)
    K = math.floor(f(yaw_range) / f(yaw_step) + 1e-9)
    return (2 * K + 1) * (2 * I + 1) ** 2


def test_prelocalize_refusals(lv, L):
    res = lv.PrelocResult()

    def run(h=None, pts=BASE, n=1000, p=None, out=C.byref(res), scores=None, **kw):
        prm = params(lv, **kw) if p is None else p
        return L.lv_prelocalize(h, pts, n, None if prm == "null" else C.byref(prm), out, scores)

    assert run() == lv.ERR_ARG and err(L) == b"prelocalize: null handle"
    assert run(n=1) == lv.ERR_ARG and err(L) == b"prelocalize: null handle"
    assert run(n=0x7fffffff, max_points=4096) == lv.ERR_ARG and err(L) == b"prelocalize: null handle"
    for kw in (dict(pts=None), dict(out=None), dict(p="null")):
        assert run(**kw) == lv.ERR_ARG and err(L) == b"prelocalize: null params, result or points", kw
    for n in (0, -1, 0x80000000):
        assert run(n=n) == lv.ERR_ARG and err(L) == b"prelocalize: n outside [1, 2^31 - 1]", n
    for radius in (-0.1, NAN, INF, -INF):
        assert run(radius=radius) == lv.ERR_ARG and err(L) == b"prelocalize: radius outside [0, inf)", radius
    for step in (0.0, -0.4, NAN, INF):
        assert run(step=step) == lv.ERR_ARG and err(L) == b"prelocalize: step not a positive finite number", step
    for yr in (-0.01, 3.1416, 4.0, NAN, INF):
        assert run(yaw_range=yr) == lv.ERR_ARG and err(L) == b"prelocalize: yaw_range outside [0, pi]", yr
    for ys in (0.0, -0.05, NAN, INF):
        assert run(yaw_step=ys) == lv.ERR_ARG and err(L) == b"prelocalize: yaw_step not a positive finite number", ys
    for mp in (0, -1, 4097):
        assert run(max_points=mp) == lv.ERR_ARG and err(L) == b"prelocalize: max_points outside [1, 4096]", mp
    # the edges that are accepted: radius 0, yaw_range 0 and pi (as a float), one point, 4096 points
    for kw in (dict(radius=0.0), dict(yaw_range=0.0), dict(yaw_range=PI32), dict(max_points=1), dict(max_points=4096)):
        assert run(**kw) == lv.ERR_ARG and err(L) == b"prelocalize: null handle", kw
    # 2^24 candidates at most: 4095^2 passes, 4097^2 = 16785409 is refused
    assert run(radius=2047.0, step=1.0, yaw_range=0.0) == lv.ERR_ARG and err(L) == b"prelocalize: null handle"
    assert run(radius=2048.0, step=1.0, yaw_range=0.0) == lv.ERR_ARG
    assert err(L) == b"prelocalize: 16785409 candidates, more than 2^24"
    assert run(radius=5.0, step=0.4, yaw_range=PI32, yaw_step=1e-4) == lv.ERR_ARG and b"more than 2^24" in err(L)


@pytest.mark.parametrize("radius,step,yaw_range,yaw_step", [
    (0.0, 0.4, 0.5, 0.05),               # radius 0: one position
    (2.0, 0.5, 0.5, 0.05),               # an exact multiple: I = 4
    (1.0, 0.25, 0.5, 0.125),             # exact multiples on both axes
    (1.2, 0.4, 0.35, 0.07),              # not exact in fp32: 1.2f / 0.4f is just above 3
    (5.0, 0.4, PI32, math.radians(2)),   # the recommended window
    (5.0, 0.4, 0.0, 0.1),                # yaw_range 0: one heading
    (0.1, 0.4, PI32, 0.01),              # step above the radius
    (2048.0, 1.0, 0.0, 1.0),             # just over 2^24: counted, refused by lv_prelocalize
    (2047.0, 1.0, 0.0, 1.0),             # just under
])
def test_preloc_count_formula(lv, radius, step, yaw_range, yaw_step):
    assert lv.preloc_count(radius, step, yaw_range, yaw_step) == formula(radius, step, yaw_range, yaw_step)


def test_preloc_count_values(lv):
    assert lv.preloc_count(0.0, 0.4, 0.0, 0.1) == 1
    assert lv.preloc_count(2.0, 0.5, 0.0, 0.1) == 81
    assert lv.preloc_count(2.0, 0.5, 0.5, 0.125) == 9 * 81
    assert lv.preloc_count(1.2, 0.4, 0.0, 0.1) == 49          # 1.2f / 0.4f = 3.00000007: I = 3
    assert lv.preloc_count(1.0, 0.1, 0.0, 0.1) == 361         # 1.0f / 0.1f = 9.99999985: I = 9, not 10
    assert lv.preloc_count(5.0, 0.4, PI32, math.radians(2)) == 181 * 625
    assert lv.preloc_count(2048.0, 1.0, 0.0, 1.0) == 4097 ** 2 == (1 << 24) + 8193


def test_preloc_count_invalid(lv, L):
    assert L.lv_preloc_count(None) == -1
    for kw in (dict(radius=-1.0), dict(radius=NAN), dict(step=0.0), dict(step=INF), dict(yaw_range=3.2), dict(yaw_range=-0.1),
               dict(yaw_step=0.0), dict(yaw_step=NAN), dict(max_points=0), dict(max_points=4097)):
        p = params(lv, **kw)
        assert L.lv_preloc_count(C.byref(p)) == -1, kw
    assert lv.preloc_count(3e38, 1e-30, 0.0, 1.0) == -1         # beyond 2^61
