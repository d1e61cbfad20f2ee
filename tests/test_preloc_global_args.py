"""lv_prelocalize_global's and lv_map_extent's argument refusals without a GPU: every refusal happens on the host before any
device work, so it is LV_ERR_ARG with a message naming the problem even with a null handle (the device pointer below is
never dereferenced)."""
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


def test_prelocalize_global_refusals(lv, L):
    res, stats = lv.PrelocResult(), lv.PrelocStats()

    def run(h=None, pts=BASE, n=1000, p=None, out=C.byref(res), st=C.byref(stats), **kw):
        prm = params(lv, **kw) if p is None else p
        return L.lv_prelocalize_global(h, pts, n, None if prm == "null" else C.byref(prm), out, st)

    assert run() == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"
    assert run(st=None) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"      # stats may be NULL
    assert run(n=1) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"
    assert run(n=0x7fffffff, max_points=4096) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"
    for kw in (dict(pts=None), dict(out=None), dict(p="null")):
        assert run(**kw) == lv.ERR_ARG and err(L) == b"prelocalize_global: null params, result or points", kw
    for n in (0, -1, 0x80000000):
        assert run(n=n) == lv.ERR_ARG and err(L) == b"prelocalize_global: n outside [1, 2^31 - 1]", n
    for radius in (-0.1, NAN, INF, -INF):
        assert run(radius=radius) == lv.ERR_ARG and err(L) == b"prelocalize_global: radius outside [0, inf)", radius
    for step in (0.0, -0.4, NAN, INF):
        assert run(step=step) == lv.ERR_ARG and err(L) == b"prelocalize_global: step not a positive finite number", step
    for yr in (-0.01, 3.1416, 4.0, NAN, INF):
        assert run(yaw_range=yr) == lv.ERR_ARG and err(L) == b"prelocalize_global: yaw_range outside [0, pi]", yr
    for ys in (0.0, -0.05, NAN, INF):
        assert run(yaw_step=ys) == lv.ERR_ARG and err(L) == b"prelocalize_global: yaw_step not a positive finite number", ys
    for mp in (0, -1, 4097):
        assert run(max_points=mp) == lv.ERR_ARG and err(L) == b"prelocalize_global: max_points outside [1, 4096]", mp
    for kw in (dict(radius=0.0), dict(yaw_range=0.0), dict(yaw_range=PI32), dict(max_points=1), dict(max_points=4096)):
        assert run(**kw) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle", kw
    # lv_prelocalize's cap of 2^24 does not apply: the whole 10 M-point SynthWorld from its centre at 0.4 m / 2 degrees
    assert lv.preloc_count(281.0, 0.4, PI32, math.radians(2.0)) > 1 << 24
    assert run(radius=281.0, step=0.4, yaw_range=PI32, yaw_step=math.radians(2.0)) == lv.ERR_ARG
    assert err(L) == b"prelocalize_global: null handle"
    # 2^40 at most: 1048575^2 = 2^40 - 2^21 + 1 passes, 1048577^2 is refused, so is a count far beyond it
    assert run(radius=524287.0, step=1.0, yaw_range=0.0) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"
    assert run(radius=524288.0, step=1.0, yaw_range=0.0) == lv.ERR_ARG
    assert err(L) == b"prelocalize_global: 1099513724929 candidates, more than 2^40"
    assert lv.preloc_count(524288.0, 1.0, 0.0, 1.0) == 1048577 ** 2 == 1099513724929
    assert run(radius=3000.0, step=0.1, yaw_range=PI32, yaw_step=0.01) == lv.ERR_ARG and b"more than 2^40" in err(L)
    assert run(radius=3e38, step=1e-30) == lv.ERR_ARG and err(L) == b"prelocalize_global: more than 2^61 candidates"
    # 2^20 headings at most (cells split positions, not headings): a heading grid lv_prelocalize accepts is refused here
    assert lv.preloc_count(0.0, 0.4, PI32, 5e-6) == 1256637 < 1 << 24
    assert run(radius=0.0, yaw_range=PI32, yaw_step=5e-6) == lv.ERR_ARG
    assert err(L) == b"prelocalize_global: 1256637 headings, more than 2^20"
    H = lv.preloc_count(0.0, 0.4, PI32, 6e-6)
    assert (1 << 19) < H < 1 << 20
    assert run(radius=0.0, yaw_range=PI32, yaw_step=6e-6) == lv.ERR_ARG and err(L) == b"prelocalize_global: null handle"


def test_top_level_is_bounded():
    """the top level of the cells returns for every window, also with more headings than the top-level cell budget"""
    import shim_binding
    S = shim_binding.lib()
    assert S.shim_pg_top_level(50, 100) == 5
    assert S.shim_pg_top_level(0, 600000) == 1               # 1 200 001 headings: one cell of one position each
    assert S.shim_pg_top_level(0, 0) == 1
    assert S.shim_pg_top_level(524287, 0) == 10              # 2^40 - 2^21 + 1 candidates: 1024 x 1024 cells of 1024^2
    for I, K in ((92, 90), (281, 90), (703, 90), (150, 90), (20000, 10)):
        L = S.shim_pg_top_level(I, K)
        C = (2 * I + 1 + (1 << L) - 1) >> L
        assert (2 * K + 1) * C * C <= 1 << 20 and L >= 1, (I, K, L)


def test_map_extent_refusals(lv, L):
    lo, hi = (C.c_double * 3)(), (C.c_double * 3)()
    assert L.lv_map_extent(None, lo, hi) == lv.ERR_ARG and err(L) == b"map_extent: null handle"
    assert L.lv_map_extent(None, None, hi) == lv.ERR_ARG and err(L) == b"map_extent: null handle"
