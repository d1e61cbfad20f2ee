"""The tick's output and mapping calls without a GPU: every argument refusal of lv_sweep_to_world_device_async and
lv_map_add_device_async happens on the host before any device call, so null pointers, a bound n_max outside [1, 2^31 - 1] and
ranges that overlap are LV_ERR_ARG with a message naming the problem even with a null handle (the device pointers below are never
dereferenced).  The bound against the handle's max_points needs a handle: tests/test_gpu_world_clouds.py covers it.

Also Mapper::hasToMap of the C++ facade (host/Modules.hpp), compiled on its own, against the reference's text (Mapper.cpp:58-61):

    bool Mapper::hasToMap(double t) {
        if (this->last_map_time < 0) this->last_map_time = t;
        return t - this->last_map_time >= Config.full_rotation_time;
    }

with Mapper::add setting last_map_time = time (Mapper.cpp:29)."""
import os
import subprocess

import numpy as np
import pytest

from test_async_tick_args import BASE, CNT, OUT, err

N = 1000
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def L(lv):
    return lv.lib()


def test_sweep_to_world_checks(lv, L):
    def run(h=None, xyz=BASE, d_n=CNT, n_max=N, out=OUT, n_out=CNT + 8):
        return L.lv_sweep_to_world_device_async(h, xyz, d_n, n_max, out, n_out)

    assert run() == lv.ERR_ARG and err(L) == b"sweep to world: null handle"
    assert run(n_max=1) == lv.ERR_ARG and err(L) == b"sweep to world: null handle"
    assert run(out=BASE) == lv.ERR_ARG and err(L) == b"sweep to world: null handle"          # in place is fine
    assert run(n_out=CNT) == lv.ERR_ARG and err(L) == b"sweep to world: null handle"         # so is the count in place
    for kw in (dict(xyz=None), dict(d_n=None), dict(out=None), dict(n_out=None)):
        assert run(**kw) == lv.ERR_ARG and b"null input, count, output or output count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max
    for kw in (dict(out=BASE + 12), dict(out=BASE - 12 * N + 4),                              # shifted outputs
               dict(n_out=BASE + 12 * N - 8), dict(n_out=OUT + 40), dict(n_out=OUT - 4),      # the count among the points
               dict(d_n=OUT + 12 * N - 4), dict(n_out=CNT + 4)):                               # the input count overwritten
        assert run(**kw) == lv.ERR_ARG and b"overlaps" in err(L), kw
    for kw in (dict(out=BASE + 12 * N), dict(out=BASE - 12 * N), dict(n_out=OUT + 12 * N), dict(n_out=OUT - 8),
               dict(d_n=BASE + 40)):                                                             # adjacent, or two inputs
        assert run(**kw) == lv.ERR_ARG and err(L) == b"sweep to world: null handle", kw


def test_map_add_async_checks(lv, L):
    def run(h=None, xyz=BASE, d_n=CNT, n_max=N, downsample=1):
        return L.lv_map_add_device_async(h, xyz, d_n, n_max, downsample)

    assert run() == lv.ERR_ARG and err(L) == b"map add async: null handle"
    assert run(downsample=0, n_max=1) == lv.ERR_ARG and err(L) == b"map add async: null handle"
    for kw in (dict(xyz=None), dict(d_n=None)):
        assert run(**kw) == lv.ERR_ARG and b"null points or count" in err(L), kw
    for n_max in (0, -1, 0x80000000):
        assert run(n_max=n_max) == lv.ERR_ARG and b"n_max outside" in err(L), n_max


# ---- Mapper::hasToMap --------------------------------------------------------------------------------------------------------------
class RefMapper:
    """Mapper.cpp:22-30 (last_map_time only) and :58-61, line for line"""

    def __init__(self, full_rotation_time):
        self.last_map_time = -1.0
        self.frt = full_rotation_time

    def add(self, time):
        self.last_map_time = time

    def hasToMap(self, t):
        if self.last_map_time < 0:
            self.last_map_time = t
        return t - self.last_map_time >= self.frt


FACADE = r"""
#include <stdio.h>
#include "Modules.hpp"
int main() {   /* reads "h <t> <frt>" (hasToMap) and "a <t>" (add) lines; prints the result and last_map_time, bit for bit */
    double last = -1, t, frt;
    char op;
    while (scanf(" %c %lf", &op, &t) == 2) {
        if (op == 'a') { last = t; continue; }
        if (scanf("%lf", &frt) != 1) return 1;
        const bool r = lv::Mapper::has_to_map(last, t, frt);
        printf("%d %a\n", r ? 1 : 0, last);
    }
    return 0;
}
"""


def test_has_to_map_follows_the_reference_text(tmp_path):
    src = tmp_path / "has_to_map.cpp"
    src.write_text(FACADE)
    exe = tmp_path / "has_to_map"
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-I" + os.path.join(ROOT, "limo-velo_b200", "host"), "-o", str(exe), str(src)])
    rng = np.random.default_rng(5)
    for frt in (0.1, 0.05, 0.0):
        ref, lines, want = RefMapper(frt), [], []
        t = 10.0
        for k in range(400):
            t = t + float(rng.choice([0.01, 0.02, 0.1, 0.0, frt, 0.03]))                 # ties at exactly full_rotation_time too
            if k % 3 == 2 and ref.hasToMap(t):                                          # the tick maps: Mapper::add(..., t2, ...)
                lines.append("h %r %r" % (t, frt))
                want.append("1 %s" % float.hex(ref.last_map_time))
                ref.add(t)
                lines.append("a %r" % t)
                continue
            if k % 3 == 2:
                lines.append("h %r %r" % (t, frt))
                want.append("0 %s" % float.hex(ref.last_map_time))
        got = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.split("\n")
        assert len(want) > 50 and "1" in {w[0] for w in want} and ("0" in {w[0] for w in want} or frt == 0.0), frt
        for g, w in zip(got, want):
            r, v = g.split()
            assert r == w.split()[0] and float.fromhex(v) == float.fromhex(w.split()[1]), (frt, g, w)
        assert len([g for g in got if g]) == len(want)
