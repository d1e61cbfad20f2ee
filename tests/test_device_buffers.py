"""The buffer and event owners of lv_buffers.h, built with g++ against a fake CUDA runtime (tests/cpu_shim/buffers.cpp), and the
rule that keeps raw allocations out of the context code.

The fake counts live allocations, flags a free of a pointer it does not hold, and fails the k-th allocation on request, so the
failure paths run here without ever exhausting a device."""
import ctypes as C
import os
import re

import pytest

import shim_binding as S

ERR_ALLOC = 2            # cudaErrorMemoryAllocation
DEVICE, PINNED = 0, 1


def counts():
    out = (C.c_int64 * 7)()
    S.lib().shim_buf_counts(out)
    return dict(zip(("device", "pinned", "events", "allocs", "frees", "foreign", "last_error"), out))


class Buf:
    def __init__(self, kind=DEVICE, h=None):
        self.L = S.lib()
        self.h = h if h is not None else self.L.shim_buf_new(kind)

    def reserve(self, n):
        return self.L.shim_buf_reserve(self.h, n)

    def size(self):
        return self.L.shim_buf_size(self.h)

    def ptr(self):
        return self.L.shim_buf_ptr(self.h)

    def delete(self):
        self.L.shim_buf_delete(self.h)


@pytest.fixture(autouse=True)
def nothing_leaks():
    """every scenario ends with nothing live, no foreign or double free and no pending error"""
    S.lib().shim_buf_fail_at(0)
    before = counts()
    assert before["device"] == before["pinned"] == before["events"] == 0
    yield
    S.lib().shim_buf_fail_at(0)
    after = counts()
    assert after["device"] == after["pinned"] == after["events"] == 0
    assert after["foreign"] == before["foreign"]
    assert after["last_error"] == 0


@pytest.mark.parametrize("kind", [DEVICE, PINNED])
def test_reserve_grows_only(kind):
    b = Buf(kind)
    assert b.size() == 0 and b.ptr() == 0
    c0 = counts()
    assert b.reserve(10) == 0
    p = b.ptr()
    assert p != 0 and b.size() == 10
    assert counts()["allocs"] == c0["allocs"] + 1
    for n in (0, 5, 10):                                  # fits: neither freed nor allocated
        assert b.reserve(n) == 0
        assert b.ptr() == p and b.size() == 10
    c1 = counts()
    assert (c1["allocs"], c1["frees"]) == (c0["allocs"] + 1, c0["frees"])
    assert b.reserve(11) == 0                             # grows: one free, then one allocation of exactly n
    c2 = counts()
    assert (c2["allocs"], c2["frees"]) == (c1["allocs"] + 1, c1["frees"] + 1)
    assert b.size() == 11 and b.ptr() != 0
    S.lib().shim_buf_reset(b.h)
    assert b.size() == 0 and b.ptr() == 0
    assert counts()["frees"] == c2["frees"] + 1
    b.delete()                                            # an empty owner frees nothing
    assert counts()["frees"] == c2["frees"] + 1


# the lazily allocated pairs of a context (d_path / h_path, d_imu / h_imu, ...): reserved one by one, each checked
SEQUENCE = [(DEVICE, 4), (PINNED, 4), (DEVICE, 1), (PINNED, 1), (DEVICE, 9)]


@pytest.mark.parametrize("k", range(1, len(SEQUENCE) + 1))
def test_failure_at_every_allocation_is_retried(k):
    bufs = [Buf(kind) for kind, _ in SEQUENCE]

    def run():
        for i, (b, (_, n)) in enumerate(zip(bufs, SEQUENCE)):
            e = b.reserve(n)
            if e:
                return i, e
        return None, 0

    S.lib().shim_buf_fail_at(k)
    failed, e = run()
    assert (failed, e) == (k - 1, ERR_ALLOC)
    assert counts()["last_error"] == 0                    # cleared: a later launcher does not report it
    for i, (b, (_, n)) in enumerate(zip(bufs, SEQUENCE)):
        assert (b.size(), b.ptr() != 0) == ((n, True) if i < k - 1 else (0, False))
    held = [b.ptr() for b in bufs[:k - 1]]
    c0 = counts()
    assert run() == (None, 0)                             # the next call allocates what is missing, and only that
    assert counts()["allocs"] == c0["allocs"] + len(SEQUENCE) - (k - 1)
    assert [b.ptr() for b in bufs[:k - 1]] == held
    assert all(b.size() == n for b, (_, n) in zip(bufs, SEQUENCE))
    for b in bufs:
        b.delete()


@pytest.mark.parametrize("kind", [DEVICE, PINNED])
def test_failed_growth_leaves_the_owner_empty(kind):
    b = Buf(kind)
    assert b.reserve(8) == 0
    c0 = counts()
    S.lib().shim_buf_fail_at(1)
    assert b.reserve(16) == ERR_ALLOC
    c1 = counts()
    assert b.size() == 0 and b.ptr() == 0                 # neither the freed pointer nor the old size survives
    assert c1["frees"] == c0["frees"] + 1 and c1["last_error"] == 0
    assert b.reserve(8) == 0 and b.size() == 8            # not "fits": allocated again
    assert counts()["allocs"] == c1["allocs"] + 1
    b.delete()


@pytest.mark.parametrize("kind", [DEVICE, PINNED])
def test_move_transfers_ownership(kind):
    L = S.lib()
    a = Buf(kind)
    assert a.reserve(7) == 0
    p = a.ptr()
    b = Buf(h=L.shim_buf_move_new(a.h))                   # move construction
    assert (b.ptr(), b.size()) == (p, 7) and (a.ptr(), a.size()) == (0, 0)
    c = Buf(kind)
    assert c.reserve(3) == 0
    c0 = counts()
    L.shim_buf_move_assign(c.h, b.h)                      # move assignment frees what c held
    assert (c.ptr(), c.size()) == (p, 7) and (b.ptr(), b.size()) == (0, 0)
    assert counts()["frees"] == c0["frees"] + 1
    L.shim_buf_move_assign(c.h, c.h)                      # self-assignment keeps the buffer
    assert (c.ptr(), c.size()) == (p, 7)
    for o in (a, b):
        o.delete()
    assert counts()["frees"] == c0["frees"] + 1
    c.delete()
    assert counts()["frees"] == c0["frees"] + 2


def test_event_created_once_destroyed_once():
    L = S.lib()
    e = L.shim_event_new()
    c0 = counts()
    S.lib().shim_buf_fail_at(1)
    assert L.shim_event_create(e) == ERR_ALLOC
    assert not L.shim_event_handle(e) and counts()["last_error"] == 0
    assert L.shim_event_create(e) == 0                    # retried
    h = L.shim_event_handle(e)
    assert h and counts()["events"] == 1
    assert L.shim_event_create(e) == 0 and L.shim_event_handle(e) == h
    assert counts()["allocs"] == c0["allocs"] + 2
    L.shim_event_delete(e)
    assert counts()["events"] == 0 and counts()["frees"] == c0["frees"] + 1
    L.shim_event_delete(L.shim_event_new())               # never created: nothing destroyed
    assert counts()["frees"] == c0["frees"] + 1


# ---- the sources: raw allocations only where no owner can hold them ------------------------------------------------------
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "limo-velo_b200", "csrc")
RAW = re.compile(r"\b(cudaMallocHost|cudaMalloc|cudaFreeHost|cudaFree|cudaEventCreate\w*|cudaEventDestroy)\s*\(")
# the caller-owned allocations of the C ABI, the profiling event pool, and the map's counters (the rest of the map is
# stream-ordered, allocated with cudaMallocAsync)
ALLOWED = {("lv_host_alloc", "cudaMallocHost"), ("lv_host_free", "cudaFreeHost"), ("lv_device_alloc", "cudaMalloc"),
           ("lv_device_free", "cudaFree"), ("prof_begin", "cudaEventCreate"), ("~lv_context", "cudaEventDestroy"),
           ("map_alloc", "cudaMalloc"), ("map_alloc", "cudaMallocHost"), ("map_free", "cudaFree"), ("map_free", "cudaFreeHost")}


def _strip(src):
    """the code without comments, string and character literals and preprocessor lines"""
    src = re.sub(r"/\*.*?\*/|//[^\n]*|\"(?:\\.|[^\"\\\n])*\"|'(?:\\.|[^'\\\n])*'",
                 lambda m: '""' if m.group(0)[0] == '"' else ("' '" if m.group(0)[0] == "'" else " "), src, flags=re.S)
    return re.sub(r"^[ \t]*#(?:[^\n]*\\\n)*[^\n]*", "", src, flags=re.M)


def _functions(code, start=0, end=None):
    """(name, body) of every function defined in code[start:end], inside namespaces, extern "C" blocks and classes too"""
    end = len(code) if end is None else end
    depth, head = 0, start
    for i in range(start, end):
        c = code[i]
        if c == "{":
            if depth == 0:
                header, open_at = code[head:i], i
            depth += 1
        elif c == "}":
            depth -= 1
            if depth == 0:
                close = header.rfind(")")
                if close < 0:                                    # a namespace, class or initializer: look inside
                    yield from _functions(code, open_at + 1, i)
                else:                                            # the name before the last parameter list
                    level, j = 0, close
                    while True:
                        level += {")": 1, "(": -1}.get(header[j], 0)
                        if level == 0:
                            break
                        j -= 1
                    yield re.search(r"(~?\w+)\s*$", header[:j]).group(1), code[open_at:i + 1]
                head = i + 1
        elif c == ";" and depth == 0:
            head = i + 1


def test_raw_allocations_only_outside_the_owners():
    found = set()
    names = set()
    for f in ("lv_capi.cu", "lv_downsample.cu", "lv_lidar_buffer.cu", "lv_map.cu"):
        code = _strip(open(os.path.join(CSRC, f)).read())
        calls = [m.group(1) for m in RAW.finditer(code)]
        in_functions = 0
        for name, body in _functions(code):
            names.add(name)
            for m in RAW.finditer(body):
                kind = "cudaEventCreate" if m.group(1).startswith("cudaEventCreate") else m.group(1)
                in_functions += 1
                found.add((name, kind))
                assert (name, kind) in ALLOWED, "%s: %s calls %s: hold the allocation in a DeviceBuf / PinnedBuf / Event" % (
                    f, name, m.group(1))
        assert in_functions == len(calls), "%s: a raw call outside every function" % f
    assert {"create_buffers", "lidar_resize", "ds_reserve", "map_points_sorted", "~lv_context"} <= names
    assert found == ALLOWED
