"""PCD map files (lv_pcd_write / lv_pcd_read, host code, no GPU): the binary round trip bit for bit, files written here with
numpy in the layouts other tools write (extra fields, padding, NaN rows, comments, no COUNT line, ascii), and every refusal."""
import ctypes as C

import numpy as np
import pytest

HEADER = ("# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\n"
          "WIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")


@pytest.fixture
def L(lv):
    return lv.lib()


def special_points():
    v = np.array([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, -2.5e-40, 3e38, -3e38, 3.4028235e38, 1.0, -1.0, 123.456], np.float32)
    rng = np.random.default_rng(7)
    pts = np.concatenate([v.reshape(-1, 3), rng.normal(0, 100, (1000, 3)).astype(np.float32)])
    return np.ascontiguousarray(pts, np.float32)


def test_round_trip_bit_exact(lv, tmp_path):
    pts = special_points()
    path = tmp_path / "map.pcd"
    lv.pcd_write(path, pts)
    raw = path.read_bytes()
    hdr = HEADER.format(n=len(pts)).encode()
    assert raw[:len(hdr)] == hdr and len(raw) == len(hdr) + 12 * len(pts)
    back = lv.pcd_read(path)
    assert back.shape == pts.shape and back.view(np.uint32).tobytes() == pts.view(np.uint32).tobytes()
    lv.pcd_write(path, np.zeros((0, 3), np.float32))            # an empty map
    assert lv.pcd_read(path).shape == (0, 3)


def write_binary(path, rec, header_lines):
    path.write_bytes(("\n".join(header_lines) + "\n").encode() + rec.tobytes())


EXTRA = np.dtype([("intensity", "<f4"), ("x", "<f4"), ("rgb", "<u4"), ("y", "<f4"), ("timestamp", "<f8"), ("z", "<f4"),
                  ("_", "u1", (4,))])


def extra_records(n=500, seed=3):
    rng = np.random.default_rng(seed)
    rec = np.zeros(n, EXTRA)
    for f in ("x", "y", "z"):
        rec[f] = rng.uniform(-50, 50, n).astype(np.float32)
    rec["intensity"] = rng.uniform(0, 255, n)
    rec["rgb"] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    rec["timestamp"] = 1.7e9 + np.arange(n) * 1e-3
    rec["_"] = 0xAB
    rec["x"][[5, 27]] = np.nan                                  # NaN rows are dropped
    rec["z"][[40]] = np.inf
    keep = np.isfinite(rec["x"]) & np.isfinite(rec["y"]) & np.isfinite(rec["z"])
    want = np.stack([rec["x"][keep], rec["y"][keep], rec["z"][keep]], axis=1).astype(np.float32)
    return rec, want


def extra_header(n, data="binary", count=True, comments=True, version="0.7", points=None, width=None, height=1):
    lines = ["# .PCD v0.7 - written by numpy"] if comments else []
    lines += ["VERSION " + version, "FIELDS intensity x rgb y timestamp z _", "SIZE 4 4 4 4 8 4 1", "TYPE F F U F F F U"]
    if count:
        lines.append("COUNT 1 1 1 1 1 1 4")
    if comments:
        lines.append("# a comment between header lines")
    lines += ["WIDTH %d" % (n if width is None else width), "HEIGHT %d" % height, "VIEWPOINT 1 2 3 1 0 0 0",
              "POINTS %d" % (n if points is None else points), "DATA " + data]
    return lines


def test_binary_with_extra_fields(lv, tmp_path):
    rec, want = extra_records()
    p = tmp_path / "extra.pcd"
    write_binary(p, rec, extra_header(len(rec), version=".7"))
    got = lv.pcd_read(p)
    assert got.tobytes() == want.tobytes() and len(got) == len(rec) - 3


def test_missing_count_line(lv, tmp_path):
    dt = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4"), ("t", "<f8")])
    rec = np.zeros(64, dt)
    rec["x"], rec["y"], rec["z"] = np.arange(64), -np.arange(64), 0.5
    rec["y"][3] = np.nan
    p = tmp_path / "nocount.pcd"
    write_binary(p, rec, ["VERSION 0.7", "FIELDS x y z intensity t", "SIZE 4 4 4 4 8", "TYPE F F F F F", "WIDTH 8", "HEIGHT 8",
                          "VIEWPOINT 0 0 0 1 0 0 0", "POINTS 64", "DATA binary"])
    got = lv.pcd_read(p)
    keep = np.arange(64) != 3
    assert got.tobytes() == np.stack([rec["x"], rec["y"], rec["z"]], 1)[keep].astype(np.float32).tobytes()


def test_ascii(lv, tmp_path):
    rec, want = extra_records(200, seed=9)
    lines = extra_header(len(rec), data="ascii")
    body = []
    for r in rec:
        vals = ["%.9g" % r["intensity"], "%.9g" % r["x"], "%d" % r["rgb"], "%.9g" % r["y"], "%.17g" % r["timestamp"], "%.9g" % r["z"]]
        vals += ["%d" % b for b in r["_"]]
        body.append(" ".join(vals))
    p = tmp_path / "ascii.pcd"
    p.write_text("\n".join(lines) + "\n" + "\n".join(body) + "\n")
    got = lv.pcd_read(p)
    assert got.tobytes() == want.tobytes()


def test_count_only_and_capacity(lv, L, tmp_path):
    pts = special_points()
    p = str(tmp_path / "m.pcd").encode()
    lv.pcd_write(tmp_path / "m.pcd", pts)
    n = C.c_int64(-1)
    assert L.lv_pcd_read(p, None, 0, C.byref(n)) == lv.OK and n.value == len(pts)
    out = np.full((len(pts), 3), 7.0, np.float32)
    assert L.lv_pcd_read(p, out.ctypes.data_as(C.POINTER(C.c_float)), len(pts) - 1, C.byref(n)) == lv.ERR_CAPACITY
    assert n.value == len(pts) and np.all(out == 7.0)
    assert b"more than cap" in L.lv_last_error()


def refusal(lv, L, path):
    n = C.c_int64(0)
    st = L.lv_pcd_read(str(path).encode(), None, 0, C.byref(n))
    return st, L.lv_last_error()


def test_refusals(lv, L, tmp_path):
    rec, _ = extra_records(50)
    cases = {
        "compressed": (extra_header(50, data="binary_compressed"), b"pcl_convert_pcd_ascii_binary"),
        "points": (extra_header(50, points=49), b"POINTS 49 != WIDTH x HEIGHT 50"),
        "short": (extra_header(50, width=60, points=60), b"data section holds 50 of 60 POINTS records"),
    }
    for name, (hdr, msg) in cases.items():
        p = tmp_path / (name + ".pcd")
        write_binary(p, rec, hdr)
        st, e = refusal(lv, L, p)
        assert st == lv.ERR_IO and msg in e, (name, e)
    # a missing or ill-typed coordinate field
    base = ["VERSION 0.7", "WIDTH 2", "HEIGHT 1", "POINTS 2", "DATA binary"]
    for fields, msg in ((["FIELDS x y", "SIZE 4 4", "TYPE F F"], b"no x, y and z fields"),
                        (["FIELDS x y z", "SIZE 4 4 8", "TYPE F F F"], b"field z is not TYPE F, SIZE 4, COUNT 1"),
                        (["FIELDS x y z", "SIZE 4 4 4", "TYPE F U F"], b"field y is not TYPE F, SIZE 4, COUNT 1"),
                        (["FIELDS x y z", "SIZE 4 4 4", "TYPE F F F", "COUNT 2 1 1"], b"field x is not TYPE F, SIZE 4, COUNT 1")):
        p = tmp_path / "bad.pcd"
        p.write_bytes(("\n".join(base[:1] + fields + base[1:]) + "\n").encode() + bytes(64))
        st, e = refusal(lv, L, p)
        assert st == lv.ERR_IO and msg in e, (fields, e)
    # an ascii file that ends early
    p = tmp_path / "short.pcd"
    p.write_text("VERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nWIDTH 3\nHEIGHT 1\nPOINTS 3\nDATA ascii\n1 2 3\n4 5 6\n")
    st, e = refusal(lv, L, p)
    assert st == lv.ERR_IO and b"data section holds 2 of 3 POINTS records" in e
    # an unreadable file
    st, e = refusal(lv, L, tmp_path / "does_not_exist.pcd")
    assert st == lv.ERR_IO and b"cannot read" in e
    # a failed open for writing
    pts = np.zeros((1, 3), np.float32)
    assert L.lv_pcd_write(str(tmp_path / "no_dir" / "m.pcd").encode(), pts.ctypes.data_as(C.POINTER(C.c_float)), 1) == lv.ERR_IO
    assert b"cannot open" in L.lv_last_error()
    assert L.lv_pcd_write(None, None, 0) == lv.ERR_ARG
