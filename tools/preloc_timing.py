"""Cost of starting a sequence in a saved map on one GPU: lv_prelocalize at the recommended window, and lv_pcd_read +
lv_map_build, on SynthWorld maps of 1 M and 10 M points.

    python tools/preloc_timing.py [--sizes 1000000,10000000] [--reps 25] [--json OUT]

lv_prelocalize synchronises, so its time is the wall time of the call (host frames and offsets, two small uploads, the kernel,
the winner's read-back), the median of --reps calls after two warm-up calls, without and with the scores array.  probes/s =
candidates x scored points / time.  The load is split into the file read (lv_pcd_read into host memory), the upload
(lv_memcpy_h2d) and the build (lv_map_build_device, then lv_synchronize).  The PCD file goes to a temporary directory.  The
card's name, power limit and maximum SM clock are read with `nvidia-smi --query-gpu` in the same run; nothing is changed on
the device.
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "nvidia-smi: no output"
    except Exception as e:
        return "nvidia-smi unavailable (%s)" % e


def median_ms(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(t), min(t), max(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--reps", type=int, default=25)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    lv = G.load_package()
    rec = dict(radius=5.0, step=0.4, yaw_range=float(np.float32(math.pi)), yaw_step=math.radians(2.0), max_points=2048)
    res = dict(gpu=gpu_info(), window=rec, candidates=lv.preloc_count(**rec), sizes=[])
    print("gpu:", res["gpu"], " window:", rec, " candidates:", res["candidates"], flush=True)
    for m in [int(s) for s in a.sizes.split(",")]:
        prm = lv.params_from_yaml(os.path.join(lv.CONFIG_DIR, "xaloc.yaml"), max_map_points=m + (m >> 4), max_points=1 << 15)
        world = lv.SynthWorld(20261016, m)
        mp = world.map()
        truth = world.pose(60.0, prm)
        sweep = world.sweep(truth, rings=32, azimuths=256, elev=(-10.0, 15.0), seed=3)
        loc = lv.Localizer(prm)
        row = dict(map_points=len(mp))
        try:
            with tempfile.TemporaryDirectory() as td:
                path = os.path.join(td, "map.pcd")
                t0 = time.perf_counter()
                lv.pcd_write(path, mp)
                row["pcd_write_ms"] = (time.perf_counter() - t0) * 1e3
                L = lv.lib()
                n = C.c_int64(0)
                host = np.zeros((len(mp), 3), np.float32)

                def read():
                    st = L.lv_pcd_read(path.encode(), host.ctypes.data_as(C.POINTER(C.c_float)), len(host), C.byref(n))
                    assert st == lv.OK and n.value == len(mp)
                row["pcd_read_ms"] = median_ms(read, 5, warm=1)
            d_map = loc.device_alloc(host.nbytes)

            def upload():
                assert L.lv_memcpy_h2d(loc.h, d_map, host.ctypes.data_as(C.c_void_p), host.nbytes) == lv.OK
            row["upload_ms"] = median_ms(upload, 5, warm=1)

            def build():
                assert L.lv_map_build_device(loc.h, C.c_void_p(d_map), len(host)) == lv.OK
                loc.synchronize()
            row["build_ms"] = median_ms(build, 5, warm=1)
            row["map_bytes"] = loc.map_info()["bytes"]
            loc.init_state()
            x0, P0 = loc.get_state()
            d = loc.upload(np.ascontiguousarray(sweep, np.float32))
            for scores in (False, True):
                def call():
                    loc.set_state(truth, P0)
                    st, out = loc.prelocalize(d, len(sweep), scores=scores, **rec)
                    assert st == lv.OK
                t = median_ms(call, a.reps)
                key = "prelocalize_scores_ms" if scores else "prelocalize_ms"
                row[key] = t
                row[key.replace("_ms", "_probes_per_s")] = res["candidates"] * rec["max_points"] / (t[0] * 1e-3)
            loc.device_free(d)
            loc.device_free(d_map)
        finally:
            loc.close()
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
