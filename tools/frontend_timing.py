"""Accumulator::process (decode -> decimate -> time sort) on the host versus lv_process_cloud_device, at the cfg1 shape
(Velodyne 64 x 1024, point_step 32) and the cfg3 shape (Ouster 128 x 2048, point_step 48), rate 4, min_dist 3:

  (a) the host front end of INTEGRATION.md B4: lv_pointcloud2_to_points_checked, lv_temporal_downsample, lv_time_sort_indices,
      the index gathers and the upload of xyz / time that lv_compensate_device needs; host clock ending in a synchronise
  (b) lv_memcpy_h2d of the raw bytes from a pinned buffer + lv_process_cloud_device; host clock ending in a synchronise
  (c) lv_process_cloud_device alone, bytes resident: CUDA events around the call on the handle's stream (the end event is
      recorded after the call's final synchronise returns, so this includes that wake-up), and the kernel + copy time of
      one call from a torch.profiler trace (written to OUT/frontend_trace_<shape>.json)

Median of --runs runs after --warmup; the card's name and power limit and the host CPU are read in the same run.  Prints
one JSON line per shape and writes them to OUT/frontend_timing.json.
    python tools/frontend_timing.py [--runs 50] [--warmup 10] [--out DIR]   (DIR defaults to <tmp>/frontend_timing)
"""
import argparse
import ctypes as C
import json
import os
import platform
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as G  # noqa: E402

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
VELO = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                 "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "<u1", "<u2", "<u4"],
                   "offsets": [0, 4, 8, 16, 20, 24, 26, 28, 32], "itemsize": 48})
SHAPES = {"cfg1_velodyne_64x1024": ("velodyne", VELO, 64, 1024), "cfg3_ouster_128x2048": ("ouster", OUSTER, 128, 2048)}
RATE, MIN_DIST, STAMP_US = 4, 3.0, 1_695_000_000_350_000


def cloud(lidar, dtype, rings, cols, seed=1):
    """a sweep in the driver's column-major firing order: one time per column"""
    rng = np.random.default_rng(seed)
    n = rings * cols
    p = np.zeros(n, dtype)
    r = rng.uniform(1.0, 80.0, n)
    az = np.repeat(np.linspace(0, 2 * np.pi, cols, endpoint=False), rings)
    el = np.tile(np.linspace(-0.4, 0.1, rings), cols)
    p["x"], p["y"], p["z"] = r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)
    p["ring"] = np.tile(np.arange(rings), cols)
    if lidar == "velodyne":
        p["time"] = np.repeat(np.linspace(0, 0.1, cols, endpoint=False), rings).astype(np.float32)
        p["intensity"] = rng.uniform(0, 255, n)
    else:
        p["t"] = np.repeat(np.arange(cols) * (100_000_000 // cols), rings).astype(np.uint32)
        p["reflectivity"] = rng.integers(0, 60000, n)
        p["range"] = (r * 1000).astype(np.uint32)
    return p


def med(xs):
    return float(np.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frontend_timing"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("frontend_timing: no CUDA device (there is nothing to measure without one)")
    os.makedirs(a.out, exist_ok=True)
    lv = G.load_package()
    L = lv.lib()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    cpu = next((ln.split(":", 1)[1].strip() for ln in open("/proc/cpuinfo") if ln.startswith("model name")), "")
    if cpu in ("", "unknown"):
        cpu = next((ln.split(":", 1)[1].strip() for ln in subprocess.run(["lscpu"], capture_output=True, text=True).stdout.splitlines()
                    if ln.startswith(("Model name", "Vendor ID"))), platform.processor() or "not reported")
    stream = torch.cuda.Stream()
    prm = lv.default_params(max_points=1 << 19, max_map_points=1 << 16)
    prm.stream = stream.cuda_stream
    loc = lv.Localizer(prm)
    fp, dp, i32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
    results = []
    for name, (lidar, dtype, rings, cols) in SHAPES.items():
        pts = cloud(lidar, dtype, rings, cols)
        n, nb, step = len(pts), pts.nbytes, dtype.itemsize
        lay = lv.cloud_layout(lidar, dtype)
        ltype = lv.LIDAR_TYPES[lidar]
        pinned = L.lv_host_alloc(nb)
        C.memmove(pinned, pts.ctypes.data, nb)
        d_msg = loc.device_alloc(nb)
        d_out = [loc.device_alloc(k * n) for k in (12, 8, 4, 4, 4)]
        d_up = [loc.device_alloc(12 * n), loc.device_alloc(8 * n)]
        xyz, t, inten, rng_ = np.empty((n, 3), np.float32), np.empty(n), np.empty(n, np.float32), np.empty(n, np.float32)
        ds_xyz, ds_idx, m = np.empty((n, 3), np.float32), np.empty(n, np.int32), C.c_int64(0)
        raw = pts.ctypes.data_as(C.POINTER(C.c_uint8))

        def host_front_end():
            lv._check(L.lv_pointcloud2_to_points_checked(ltype, C.byref(lay), raw, C.c_int64(nb), C.c_int64(n), C.c_uint64(STAMP_US), 0, 1,
                                                         C.c_double(0.1), xyz.ctypes.data_as(fp), t.ctypes.data_as(dp),
                                                         inten.ctypes.data_as(fp), rng_.ctypes.data_as(fp)))
            lv._check(L.lv_temporal_downsample(loc.h, xyz.ctypes.data_as(fp), C.c_int64(n), C.c_int32(RATE), C.c_double(MIN_DIST),
                                               ds_xyz.ctypes.data_as(fp), ds_idx.ctypes.data_as(i32p), C.byref(m)))
            k = m.value
            idx = ds_idx[:k]
            tk = np.ascontiguousarray(t[idx])
            order = np.empty(k, np.int32)
            lv._check(L.lv_time_sort_indices(tk.ctypes.data_as(dp), C.c_int64(k), order.ctypes.data_as(i32p)))
            sx, st = np.ascontiguousarray(ds_xyz[order]), np.ascontiguousarray(tk[order])
            _ = inten[idx][order], rng_[idx][order], idx[order]              # what rides along for the caller
            lv._check(L.lv_memcpy_h2d(loc.h, C.c_void_p(d_up[0]), sx.ctypes.data_as(C.c_void_p), sx.nbytes))
            lv._check(L.lv_memcpy_h2d(loc.h, C.c_void_p(d_up[1]), st.ctypes.data_as(C.c_void_p), st.nbytes))
            return k

        def device_call():
            return loc.process_cloud_device(lidar, lay, d_msg, nb, n, STAMP_US, 0, 1, 0.1, RATE, MIN_DIST, *d_out)

        def upload_and_process():
            lv._check(L.lv_memcpy_h2d(loc.h, C.c_void_p(d_msg), C.c_void_p(pinned), nb))
            return device_call()

        k_host = host_front_end()
        k_dev = upload_and_process()
        got_t = loc.download(d_out[1], np.empty(k_dev))
        assert k_host == k_dev and (got_t.view(np.uint64) == np.sort(t[ds_idx[:k_host]], kind="stable").view(np.uint64)).all()
        ta, tb, tc = [], [], []
        for i in range(a.warmup + a.runs):
            t0 = time.perf_counter(); host_front_end(); t1 = time.perf_counter()
            upload_and_process(); t2 = time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream); device_call(); e1.record(stream); e1.synchronize()
            if i >= a.warmup:
                ta.append((t1 - t0) * 1e3); tb.append((t2 - t1) * 1e3); tc.append(e0.elapsed_time(e1))
        # one profiled pass: where the device time of a call goes
        trace = os.path.join(a.out, "frontend_trace_%s.json" % name)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
            for _ in range(5):
                upload_and_process()
        prof.export_chrome_trace(trace)
        ev = [e for e in json.load(open(trace))["traceEvents"] if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
        per = {}
        for e in ev:
            key = e["name"][:60]
            per[key] = per.get(key, 0.0) + e["dur"] / 5.0
        kern_us = sum(v for kk, v in per.items() if not kk.startswith("Memcpy"))
        out_bytes = 32 * k_dev                       # xyz 12, time 8, intensity 4, range 4, index 4 per kept point
        bound_us = (nb + out_bytes) / HBM_BYTES_PER_S * 1e6
        r = dict(shape=name, n=n, point_step=step, kept=k_dev, card=card, host_cpu=cpu, runs=a.runs,
                 a_host_front_end_ms=med(ta), b_upload_plus_device_ms=med(tb), c_device_call_events_ms=med(tc),
                 c_kernels_per_call_us=kern_us, device_time_per_call_us=dict(sorted(per.items(), key=lambda kv: -kv[1])),
                 message_bytes_per_point=step, output_bytes_per_point=out_bytes / n,
                 hbm_bound_us=bound_us, kernels_over_hbm_bound=kern_us / bound_us,
                 spread_ms=dict(a=[float(np.percentile(ta, 10)), float(np.percentile(ta, 90))],
                                b=[float(np.percentile(tb, 10)), float(np.percentile(tb, 90))],
                                c=[float(np.percentile(tc, 10)), float(np.percentile(tc, 90))]))
        print(json.dumps(r), flush=True)
        results.append(r)
        for d in [d_msg] + d_out + d_up:
            loc.device_free(d)
        L.lv_host_free(pinned)
    loc.close()
    json.dump(results, open(os.path.join(a.out, "frontend_timing.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
