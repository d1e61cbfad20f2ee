"""Device time per call of the Ouster packet front end (lv_process_ouster_packets_device_async) on the packets of one lidar UDP
profile (--profile, LEGACY by default) against the PointCloud2 front end
(lv_process_cloud_device_async, os_cloud_node's layout of 48 bytes per point) on the same points: one OS1-64 1024x10 frame (64
packets, 65 536 slots), one OS1-128 2048x10 frame (128 packets, 262 144 slots), and a single OS1-64 packet (the per-call fixed cost
that makes batching the packets of a frame worth it).  10 % of the pixels without a return, rate 4, min_dist 3, the message bytes
resident in HBM.  The PointCloud2 holds the points the packets decode to, in slot order, with t = column time - the first point's
column time.  The packets of the other profiles carry the columns of the LEGACY ones (ouster_profile_cases.encode_profile).

CUDA events around --iters back-to-back async calls on the handle's stream (no host wait between them), --runs times, the two
front ends alternated; the median of the per-call time is reported, with the spread (max - min) of the runs.  The card's name, power
limit and maximum SM clock are read in the same run.  Prints one JSON line per shape and writes them to
OUT/ouster_timing_<PROFILE>.json.
    python tools/ouster_timing.py [--profile NAME] [--runs 15] [--iters 50] [--warmup 10] [--out DIR]
(NAME: LEGACY, RNG19_RFL8_SIG16_NIR16, RNG19_RFL8_SIG16_NIR16_DUAL or RNG15_RFL8_NIR8; DIR defaults to <tmp>/ouster_timing)
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import __graft_entry__ as G  # noqa: E402
import ouster_cases as OC  # noqa: E402
import ouster_profile_cases as OP  # noqa: E402

OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2", "<u1", "<u2", "<u4"],
                   "offsets": [0, 4, 8, 16, 20, 24, 26, 28, 32], "itemsize": 48})
RATE, MIN_DIST = 4, 3.0
SHAPES = ((64, 1024, 64), (128, 2048, 128), (1, 1024, 64))   # (packets, W, H)


def frame(lv, cal, profile, n_packets, W, H, seed=1):
    """the packets, the PointCloud2 of the points they decode to, and its header stamp (us)"""
    rng = np.random.default_rng(seed)
    legacy = OC.packets(rng, n_packets, W, H, m0=0, invalid=0.0, bad_m=0.0, zero=0.1)
    pk = OP.encode_profile(legacy, profile, rng)
    xyz, t, inten, rg, idx = lv.ouster_to_points(pk.tobytes(), cal, profile)
    ts = legacy.reshape(-1)["ts"][idx // H]
    stamp_us = int(ts[0]) // 1000
    cloud = np.zeros(len(t), OUSTER)
    cloud["x"], cloud["y"], cloud["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    cloud["t"] = (ts - np.uint64(stamp_us * 1000)).astype(np.uint32)
    cloud["reflectivity"] = inten.astype(np.uint16)
    cloud["ring"] = idx % H
    cloud["range"] = rg.astype(np.uint32)
    return pk, cloud, stamp_us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", default="LEGACY", choices=OP.PROFILE_NAMES)
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "ouster_timing"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ouster_timing: no CUDA device (there is nothing to measure without one)")
    os.makedirs(a.out, exist_ok=True)
    lv = G.load_package()
    profile = OP.PROFILE_NAMES.index(a.profile)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    stream = torch.cuda.Stream()
    prm = lv.default_params(max_points=1 << 19, max_map_points=1 << 16)
    prm.stream = stream.cuda_stream
    loc = lv.Localizer(prm)
    results = []
    for n_packets, W, H in SHAPES:
        cal = OC.calibration(lv, W, H, OC.ORIGIN_MM, np.random.default_rng(2))
        pk, cloud, stamp_us = frame(lv, cal, profile, n_packets, W, H)
        n = 16 * H * n_packets
        d_pk, d_cloud = loc.upload(np.frombuffer(pk.tobytes(), np.uint8)), loc.upload(cloud)
        outs = [loc.device_alloc(k * n) for k in (12, 8, 4, 4, 4)]
        d_n = loc.device_alloc(8)
        lay = lv.cloud_layout("ouster", OUSTER)
        calls = {
            "ouster_packets": lambda: loc.process_ouster_device_async(d_pk, pk.nbytes, n_packets, cal, RATE, MIN_DIST, outs[0], outs[1],
                                                                      d_n, *outs[2:], profile=profile),
            "pointcloud2": lambda: loc.process_cloud_device_async("ouster", lay, d_cloud, cloud.nbytes, len(cloud), stamp_us, 1, 1, 0.1,
                                                                   RATE, MIN_DIST, outs[0], outs[1], d_n, *outs[2:]),
        }
        kept = {}
        for name, call in calls.items():
            for _ in range(a.warmup):
                call()
            loc.synchronize()
            kept[name] = int(loc.download(d_n, np.zeros(1, np.int64))[0])
        per_call = {k: [] for k in calls}
        for _ in range(a.runs):
            for name, call in calls.items():                            # alternated, so both see the same machine state
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.iters):
                    call()
                e1.record(stream)
                e1.synchronize()
                per_call[name].append(e0.elapsed_time(e1) * 1e3 / a.iters)
        assert loc.async_status()[0] == lv.OK
        r = dict(profile=a.profile, packets=n_packets, bytes=pk.nbytes, W=W, H=H, slots=n, points=len(cloud), card=card, rate=RATE,
                 min_dist=MIN_DIST, kept=kept,
                 us_per_call={k: float(np.median(v)) for k, v in per_call.items()},
                 us_spread={k: float(np.max(v) - np.min(v)) for k, v in per_call.items()})
        print(json.dumps(r))
        results.append(r)
        for d in [d_pk, d_cloud, d_n] + outs:
            loc.device_free(d)
    loc.close()
    with open(os.path.join(a.out, "ouster_timing_%s.json" % a.profile), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
