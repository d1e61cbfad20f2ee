"""Device time per scan of the Velodyne packet front end (lv_process_velodyne_device_async) against the PointCloud2 front end
(lv_process_cloud_device_async, the velodyne_pointcloud layout of 32 bytes per point) on the same points: 76 packets (one 10 Hz
rotation of a VLP-16, 29 184 slots) and 754 packets (one second of packets), 10 % of the slots without a return, rate 4, min_dist 3,
the message bytes resident in HBM.  The PointCloud2 holds the points the packets decode to, in slot order, with their times
relative to the first packet's stamp.

CUDA events around --iters back-to-back async calls on the handle's stream (no host wait between them), --runs times, the two
front ends alternated; the median of the per-call time is reported.  The card's name, power limit and maximum SM clock are read in
the same run.  Prints one JSON line per shape and writes them to OUT/velodyne_timing.json.
    python tools/velodyne_timing.py [--runs 15] [--iters 50] [--warmup 10] [--out DIR]   (DIR defaults to <tmp>/velodyne_timing)
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
import velodyne_cases as VC  # noqa: E402

VELO = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                 "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
RATE, MIN_DIST = 4, 3.0


def scan(lv, cal, n_packets, seed=1):
    """the packets, and the PointCloud2 of the points they decode to"""
    pk = VC.packets(np.random.default_rng(seed), n_packets, step=40)
    xyz, t, inten, _, idx = lv.velodyne_to_points(pk.tobytes(), cal)
    velo = np.zeros(len(t), VELO)
    velo["x"], velo["y"], velo["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    velo["intensity"] = inten
    velo["ring"] = idx % 16
    velo["time"] = (t - t[0]).astype(np.float32)
    return pk, velo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "velodyne_timing"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("velodyne_timing: no CUDA device (there is nothing to measure without one)")
    os.makedirs(a.out, exist_ok=True)
    lv = G.load_package()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    stream = torch.cuda.Stream()
    prm = lv.default_params(max_points=1 << 19, max_map_points=1 << 16)
    prm.stream = stream.cuda_stream
    loc = lv.Localizer(prm)
    cal = lv.velodyne_calibration("vlp16")
    results = []
    for n_packets in (76, 754):
        pk, velo = scan(lv, cal, n_packets)
        n = 384 * n_packets
        d_pk, d_velo = loc.upload(np.frombuffer(pk.tobytes(), np.uint8)), loc.upload(velo)
        outs = [loc.device_alloc(k * n) for k in (12, 8, 4, 4, 4)]
        d_n = loc.device_alloc(8)
        lay = lv.cloud_layout("velodyne", VELO)
        stamp_us = int(pk["sec"][0]) * 1_000_000 + int(pk["nsec"][0]) // 1000
        calls = {
            "velodyne_packets": lambda: loc.process_velodyne_device_async(d_pk, pk.nbytes, n_packets, cal, RATE, MIN_DIST, outs[0], outs[1],
                                                                          d_n, *outs[2:]),
            "pointcloud2": lambda: loc.process_cloud_device_async("velodyne", lay, d_velo, velo.nbytes, len(velo), stamp_us, 1, 1, 0.1, RATE,
                                                                   MIN_DIST, outs[0], outs[1], d_n, *outs[2:]),
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
        r = dict(packets=n_packets, slots=n, points=len(velo), card=card, rate=RATE, min_dist=MIN_DIST, kept=kept,
                 us_per_scan={k: float(np.median(v)) for k, v in per_call.items()},
                 us_spread={k: float(np.max(v) - np.min(v)) for k, v in per_call.items()})
        print(json.dumps(r))
        results.append(r)
        for d in [d_pk, d_velo, d_n] + outs:
            loc.device_free(d)
    loc.close()
    with open(os.path.join(a.out, "velodyne_timing.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
