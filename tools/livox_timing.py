"""Device time per message of the Livox front end (lv_process_livox_device_async) against the PointCloud2 front end
(lv_process_cloud_device_async, the Velodyne layout of 32 bytes per point) at the same point count, 24 000 and 240 000 points
(a Livox Avia / Mid-70 message at 10 Hz, and ten of them), rate 4, min_dist 3, the message bytes resident in HBM.  The Livox
records carry tag 0x10 (second return) on 10 % of the points and the call uses mask 0x20, so the tag select keeps all of them
but the rank pass runs in full.

CUDA events around --iters back-to-back async calls on the handle's stream (no host wait between them), --runs times; the median
of the per-call time is reported.  The card's name and power limit are read in the same run.  Prints one JSON line per shape and
writes them to OUT/livox_timing.json.
    python tools/livox_timing.py [--runs 15] [--iters 50] [--warmup 10] [--out DIR]   (DIR defaults to <tmp>/livox_timing)
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
import livox_cases as LC  # noqa: E402

VELO = np.dtype({"names": ["x", "y", "z", "intensity", "ring", "time"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                 "offsets": [0, 4, 8, 16, 20, 24], "itemsize": 32})
RATE, MIN_DIST, MASK = 4, 3.0, 0x20
TB = 1_712_345_678 * 10**9


def messages(n, seed=1):
    """the same points as a Livox message (times in firing order over 0.1 s) and as a Velodyne PointCloud2"""
    rng = np.random.default_rng(seed)
    recs = LC.records(rng, n)
    recs["offset_time"] = np.sort(recs["offset_time"])
    recs["tag"] = np.where(rng.random(n) < 0.1, 0x10, 0x00)
    velo = np.zeros(n, VELO)
    velo["x"], velo["y"], velo["z"] = recs["x"], recs["y"], recs["z"]
    velo["intensity"] = recs["reflectivity"]
    velo["time"] = (recs["offset_time"] * 1e-9).astype(np.float32)
    return recs, velo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=15)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "livox_timing"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("livox_timing: no CUDA device (there is nothing to measure without one)")
    os.makedirs(a.out, exist_ok=True)
    lv = G.load_package()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    stream = torch.cuda.Stream()
    prm = lv.default_params(max_points=1 << 19, max_map_points=1 << 16)
    prm.stream = stream.cuda_stream
    loc = lv.Localizer(prm)
    results = []
    for n in (24_000, 240_000):
        recs, velo = messages(n)
        d_livox, d_velo = loc.upload(recs), loc.upload(velo)
        outs = [loc.device_alloc(k * n) for k in (12, 8, 4, 4, 4)]
        d_n = loc.device_alloc(8)
        lay = lv.cloud_layout("velodyne", VELO)
        calls = {
            "livox": lambda: loc.process_livox_device_async(d_livox, recs.nbytes, n, TB, MASK, RATE, MIN_DIST, outs[0], outs[1], d_n, *outs[2:]),
            "pointcloud2": lambda: loc.process_cloud_device_async("velodyne", lay, d_velo, velo.nbytes, n, 0, 0, 1, 0.1, RATE, MIN_DIST,
                                                                   outs[0], outs[1], d_n, *outs[2:]),
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
        r = dict(points=n, card=card, rate=RATE, min_dist=MIN_DIST, tag_reject_mask=MASK, kept=kept,
                 us_per_message={k: float(np.median(v)) for k, v in per_call.items()},
                 us_spread={k: float(np.max(v) - np.min(v)) for k, v in per_call.items()})
        print(json.dumps(r))
        results.append(r)
        for d in [d_livox, d_velo, d_n] + outs:
            loc.device_free(d)
    loc.close()
    with open(os.path.join(a.out, "livox_timing.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
