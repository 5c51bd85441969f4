"""Cost of keeping the current scan's cloud (Pipeline(keep_cloud=True)): ms per scan of Pipeline.computeRecords on
synthetic 64 x 2048-ray sequences (KITTI float32 16-byte records, the inclusive gate, a per-point stamp in the fourth
column), four arms:
  off     keep_cloud=False;
  keep    keep_cloud=True, nothing read back;
  host    keep_cloud=True and currentCloudArray() + currentCloudIndices() after every scan;
  device  keep_cloud=True and currentCloudArray(device=True) + currentCloudIndices(device=True) + a sync after every scan.
Each arm runs without a deskew, with the azimuth deskew and with the time-stamp deskew, with and without look-ahead
(prefetchRecords).  The arms alternate, twice, in one process; every run of a configuration must give the same poses bit
for bit (the script exits non-zero otherwise).  Prints the card and its power limit, and one JSON line per configuration
with ms per scan and kernel launches per scan of each arm.

    python scripts/cloud_bench.py [--scans 200] [--out /tmp/cloud_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mad_icp_b200 import synth  # noqa: E402

HZ = 10.0
GATE = dict(min_range=0.7, max_range=120.0)
ARMS = ("off", "keep", "host", "device")


def sequence(n):
    """n scans of 64 x 2048 rays along a street, unfiltered, stamped (float32 seconds, <= 0) by their azimuth"""
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=64, azimuths=2048, seed=100 + i, r_min=0.0, r_max=np.inf)
        a = np.zeros((p.shape[0], 4), np.float32)
        a[:, :3] = p
        a[:, 3] = -(np.pi - np.arctan2(p[:, 1], p[:, 0])) / (2 * np.pi) / HZ
        out.append(a)
    return out


def run(arm, scans, deskew, ahead):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=HZ, deskew=deskew != "none", b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                 num_keyframes=16, num_threads=8, realtime=False, keep_cloud=arm != "off")
    kw = dict(GATE)
    if deskew == "time":
        kw.update(time_field=3, time_scale=1.0)
    poses = []
    torch.cuda.synchronize()
    l0 = p._kernelLaunches()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        if ahead and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 32, len(scans))):
                assert p.prefetchRecords(scans[k], deskew_ahead=True, **kw)
        p.computeRecords(0.1 * i, scans[i], **kw)
        if arm == "host":
            p.currentCloudArray()
            p.currentCloudIndices()
        elif arm == "device":
            p.currentCloudArray(device=True)
            p.currentCloudIndices(device=True)
            torch.cuda.synchronize()
        poses.append(p.currentPose().copy())
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / len(scans)
    return ms, (p._kernelLaunches() - l0) / len(scans), np.array(poses)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in q.split(",")]
        return name, limit
    except Exception as e:  # (the table is still printed; the card is then "unknown")
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "cloud_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    scans = sequence(args.scans)
    lines, ok = [], True
    for deskew in ("none", "azimuth", "time"):
        for ahead in (False, True):
            for arm in ARMS:
                run(arm, scans[:4], deskew, ahead)  # warm-up of the shapes and lanes
            ms, launches, ref = {a: [] for a in ARMS}, {}, None
            for _ in range(2):
                for arm in ARMS:
                    t, n, poses = run(arm, scans, deskew, ahead)
                    ms[arm].append(round(t, 3))
                    launches[arm] = round(n, 2)
                    if ref is None:
                        ref = poses
                    ok = ok and poses.tobytes() == ref.tobytes()
            row = dict(deskew=deskew, lookahead=ahead, points=int(scans[0].shape[0]), scans=args.scans, ms_per_scan=ms,
                       launches_per_scan=launches, poses_identical=ok, card=name, power_limit=limit)
            print(json.dumps(row), flush=True)
            lines.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    if not ok:
        print("poses differ between arms", flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
