"""Deskew by per-point time stamps vs the azimuth deskew vs no deskew: ms per scan of Pipeline.computeRecords on
synthetic 64 x 2048-ray sequences (KITTI float32 16-byte records with the inclusive gate, the stamp in the fourth column;
Ouster-like 48-byte float32 records with NaN rows, the strict gate and NaN drop, the stamp after z), three arms:
  azimuth  deskew=True, no time field: the host sorts the kept points by azimuth (Pipeline::deskew's order);
  time     deskew=True, time_field: each point's chunk from its own stamp, all on the device;
  none     deskew=False.
Each arm runs on host records and on CUDA tensors, with and without look-ahead (prefetchRecords, deskew_ahead).  The arms
alternate, twice, in one process; each arm's repeats must give the same poses bit for bit.  Prints the card and its
power limit with the table (one JSON line per configuration; --out also writes them to a file).

    python scripts/time_deskew_bench.py [--scans 30] [--out /tmp/time_deskew.json]
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
GATE = {"kitti": dict(min_range=0.7, max_range=120.0), "ouster": dict(min_range=0.7, max_range=120.0, inclusive=False,
                                                                        drop_nan=True)}


def sequence(n, layout):
    """n scans of 64 x 2048 rays along a street, unfiltered, each point stamped (float32 seconds, <= 0) by its azimuth as
    a counter-clockwise sweep ending at +pi would stamp it"""
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=64, azimuths=2048, seed=100 + i, r_min=0.0, r_max=np.inf)
        t = (-(np.pi - np.arctan2(p[:, 1], p[:, 0])) / (2 * np.pi) / HZ).astype(np.float32)
        if layout == "kitti":
            a = np.zeros((p.shape[0], 4), np.float32)
            a[:, :3], a[:, 3] = p, t
        else:
            rs = np.random.RandomState(i)
            at = np.sort(rs.randint(0, p.shape[0], size=2000))
            p, t = np.insert(p, at, np.nan, axis=0), np.insert(t, at, 0.0)
            a = np.zeros((p.shape[0], 12), np.float32)  # 48-byte records: x y z at bytes 16 / 20 / 24, the stamp at 32
            a[:, 4:7], a[:, 7], a[:, 8] = p, 0.5, t
        out.append(a)
    return out


def view(a, layout):
    return a if layout == "kitti" else a[:, 4:9]  # (x, y, z, intensity, t): the stamp is column 3 / 4 of the view


def run(arm, scans, layout, ahead):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=HZ, deskew=arm != "none", b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                 num_keyframes=16, num_threads=8, realtime=False)
    kw = dict(GATE[layout])
    if arm == "time":
        kw.update(time_field=3 if layout == "kitti" else 4, time_scale=1.0)
    poses = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        if ahead and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 32, len(scans))):
                assert p.prefetchRecords(view(scans[k], layout), deskew_ahead=True, **kw)
        p.computeRecords(0.1 * i, view(scans[i], layout), **kw)
        poses.append(p.currentPose().copy())
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / len(scans), np.array(poses)


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
    ap.add_argument("--scans", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "time_deskew_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    lines = []
    for layout in ("kitti", "ouster"):
        host = sequence(args.scans, layout)
        inputs = {"host": host, "cuda": [torch.from_numpy(a).cuda() for a in host]}
        for src, scans in inputs.items():
            for ahead in (False, True):
                for arm in ("azimuth", "time", "none"):
                    run(arm, scans[:4], layout, ahead)  # warm-up of the shapes and lanes
                ms = {"azimuth": [], "time": [], "none": []}
                ref = {}
                for _ in range(2):
                    for arm in ("azimuth", "time", "none"):
                        t, poses = run(arm, scans, layout, ahead)
                        ms[arm].append(t)
                        ref.setdefault(arm, poses)
                        assert poses.tobytes() == ref[arm].tobytes(), (layout, src, ahead, arm)
                row = dict(layout=layout, input=src, points=int(host[0].shape[0]), lookahead=ahead, scans=args.scans,
                           ms_per_scan={k: [round(v, 3) for v in vals] for k, vals in ms.items()},
                           poses_identical_within_arm=True, card=name, power_limit=limit)
                print(json.dumps(row), flush=True)
                lines.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
