"""Scans handed over from host memory vs from the GPU: ms per scan of Pipeline.computeRecords on synthetic 64 x 2048-ray
sequences (KITTI float32 16-byte records with the inclusive gate; Ouster-like 48-byte float32 records with NaN rows, the
strict gate and NaN drop), deskew off and on, look-ahead off and on (prefetchRecords, deskew_ahead), three arms:
  numpy   the records as a host numpy array;
  cpu     the records as a CUDA tensor that the caller first brings over with tensor.cpu().numpy() (in the timed loop);
  cuda    the CUDA tensor itself, read in place.
The arms alternate, twice, in one process; every arm must give the same poses bit for bit.  Prints the card and its
power limit with the table (one JSON line per configuration; --out also writes them to a file).

    python scripts/device_input_bench.py [--scans 40] [--out /tmp/device_input.json]
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

GATE = {"kitti": dict(min_range=0.7, max_range=120.0), "ouster": dict(min_range=0.7, max_range=120.0, inclusive=False,
                                                                        drop_nan=True)}


def sequence(n, layout, seed=0):
    """n scans of 64 x 2048 rays along a street, unfiltered (r in [0, inf)), with NaN rows for the Ouster layout"""
    scene = synth.StreetScene(seed=7 + seed, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=64, azimuths=2048, seed=100 + i, r_min=0.0, r_max=np.inf)
        if layout == "kitti":
            a = np.zeros((p.shape[0], 4), np.float32)
            a[:, :3], a[:, 3] = p, 0.5
            out.append(a)
        else:
            rs = np.random.RandomState(i)
            p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=2000)), np.nan, axis=0)
            a = np.zeros((p.shape[0], 12), np.float32)  # 48-byte records, x y z at bytes 16 / 20 / 24
            a[:, 4:7], a[:, 7] = p, 0.5
            out.append(a)
    return out


def view(a, layout):
    return a[:, :3] if layout == "kitti" else a[:, 4:7]


def run(arm, host, dev, layout, deskew, ahead):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                 num_threads=8, realtime=False)
    gate = GATE[layout]

    def scan(i):
        if arm == "numpy":
            return view(host[i], layout)
        if arm == "cpu":
            return view(dev[i].cpu().numpy(), layout)
        return view(dev[i], layout)

    poses = []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(len(host)):
        if ahead and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 32, len(host))):
                assert p.prefetchRecords(scan(k), deskew_ahead=True, **gate)
        p.computeRecords(0.1 * i, scan(i), **gate)
        poses.append(p.currentPose().copy())
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / len(host), np.array(poses)


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
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "device_input_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    lines = []
    for layout in ("kitti", "ouster"):
        host = sequence(args.scans, layout)
        dev = [torch.from_numpy(a).cuda() for a in host]
        for deskew in (False, True):
            for ahead in (False, True):
                run("cuda", host[:4], dev[:4], layout, deskew, ahead)  # warm-up of the shapes and lanes
                ms = {"numpy": [], "cpu": [], "cuda": []}
                ref = None
                for _ in range(2):
                    for arm in ("numpy", "cpu", "cuda"):
                        t, poses = run(arm, host, dev, layout, deskew, ahead)
                        ms[arm].append(t)
                        if ref is None:
                            ref = poses
                        assert poses.tobytes() == ref.tobytes(), (layout, deskew, ahead, arm)
                row = dict(layout=layout, points=int(host[0].shape[0]), deskew=deskew, lookahead=ahead, scans=args.scans,
                           ms_per_scan={k: [round(v, 3) for v in vals] for k, vals in ms.items()}, poses_identical=True,
                           card=name, power_limit=limit)
                print(json.dumps(row), flush=True)
                lines.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
