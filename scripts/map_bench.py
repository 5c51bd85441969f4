"""Cost of the voxel map (Pipeline(map_voxel_size=v, map_points_per_voxel=K)): ms per scan of Pipeline.computeRecords on
a synthetic 64 x 2048-ray KITTI sequence (float32 16-byte records, the inclusive gate, no deskew), five arms:
  off       no map, keep_cloud=False (the pipeline as it is without the feature);
  keep      no map, keep_cloud=True (what the map needs of the context, without the map);
  v0.2K1    map_voxel_size=0.2, map_points_per_voxel=1;
  v0.5K1    map_voxel_size=0.5, map_points_per_voxel=1;
  v0.2K8    map_voxel_size=0.2, map_points_per_voxel=8.
Each arm runs with and without look-ahead (prefetchRecords); the arms alternate, twice, in one process, and every run
must give the same poses bit for bit (the script exits non-zero otherwise).  After each map run of the whole sequence it
reports the map size, the time of mapArray() and of mapArray(device=True) plus a synchronisation, and the kernel launches
per insert (the launches of the arm minus those of `keep`, per scan).  Prints the card and its power limit, and one JSON
line per configuration.

    python scripts/map_bench.py [--scans 400] [--out /tmp/map_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from multiprocessing import Pool

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from mad_icp_b200 import synth  # noqa: E402

HZ = 10.0
GATE = dict(min_range=0.7, max_range=120.0)
ARMS = {"off": dict(), "keep": dict(keep_cloud=True), "v0.2K1": dict(map_voxel_size=0.2, map_points_per_voxel=1),
        "v0.5K1": dict(map_voxel_size=0.5, map_points_per_voxel=1), "v0.2K8": dict(map_voxel_size=0.2, map_points_per_voxel=8)}


def scan(args):
    i, n = args
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
    p = synth.lidar_scan(scene, base, beams=64, azimuths=2048, seed=100 + i, r_min=0.0, r_max=np.inf)
    a = np.zeros((p.shape[0], 4), np.float32)
    a[:, :3] = p
    return a


def sequence(n):
    """n scans of 64 x 2048 rays along a street, unfiltered (about a second of numpy per scan: built in a pool)"""
    with Pool(max(1, min(os.cpu_count() or 1, 32))) as pool:
        return pool.map(scan, [(i, n) for i in range(n)])


def run(arm, scans, ahead, read_map=False):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=HZ, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                 num_threads=8, realtime=False, **ARMS[arm])
    poses = []
    torch.cuda.synchronize()
    l0 = p._kernelLaunches()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        if ahead and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 32, len(scans))):
                assert p.prefetchRecords(scans[k], **GATE)
        p.computeRecords(0.1 * i, scans[i], **GATE)
        poses.append(p.currentPose().copy())
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / len(scans)
    out = dict(ms=ms, launches=(p._kernelLaunches() - l0) / len(scans), poses=np.array(poses))
    if read_map and "map_voxel_size" in ARMS[arm]:
        out["map_points"] = p.mapSize()
        out["map_dropped"] = p.mapDropped()
        t = time.perf_counter()
        host = p.mapArray()
        out["mapArray_ms"] = (time.perf_counter() - t) * 1e3
        torch.cuda.synchronize()
        t = time.perf_counter()
        dev = p.mapArray(device=True)
        torch.cuda.synchronize()
        out["mapArray_device_ms"] = (time.perf_counter() - t) * 1e3
        out["device_equals_host"] = bool(np.array_equal(dev.cpu().numpy().view(np.int64), host.view(np.int64)))
    return out


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
    ap.add_argument("--scans", type=int, default=400)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "map_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    scans = sequence(args.scans)
    lines, ok = [], True
    for ahead in (False, True):
        for arm in ARMS:
            run(arm, scans[:8], ahead)  # warm-up of the shapes and lanes
        ms, launches, ref, reads = {a: [] for a in ARMS}, {}, None, {}
        for rep in range(2):
            for arm in ARMS:
                r = run(arm, scans, ahead, read_map=rep == 1)
                ms[arm].append(round(r["ms"], 3))
                launches[arm] = round(r["launches"], 2)
                if ref is None:
                    ref = r["poses"]
                ok = ok and r["poses"].tobytes() == ref.tobytes()
                if "map_points" in r:
                    reads[arm] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()
                                  if k.startswith("map") or k == "device_equals_host"}
                    ok = ok and r["device_equals_host"]
        per_insert = {a: round(launches[a] - launches["keep"], 2) for a in ARMS if a not in ("off", "keep")}
        row = dict(lookahead=ahead, points=int(scans[0].shape[0]), scans=args.scans, ms_per_scan=ms,
                   launches_per_scan=launches, launches_per_insert=per_insert, map=reads, poses_identical=ok, card=name,
                   power_limit=limit)
        print(json.dumps(row), flush=True)
        lines.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    if not ok:
        print("poses differ between arms, or the device map differs from the host map", flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
