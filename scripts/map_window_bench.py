"""Cost and effect of the voxel map's window (Pipeline(map_max_distance=D), madicp_map_remove_far) on a drive of synthetic
64 x 2048-ray KITTI scans (float32 16-byte records, the inclusive gate, no deskew, 0.8 m per scan), four arms:
  off          no map;
  v0.5K20      map_voxel_size=0.5, map_points_per_voxel=20, no window (the map grows with the drive);
  v0.5K20D50   the same with map_max_distance=50;
  v0.2K1D50    map_voxel_size=0.2, map_points_per_voxel=1, map_max_distance=50.
Each arm runs with and without look-ahead (prefetchRecords); the arms alternate, twice, in one process, and every run
must give the same poses bit for bit (the script exits non-zero otherwise).  Reported per arm: ms per scan of
computeRecords, kernel launches per scan, the map size at 25 / 50 / 100 % of the drive, and the time of
mapArray(device=True) plus a synchronisation at the end.  Then the removal alone, at engine level on a map of about a
million rows: ms per madicp_map_remove_far call that removes nothing, and per call that removes an outer shell of voxels
(so nearly every row is compacted), host clock around 50 calls that end in a device synchronisation.  Prints the card
and its power limit, and one JSON line per configuration.

    python scripts/map_window_bench.py [--scans 1000] [--out /tmp/map_window_bench.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from map_bench import GATE, HZ, card, sequence  # noqa: E402

ARMS = {"off": dict(),
        "v0.5K20": dict(map_voxel_size=0.5, map_points_per_voxel=20),
        "v0.5K20D50": dict(map_voxel_size=0.5, map_points_per_voxel=20, map_max_distance=50.0),
        "v0.2K1D50": dict(map_voxel_size=0.2, map_points_per_voxel=1, map_max_distance=50.0)}


def run(arm, scans, ahead, read_map=False):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=HZ, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                 num_threads=8, realtime=False, **ARMS[arm])
    has_map = "map_voxel_size" in ARMS[arm]
    marks = {len(scans) // 4: "25%", len(scans) // 2: "50%", len(scans): "100%"}
    poses, sizes = [], {}
    torch.cuda.synchronize()
    l0 = p._kernelLaunches()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        if ahead and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 32, len(scans))):
                assert p.prefetchRecords(scans[k], **GATE)
        p.computeRecords(0.1 * i, scans[i], **GATE)
        poses.append(p.currentPose().copy())
        if read_map and has_map and i + 1 in marks:  # (outside the timed runs)
            sizes[marks[i + 1]] = p.mapSize()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / len(scans)
    out = dict(ms=ms, launches=(p._kernelLaunches() - l0) / len(scans), poses=np.array(poses))
    if read_map and has_map:
        out["map_size"] = sizes
        torch.cuda.synchronize()
        t = time.perf_counter()
        dev = p.mapArray(device=True)
        torch.cuda.synchronize()
        out["mapArray_device_ms"] = (time.perf_counter() - t) * 1e3
        out["device_equals_host"] = bool(np.array_equal(dev.cpu().numpy().view(np.int64), p.mapArray().view(np.int64)))
    return out


def removal_cost(scans, calls=50):
    """ms per remove_far call on a map of about a million rows: removing nothing, and removing an outer shell each call"""
    import torch
    from mad_icp_b200 import Registrar, synth
    reg = Registrar(device=0, max_keyframes=2)
    reg.keep_cloud(True)
    out = {}
    for what in ("nothing", "shell"):
        m = reg.voxel_map(0.05, 32)
        for i, a in enumerate(scans[:8]):
            P = np.asarray(a[:, :3], np.float64)
            P = P[np.isfinite(P).all(axis=1) & (np.linalg.norm(P, axis=1) >= GATE["min_range"])]
            m.insert(reg.build_tree(P), synth.pose_xyyaw(0.8 * i, 0.0, 0.0), scan=i)
        rows0 = m.size()
        D0 = 130.0
        m.remove_far([0.0, 0.0, 0.0], D0)  # (warm-up)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for k in range(calls):
            m.remove_far([0.0, 0.0, 0.0], D0 if what == "nothing" else D0 - 1.5 * (k + 1))
        torch.cuda.synchronize()
        out[what] = dict(ms_per_call=round((time.perf_counter() - t) * 1e3 / calls, 4), rows_before=rows0,
                         rows_after=m.size())
        m.free()
    reg.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "map_window_bench needs a GPU"
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
                if "map_size" in r:
                    reads[arm] = dict(size=r["map_size"], mapArray_device_ms=round(r["mapArray_device_ms"], 3))
                    ok = ok and r["device_equals_host"]
        row = dict(lookahead=ahead, points=int(scans[0].shape[0]), scans=args.scans, ms_per_scan=ms,
                   launches_per_scan=launches, map=reads, poses_identical=ok, card=name, power_limit=limit)
        print(json.dumps(row), flush=True)
        lines.append(row)
    row = dict(removal=removal_cost(scans), card=name, power_limit=limit)
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
