"""Cost and effect of carving the voxel map along each scan's rays (Pipeline(map_carve=r), madicp_map_carve) on a drive of
synthetic 64 x 2048-ray KITTI scans (float32 16-byte records, the inclusive gate, no deskew, 0.8 m per scan), six arms:
  v0.2K1 / v0.2K1C0.75 / v0.2K1C1     map_voxel_size=0.2, map_points_per_voxel=1, map_carve 0 (off), 0.75, 1;
  v0.5K20 / v0.5K20C0.75 / v0.5K20C1  map_voxel_size=0.5, map_points_per_voxel=20, likewise.
The arms alternate, twice, in one process, and every run must give the same poses bit for bit (the script exits non-zero
otherwise).  Reported per arm: ms per scan of computeRecords, kernel launches per scan, and the map's rows at 25 / 50 /
100 % of the drive (no object moves in this scene, so every row a carve takes is erosion of static surfaces).  Then the
carve alone: the drive replayed at engine level (each scan's kept cloud, built into a device tree, inserted and carved
under the first run's poses), the carve's 7 launches timed with CUDA events on the context's stream; median, min and max
over the last 100 scans, with the ray steps of those scans counted on the host.  Prints the card and its power limit,
and one JSON line per configuration.

    python scripts/map_carve_bench.py [--scans 1000] [--out /tmp/map_carve_bench.json]
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

MAPS = {"v0.2K1": dict(map_voxel_size=0.2, map_points_per_voxel=1),
        "v0.5K20": dict(map_voxel_size=0.5, map_points_per_voxel=20)}
ARMS = {f"{m}{'' if r == 0 else f'C{r:g}'}": dict(MAPS[m], map_carve=r) for m in MAPS for r in (0.0, 0.75, 1.0)}


def run(arm, scans, read_map=False):
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    p = Pipeline(sensor_hz=HZ, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                 num_threads=8, realtime=False, **ARMS[arm])
    marks = {len(scans) // 4: "25%", len(scans) // 2: "50%", len(scans): "100%"}
    poses, sizes = [], {}
    torch.cuda.synchronize()
    l0 = p._kernelLaunches()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        p.computeRecords(0.1 * i, scans[i], **GATE)
        poses.append(p.currentPose().copy())
        if read_map and i + 1 in marks:  # (outside the timed runs)
            sizes[marks[i + 1]] = p.mapSize()
    torch.cuda.synchronize()
    out = dict(ms=(time.perf_counter() - t0) * 1e3 / len(scans), launches=(p._kernelLaunches() - l0) / len(scans),
               poses=np.array(poses))
    if read_map:
        out["map_size"] = sizes
    return out


def ray_steps(P, origin, v, reach):
    """the carved steps of one scan's rays (each one table probe)"""
    kb = np.floor(P / v).astype(np.int64)
    n = np.abs(kb - np.floor(origin / v).astype(np.int64)).max(axis=1)
    n = n[(n > 0) & (n <= 16384)]
    return int(np.ceil(reach * n.astype(np.float64)).sum())


def carve_alone(scans, poses, last=100):
    """the carve's kernels, CUDA events around each call on the context's stream, over the last `last` scans"""
    import torch
    from mad_icp_b200 import Registrar
    reg = Registrar(device=0, max_keyframes=2)
    reg.keep_cloud(True)
    stream = torch.cuda.ExternalStream(reg.stream)
    kept = []
    for a in scans:
        P = np.asarray(a[:, :3], np.float64)
        r = np.linalg.norm(P, axis=1)
        kept.append(np.ascontiguousarray(P[np.isfinite(r) & (r >= GATE["min_range"]) & (r <= GATE["max_range"])]))
    out = {}
    for name, (v, K) in (("v0.2K1", (0.2, 1)), ("v0.5K20", (0.5, 20))):
        for reach in (0.75, 1.0):
            m = reg.voxel_map(v, K)
            ev = []
            for i, P in enumerate(kept):
                t = reg.build_tree(P)
                m.insert(t, poses[i], scan=i)
                timed = i >= len(kept) - last
                if timed:
                    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                    e[0].record(stream)
                m.carve(t, poses[i], reach)
                if timed:
                    e[1].record(stream)
                    ev.append(e)
            torch.cuda.synchronize()
            ms = np.array([e[0].elapsed_time(e[1]) for e in ev])
            steps = [ray_steps((poses[i][:3, :3] @ kept[i].T).T + poses[i][:3, 3], poses[i][:3, 3], v, reach)
                     for i in range(len(kept) - last, len(kept))]
            out[f"{name}C{reach:g}"] = dict(ms_median=round(float(np.median(ms)), 4), ms_min=round(float(ms.min()), 4),
                                            ms_max=round(float(ms.max()), 4), rows_at_end=m.size(),
                                            ray_steps_median=int(np.median(steps)), points=int(kept[-1].shape[0]))
            m.free()
    reg.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "map_carve_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    scans = sequence(args.scans)
    for arm in ARMS:
        run(arm, scans[:8])  # warm-up of the shapes and lanes
    ms, launches, ref, sizes, ok = {a: [] for a in ARMS}, {}, None, {}, True
    for rep in range(2):
        for arm in ARMS:
            r = run(arm, scans, read_map=rep == 1)
            ms[arm].append(round(r["ms"], 3))
            launches[arm] = round(r["launches"], 2)
            if ref is None:
                ref = r["poses"]
            ok = ok and r["poses"].tobytes() == ref.tobytes()
            if "map_size" in r:
                sizes[arm] = r["map_size"]
    lines = [dict(points=int(scans[0].shape[0]), scans=args.scans, ms_per_scan=ms, launches_per_scan=launches,
                  map_rows=sizes, poses_identical=ok, card=name, power_limit=limit)]
    print(json.dumps(lines[-1]), flush=True)
    lines.append(dict(carve=carve_alone(scans, list(ref)), card=name, power_limit=limit))
    print(json.dumps(lines[-1]), flush=True)
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
