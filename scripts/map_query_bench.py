"""Cost of the voxel map's nearest-row query (Pipeline.mapNearest, madicp_map_nearest_dev) on the drive of
map_window_bench.py: synthetic 64 x 2048-ray KITTI scans (float32 16-byte records, the inclusive gate, no deskew, 0.8 m
per scan), three maps:
  v0.5K20      map_voxel_size=0.5, map_points_per_voxel=20, no window (the map grows with the drive);
  v0.5K20D50   the same with map_max_distance=50;
  v0.2K1D50    map_voxel_size=0.2, map_points_per_voxel=1, map_max_distance=50.
The queries are each scan's kept cloud in the map frame (currentCloudArray(frame="map", device=True)), with scan_below =
the scan's number.  Per map:
  - per-scan cost: a pipeline that queries every scan (at r = v) against one that does not, alternating, twice, in one
    process; the poses must be identical (the script exits non-zero otherwise);
  - index and query: in a third drive, CUDA events on torch's stream around three calls after every scan: the first
    query (the index build and the query), the same query again, and a query at r = 4 v; index = first - second;
    medians over the last 100 scans;
  - on the final map: ms per query call at r = v and r = 4 v, host clock around 50 calls that end in a synchronisation.
Prints the card and its power limit, and one JSON line per map.

    python scripts/map_query_bench.py [--scans 1000] [--out /tmp/map_query_bench.json]
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

MAPS = {"v0.5K20": dict(map_voxel_size=0.5, map_points_per_voxel=20),
        "v0.5K20D50": dict(map_voxel_size=0.5, map_points_per_voxel=20, map_max_distance=50.0),
        "v0.2K1D50": dict(map_voxel_size=0.2, map_points_per_voxel=1, map_max_distance=50.0)}


def pipeline(arm):
    from mad_icp_b200.pybind.pypeline import Pipeline
    return Pipeline(sensor_hz=HZ, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
                    num_threads=8, realtime=False, keep_cloud=True, **MAPS[arm])


def drive(arm, scans, query, events=False):
    import torch
    v = MAPS[arm]["map_voxel_size"]
    p = pipeline(arm)
    poses, ev, hits = [], [], 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(len(scans)):
        scan = p.currentID()
        p.computeRecords(0.1 * i, scans[i], **GATE)
        poses.append(p.currentPose().copy())
        if query:
            Q = p.currentCloudArray(frame="map", device=True)
            if events:
                e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                e[0].record()
                row, _ = p.mapNearest(Q, v, scan_below=scan)
                e[1].record()
                p.mapNearest(Q, v, scan_below=scan)
                e[2].record()
                p.mapNearest(Q, 4 * v, scan_below=scan)
                e[3].record()
                ev.append(e)
                if i == len(scans) - 1:
                    hits = float((row >= 0).float().mean())
            else:
                p.mapNearest(Q, v, scan_below=scan)
    torch.cuda.synchronize()
    out = dict(ms=(time.perf_counter() - t0) * 1e3 / len(scans), poses=np.array(poses), p=p)
    if events:
        t = np.array([[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])] for e in ev[-100:]])
        out.update(index_ms=float(np.median(t[:, 0] - t[:, 1])), first_query_ms=float(np.median(t[:, 0])),
                   query_ms_r_v=float(np.median(t[:, 1])), query_ms_r_4v=float(np.median(t[:, 2])),
                   hit_share_r_v_last_scan=round(hits, 4))
    return out


def final_map_calls(p, v, calls=50):
    import torch
    Q = p.currentCloudArray(frame="map", device=True)
    out = {}
    for name, r in (("r_v", v), ("r_4v", 4 * v)):
        for _ in range(3):
            p.mapNearest(Q, r)  # (warm-up)
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(calls):
            p.mapNearest(Q, r)
        torch.cuda.synchronize()
        out[name] = round((time.perf_counter() - t) * 1e3 / calls, 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "map_query_bench needs a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    scans = sequence(args.scans)
    lines, ok = [], True
    for arm in MAPS:
        v = MAPS[arm]["map_voxel_size"]
        for q in (False, True):
            drive(arm, scans[:8], q)  # warm-up
        ms, ref = {"no_query": [], "query": []}, None
        for rep in range(2):
            for q in (False, True):
                r = drive(arm, scans, q)
                ms["query" if q else "no_query"].append(round(r["ms"], 3))
                ref = r["poses"] if ref is None else ref
                ok = ok and r["poses"].tobytes() == ref.tobytes()
                del r
        r = drive(arm, scans, True, events=True)
        ok = ok and r["poses"].tobytes() == ref.tobytes()
        p = r.pop("p")
        row = dict(map=arm, scans=args.scans, points=int(scans[0].shape[0]), map_rows=p.mapSize(),
                   queries=int(p.currentCloudArray().shape[0]), ms_per_scan=ms,
                   per_scan_query_cost_ms=round(float(np.mean(ms["query"]) - np.mean(ms["no_query"])), 3),
                   spread_ms=dict(no_query=round(max(ms["no_query"]) - min(ms["no_query"]), 3),
                                  query=round(max(ms["query"]) - min(ms["query"]), 3)),
                   **{k: round(x, 4) if isinstance(x, float) else x for k, x in r.items() if k not in ("ms", "poses")},
                   final_map_ms_per_call=final_map_calls(p, v), poses_identical=ok, card=name, power_limit=limit)
        del p
        print(json.dumps(row), flush=True)
        lines.append(row)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")
    if not ok:
        print("poses differ between a pipeline that queries and one that does not", flush=True)
        sys.exit(1)


if __name__ == "__main__":
    main()
