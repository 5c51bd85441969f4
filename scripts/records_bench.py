"""Raw records straight to the device vs the dataset readers' numpy filtering (apps/utils/kitti_reader.py:82-88,
apps/utils/point_cloud2.py:77-87) followed by Pipeline.compute.  A synthetic KITTI-shape sequence (64 x 2048 rays,
no range gate at the source) is laid out two ways:
  kitti   float32 N x 4 records (16 bytes), gate 0.7 <= r <= 120 (the KITTI config)
  ouster  48-byte PointCloud2 records, x/y/z float32 at 16/20/24, NaN rows for missing returns, NaN drop + gate
          0 < r < 50 (the vbr_os0 config; its reader hands float64 to compute)
  kitti+correction  the kitti layout with the KITTI config's apply_correction: the reader's scipy rotation of the kept
          points (kitti_reader.py:72-79, 90-91) + compute, against computeRecords(apply_correction=True)
and run four ways: reader + compute, reader + prefetch, computeRecords, prefetchRecords (look-ahead batches of 16).
Two deskewed layouts (the mulran / vbr_os1 configs deskew) run three ways: reader + compute, computeRecords, and
prefetchRecords(deskew_ahead=True) (look-ahead plans, 16 at a time):
  kitti+deskew   the kitti layout, deskewed at 10 Hz
  ouster+deskew  the ouster layout with vbr_os1's strict gate 1.3 < r < 120, deskewed at 20 Hz
Reports host wall time per scan (reader included), scans/s and H2D bytes per scan, plus the GPU name and power limit.
With MADICP_PIPELINE_TIMING set every pipeline prints its per-phase means to stderr when it is destroyed.
Usage: python scripts/records_bench.py [n_scans=1000] [out.json] [layouts=all, comma-separated] [ways=all: any of
reader,records,prefetch]"""
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from scipy.spatial.transform import Rotation

from mad_icp_b200 import synth

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
out_path = sys.argv[2] if len(sys.argv) > 2 and sys.argv[2] != "-" else None
scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [16, 20, 24, 28, 32, 40], "itemsize": 48})


def make_scan(i):
    base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
    p = synth.lidar_scan(scene, base, beams=64, azimuths=2048, seed=100 + i, r_min=0.0, r_max=np.inf)
    rs = np.random.RandomState(i)
    holes = np.sort(rs.randint(0, p.shape[0], size=p.shape[0] // 20))  # missing returns
    return np.insert(p, holes, np.nan, axis=0).astype(np.float32)


if n > 64:
    import multiprocessing as mp
    with mp.get_context("fork").Pool(min(32, os.cpu_count() or 1)) as pool:
        raw = pool.map(make_scan, range(n), chunksize=4)
else:
    raw = [make_scan(i) for i in range(n)]
kitti = []
ouster = []
for p in raw:
    k = np.zeros((p.shape[0], 4), np.float32)
    k[:, :3] = p
    kitti.append(k.tobytes())  # what np.fromfile reads
    o = np.zeros(p.shape[0], OUSTER)
    o["x"], o["y"], o["z"] = p[:, 0], p[:, 1], p[:, 2]
    ouster.append(o.tobytes())  # what msg.data holds
del raw

from mad_icp_b200.pybind.pypeline import Pipeline  # noqa: E402  (after the fork)


def read_kitti(buf):  # kitti_reader.py:82-88
    cloud = np.frombuffer(buf, np.float32).reshape(-1, 4)[:, :3]
    norms = np.linalg.norm(cloud, axis=1)
    return cloud[(norms >= 0.7) & (norms <= 120.0)]


def read_kitti_corrected(buf):  # kitti_reader.py:72-79, 82-91 with apply_correction
    points = read_kitti(buf)
    rotation_vectors = np.cross(points, np.array([0., 0., 1.]))
    norms = np.linalg.norm(rotation_vectors, axis=1).reshape(-1, 1)
    rotation_vectors_normalized = rotation_vectors / norms
    return Rotation.from_rotvec(np.radians(0.205) * rotation_vectors_normalized).apply(points)


def read_ouster(buf, lo=0.0, hi=50.0):  # point_cloud2.py:77-87, 96
    s = np.frombuffer(buf, OUSTER)
    pts = np.column_stack([s["x"], s["y"], s["z"]])
    pts = pts[~np.any(np.isnan(pts), axis=1)]
    norms = np.linalg.norm(pts, axis=1)
    return pts[(norms > lo) & (norms < hi)].astype(np.float64)


# name: (buffers, reader, records view, gate, pipeline settings)
LAYOUTS = {
    "kitti": (kitti, read_kitti, lambda b: np.frombuffer(b, np.float32).reshape(-1, 4)[:, :3],
              dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False), {}),
    "ouster": (ouster, read_ouster, lambda b: np.frombuffer(b, OUSTER),
               dict(min_range=0.0, max_range=50.0, inclusive=False, drop_nan=True), {}),
    "kitti+correction": (kitti, read_kitti_corrected, lambda b: np.frombuffer(b, np.float32).reshape(-1, 4)[:, :3],
                         dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False, apply_correction=True), {}),
    "kitti+deskew": (kitti, read_kitti, lambda b: np.frombuffer(b, np.float32).reshape(-1, 4)[:, :3],
                     dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False), dict(deskew=True)),
    "ouster+deskew": (ouster, lambda b: read_ouster(b, 1.3, 120.0), lambda b: np.frombuffer(b, OUSTER),
                      dict(min_range=1.3, max_range=120.0, inclusive=False, drop_nan=True),
                      dict(deskew=True, sensor_hz=20.0)),
}
kw = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
          num_threads=min(16, os.cpu_count() or 1), realtime=False)


def run(layout, records, prefetch):
    bufs, reader, view, gate, settings = LAYOUTS[layout]
    cfg = dict(kw, **settings)
    ahead = dict(deskew_ahead=True) if cfg["deskew"] else {}  # (a deskewed pipeline plans its look-ahead scans)
    p = Pipeline(**cfg)
    sys.stderr.write(f"[{layout} {'records' if records else 'reader+compute'}{' +prefetch' if prefetch else ''}] ")
    h2d = 0
    poses = []
    t0 = None
    for i, b in enumerate(bufs):
        if i == 1:
            t0 = time.perf_counter()
        if records:
            a = view(b)
            if prefetch and i >= 1 and p.prefetched() == 0:
                for k in range(i, min(i + 16, len(bufs))):
                    assert p.prefetchRecords(view(bufs[k]), **gate, **ahead)
            p.computeRecords(i / cfg["sensor_hz"], a, **gate)
            h2d += a.shape[0] * (48 if layout.startswith("ouster") else 16) - (20 if layout.startswith("ouster") else 4)
        else:
            pts = reader(b)
            if prefetch and i >= 1 and p.prefetched() == 0:
                for k in range(i, min(i + 16, len(bufs))):
                    p.prefetch(reader(bufs[k]))
            p.compute(i / cfg["sensor_hz"], pts)
            h2d += pts.nbytes
        poses.append(p.currentPose())
    dt = time.perf_counter() - t0
    del p  # (prints its phases now, with MADICP_PIPELINE_TIMING)
    sys.stderr.flush()
    return dict(ms_per_scan=1e3 * dt / (len(bufs) - 1), scans_per_s=(len(bufs) - 1) / dt, h2d_bytes_per_scan=h2d / len(bufs),
                poses=np.array(poses))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


layouts = sys.argv[3].split(",") if len(sys.argv) > 3 and sys.argv[3] != "all" else list(LAYOUTS)
ways = sys.argv[4].split(",") if len(sys.argv) > 4 else ["reader", "records", "prefetch"]
result = dict(gpu=gpu_info(), n_scans=n, runs={})
print("GPU:", result["gpu"])
for layout in layouts:
    base = None
    deskew = LAYOUTS[layout][4].get("deskew", False)
    for prefetch in (False, True):
        for records in (False, True):
            if (prefetch and ("prefetch" not in ways or (deskew and not records)) or
                    (not prefetch and ("records" if records else "reader") not in ways)):
                continue  # (deskewed: look-ahead plans take records)
            name = f"{layout} {'records' if records else 'reader+compute'}{' +prefetch' if prefetch else ''}"
            r = run(layout, records, prefetch)
            if base is None:
                base = r["poses"]
            same = bool((r["poses"] == base).all())
            r["poses_sha256"] = hashlib.sha256(np.ascontiguousarray(r.pop("poses")).tobytes()).hexdigest()
            r["poses_equal_reader_compute"] = same
            result["runs"][name] = r
            print(f"{name:34s} {r['ms_per_scan']:7.3f} ms/scan  {r['scans_per_s']:7.1f} scans/s  "
                  f"H2D {r['h2d_bytes_per_scan'] / 1e6:6.2f} MB/scan  poses identical: {same}", flush=True)
if out_path:
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(result, f, indent=1)
