"""Launch and batching census of every route a scan takes through Pipeline: compute (VectorEigen3d, float64 and float32
arrays, CUDA tensors), computeRecords (host and device records, gated and ungated, with and without the vertical
correction, a time field and the deskew), prefetch / prefetchRecords at look-ahead depths 1 and 5 (with and without
deskew_ahead on a deskewing pipeline), and look-ahead sequences that mix the kinds of scan a batch keeps apart: float32
and float64 clouds, host records, and device records ready on different streams.  Each route runs with kept clouds off
and on, with device-built trees and, where the scans are host memory, with host-built ones (MADICP_GPU_BUILD=0).

For every scan of an eight-scan sequence a route notes the kernel launches (Pipeline._kernelLaunches()) of that scan's
prefetch and compute calls, the size of every look-ahead batch built meanwhile with the number of its scans that had
been uploaded ahead ("N scans (k staged)", printed under MADICP_BUILD_TIMING=1; the entry point's name is not part of
the census), and how many scans are queued afterwards.  How the Pipeline hands scans to the library may change; what
reaches the device may not, so every entry of the table must stay as it is.  Poses, clouds and leaves of these routes
are compared bit for bit elsewhere (test_gpu_cloud_out.py, test_deskew_lookahead.py, test_gpu_device_input.py,
test_records.py).

`python tests/test_pipeline_routes.py` runs every route on the GPU and prints the table."""
import contextlib
import hashlib
import itertools
import json
import os
import re
import sys
import tempfile
from unittest import mock

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from mad_icp_b200 import records, synth  # noqa: E402

N_SCANS = 8
GATE = dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False)
PACKED = ("vec", "f64", "f32", "cuda32", "cuda64")
ONOFF = (0, 1)
# look-ahead sequences of mixed kinds (one source per scan); "-s2": device memory ready on a second stream
MIXES = {
    "packed": ("f64", "f32", "f64", "f64", "f32", "f32", "vec", "f64"),
    "records": ("host", "host-ungated", "dev", "dev", "dev-s2", "host", "cuda32", "dev-s2"),
    "all": ("f64", "host", "f64", "dev", "f32", "host", "host", "cuda64"),
}


def _route(**kw):
    return kw


ROUTES = (
    [_route(api="compute", src=s, deskew=d, keep=k, build=b)
     for s, d, k, b in itertools.product(PACKED, ONOFF, ONOFF, ("gpu", "host"))]
    + [_route(api="records", src=s, gate=g, corr=c, time=t, deskew=d, keep=k, build=b)
       for s, g, c, t, d, k, b in itertools.product(("host", "dev"), ONOFF, ONOFF, ONOFF, ONOFF, ONOFF, ("gpu", "host"))]
    + [_route(api="prefetch", src=s, depth=n, deskew=d, ahead=a, keep=k)
       for s, n, (d, a), k in itertools.product(PACKED, (1, 5), ((0, 0), (1, 0), (1, 1)), ONOFF)]
    + [_route(api="prefetchRecords", src=s, gate=g, corr=c, time=t, depth=n, deskew=d, ahead=a, keep=k)
       for s, (g, c, t), n, (d, a), k in itertools.product(("host", "dev"), ((1, 0, 0), (0, 0, 0), (1, 1, 1)), (1, 5),
                                                            ((0, 0), (1, 0), (1, 1)), ONOFF)]
    + [_route(api="mixed", mix=m, depth=n, keep=k) for m, n, k in itertools.product(MIXES, (5, 8), ONOFF)])


def route_id(r):
    return "-".join([r["api"]] + [f"{k}={v}" for k, v in r.items() if k != "api"])


def _sequence():
    """KITTI float32 N x 4 records on a street, column 3 a time stamp in seconds; every 97th point pushed beyond the
    range gate's 120 m"""
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * N_SCANS)
    out = []
    for i in range(N_SCANS):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        p[::97] *= 200.0
        a = np.zeros((p.shape[0], 4), np.float32)
        a[:, :3] = p
        a[:, 3] = np.linspace(-0.1, 0.0, p.shape[0])
        out.append(a)
    return out


def _ungated_layout(layout):
    """records.layout without a range gate (what the Python API never asks for on records)"""
    def wrap(*args, **kw):
        t = list(layout(*args, **kw))
        t[9] = records.RANGE_NONE
        return tuple(t)
    return wrap


@contextlib.contextmanager
def _stderr_into(lines):
    """what the library writes to file descriptor 2 meanwhile, appended to `lines`"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            yield
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            f.seek(0)
            lines.extend(f.read().decode(errors="replace").splitlines())


BATCH = re.compile(r": (\d+) scans \((\d+) staged\)")


class Scans:
    """The sequence in every form a route hands it over in"""

    def __init__(self, seq):
        self.seq = seq
        self.kept = [a[(np.linalg.norm(a[:, :3].astype(np.float64), axis=1) >= 0.7)
                       & (np.linalg.norm(a[:, :3].astype(np.float64), axis=1) <= 120.0)][:, :3] for a in seq]

    def packed(self, src, i):
        import torch
        from mad_icp_b200.pybind.pypeline import VectorEigen3d
        x = np.ascontiguousarray(self.kept[i], np.float32 if src in ("f32", "cuda32") else np.float64)
        if src == "vec":
            return VectorEigen3d(x)
        return torch.from_numpy(x).cuda() if src.startswith("cuda") else x

    def records(self, src, i):
        import torch
        return torch.from_numpy(self.seq[i]).cuda() if src.startswith("dev") else self.seq[i]


def _kwargs(route, src):
    """computeRecords / prefetchRecords keywords of a records route"""
    kw = dict(GATE, apply_correction=bool(route.get("corr", 0)))
    if route.get("time", 0):
        kw.update(time_field=3, time_scale=1.0)
    return kw


def run(route, scans, digest=None):
    """The census entries of one route over the sequence; with `digest` (a hashlib object) every pose, keyframe ID,
    inlier ratio, kept cloud and the model's leaves go into it"""
    import torch
    from mad_icp_b200.pybind.pypeline import Pipeline
    api = route["api"]
    deskew = bool(route.get("deskew", 0))
    env = {"MADICP_GPU_BUILD": "0" if route.get("build") == "host" else "1", "MADICP_BUILD_TIMING": "1"}
    with mock.patch.dict(os.environ, env):
        p = Pipeline(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                     num_keyframes=4, num_threads=4, realtime=False, keep_cloud=bool(route["keep"]))
    s2 = torch.cuda.Stream()
    if api == "mixed":
        srcs = MIXES[route["mix"]]
    else:
        srcs = (route["src"],) * N_SCANS
    is_records = api in ("records", "prefetchRecords")
    depth = route.get("depth", 0)

    def hand(i, call):
        """scan i through `call` ("compute" or "prefetch") in its route's form"""
        src = srcs[i]
        rec = is_records or (api == "mixed" and src.startswith(("host", "dev")))
        ungated = (is_records and not route["gate"]) or src == "host-ungated"
        ctx = torch.cuda.stream(s2) if src.endswith("-s2") else contextlib.nullcontext()
        with ctx, mock.patch.object(records, "layout", _ungated_layout(records.layout) if ungated else records.layout):
            if rec:
                x, kw = scans.records(src, i), _kwargs(route, src)
                if call == "compute":
                    return p.computeRecords(0.1 * i, x, **kw)
                return p.prefetchRecords(x, **kw, deskew_ahead=bool(route.get("ahead", 0)))
            x = scans.packed(src, i)
            if call == "compute":
                return p.compute(0.1 * i, x)
            return p.prefetch(x, deskew_ahead=bool(route.get("ahead", 0)))

    out, queued = [], 0
    with mock.patch.dict(os.environ, {"MADICP_BUILD_TIMING": "1"}):
        for i in range(N_SCANS):
            lines = []
            l0 = p._kernelLaunches()
            with _stderr_into(lines):
                while depth and queued < min(i + depth, N_SCANS):
                    if not hand(queued, "prefetch"):
                        break
                    queued += 1
                hand(i, "compute")
                torch.cuda.synchronize()
            e = str(p._kernelLaunches() - l0)
            batches = [f"{m.group(1)}/{m.group(2)}" for m in map(BATCH.search, lines) if m]
            if batches:
                e += "[" + ",".join(batches) + "]"
            if depth:
                e += f"q{p.prefetched()}"
            out.append(e)
            if digest is not None:
                digest.update(p.currentPose().tobytes())
                digest.update(np.array([p.keyframeID(), p.inliersRatio()]).tobytes())
                if route["keep"]:
                    digest.update(p.currentCloudArray(frame="sensor").tobytes())
                    digest.update(p.currentCloudIndices().tobytes())
            queued = max(queued, i + 1)
    if digest is not None:
        digest.update(p.modelLeavesArray().tobytes())
    return " ".join(out)


# route id -> the census of its eight scans ("launches[batch size/staged,...]q<queued after the scan>"), recorded on
# an NVIDIA H100 80GB HBM3 (700 W power limit)
CENSUS = {
    'compute-src=vec-deskew=0-keep=0-build=gpu': '281 271 283 283 287 283 283 287',
    'compute-src=vec-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=vec-deskew=0-keep=1-build=gpu': '282 272 284 284 288 284 284 288',
    'compute-src=vec-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=vec-deskew=1-keep=0-build=gpu': '281 271 285 285 289 285 285 289',
    'compute-src=vec-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=vec-deskew=1-keep=1-build=gpu': '282 272 285 285 289 285 285 289',
    'compute-src=vec-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f64-deskew=0-keep=0-build=gpu': '281 271 283 283 287 283 283 287',
    'compute-src=f64-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f64-deskew=0-keep=1-build=gpu': '282 272 284 284 288 284 284 288',
    'compute-src=f64-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f64-deskew=1-keep=0-build=gpu': '281 271 285 285 289 285 285 289',
    'compute-src=f64-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f64-deskew=1-keep=1-build=gpu': '282 272 285 285 289 285 285 289',
    'compute-src=f64-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f32-deskew=0-keep=0-build=gpu': '281 271 283 283 287 283 283 287',
    'compute-src=f32-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f32-deskew=0-keep=1-build=gpu': '282 272 284 284 288 284 284 288',
    'compute-src=f32-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f32-deskew=1-keep=0-build=gpu': '281 271 285 285 289 285 285 289',
    'compute-src=f32-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=f32-deskew=1-keep=1-build=gpu': '282 272 285 285 289 285 285 289',
    'compute-src=f32-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda32-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'compute-src=cuda32-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda32-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'compute-src=cuda32-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda32-deskew=1-keep=0-build=gpu': '286 276 289 289 293 289 289 293',
    'compute-src=cuda32-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda32-deskew=1-keep=1-build=gpu': '287 277 291 291 295 291 291 295',
    'compute-src=cuda32-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda64-deskew=0-keep=0-build=gpu': '282 272 284 284 288 284 284 288',
    'compute-src=cuda64-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda64-deskew=0-keep=1-build=gpu': '283 273 285 285 289 285 285 289',
    'compute-src=cuda64-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda64-deskew=1-keep=0-build=gpu': '282 272 289 289 293 289 289 293',
    'compute-src=cuda64-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'compute-src=cuda64-deskew=1-keep=1-build=gpu': '283 273 291 291 295 291 291 295',
    'compute-src=cuda64-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=0-time=0-deskew=0-keep=0-build=gpu': '281 303 299 299 303 299 299 303',
    'records-src=host-gate=0-corr=0-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=0-time=0-deskew=0-keep=1-build=gpu': '282 304 300 300 304 300 300 304',
    'records-src=host-gate=0-corr=0-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=0-time=0-deskew=1-keep=0-build=gpu': '281 303 301 305 285 301 301 305',
    'records-src=host-gate=0-corr=0-time=0-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=0-time=0-deskew=1-keep=1-build=gpu': '282 304 301 305 285 301 301 305',
    'records-src=host-gate=0-corr=0-time=0-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=0-time=1-deskew=0-keep=0-build=gpu': '281 303 299 299 303 299 299 303',
    'records-src=host-gate=0-corr=0-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=0-time=1-deskew=0-keep=1-build=gpu': '282 304 300 300 304 300 300 304',
    'records-src=host-gate=0-corr=0-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=0-time=1-deskew=1-keep=0-build=gpu': '281 303 304 308 304 304 304 308',
    'records-src=host-gate=0-corr=0-time=1-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=0-time=1-deskew=1-keep=1-build=gpu': '282 304 305 309 305 305 305 309',
    'records-src=host-gate=0-corr=0-time=1-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=1-time=0-deskew=0-keep=0-build=gpu': '283 305 301 301 305 301 301 305',
    'records-src=host-gate=0-corr=1-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=1-time=0-deskew=0-keep=1-build=gpu': '284 306 302 302 306 302 302 306',
    'records-src=host-gate=0-corr=1-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=1-time=0-deskew=1-keep=0-build=gpu': '283 305 301 305 285 301 301 305',
    'records-src=host-gate=0-corr=1-time=0-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=1-time=0-deskew=1-keep=1-build=gpu': '284 306 301 305 285 301 301 305',
    'records-src=host-gate=0-corr=1-time=0-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=host-gate=0-corr=1-time=1-deskew=0-keep=0-build=gpu': '283 305 301 301 305 301 301 305',
    'records-src=host-gate=0-corr=1-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=1-time=1-deskew=0-keep=1-build=gpu': '284 306 302 302 306 302 302 306',
    'records-src=host-gate=0-corr=1-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=1-time=1-deskew=1-keep=0-build=gpu': '283 305 304 304 308 304 304 308',
    'records-src=host-gate=0-corr=1-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=0-corr=1-time=1-deskew=1-keep=1-build=gpu': '284 306 305 305 309 305 305 309',
    'records-src=host-gate=0-corr=1-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=0-deskew=0-keep=0-build=gpu': '284 274 286 286 290 286 286 290',
    'records-src=host-gate=1-corr=0-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=0-deskew=0-keep=1-build=gpu': '285 275 287 287 291 287 287 291',
    'records-src=host-gate=1-corr=0-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=0-deskew=1-keep=0-build=gpu': '284 274 285 285 289 285 285 289',
    'records-src=host-gate=1-corr=0-time=0-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=0-deskew=1-keep=1-build=gpu': '285 275 285 285 289 285 285 289',
    'records-src=host-gate=1-corr=0-time=0-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=1-deskew=0-keep=0-build=gpu': '284 274 286 286 290 286 286 290',
    'records-src=host-gate=1-corr=0-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=1-deskew=0-keep=1-build=gpu': '285 275 287 287 291 287 287 291',
    'records-src=host-gate=1-corr=0-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=1-deskew=1-keep=0-build=gpu': '284 274 288 288 292 288 288 292',
    'records-src=host-gate=1-corr=0-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=0-time=1-deskew=1-keep=1-build=gpu': '285 275 289 289 293 289 289 293',
    'records-src=host-gate=1-corr=0-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=0-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=host-gate=1-corr=1-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=0-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=host-gate=1-corr=1-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=0-deskew=1-keep=0-build=gpu': '286 276 285 285 289 285 285 289',
    'records-src=host-gate=1-corr=1-time=0-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=0-deskew=1-keep=1-build=gpu': '287 277 285 285 289 285 285 289',
    'records-src=host-gate=1-corr=1-time=0-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=1-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=host-gate=1-corr=1-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=1-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=host-gate=1-corr=1-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=1-deskew=1-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=host-gate=1-corr=1-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=host-gate=1-corr=1-time=1-deskew=1-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=host-gate=1-corr=1-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=0-time=0-deskew=0-keep=0-build=gpu': '286 308 304 304 308 304 304 308',
    'records-src=dev-gate=0-corr=0-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=0-time=0-deskew=0-keep=1-build=gpu': '287 309 305 305 309 305 305 309',
    'records-src=dev-gate=0-corr=0-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=0-time=0-deskew=1-keep=0-build=gpu': '286 308 305 309 289 305 305 309',
    'records-src=dev-gate=0-corr=0-time=0-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=0-time=0-deskew=1-keep=1-build=gpu': '287 309 307 311 291 307 307 311',
    'records-src=dev-gate=0-corr=0-time=0-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=0-time=1-deskew=0-keep=0-build=gpu': '286 308 304 304 308 304 304 308',
    'records-src=dev-gate=0-corr=0-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=0-time=1-deskew=0-keep=1-build=gpu': '287 309 305 305 309 305 305 309',
    'records-src=dev-gate=0-corr=0-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=0-time=1-deskew=1-keep=0-build=gpu': '286 308 304 308 304 304 304 308',
    'records-src=dev-gate=0-corr=0-time=1-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=0-time=1-deskew=1-keep=1-build=gpu': '287 309 305 309 305 305 305 309',
    'records-src=dev-gate=0-corr=0-time=1-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=1-time=0-deskew=0-keep=0-build=gpu': '286 308 304 304 308 304 304 308',
    'records-src=dev-gate=0-corr=1-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=1-time=0-deskew=0-keep=1-build=gpu': '287 309 305 305 309 305 305 309',
    'records-src=dev-gate=0-corr=1-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=1-time=0-deskew=1-keep=0-build=gpu': '286 308 305 309 289 305 305 309',
    'records-src=dev-gate=0-corr=1-time=0-deskew=1-keep=0-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=1-time=0-deskew=1-keep=1-build=gpu': '287 309 307 311 291 307 307 311',
    'records-src=dev-gate=0-corr=1-time=0-deskew=1-keep=1-build=host': '0 6 2 6 2 2 2 6',
    'records-src=dev-gate=0-corr=1-time=1-deskew=0-keep=0-build=gpu': '286 308 304 304 308 304 304 308',
    'records-src=dev-gate=0-corr=1-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=1-time=1-deskew=0-keep=1-build=gpu': '287 309 305 305 309 305 305 309',
    'records-src=dev-gate=0-corr=1-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=1-time=1-deskew=1-keep=0-build=gpu': '286 308 304 304 308 304 304 308',
    'records-src=dev-gate=0-corr=1-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=0-corr=1-time=1-deskew=1-keep=1-build=gpu': '287 309 305 305 309 305 305 309',
    'records-src=dev-gate=0-corr=1-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=0-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=0-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=0-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=0-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=0-deskew=1-keep=0-build=gpu': '286 276 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=0-time=0-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=0-deskew=1-keep=1-build=gpu': '287 277 291 291 295 291 291 295',
    'records-src=dev-gate=1-corr=0-time=0-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=1-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=0-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=1-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=0-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=1-deskew=1-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=0-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=0-time=1-deskew=1-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=0-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=0-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=1-time=0-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=0-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=1-time=0-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=0-deskew=1-keep=0-build=gpu': '286 276 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=1-time=0-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=0-deskew=1-keep=1-build=gpu': '287 277 291 291 295 291 291 295',
    'records-src=dev-gate=1-corr=1-time=0-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=1-deskew=0-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=1-time=1-deskew=0-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=1-deskew=0-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=1-time=1-deskew=0-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=1-deskew=1-keep=0-build=gpu': '286 276 288 288 292 288 288 292',
    'records-src=dev-gate=1-corr=1-time=1-deskew=1-keep=0-build=host': '0 6 2 2 6 2 2 6',
    'records-src=dev-gate=1-corr=1-time=1-deskew=1-keep=1-build=gpu': '287 277 289 289 293 289 289 293',
    'records-src=dev-gate=1-corr=1-time=1-deskew=1-keep=1-build=host': '0 6 2 2 6 2 2 6',
    'prefetch-src=vec-depth=1-deskew=0-ahead=0-keep=0': '280[1/1]q0 270[1/1]q0 282[1/1]q0 282[1/1]q0 286[1/1]q0 282[1/1]q0 282[1/1]q0 286[1/1]q0',
    'prefetch-src=vec-depth=1-deskew=0-ahead=0-keep=1': '281[1/1]q0 271[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0',
    'prefetch-src=vec-depth=1-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=1-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=1-deskew=1-ahead=1-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=1-deskew=1-ahead=1-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=5-deskew=0-ahead=0-keep=0': '280[5/5]q4 6q4 2q4 2q4 6q3 282[3/3]q2 2q1 6q0',
    'prefetch-src=vec-depth=5-deskew=0-ahead=0-keep=1': '281[5/5]q4 6q4 2q4 2q4 6q3 283[3/3]q2 2q1 6q0',
    'prefetch-src=vec-depth=5-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=5-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=vec-depth=5-deskew=1-ahead=1-keep=0': '281q4 271q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=vec-depth=5-deskew=1-ahead=1-keep=1': '282q4 272q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=f64-depth=1-deskew=0-ahead=0-keep=0': '280[1/1]q0 270[1/1]q0 282[1/1]q0 282[1/1]q0 286[1/1]q0 282[1/1]q0 282[1/1]q0 286[1/1]q0',
    'prefetch-src=f64-depth=1-deskew=0-ahead=0-keep=1': '281[1/1]q0 271[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0',
    'prefetch-src=f64-depth=1-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=1-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=1-deskew=1-ahead=1-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=1-deskew=1-ahead=1-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=5-deskew=0-ahead=0-keep=0': '280[5/5]q4 6q4 2q4 2q4 6q3 282[3/3]q2 2q1 6q0',
    'prefetch-src=f64-depth=5-deskew=0-ahead=0-keep=1': '281[5/5]q4 6q4 2q4 2q4 6q3 283[3/3]q2 2q1 6q0',
    'prefetch-src=f64-depth=5-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=5-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f64-depth=5-deskew=1-ahead=1-keep=0': '281q4 271q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=f64-depth=5-deskew=1-ahead=1-keep=1': '282q4 272q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=f32-depth=1-deskew=0-ahead=0-keep=0': '281[1/1]q0 271[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0 283[1/1]q0 283[1/1]q0 287[1/1]q0',
    'prefetch-src=f32-depth=1-deskew=0-ahead=0-keep=1': '282[1/1]q0 272[1/1]q0 284[1/1]q0 284[1/1]q0 288[1/1]q0 284[1/1]q0 284[1/1]q0 288[1/1]q0',
    'prefetch-src=f32-depth=1-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=1-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=1-deskew=1-ahead=1-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=1-deskew=1-ahead=1-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=5-deskew=0-ahead=0-keep=0': '281[5/5]q4 6q4 2q4 2q4 6q3 283[3/3]q2 2q1 6q0',
    'prefetch-src=f32-depth=5-deskew=0-ahead=0-keep=1': '282[5/5]q4 6q4 2q4 2q4 6q3 284[3/3]q2 2q1 6q0',
    'prefetch-src=f32-depth=5-deskew=1-ahead=0-keep=0': '281q0 271q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=5-deskew=1-ahead=0-keep=1': '282q0 272q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetch-src=f32-depth=5-deskew=1-ahead=1-keep=0': '281q4 271q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=f32-depth=5-deskew=1-ahead=1-keep=1': '282q4 272q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetch-src=cuda32-depth=1-deskew=0-ahead=0-keep=0': '286[1/0]q0 276[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0',
    'prefetch-src=cuda32-depth=1-deskew=0-ahead=0-keep=1': '287[1/0]q0 277[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0',
    'prefetch-src=cuda32-depth=1-deskew=1-ahead=0-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda32-depth=1-deskew=1-ahead=0-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda32-depth=1-deskew=1-ahead=1-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda32-depth=1-deskew=1-ahead=1-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda32-depth=5-deskew=0-ahead=0-keep=0': '286[5/0]q4 6q4 2q4 2q4 6q3 288[3/0]q2 2q1 6q0',
    'prefetch-src=cuda32-depth=5-deskew=0-ahead=0-keep=1': '287[5/0]q4 6q4 2q4 2q4 6q3 289[3/0]q2 2q1 6q0',
    'prefetch-src=cuda32-depth=5-deskew=1-ahead=0-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda32-depth=5-deskew=1-ahead=0-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda32-depth=5-deskew=1-ahead=1-keep=0': '302q4 276q4 289q4 289q4 289q3 285q2 285q1 289q0',
    'prefetch-src=cuda32-depth=5-deskew=1-ahead=1-keep=1': '307q4 277q4 291q4 291q4 290q3 286q2 286q1 290q0',
    'prefetch-src=cuda64-depth=1-deskew=0-ahead=0-keep=0': '282[1/0]q0 272[1/0]q0 284[1/0]q0 284[1/0]q0 288[1/0]q0 284[1/0]q0 284[1/0]q0 288[1/0]q0',
    'prefetch-src=cuda64-depth=1-deskew=0-ahead=0-keep=1': '283[1/0]q0 273[1/0]q0 285[1/0]q0 285[1/0]q0 289[1/0]q0 285[1/0]q0 285[1/0]q0 289[1/0]q0',
    'prefetch-src=cuda64-depth=1-deskew=1-ahead=0-keep=0': '282q0 272q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda64-depth=1-deskew=1-ahead=0-keep=1': '283q0 273q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda64-depth=1-deskew=1-ahead=1-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda64-depth=1-deskew=1-ahead=1-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda64-depth=5-deskew=0-ahead=0-keep=0': '282[5/0]q4 6q4 2q4 2q4 6q3 284[3/0]q2 2q1 6q0',
    'prefetch-src=cuda64-depth=5-deskew=0-ahead=0-keep=1': '283[5/0]q4 6q4 2q4 2q4 6q3 285[3/0]q2 2q1 6q0',
    'prefetch-src=cuda64-depth=5-deskew=1-ahead=0-keep=0': '282q0 272q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetch-src=cuda64-depth=5-deskew=1-ahead=0-keep=1': '283q0 273q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetch-src=cuda64-depth=5-deskew=1-ahead=1-keep=0': '302q4 276q4 289q4 289q4 289q3 285q2 285q1 289q0',
    'prefetch-src=cuda64-depth=5-deskew=1-ahead=1-keep=1': '307q4 277q4 291q4 291q4 290q3 286q2 286q1 290q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=0': '284[1/1]q0 274[1/1]q0 286[1/1]q0 286[1/1]q0 290[1/1]q0 286[1/1]q0 286[1/1]q0 290[1/1]q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=1': '285[1/1]q0 275[1/1]q0 287[1/1]q0 287[1/1]q0 291[1/1]q0 287[1/1]q0 287[1/1]q0 291[1/1]q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=0': '284q0 274q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=1': '285q0 275q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=0': '284q0 274q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=1': '285q0 275q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=0': '284[5/5]q4 6q4 2q4 2q4 6q3 286[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=1': '285[5/5]q4 6q4 2q4 2q4 6q3 287[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=0': '284q0 274q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=1': '285q0 275q0 285q0 285q0 289q0 285q0 285q0 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=0': '284q4 274q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=host-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=1': '285q4 275q4 285q4 285q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=0': '281[1/1]q0 303[1/1]q0 299[1/1]q0 299[1/1]q0 303[1/1]q0 299[1/1]q0 299[1/1]q0 303[1/1]q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=1': '282[1/1]q0 304[1/1]q0 300[1/1]q0 300[1/1]q0 304[1/1]q0 300[1/1]q0 300[1/1]q0 304[1/1]q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=0': '281q0 303q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=1': '282q0 304q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=0': '281q0 303q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=1': '282q0 304q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=0': '297[5/5]q4 6q4 2q4 2q4 6q3 299[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=1': '298[5/5]q4 6q4 2q4 2q4 6q3 300[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=0': '281q0 303q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=1': '282q0 304q0 301q0 305q0 285q0 301q0 301q0 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=0': '281q4 303q4 301q4 305q4 285q3 301q2 301q1 305q0',
    'prefetchRecords-src=host-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=1': '282q4 304q4 301q4 305q4 285q3 301q2 301q1 305q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=0-ahead=0-keep=0': '286[1/1]q0 276[1/1]q0 288[1/1]q0 288[1/1]q0 292[1/1]q0 288[1/1]q0 288[1/1]q0 292[1/1]q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=0-ahead=0-keep=1': '287[1/1]q0 277[1/1]q0 289[1/1]q0 289[1/1]q0 293[1/1]q0 289[1/1]q0 289[1/1]q0 293[1/1]q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=0-keep=0': '286q0 276q0 288q0 288q0 292q0 288q0 288q0 292q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=0-keep=1': '287q0 277q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=1-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=1-keep=1': '287q0 277q0 290q0 290q0 294q0 290q0 290q0 294q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=0-ahead=0-keep=0': '286[5/5]q4 6q4 2q4 2q4 6q3 288[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=0-ahead=0-keep=1': '287[5/5]q4 6q4 2q4 2q4 6q3 289[3/3]q2 2q1 6q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=0-keep=0': '286q0 276q0 288q0 288q0 292q0 288q0 288q0 292q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=0-keep=1': '287q0 277q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=1-keep=0': '302q4 276q4 289q4 289q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=host-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=1-keep=1': '307q4 277q4 290q4 290q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=0': '286[1/0]q0 276[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=1': '287[1/0]q0 277[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=0': '286[5/0]q4 6q4 2q4 2q4 6q3 288[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=1': '287[5/0]q4 6q4 2q4 2q4 6q3 289[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=1': '287q0 277q0 291q0 291q0 295q0 291q0 291q0 295q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=0': '302q4 276q4 289q4 289q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=dev-gate=1-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=1': '307q4 277q4 291q4 291q4 290q3 286q2 286q1 290q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=0': '286[1/0]q0 308[1/0]q0 304[1/0]q0 304[1/0]q0 308[1/0]q0 304[1/0]q0 304[1/0]q0 308[1/0]q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=0-ahead=0-keep=1': '287[1/0]q0 309[1/0]q0 305[1/0]q0 305[1/0]q0 309[1/0]q0 305[1/0]q0 305[1/0]q0 309[1/0]q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=0': '286q0 308q0 305q0 309q0 289q0 305q0 305q0 309q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=0-keep=1': '287q0 309q0 307q0 311q0 291q0 307q0 307q0 311q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=0': '286q0 308q0 305q0 309q0 289q0 305q0 305q0 309q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=1-deskew=1-ahead=1-keep=1': '287q0 309q0 307q0 311q0 291q0 307q0 307q0 311q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=0': '302[5/0]q4 6q4 2q4 2q4 6q3 304[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=0-ahead=0-keep=1': '303[5/0]q4 6q4 2q4 2q4 6q3 305[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=0': '286q0 308q0 305q0 309q0 289q0 305q0 305q0 309q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=0-keep=1': '287q0 309q0 307q0 311q0 291q0 307q0 307q0 311q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=0': '302q4 308q4 305q4 309q4 285q3 301q2 301q1 305q0',
    'prefetchRecords-src=dev-gate=0-corr=0-time=0-depth=5-deskew=1-ahead=1-keep=1': '307q4 309q4 307q4 311q4 286q3 302q2 302q1 306q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=0-ahead=0-keep=0': '286[1/0]q0 276[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0 288[1/0]q0 288[1/0]q0 292[1/0]q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=0-ahead=0-keep=1': '287[1/0]q0 277[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0 289[1/0]q0 289[1/0]q0 293[1/0]q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=0-keep=0': '286q0 276q0 288q0 288q0 292q0 288q0 288q0 292q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=0-keep=1': '287q0 277q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=1-keep=0': '286q0 276q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=1-deskew=1-ahead=1-keep=1': '287q0 277q0 290q0 290q0 294q0 290q0 290q0 294q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=0-ahead=0-keep=0': '286[5/0]q4 6q4 2q4 2q4 6q3 288[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=0-ahead=0-keep=1': '287[5/0]q4 6q4 2q4 2q4 6q3 289[3/0]q2 2q1 6q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=0-keep=0': '286q0 276q0 288q0 288q0 292q0 288q0 288q0 292q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=0-keep=1': '287q0 277q0 289q0 289q0 293q0 289q0 289q0 293q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=1-keep=0': '302q4 276q4 289q4 289q4 289q3 285q2 285q1 289q0',
    'prefetchRecords-src=dev-gate=1-corr=1-time=1-depth=5-deskew=1-ahead=1-keep=1': '307q4 277q4 290q4 290q4 289q3 285q2 285q1 289q0',
    'mixed-mix=packed-depth=5-keep=0': '280[1/1]q4 271[1/1]q4 282[2/2]q4 2q4 287[2/2]q3 2q2 282[2/2]q1 6q0',
    'mixed-mix=packed-depth=5-keep=1': '281[1/1]q4 272[1/1]q4 283[2/2]q4 2q4 288[2/2]q3 2q2 283[2/2]q1 6q0',
    'mixed-mix=packed-depth=8-keep=0': '280[1/1]q7 271[1/1]q6 282[2/2]q5 2q4 287[2/2]q3 2q2 282[2/2]q1 6q0',
    'mixed-mix=packed-depth=8-keep=1': '281[1/1]q7 272[1/1]q6 283[2/2]q5 2q4 288[2/2]q3 2q2 283[2/2]q1 6q0',
    'mixed-mix=records-depth=5-keep=0': '300[2/2]q4 6q4 288[2/0]q4 2q4 292[1/0]q3 286[1/1]q2 288[1/0]q1 292[1/0]q0',
    'mixed-mix=records-depth=5-keep=1': '301[2/2]q4 6q4 289[2/0]q4 2q4 293[1/0]q3 287[1/1]q2 289[1/0]q1 293[1/0]q0',
    'mixed-mix=records-depth=8-keep=0': '300[2/2]q7 6q6 288[2/0]q5 2q4 292[1/0]q3 286[1/1]q2 288[1/0]q1 292[1/0]q0',
    'mixed-mix=records-depth=8-keep=1': '301[2/2]q7 6q6 289[2/0]q5 2q4 293[1/0]q3 287[1/1]q2 289[1/0]q1 293[1/0]q0',
    'mixed-mix=all-depth=5-keep=0': '280[1/1]q4 274[1/1]q4 282[1/1]q4 288[1/0]q4 287[1/1]q3 286[2/2]q2 2q1 288[1/0]q0',
    'mixed-mix=all-depth=5-keep=1': '281[1/1]q4 275[1/1]q4 283[1/1]q4 289[1/0]q4 288[1/1]q3 287[2/2]q2 2q1 289[1/0]q0',
    'mixed-mix=all-depth=8-keep=0': '280[1/1]q7 274[1/1]q6 282[1/1]q5 288[1/0]q4 287[1/1]q3 286[2/2]q2 2q1 288[1/0]q0',
    'mixed-mix=all-depth=8-keep=1': '281[1/1]q7 275[1/1]q6 283[1/1]q5 289[1/0]q4 288[1/1]q3 287[2/2]q2 2q1 289[1/0]q0',
}


@pytest.fixture(scope="module")
def scans(built):
    return Scans(_sequence())


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES, ids=route_id)
def test_route_census(scans, route):
    assert run(route, scans) == CENSUS[route_id(route)]


def record(outputs=None):
    """Runs every route; prints the census table, and with `outputs` writes a digest of every route's results there"""
    import __graft_entry__ as g
    g.build()
    s = Scans(_sequence())
    table, digests = {}, {}
    for r in ROUTES:
        h = hashlib.sha256()
        table[route_id(r)] = run(r, s, h)
        digests[route_id(r)] = h.hexdigest()
    print("CENSUS = {")
    for k, v in table.items():
        print(f"    {k!r}: {v!r},")
    print("}")
    if outputs:
        with open(outputs, "w") as f:
            json.dump(dict(census=table, digests=digests), f, indent=1)


if __name__ == "__main__":
    record(sys.argv[1] if len(sys.argv) > 1 else None)
