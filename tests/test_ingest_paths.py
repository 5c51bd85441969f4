"""Launch census of every route a scan takes to the device: madicp_ingest (float32, float64), host and device records
(gated and ungated), host and device plans consumed by madicp_ingest_plan, and madtree_gpu_build.  Each route runs
without a deskew, with the azimuth deskew and with the time-stamp deskew where it takes one, with the vertical
correction off and on, and with kept clouds off and on.  The counts are Registrar.kernel_launches() deltas recorded on
an H100; a refactor of the ingest must launch the same kernels, so it leaves every count as it is.  Clouds, indices,
trees and poses of these routes are checked bit for bit elsewhere (test_records.py, test_gpu_device_input.py,
test_time_deskew.py, test_gpu_cloud_out.py)."""
import itertools
from unittest import mock

import numpy as np
import pytest

from mad_icp_b200 import engine, records, synth

GATE = dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False)
DSK = dict(deskew=True, T_prev=synth.pose_xyyaw(0.0, 0.0, 0.0), T_now=synth.pose_xyyaw(0.8, 0.05, 0.03), sensor_hz=10.0)
ONOFF = (False, True)


def _records():
    """KITTI float32 N x 4 records on a street, column 3 a time stamp in seconds"""
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.0, 1.0, 0.0), beams=16, azimuths=512, seed=100, r_min=0.0, r_max=np.inf)
    a = np.zeros((p.shape[0], 4), np.float32)
    a[:, :3] = p
    a[:, 3] = np.linspace(-0.1, 0.0, p.shape[0])
    return a


def _ungated(describe):
    """records.describe without a range gate (what Registrar.ingest_records never asks for itself)"""
    def wrap(*args, **kw):
        d = describe(*args, **kw)
        d.range_mode = records.RANGE_NONE
        return d
    return wrap


ROUTES = (
    [("ingest", dt, dsk, keep) for dt, dsk, keep in itertools.product(("f32", "f64"), ("none", "azimuth"), ONOFF)]
    + [("records", src, gate, dsk, corr, keep) for src, gate, dsk, corr, keep in
       itertools.product(("host", "dev"), ("gated", "ungated"), ("none", "azimuth", "time"), ONOFF, ONOFF)]
    + [("plan", src, kind, dsk, corr, keep) for src, kind, dsk, corr, keep in
       itertools.product(("host", "dev"), ("azimuth", "time"), ONOFF, ONOFF, ONOFF)]
    + [("build", keep) for keep in ONOFF])


def route_id(route):
    return "-".join(str(x) for x in route)


def launches(reg, a, route):
    """kernel launches of one run of `route` on the records `a`"""
    import torch
    kind, keep = route[0], route[-1]
    src = torch.from_numpy(a).cuda() if kind in ("records", "plan") and route[1] == "dev" else a
    reg.keep_cloud(keep)
    try:
        before = reg.kernel_launches
        if kind == "ingest":
            _, dt, dsk, _ = route
            xyz = np.ascontiguousarray(a[:, :3], np.float32 if dt == "f32" else np.float64)
            reg.ingest(xyz, **(DSK if dsk == "azimuth" else {}))
        elif kind == "records":
            _, _, gate, dsk, corr, _ = route
            kw = dict(GATE, apply_correction=corr, **({} if dsk == "none" else DSK))
            if dsk == "time":
                kw["time_field"] = 3
            with mock.patch.object(engine, "describe", _ungated(records.describe) if gate == "ungated" else records.describe):
                reg.ingest_records(src, **kw)
        elif kind == "plan":
            _, _, plan_kind, dsk, corr, _ = route
            plan = reg.plan_records(src, **GATE, apply_correction=corr, **({"time_field": 3} if plan_kind == "time" else {}))
            reg.ingest_plan(plan, **(DSK if dsk else {}))
        else:
            reg.build_tree(np.ascontiguousarray(a[:, :3], np.float64))
        if route[1] == "dev":
            torch.cuda.synchronize()
        return reg.kernel_launches - before
    finally:
        reg.keep_cloud(False)


# route id -> launches, recorded on an NVIDIA H100 80GB HBM3 (700 W power limit)
CENSUS = {
    "ingest-f32-none-False": 1, "ingest-f32-none-True": 2, "ingest-f32-azimuth-False": 1, "ingest-f32-azimuth-True": 1,
    "ingest-f64-none-False": 1, "ingest-f64-none-True": 2, "ingest-f64-azimuth-False": 1, "ingest-f64-azimuth-True": 1,
    "records-host-gated-none-False-False": 4, "records-host-gated-none-False-True": 5,
    "records-host-gated-none-True-False": 4, "records-host-gated-none-True-True": 5,
    "records-host-gated-azimuth-False-False": 1, "records-host-gated-azimuth-False-True": 1,
    "records-host-gated-azimuth-True-False": 1, "records-host-gated-azimuth-True-True": 1,
    "records-host-gated-time-False-False": 4, "records-host-gated-time-False-True": 5,
    "records-host-gated-time-True-False": 4, "records-host-gated-time-True-True": 5,
    "records-host-ungated-none-False-False": 1, "records-host-ungated-none-False-True": 2,
    "records-host-ungated-none-True-False": 1, "records-host-ungated-none-True-True": 2,
    "records-host-ungated-azimuth-False-False": 1, "records-host-ungated-azimuth-False-True": 1,
    "records-host-ungated-azimuth-True-False": 1, "records-host-ungated-azimuth-True-True": 1,
    "records-host-ungated-time-False-False": 4, "records-host-ungated-time-False-True": 5,
    "records-host-ungated-time-True-False": 4, "records-host-ungated-time-True-True": 5,
    "records-dev-gated-none-False-False": 4, "records-dev-gated-none-False-True": 5,
    "records-dev-gated-none-True-False": 4, "records-dev-gated-none-True-True": 5,
    "records-dev-gated-azimuth-False-False": 5, "records-dev-gated-azimuth-False-True": 7,
    "records-dev-gated-azimuth-True-False": 5, "records-dev-gated-azimuth-True-True": 7,
    "records-dev-gated-time-False-False": 4, "records-dev-gated-time-False-True": 5,
    "records-dev-gated-time-True-False": 4, "records-dev-gated-time-True-True": 5,
    "records-dev-ungated-none-False-False": 4, "records-dev-ungated-none-False-True": 5,
    "records-dev-ungated-none-True-False": 4, "records-dev-ungated-none-True-True": 5,
    "records-dev-ungated-azimuth-False-False": 5, "records-dev-ungated-azimuth-False-True": 7,
    "records-dev-ungated-azimuth-True-False": 5, "records-dev-ungated-azimuth-True-True": 7,
    "records-dev-ungated-time-False-False": 4, "records-dev-ungated-time-False-True": 5,
    "records-dev-ungated-time-True-False": 4, "records-dev-ungated-time-True-True": 5,
    "plan-host-azimuth-False-False-False": 4, "plan-host-azimuth-False-False-True": 5,
    "plan-host-azimuth-False-True-False": 4, "plan-host-azimuth-False-True-True": 5,
    "plan-host-azimuth-True-False-False": 1, "plan-host-azimuth-True-False-True": 1,
    "plan-host-azimuth-True-True-False": 1, "plan-host-azimuth-True-True-True": 1,
    "plan-host-time-False-False-False": 4, "plan-host-time-False-False-True": 5, "plan-host-time-False-True-False": 4,
    "plan-host-time-False-True-True": 5, "plan-host-time-True-False-False": 5, "plan-host-time-True-False-True": 6,
    "plan-host-time-True-True-False": 5, "plan-host-time-True-True-True": 6, "plan-dev-azimuth-False-False-False": 4,
    "plan-dev-azimuth-False-False-True": 5, "plan-dev-azimuth-False-True-False": 4,
    "plan-dev-azimuth-False-True-True": 5, "plan-dev-azimuth-True-False-False": 5,
    "plan-dev-azimuth-True-False-True": 7, "plan-dev-azimuth-True-True-False": 5, "plan-dev-azimuth-True-True-True": 7,
    "plan-dev-time-False-False-False": 4, "plan-dev-time-False-False-True": 5, "plan-dev-time-False-True-False": 4,
    "plan-dev-time-False-True-True": 5, "plan-dev-time-True-False-False": 5, "plan-dev-time-True-False-True": 6,
    "plan-dev-time-True-True-False": 5, "plan-dev-time-True-True-True": 6, "build-False": 264, "build-True": 265
}


@pytest.fixture(scope="module")
def scan_and_reg(built):
    from mad_icp_b200 import Registrar
    return _records(), Registrar(device=0, max_keyframes=4)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES, ids=route_id)
def test_launch_census(scan_and_reg, route):
    a, reg = scan_and_reg
    assert launches(reg, a, route) == CENSUS[route_id(route)]
