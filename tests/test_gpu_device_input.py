"""Scans that already live on the GPU: CUDA tensors handed to the record entry points are read in place (the _dev calls
of include/madicp_b200.h) and must give what the same arrays give from host memory, bit for bit -- kept clouds, device
trees, plans, forests, whole Pipeline sequences and the tree search.  Every device array here is
torch.from_numpy(a).cuda() of the host array it is compared with."""
import ctypes as C
import os

import numpy as np
import pytest

from mad_icp_b200 import MadIcpError, _capi, records, synth
from util import bits_equal

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GATE = dict(min_range=0.7, max_range=120.0)


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _scan(seed, beams=32, azimuths=1024):
    """a synthetic sweep without the range gate + NaN / zero / too-near / too-far rows, N x 3 float64"""
    scene = synth.StreetScene(seed=7)
    p = synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), beams, azimuths, seed=seed, r_min=0.0,
                         r_max=np.inf)
    rs = np.random.RandomState(seed)
    bad = np.concatenate([np.full((7, 3), np.nan), np.zeros((5, 3)), rs.normal(size=(40, 3)) * 0.2,
                          rs.normal(size=(40, 3)) * 300, [[np.nan, 1, 2], [3, np.nan, 4], [5, 6, np.nan]]])
    return np.insert(p, np.sort(rs.randint(0, p.shape[0], size=bad.shape[0])), bad, axis=0)


def _records(p, layout, dtype, shift=0):
    """(host view, device view) of the same records: KITTI (x y z i, 16 / 32-byte rows) or Ouster-like 48-byte rows (x, y,
    z at bytes 16 / 8 of the row); shift: the base address moved by that many bytes (a storage offset), in both"""
    cols, at = {("kitti", 4): (4, 0), ("kitti", 8): (4, 0), ("ouster", 4): (12, 4), ("ouster", 8): (6, 1)}[
        (layout, np.dtype(dtype).itemsize)]
    e = np.dtype(dtype).itemsize
    flat = np.zeros(p.shape[0] * cols + shift // e, dtype)
    a = flat[shift // e:].reshape(-1, cols)
    a[:, at:at + 3] = p
    a[:, at + 3:] = 0.5
    t = torch.from_numpy(flat).cuda()[shift // e:].view(-1, cols)
    assert t.data_ptr() % 16 == shift  # (the caching allocator hands out 512-byte aligned blocks)
    return a[:, at:at + 3], t[:, at:at + 3]


def _gate(layout):
    return dict(GATE, inclusive=layout == "kitti", drop_nan=layout != "kitti")


DESKEW = dict(deskew=True, T_prev=synth.pose_xyyaw(0, 0, 0), T_now=synth.pose_xyyaw(0.8, 0.05, 0.03), sensor_hz=10.0,
              num_threads=4)


def _tree(dt):
    r, lr = dt.records(), dt.leaf_records()
    return r, lr


def _same_tree(a, b):
    assert all(bits_equal(a[0][k], b[0][k]) for k in ("mean", "dir", "bbox0"))
    assert (a[0]["link"] == b[0]["link"]).all() and (a[0]["num_points"] == b[0]["num_points"]).all() and (a[1] == b[1]).all()


CASES = [(lay, dt, s) for lay in ("kitti", "ouster") for dt in (np.float32, np.float64)
         for s in ((0, 4, 8, 12) if dt == np.float32 else (0, 8))]


@pytest.mark.parametrize("layout,dtype,shift", CASES)
@pytest.mark.parametrize("corr", [False, True])
@pytest.mark.parametrize("deskew", [False, True])
def test_ingest_and_tree_equal_host(reg, layout, dtype, shift, corr, deskew):
    h, d = _records(_scan(3), layout, dtype, shift)
    kw = dict(_gate(layout), apply_correction=corr, **(DESKEW if deskew else {}))
    want = reg.ingest_records(h, want_points=True, **kw)
    want_tree = _tree(reg.build_tree())
    got = reg.ingest_records(d, want_points=True, **kw)
    got_tree = _tree(reg.build_tree())
    assert got.shape == want.shape and bits_equal(got, want)
    assert reg.ingest_records(d, **kw) == want.shape[0]
    _same_tree(got_tree, want_tree)


@pytest.mark.parametrize("count", [1, 7, 32])
def test_forest_of_device_scans(reg, count):
    scans = []
    for k in range(count):
        p = _scan(20 + k)[: 4000 + 997 * k]  # mixed sizes
        scans.append(_records(p, "kitti" if k % 2 else "ouster", np.float32, 4 * (k % 4)))
    gate = dict(GATE)
    corr = [bool(k % 3 == 0) for k in range(count)]
    want = [_tree(t) for t in reg.build_trees_records([h for h, _ in scans], apply_correction=corr, **gate)]
    got = [_tree(t) for t in reg.build_trees_records([d for _, d in scans], apply_correction=corr, **gate)]
    for g, w in zip(got, want):
        _same_tree(g, w)
    if count > 3:  # a scan the gate leaves empty fails the call with its index; the next call works
        bad = list(scans)
        bad[3] = _records(np.full((500, 3), 500.0), "kitti", np.float32)
        with pytest.raises(MadIcpError, match="scan 3 has no point inside the range gate"):
            reg.build_trees_records([d for _, d in bad], **gate)
        again = [_tree(t) for t in reg.build_trees_records([d for _, d in scans], apply_correction=corr, **gate)]
        for g, w in zip(again, want):
            _same_tree(g, w)


@pytest.mark.parametrize("layout", ["kitti", "ouster"])
@pytest.mark.parametrize("corr", [False, True])
@pytest.mark.parametrize("deskew", [False, True])
def test_plans_of_device_records(reg, layout, corr, deskew):
    h, d = _records(_scan(9), layout, np.float32, 4 if layout == "kitti" else 0)
    kw = dict(_gate(layout), apply_correction=corr)
    ing = dict(DESKEW) if deskew else {}
    ing.pop("num_threads", None)
    want = reg.ingest_plan(reg.plan_records(h, num_threads=2, **kw), want_points=True, **ing)
    want_tree = _tree(reg.build_tree())
    plans = [reg.plan_records(d, num_threads=2, **kw) for _ in range(3)]  # several in flight, consumed in any order
    for pl in (plans[1], plans[0]):
        got = reg.ingest_plan(pl, want_points=True, **ing)
        assert bits_equal(got, want)
        _same_tree(_tree(reg.build_tree()), want_tree)
    plans[2].free()


def _pipeline(**kw):
    from mad_icp_b200.pybind.pypeline import Pipeline
    args = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
                num_threads=4, realtime=False)
    args.update(kw)
    return Pipeline(**args)


def _sequence(n):
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        rs = np.random.RandomState(i)
        bad = np.concatenate([np.full((3, 3), np.nan), rs.normal(size=(20, 3)) * 0.3, rs.normal(size=(20, 3)) * 400.0])
        p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=bad.shape[0])), bad, axis=0)
        a = np.zeros((p.shape[0], 4), np.float32)
        a[:, :3], a[:, 3] = p, 0.5
        out.append(a)
    return out


SEQ = {}


def _seq():
    if not SEQ:
        recs = _sequence(40)
        clouds = [np.ascontiguousarray(a[:, :3][records.range_mask(a[:, :3], **GATE).astype(bool)]) for a in recs]
        SEQ["records"] = [(a[:, :3], torch.from_numpy(a).cuda()[:, :3]) for a in recs]
        SEQ["compute"] = [(c, torch.from_numpy(c).cuda()) for c in clouds]
    return SEQ


def _run(api, deskew, hz, depth, dev, gpu_build=True):
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        p = _pipeline(sensor_hz=hz, deskew=deskew)
    finally:
        os.environ.pop("MADICP_GPU_BUILD")
    seq = _seq()[api]
    out = []
    for i in range(len(seq)):
        if depth and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + depth, len(seq))):
                x = seq[k][1 if dev else 0]
                ok = p.prefetchRecords(x, deskew_ahead=True, **GATE) if api == "records" else p.prefetch(x, deskew_ahead=True)
                assert ok == gpu_build
        x = seq[i][1 if dev else 0]
        if api == "records":
            p.computeRecords(i / hz, x, **GATE)
        else:
            p.compute(i / hz, x)
        out.append((p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())))
    return out


def _same_run(got, want):
    assert sum(o[1] for o in want) >= 3
    for i, (g, w) in enumerate(zip(got, want)):
        assert bits_equal(g[0], w[0]), i
        assert g[1:] == w[1:], i


@pytest.mark.parametrize("api", ["records", "compute"])
@pytest.mark.parametrize("deskew,hz", [(False, 10.0), (True, 10.0), (True, 20.0)])
def test_pipeline_sequences_equal_host(built, api, deskew, hz):
    want = _run(api, deskew, hz, 0, dev=False)
    for depth in (0, 1, 5, 32):
        _same_run(_run(api, deskew, hz, depth, dev=True), want)
    host_built = _run(api, deskew, hz, 0, dev=False, gpu_build=False)
    _same_run(_run(api, deskew, hz, 5, dev=True, gpu_build=False), host_built)


def test_producer_stream_is_waited_for(reg):
    """records written on a side stream behind a long sleep and handed over without a synchronisation"""
    h, _ = _records(_scan(4), "kitti", np.float32)
    src = torch.from_numpy(np.ascontiguousarray(h)).cuda()
    want = reg.ingest_records(h, want_points=True, **GATE)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.full_like(src, float("nan"))
        torch.cuda._sleep(200_000_000)
        t.copy_(src)
        got = reg.ingest_records(t, want_points=True, **GATE)  # (torch's current stream: the side stream)
    assert bits_equal(got, want)
    assert records.describe(t, stream=side, **GATE).stream == side.cuda_stream
    # the same through the Pipeline
    p1, p2 = _pipeline(), _pipeline()
    p1.computeRecords(0.0, h, **GATE)
    with torch.cuda.stream(side):
        t3 = torch.full_like(src, float("nan"))
        torch.cuda._sleep(200_000_000)
        t3.copy_(src)
        p2.computeRecords(0.0, t3, **GATE)
    assert bits_equal(np.asarray(p1.currentLeaves()), np.asarray(p2.currentLeaves()))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_search_cloud_arrays_on_device(built, dtype):
    from mad_icp_b200.pybind.pymadtree import MADtree
    t = MADtree()
    t.build(np.ascontiguousarray(_scan(6)[records.range_mask(_scan(6), **GATE).astype(bool)]), 0.2, 0.1, 2)
    q = (np.random.RandomState(1).uniform(-40, 40, size=(20000, 3))).astype(dtype)
    want = t.searchCloudArrays(q)
    qd = torch.from_numpy(q).cuda()
    got = t.searchCloudArrays(qd)
    for g, w in zip(got, want):
        assert isinstance(g, torch.Tensor) and g.dtype == torch.float64 and g.device == qd.device
        assert bits_equal(g.cpu().numpy(), w)
    wide = torch.zeros((20000, 4), dtype=qd.dtype, device="cuda")
    wide[:, :3] = qd
    got = t.searchCloudArrays(wide[:, :3])  # a strided view, read in place
    for g, w in zip(got, want):
        assert bits_equal(g.cpu().numpy(), w)


def test_host_pointer_and_other_device_are_rejected(reg):
    h, _ = _records(_scan(2), "kitti", np.float32)
    d = records.describe(h, **GATE)
    kept = C.c_int64(0)
    rc = _capi.lib().madicp_ingest_points_dev(reg._h, C.byref(d), None, 0, None, None, 10.0, 1, None, C.byref(kept), None)
    assert rc == -1 and "device memory" in _capi.lib().madicp_last_error().decode()
    pinned = torch.from_numpy(np.ascontiguousarray(h)).pin_memory()
    d = records.describe(np.ascontiguousarray(h), **GATE)
    d.data = pinned.data_ptr()
    assert _capi.lib().madicp_ingest_points_dev(reg._h, C.byref(d), None, 0, None, None, 10.0, 1, None, None, None) == -1
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU: the other-device case needs two")
    other = torch.from_numpy(np.ascontiguousarray(h)).to("cuda:1")
    with pytest.raises(MadIcpError, match="another device"):
        reg.ingest_records(other, **GATE)
