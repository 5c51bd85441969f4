"""Leaf means gathered on the device (madtree_gpu_leaf_means, madtree_gpu_leaf_means_dev): the scan's and the model's
leaves as numpy arrays or CUDA tensors, bit for bit what currentLeaves() / modelLeaves() return and what the host-built
path (MADICP_GPU_BUILD=0, FlatTree) computes.  The CPU section checks the bindings and the argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

from mad_icp_b200 import MadIcpError, _capi, synth
from util import bits_equal


# ---------------------------------------------------------------------------------------------------------- CPU
def test_leaf_gather_symbols_are_bound(built):
    lib = _capi.lib()
    for name in ("madtree_gpu_leaf_means", "madtree_gpu_leaf_means_dev"):
        assert name in _capi.SYMBOLS and getattr(lib, name).argtypes
    from mad_icp_b200.pybind.pypeline import Pipeline
    for name in ("currentLeavesArray", "modelLeavesArray"):
        assert hasattr(Pipeline, name)


def test_leaf_gather_rejects_bad_arguments_without_a_gpu(built):
    lib = _capi.lib()
    one = (C.c_void_p * 1)()
    out = np.empty((4, 3))
    for fn, extra in ((lib.madtree_gpu_leaf_means, ()), (lib.madtree_gpu_leaf_means_dev, (None,))):
        assert fn(None, None, 1, _capi.as_d(out), *extra) == -1  # null table
        assert "count >= 0" in lib.madicp_last_error().decode()
        assert fn(one, None, -1, _capi.as_d(out), *extra) == -1  # count < 0
        assert fn(one, None, 1, None, *extra) == -1  # null output
        assert "no output" in lib.madicp_last_error().decode()
        assert fn(one, None, 1, _capi.as_d(out), *extra) == -1  # a NULL tree
        assert "is NULL" in lib.madicp_last_error().decode()
        assert fn(one, None, 0, _capi.as_d(out), *extra) == 0  # count == 0: nothing to do


# ---------------------------------------------------------------------------------------------------------- GPU
GATE = dict(min_range=0.7, max_range=120.0)


def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


def _cloud(seed, beams=32, azimuths=1024):
    scene = synth.StreetScene(seed=7)
    return synth.lidar_scan(scene, synth.pose_xyyaw(0.4 * seed, 1.0, 0.02 * seed), beams, azimuths, seed=seed)


def _tilted(x, y, yaw, z, rx, ry):
    T = synth.pose_xyyaw(x, y, yaw, z=z)
    T[:3, :3] = T[:3, :3] @ synth.euler_xyz(rx, ry, 0.0)
    return T


POSES = [_tilted(3.5, -1.25, 0.3, 0.2, 0.01, -0.02), synth.pose_xyyaw(-12.0, 4.0, -1.1)]


@pytest.mark.gpu
@pytest.mark.parametrize("pose", [None, 0, 1])
def test_device_tree_leaf_means_equal_flat_tree(reg, pose):
    from mad_icp_b200 import FlatTree
    torch = _torch()
    c = _cloud(3)
    dt, ft = reg.build_tree(c), FlatTree(c)
    T = None if pose is None else POSES[pose]
    if T is not None:
        ft.apply_transform(T)
    want = ft.leaf_means()
    got = dt.leaf_means(T)
    assert got.shape == want.shape == (dt.num_leaves, 3) and bits_equal(got, want)
    gd = dt.leaf_means(T, device=True)
    assert isinstance(gd, torch.Tensor) and gd.dtype == torch.float64 and gd.device == torch.device("cuda", 0)
    assert bits_equal(gd.cpu().numpy(), want)


@pytest.mark.gpu
def test_batch_of_posed_and_unposed_trees_is_the_concatenation(reg):
    from mad_icp_b200.engine import leaf_means
    trees = [reg.build_tree(_cloud(s)) for s in (1, 2, 3, 4)]
    poses = [POSES[0], None, POSES[1], None]
    want = np.concatenate([t.leaf_means(T) for t, T in zip(trees, poses)])
    assert bits_equal(leaf_means(trees, poses), want)
    assert bits_equal(leaf_means(trees, poses, device=True).cpu().numpy(), want)
    assert bits_equal(leaf_means(trees), np.concatenate([t.leaf_means() for t in trees]))
    assert leaf_means([], device=False).shape == (0, 3)


@pytest.mark.gpu
def test_unposed_tree_keeps_negative_zero(reg):
    from mad_icp_b200 import FlatTree
    c = _cloud(5)
    c[c[:, 2] < np.quantile(c[:, 2], 0.2), 2] = -0.0  # the lowest points drop onto the plane z = -0.0
    c[::7, 0] = -0.0
    want = FlatTree(c).leaf_means()
    dt = reg.build_tree(c)
    for got in (dt.leaf_means(), dt.leaf_means(device=True).cpu().numpy()):
        assert bits_equal(got, want)
        assert (np.signbit(got) & (got == 0)).sum() > 10
    # (an identity pose is arithmetic: -0.0 + 0.0 = +0.0)
    posed = dt.leaf_means(np.eye(4))
    assert not (np.signbit(posed) & (posed == 0))[:, 2].any()


@pytest.mark.gpu
def test_bad_outputs_and_mixed_contexts_are_rejected(reg):
    from mad_icp_b200 import Registrar
    from mad_icp_b200.engine import leaf_means
    torch = _torch()
    lib = _capi.lib()
    dt = reg.build_tree(_cloud(2))
    tab = (C.c_void_p * 1)(dt._h)
    host = np.empty((dt.num_leaves, 3))
    assert lib.madtree_gpu_leaf_means_dev(tab, None, 1, C.c_void_p(host.ctypes.data), None) == -1
    assert "device memory" in lib.madicp_last_error().decode()
    buf = torch.empty(dt.num_leaves * 3 + 1, dtype=torch.float64, device="cuda")
    assert lib.madtree_gpu_leaf_means_dev(tab, None, 1, C.c_void_p(buf.data_ptr() + 4), None) == -1
    assert "aligned" in lib.madicp_last_error().decode()
    other = Registrar(device=0, max_keyframes=1)
    ot = other.build_tree(_cloud(4))
    for device in (False, True):
        with pytest.raises(MadIcpError, match="different contexts"):
            leaf_means([dt, ot], device=device)
    del ot


# ------------------------------------------------------------------------------------------------ pipelines
def _pipeline(deskew=False, gpu_build=True):
    from mad_icp_b200.pybind.pypeline import Pipeline
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        return Pipeline(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                        num_keyframes=4, num_threads=4, realtime=False)
    finally:
        os.environ.pop("MADICP_GPU_BUILD")


SEQ = []


def _seq():
    """40 scans along a street, 32 x 1024 rays, N x 3 float64 (the range gate already applied)"""
    if not SEQ:
        scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * 40)
        for i in range(40):
            base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
            SEQ.append(synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i))
    return SEQ


def _leaves(p):
    return np.asarray(p.currentLeaves()), np.asarray(p.modelLeaves())


def _host_run(deskew):
    """currentLeaves / modelLeaves after every scan of a host-built pipeline (the independent path)"""
    p = _pipeline(deskew, gpu_build=False)
    out = []
    for i, c in enumerate(_seq()):
        p.compute(0.1 * i, c)
        cur, model = _leaves(p)
        assert bits_equal(p.currentLeavesArray(), cur) and bits_equal(p.modelLeavesArray(), model)
        out.append((cur, model))
    dev = p.modelLeavesArray(device=True)  # (copied up once)
    assert bits_equal(dev.cpu().numpy(), out[-1][1])
    return out


HOST = {}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["compute", "prefetch", "deskew_ahead", "cuda_input"])
def test_pipeline_leaves_equal_lists_and_host_path(built, mode):
    torch = _torch()
    deskew = mode == "deskew_ahead"
    if deskew not in HOST:
        HOST[deskew] = _host_run(deskew)
    want = HOST[deskew]
    p = _pipeline(deskew)
    assert p.currentLeavesArray().shape == (0, 3) and p.modelLeavesArray().shape == (0, 3)
    assert tuple(p.modelLeavesArray(device=True).shape) == (0, 3)
    seq = _seq()
    dev = [torch.from_numpy(c).cuda() for c in seq] if mode == "cuda_input" else None
    updates = 0
    for i in range(len(seq)):
        if mode in ("prefetch", "deskew_ahead") and i >= 1 and p.prefetched() == 0:
            for k in range(i, min(i + 8, len(seq))):
                assert p.prefetch(seq[k], deskew_ahead=deskew)
        p.compute(0.1 * i, dev[i] if dev else seq[i])
        updates += bool(p.isMapUpdated())
        cur, model = _leaves(p)
        cur_a, model_a = p.currentLeavesArray(), p.modelLeavesArray()
        cur_d, model_d = p.currentLeavesArray(device=True), p.modelLeavesArray(device=True)
        assert isinstance(cur_a, np.ndarray) and cur_a.dtype == np.float64 and cur_a.shape == cur.shape
        assert model_d.dtype == torch.float64 and model_d.device == torch.device("cuda", 0)
        assert bits_equal(cur_a, cur) and bits_equal(model_a, model), i
        assert bits_equal(cur_d.cpu().numpy(), cur) and bits_equal(model_d.cpu().numpy(), model), i
        assert bits_equal(cur, want[i][0]) and bits_equal(model, want[i][1]), i
    assert updates > 5 and p.numKeyframes() == 4  # promotions and evictions both happened


@pytest.mark.gpu
def test_device_gather_waits_for_the_consumer_stream(built):
    torch = _torch()
    p = _pipeline()
    for i, c in enumerate(_seq()[:12]):
        p.compute(0.1 * i, c)
    want = p.modelLeavesArray()
    n = want.shape[0]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        junk = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        torch.cuda._sleep(200_000_000)
        junk.fill_(float("nan"))  # behind the sleep, in memory the gather's output is likely to reuse
        del junk
        got = p.modelLeavesArray(device=True)
        copy = got.clone()  # (ordered after the gather on the consumer stream, no host sync)
    side.synchronize()
    assert bits_equal(got.cpu().numpy(), want) and bits_equal(copy.cpu().numpy(), want)


@pytest.mark.gpu
def test_gather_with_the_next_scans_prefetched_is_the_current_scan(built):
    torch = _torch()
    seq = _seq()
    for deskew in (False, True):
        p = _pipeline(deskew)
        p.compute(0.0, seq[0])
        for i in range(1, 10):
            if p.prefetched() == 0:
                for k in range(i, min(i + 4, len(seq))):
                    assert p.prefetch(seq[k], deskew_ahead=True)
            p.compute(0.1 * i, seq[i])
            want_cur, want_model = _leaves(p)
            assert p.prefetched() > 0 or i % 4 == 0
            cur = p.currentLeavesArray(device=True)
            model = p.modelLeavesArray(device=True)
            torch.cuda.current_stream().synchronize()
            assert bits_equal(cur.cpu().numpy(), want_cur) and bits_equal(model.cpu().numpy(), want_model), (deskew, i)
