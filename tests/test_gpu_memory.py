"""A context gives back every byte of device memory it took: when madicp_create fails half way, and at madicp_destroy
after every lazily sized buffer has grown.  Measured as the device's free memory (torch.cuda.mem_get_info) before and
after.  The GPU may be shared, so other processes move that count: a measurement is repeated up to three times and
passes on the first run that lost less than SLACK.  A leak loses memory in every run."""
import gc

import numpy as np
import pytest

from mad_icp_b200 import MadIcpError, synth

pytestmark = pytest.mark.gpu

SLACK = 4 << 20  # bytes
T_PREV = synth.pose_xyyaw(0.0, 0.0, 0.0)
T_NOW = synth.pose_xyyaw(0.8, 0.05, 0.03)


def _free_bytes():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info(0)[0]


def _loss(run):
    """Device memory lost by run(), after one unmeasured run has loaded every kernel it launches."""
    run()
    losses = []
    for _ in range(3):
        before = _free_bytes()
        run()
        losses.append(before - _free_bytes())
        if losses[-1] < SLACK:
            break
    return losses


def test_failed_create_gives_back_everything(built, monkeypatch):
    from mad_icp_b200 import Registrar
    monkeypatch.setenv("MADICP_GN_SHAPE", "100,1")  # read at create, after the context's buffers are allocated

    def run():
        for _ in range(32):
            with pytest.raises(MadIcpError, match="unsupported persistent-kernel shape"):
                Registrar(max_keyframes=64)

    losses = _loss(run)
    assert losses[-1] < SLACK, f"32 failed creates lost {[x >> 20 for x in losses]} MB"


def _scan(seed):
    scene = synth.StreetScene(seed=7)
    return synth.lidar_scan(scene, synth.pose_xyyaw(0.3 * seed, 1.0, 0.01 * seed), 32, 1024, seed=seed)


def _kitti_records(seed):
    p = _scan(seed)
    a = np.zeros((p.shape[0], 4), np.float32)
    a[:, :3] = p
    return a


def _grown_context():
    """A context whose every lazily sized buffer has grown, then destroyed."""
    import torch
    from mad_icp_b200 import Registrar
    from mad_icp_b200.engine import leaf_means
    rs = np.random.RandomState(3)
    reg = Registrar(max_keyframes=3)
    small = synth.registration_case(K=1, beams=8, azimuths=256, seed=21)
    reg.keep_cloud(True)
    kf = reg.build_tree(small["scans"][0])
    reg.put_keyframe(0, kf, small["kf_poses"][0])
    big = np.concatenate([synth.four_walls(points_per_wall=60000, rng=rs) * [10, 10, 3],
                          rs.uniform(-1, 41, (60000, 3)) * [1, 1, 0.1]])
    big_tree = reg.build_tree(big, b_max=0.05)
    assert big_tree.num_nodes > 70000
    reg.put_keyframe(2, big_tree)  # past the first pool slot: the pool is re-homed
    query = reg.build_tree(small["query"])
    reg.set_moving_tree(query)
    reg.debug_timing(True, fetch=False)
    reg.register(small["T_guess"], iters=5)
    reg.debug_timing(False, fetch=False)
    reg.register(small["T_guess"], iters=5)
    reg.search_cloud(0, small["query"])
    leaf_means([kf, big_tree, query], [small["kf_poses"][0], None, None])
    leaf_means([kf, big_tree, query], device=True)
    kf.cloud(small["kf_poses"][0])
    kf.cloud(device=True)
    plan = reg.plan_records(_kitti_records(3), min_range=0.7, max_range=120.0, num_threads=2)
    reg.ingest_plan(plan, deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=10.0)
    batch = reg.build_trees([_scan(4), _scan(5)])
    torch.cuda.synchronize()
    del kf, big_tree, query, batch, plan
    reg.close()


def test_grown_context_gives_back_everything(built):
    losses = _loss(_grown_context)
    assert losses[-1] < SLACK, f"a grown context lost {[x >> 20 for x in losses]} MB"
