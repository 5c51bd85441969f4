"""GPU registration at its capacity edges -- up to 64 keyframes (kMaxSlots) and 2^20 moving leaves (kMatchedCap) --
against an exact reference, and the work partition of the persistent kernel that those sizes reach.

CPU part (no device): the stretches gn_stretch hands the CTAs of k_gn_loop tile the moving leaves exactly once, and
the shared-memory item map the launch reserves (gn_map_bytes) holds every entry the kernel writes: a warp writes
whole groups of 32, so CTA b needs ceil(K * n_b / 32) * 32 entries.

GPU part (`-m gpu`): per case, correspondences against the oracle's (teacher-forced at the guess and at round 4),
matched flags, and H/b against the EXACT sum of the per-pair terms of mad_icp.cpp:81-101, restated here in float64
numpy on the oracle's leaves and summed with math.fsum.  The bar is elementwise:

    |H_gpu - H_exact| <= REL * sum |terms|        REL = 2e-13 ~ 1800 u  (u = 2^-53)

Derivation.  Every term reaches the result through one chain of additions: the items of one warp, one DMMA
accumulation each (counted as one rounding per item: the k = 4 products of an m8n8k4 step are at worst added one by
one), the warps of the CTA (<= 32), then the CTA tiles -- in k_gn_loop up to G/16 per strand plus 16 strands, in
k_linearize up to G/4 per strand plus 4.  A chain of n roundings errs by at most n * u * sum |terms| (to first
order), and the GPU's own evaluation of a term differs from this file's by a few ulp of the term.  _chain() counts n
for every (case, shape) tested here and the tests assert that n + 16 <= 1800; the largest is the 2 x 2^20 case at
(512, 1): 2^21 items over 132 x 16 warps, ~1000 + 16 + 9 + 16.  One pair is ~1 / (K * L) >= 5e-7 of sum |terms|,
so a lost or doubled pair fails at every size tested.
"""
import ctypes as C
import math

import numpy as np
import pytest

from mad_icp_b200 import FlatTree, MadIcpError, Registrar, _capi, synth
from util import POSE_M, POSE_RAD, bits_equal, pose_error

U = 2.0 ** -53
REL = 2e-13
MAX_CHAIN = int(REL / U) - 16
P32 = C.POINTER(C.c_uint32)


# ------------------------------------------------------------------ CPU: the partition and the map reservation
def _stretches(L, G):
    """(lo, n) of the four stretches of every CTA, [G, 4] int64 each, from the library's gn_stretch."""
    lib = _capi.lib()
    lo, n = np.zeros((G, 4), np.uint32), np.zeros((G, 4), np.uint32)
    base_lo, base_n = lo.ctypes.data, n.ctypes.data
    for b in range(G):
        share = lib.madicp_debug_gn_stretch(L, G, b, C.cast(base_lo + 16 * b, P32), C.cast(base_n + 16 * b, P32))
        assert share >= 0
    return lo.astype(np.int64), n.astype(np.int64)


def _map_bytes(K, L, G):
    return _capi.check(_capi.lib().madicp_debug_gn_map_bytes(K, L, G), "madicp_debug_gn_map_bytes")


GRIDS = [114, 132, 264, 528]  # H100 PCIe / SXM at 1 CTA per SM, SXM at 2 and 4
SWEEP_L = sorted(set(list(range(1, 3001)) + list(range(3001, (1 << 20) + 1, 997)) + [1 << 20] +
                     list(range(429716, 522438, 1009)) + [429716, 522437] + list(range(300000, 320001, 499))))
MAP_K = [1, 2, 3, 16, 17, 32, 63, 64]


def test_stretches_tile_the_moving_leaves_and_the_map_holds_every_share(built):
    maps, short = 0, []
    for G in GRIDS:
        for L in SWEEP_L:
            lo, n = _stretches(L, G)
            flat_lo, flat_n = lo.ravel(), n.ravel()
            assert ((flat_lo >= 0) & (flat_lo + flat_n <= L)).all(), (G, L)
            nz = flat_n > 0
            order = np.argsort(flat_lo[nz], kind="stable")
            s_lo, s_hi = flat_lo[nz][order], (flat_lo + flat_n)[nz][order]
            # sorted non-empty stretches: the first starts at 0, each starts where the previous ended, the last ends at L
            assert s_lo[0] == 0 and s_hi[-1] == L and (s_lo[1:] == s_hi[:-1]).all(), (G, L)
            share = n.sum(axis=1)
            assert share.sum() == L
            for K in MAP_K:
                mb = _map_bytes(K, L, G)
                if mb:
                    maps += 1
                    written = -(-K * int(share.max()) // 32) * 32  # entries the map loop writes in the largest share
                    if mb // 4 < written:
                        short.append((G, L, K, mb // 4, written))
                    assert mb % 4 == 0 and mb <= 16 * 1024, (G, L, K, mb)
    assert not short, f"{len(short)} (G, L, K, reserved, written), first: {short[:8]}"
    assert maps > 10000  # the map is taken over most of the small-L range


def test_map_reservation_at_the_first_share_above_the_old_estimate(built):
    """L = 429 716 on 132 CTAs: a CTA of weight 8 draws 3 268 leaves, more than floor(L/G) + 8 = 3 263 that the
    reservation K*(floor(L/G) + 8) + 32 entries assumed; with K = 1 its map loop writes 3 296 entries."""
    _, n = _stretches(429716, 132)
    assert int(n.sum(axis=1).max()) == 3268
    assert _map_bytes(1, 429716, 132) // 4 >= 3296


def test_partition_entry_points_reject_bad_arguments(built):
    lib = _capi.lib()
    a, b = (C.c_uint32 * 4)(), (C.c_uint32 * 4)()
    for L, G, blk in ((0, 132, 0), (1 << 31, 132, 0), (100, 0, 0), (100, 132, 132), (100, 132, -1)):
        assert lib.madicp_debug_gn_stretch(L, G, blk, a, b) < 0, (L, G, blk)
    assert lib.madicp_debug_gn_stretch(100, 132, 131, None, b) < 0
    for K, L, G in ((0, 100, 132), (65, 100, 132), (1, 0, 132), (1, 100, 0)):
        assert lib.madicp_debug_gn_map_bytes(K, L, G) < 0, (K, L, G)
    assert _map_bytes(1, (1 << 26) + 5, 132) == 0  # past the 26-bit leaf field of a map entry


# ------------------------------------------------------------------ GPU: exact reference
DEFAULT = dict(min_ball=0.2, rho_ker=0.1, b_ratio=0.02)
SHAPES = [(1024, 1), (512, 1), (512, 2), (256, 4)]


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _chain(K, L, threads, ctas, sms):
    """Longest addition chain of a term into H/b (module docstring) for k_gn_loop at (threads, ctas) and k_linearize."""
    G = ctas * sms
    share = -(-8 * L // (8 * G - 3)) + 3 if G >= 8 else -(-L // G) + 3
    warps = threads // 32
    gn = -(-K * share // (32 * warps)) * 32 + warps + -(-G // 16) + 16
    lin_grid = min(-(-K * L // 256), 8 * sms)
    lin = -(-K * L // (256 * lin_grid)) * 32 + 8 + -(-lin_grid // 4) + 4
    return max(gn, lin)


def _terms(kf, means, X, idx, P=DEFAULT):
    """Per-pair factors of mad_icp.cpp:81-101 in float64 with the reference's operation order: flags [L] (any keyframe
    accepted the leaf) and, per keyframe, (sJ, J, e) of its accepted pairs: the terms are sJ_r * J_c and sJ_r * e."""
    X = np.asarray(X, dtype=np.float64)[:3]
    R, t = X[:, :3], X[:, 3]
    m = means
    ml = ((R[:, 0] * m[:, :1] + R[:, 1] * m[:, 1:2]) + R[:, 2] * m[:, 2:3]) + t
    ball = P["min_ball"] + P["b_ratio"] * np.sqrt((m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1]) + m[:, 2] * m[:, 2])
    rho = math.sqrt(P["rho_ker"])
    flags = np.zeros(m.shape[0], bool)
    out = []
    for k, (fmeans, fnormals, fbbox0) in enumerate(kf):
        f = idx[k]
        d = ml - fmeans[f]
        ok = ~(np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) > ball)
        flags |= ok
        d, n, q, bb = d[ok], fnormals[f][ok], m[ok], fbbox0[f][ok]
        e = (d[:, 0] * n[:, 0] + d[:, 1] * n[:, 1]) + d[:, 2] * n[:, 2]
        J = np.empty((e.size, 6))
        for j in range(3):
            J[:, j] = (n[:, 0] * R[0, j] + n[:, 1] * R[1, j]) + n[:, 2] * R[2, j]
        zero = np.zeros(e.size)
        S = [[zero, -q[:, 2], q[:, 1]], [q[:, 2], zero, -q[:, 0]], [-q[:, 1], q[:, 0], zero]]  # skew(moving mean)
        nJ = -J[:, :3]
        for j in range(3):
            J[:, 3 + j] = (nJ[:, 0] * S[0][j] + nJ[:, 1] * S[1][j]) + nJ[:, 2] * S[2][j]
        chi = np.abs(e)
        scale = np.where(chi > rho, rho / np.where(chi > rho, chi, 1.0), 1.0)
        w = 1.0 - bb / P["min_ball"]
        scale = scale * (w * w)
        out.append((scale[:, None] * J, J, e))
    return flags, out


def _exact(factors):
    """Every entry's terms summed exactly (math.fsum: rounded once) and the sum of their magnitudes."""
    s, a = np.zeros(42), np.zeros(42)
    for j in range(42):
        r, c = divmod(j, 6) if j < 36 else (j - 36, None)
        cols = [sJ[:, r] * (J[:, c] if c is not None else e) for sJ, J, e in factors]
        s[j] = math.fsum(v for col in cols for v in col.tolist())
        a[j] = sum(float(np.abs(col).sum()) for col in cols)
    return s[:36].reshape(6, 6), s[36:], a[:36].reshape(6, 6), a[36:]


def _check_exact(H, b, ex, what):
    Hx, bx, Ha, ba = ex
    eh, eb = np.abs(H - Hx), np.abs(b - bx)
    bad_h, bad_b = eh > REL * Ha, eb > REL * ba
    assert not bad_h.any() and not bad_b.any(), (
        what, [(int(r), int(c), float(eh[r, c] / max(Ha[r, c], 1e-300))) for r, c in zip(*np.nonzero(bad_h))][:6],
        [(int(r), float(eb[r] / max(ba[r], 1e-300))) for r in np.flatnonzero(bad_b)][:6])


class Case:
    def __init__(self, name, reg, otrees, kf_leaves, oq, means, X0):
        self.name, self.reg, self.otrees, self.kf, self.oq, self.means, self.X0 = name, reg, otrees, kf_leaves, oq, means, X0
        self.K, self.L = len(otrees), means.shape[0]


@pytest.fixture(scope="module")
def world(oracle):
    """64 keyframe scans (32 x 1024 beams) along a street long enough for all of them, their trees on both sides, and
    a pool of 2^20 distinct map-frame points near the first two keyframes' surfaces."""
    scene = synth.StreetScene(seed=7, x_max=60.0 + 2.0 * 64)
    base = synth.keyframe_poses(64)
    fts, ots, leaves = [], [], []
    for k in range(64):
        scan = synth.lidar_scan(scene, base[k], beams=32, azimuths=1024, seed=500 + k)
        P = synth.sensor_pose(base[k])
        ft, ot = FlatTree(scan), oracle.OracleTree(scan)
        ft.apply_transform(P)
        ot.apply_transform(P)
        fts.append(ft)
        ots.append(ot)
        means, normals, bbox0, _ = ot.leaves()
        leaves.append((means, normals, bbox0))
    q_base = base[32] @ synth.pose_xyyaw(0.8, 0.0, 0.02)
    T_true = synth.sensor_pose(q_base)
    small = synth.lidar_scan(scene, q_base, beams=16, azimuths=1024, seed=2000)  # ~5.7k leaves: 64 x them take the map
    large = synth.lidar_scan(scene, q_base, beams=64, azimuths=2048, seed=2001)
    # single-point moving leaves: points of keyframes 0 and 1 (map frame) jittered, in the frame of a pose near them
    rs = np.random.RandomState(11)
    src = np.concatenate([leaves[0][0], leaves[1][0]])
    pts = src[rs.randint(0, src.shape[0], (1 << 20))] + rs.normal(0.0, 0.03, ((1 << 20), 3))
    T_pts = synth.sensor_pose(base[0] @ synth.pose_xyyaw(1.0, 0.0, 0.01))
    pts = (pts - T_pts[:3, 3]) @ T_pts[:3, :3]
    return dict(fts=fts, ots=ots, leaves=leaves, T_true=T_true, small=small, large=large, pts=pts, T_pts=T_pts)


def _keyframe_case(w, oracle, K, which):
    slots = sorted(set(np.round(np.linspace(0, 63, K)).astype(int).tolist())) if K < 64 else list(range(64))
    if K == 32:
        slots = list(range(1, 64, 2))
    assert len(slots) == K and slots[-1] == 63
    reg = Registrar(device=0, max_keyframes=64)
    for s in slots:
        reg.put_keyframe(s, w["fts"][s])
    assert reg.active_slots() == slots
    scan = w[which]
    fq, oq = FlatTree(scan), oracle.OracleTree(scan)
    means = fq.leaf_means()
    reg.set_moving(means)
    X0 = w["T_true"] @ synth.pose_xyyaw(0.3, 0.0, 0.01)
    return Case(f"K{K}_{which}", reg, [w["ots"][s] for s in slots], [w["leaves"][s] for s in slots], oq, means, X0)


def _leaf_case(w, oracle, K, L):
    pts = w["pts"][:L]
    fq, oq = FlatTree(pts, b_max=1e-5, b_min=1e-5), oracle.OracleTree(pts, b_max=1e-5, b_min=1e-5)
    assert fq.num_leaves == L and oq.num_leaves == L
    means = fq.leaf_means()
    assert bits_equal(means, oq.leaves()[0])
    reg = Registrar(device=0, max_keyframes=2)
    for k in range(K):
        reg.put_keyframe(k, w["fts"][k])
    reg.set_moving(means)
    X0 = w["T_pts"] @ synth.pose_xyyaw(0.05, 0.0, 0.005)
    return Case(f"K{K}_L{L}", reg, w["ots"][:K], w["leaves"][:K], oq, means, X0)


def _leaf_counts():
    G = 132  # the H100 SXM grid at one CTA per SM; the cases are about the sizes, any H100 runs them
    return [(2, 1), (2, 31), (2, 33), (2, G - 1), (2, G + 1), (2, 4 * G + 3), (2, (1 << 16) + 1), (1, 429716),
            (2, 1 << 20)]


CASES = ([("kf", 17, "small"), ("kf", 32, "small"), ("kf", 64, "small"), ("kf", 64, "large")] +
         [("leaf", K, L) for K, L in _leaf_counts()])
CASE_IDS = [f"{a}{b}-{c}" for a, b, c in CASES]


def _build(w, oracle, spec):
    kind, a, b = spec
    return _keyframe_case(w, oracle, a, b) if kind == "kf" else _leaf_case(w, oracle, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("spec", CASES, ids=CASE_IDS)
def test_capacity_case_against_the_exact_reference(world, oracle, spec):
    cs = _build(world, oracle, spec)
    reg, K, L = cs.reg, cs.K, cs.L
    sms = _sm_count()
    G = sms  # automatic shapes: one CTA per SM
    if spec[0] == "kf" and spec[1] == 64:  # both sides of the item map at 64 keyframes
        assert (_map_bytes(K, L, G) > 0) == (spec[2] == "small"), (L, _map_bytes(K, L, G))
    for shape in SHAPES:
        assert _chain(K, L, *shape, sms) <= MAX_CHAIN, (shape, _chain(K, L, *shape, sms))
    ref = oracle.icp_run(cs.otrees, cs.oq, cs.X0, iters=5, num_threads=min(16, oracle.max_threads()))
    for it in (0, 4):
        X = ref["X_hist"][it]
        idx = reg.search(X)
        assert (idx == ref["idx_hist"][it]).all(), (cs.name, it, int((idx != ref["idx_hist"][it]).sum()))
        flags, factors = _terms(cs.kf, cs.means, X, idx)
        want = oracle.icp_linearize(cs.otrees, cs.oq, X)[2] if it == 0 else ref["matched"]
        assert (flags == want.astype(bool)).all(), (cs.name, it, int((flags != want).sum()))
        assert it > 0 or flags.any(), cs.name
        ex = _exact(factors)
        H, b, m = reg.linearize(X)
        assert (m == want).all(), (cs.name, it)
        _check_exact(H, b, ex, (cs.name, it, "linearize"))
        one = reg.register(X, iters=1)  # round 0 of the persistent kernel at X
        assert (one["matched"] == want).all() and one["n_matched"] == int(want.sum()), (cs.name, it)
        _check_exact(one["H"], one["b"], ex, (cs.name, it, "register"))
        if it == 4:
            for shape in SHAPES:  # every shape (with and without the item map) under the same exact bar
                reg.set_gn_grid(*shape)
                s1, s2 = reg.register(X, iters=1), reg.register(X, iters=1)
                assert bits_equal(s1["H"], s2["H"]) and bits_equal(s1["b"], s2["b"]), (cs.name, shape)
                assert (s1["matched"] == want).all() and s1["n_matched"] == int(want.sum()), (cs.name, shape)
                _check_exact(s1["H"], s1["b"], ex, (cs.name, shape))
                f1, f2 = reg.register(cs.X0, iters=5), reg.register(cs.X0, iters=5)
                assert bits_equal(f1["X"], f2["X"]) and bits_equal(f1["H"], f2["H"]), (cs.name, shape)
            reg.set_gn_grid(0, 1)
    out = reg.register(cs.X0, iters=5)
    if L >= 6:  # one moving leaf constrains one direction of six: its pose follows the rounding of a singular solve
        ang, dt = pose_error(out["X"], ref["X"])
        assert ang < POSE_RAD and dt < POSE_M, (cs.name, ang, dt)
    assert np.isfinite(out["X"]).all()
    assert (out["matched"] == ref["matched"]).mean() > 0.9999 and out["n_matched"] == int(out["matched"].sum())
    runs = []
    for mode in (0, 1, 2):
        reg.set_memo(mode)
        runs.append(reg.register(cs.X0, iters=5))
        runs[-1]["trace"] = reg.register_trace()
    reg.set_memo(True)
    for mode, r in enumerate(runs[1:], start=1):
        for key in ("X", "H", "b", "trace"):
            assert bits_equal(r[key], runs[0][key]), (cs.name, mode, key)
        assert (r["matched"] == runs[0]["matched"]).all()


@pytest.mark.gpu
def test_shrinking_within_one_context(world):
    """One context registers 2^20 moving leaves, then 1 000, then 17: the kernel zeroes the flags of the next call up
    to the buffer's capacity, so no stale flag in [L, round16(L)) reaches n_matched (16 flags per load).  Then the
    model goes from 64 keyframes down to 1 and still gives what a fresh single-keyframe context gives."""
    pts, X0 = world["pts"], world["T_pts"]
    reg = Registrar(device=0, max_keyframes=64)
    reg.put_keyframe(0, world["fts"][0])
    reg.put_keyframe(1, world["fts"][1])
    for L in (1 << 20, 1000, 17):
        reg.set_moving(pts[:L])
        out = reg.register(X0, iters=3)
        assert out["matched"].shape == (L,) and set(np.unique(out["matched"]).tolist()) <= {0, 1}
        assert out["n_matched"] == int(out["matched"].sum()) > 0, L
    means = FlatTree(world["small"]).leaf_means()
    for s in range(2, 64):
        reg.put_keyframe(s, world["fts"][s])
    reg.set_moving(means)
    X = world["T_true"]
    full = reg.register(X, iters=3)
    assert reg.num_keyframes == 64 and full["n_matched"] == int(full["matched"].sum())
    for s in range(63):
        reg.drop_keyframe(s)
    assert reg.active_slots() == [63]
    got = reg.register(X, iters=3)
    fresh = Registrar(device=0, max_keyframes=1)
    fresh.put_keyframe(0, world["fts"][63])
    fresh.set_moving(means)
    want = fresh.register(X, iters=3)
    for key in ("X", "H", "b"):
        assert bits_equal(got[key], want[key]), key
    assert (got["matched"] == want["matched"]).all() and got["n_matched"] == want["n_matched"]


@pytest.mark.gpu
def test_capacity_limits_are_rejected(world):
    with pytest.raises(MadIcpError, match="max_keyframes"):
        Registrar(device=0, max_keyframes=65)
    reg = Registrar(device=0, max_keyframes=1)
    reg.put_keyframe(0, world["fts"][0])
    extra = np.concatenate([world["pts"], world["pts"][:1] + 1.0])
    with pytest.raises(MadIcpError, match="1048576"):
        reg.set_moving(extra)
    reg.set_moving(world["pts"])  # exactly the capacity
    assert reg.register(world["T_pts"], iters=2)["matched"].shape == (1 << 20,)
