"""Every Gauss-Newton round of the persistent kernel against the exact sum of its terms, and a live context against a
fresh one after any history of calls.

Round 0 of k_gn_loop is held to the exact bar in tests/test_gpu_capacity.py; rounds 1 and later run other code: the
pose comes from epoch-tagged cells, CTA 0 polls every CTA's epoch-tagged tile, the path memo charges each item with the
move since s_Xp and kept items read their planarity weight from the ww table, the matched flags are recorded from
clear_from on into one of two buffers, and the walk counters go to one of two halves.  A small fault there (a stale
tile, one item dropped after round 0) moves the pose by far less than the oracle bars can see and is shared by every
memo mode.  Here the H/b of round n - 1 is recovered through the API -- register(X0, n) returns the H/b of its last
round, at trace[n - 1] of the longer run -- and held, round by round, to

    |H_gpu - H_exact| <= REL * sum |terms|        (test_gpu_capacity: REL = 2e-13, the _chain bound asserted)

with H_exact the math.fsum of the per-pair terms of mad_icp.cpp:81-101 at that round's pose and the oracle's indices.

A context carries state from call to call: the parity of call_seq (matched buffer and walk counters), the pose and tile
epochs, the memo arrays sized from capacities, the keyframe pool, the moving-leaf buffers, the parameters, the shape,
the calibrated pass costs and the debug timing buffers.  A seeded script of ~40 operations drives one context through
all of them and, after every registration, compares it bit for bit with a fresh context set up to the same state.

CPU part (no device): the exact per-round reference equals the oracle's own per-round H/b, and the script is
deterministic and only reaches legal states.
"""
import numpy as np
import pytest

from mad_icp_b200 import FlatTree, Registrar, synth
from test_gpu_capacity import MAX_CHAIN, REL, _chain, _check_exact, _exact, _terms
from util import bits_equal

SMALL = dict(K=2, beams=16, azimuths=512, seed=3)  # the lidar_small case of tests/golden
PARAMS = {"default": (0.2, 0.1, 0.02), "gate": (0.2, 0.3, 0.05), "reweigh": (0.1, 0.05, 0.01)}  # as test_gpu_params
AUTO_THREADS = (768, 896, 704, 640, 512)  # the shapes the automatic choice picks from (ctx.hpp kAutoShapes), 1 CTA / SM


def _pdict(P):
    return dict(zip(("min_ball", "rho_ker", "b_ratio"), P))


def _keyframes(oracle, c):
    """Map-frame trees of a case's keyframes, GPU and oracle side, and the oracle's leaves (means, normals, bbox0)."""
    fts, ots, leaves = [], [], []
    for scan, P in zip(c["scans"], c["kf_poses"]):
        ft, ot = FlatTree(scan), oracle.OracleTree(scan)
        ft.apply_transform(P)
        ot.apply_transform(P)
        fts.append(ft)
        ots.append(ot)
        leaves.append(ot.leaves()[:3])
    return fts, ots, leaves


class Case:
    def __init__(self, oracle, c, max_keyframes):
        self.c = c
        self.fts, self.ots, self.kf = _keyframes(oracle, c)
        self.oq = oracle.OracleTree(c["query"])
        self.means = FlatTree(c["query"]).leaf_means()
        assert bits_equal(self.means, self.oq.leaves()[0])
        self.reg = Registrar(device=0, max_keyframes=max_keyframes)
        for k, ft in enumerate(self.fts):
            self.reg.put_keyframe(k, ft)
        self.reg.set_moving(self.means)
        self.K, self.L = len(self.fts), self.means.shape[0]
        self._exact = {}

    def exact(self, oracle, X, P):
        """(oracle indices, flags, exact sums) at pose X under parameters P, cached by the pose's bits."""
        key = (np.asarray(X, dtype=np.float64)[:3].tobytes(), P)
        if key not in self._exact:
            idx = oracle.icp_run(self.ots, self.oq, X, iters=1, num_threads=min(16, oracle.max_threads()),
                                 **_pdict(P))["idx_hist"][0]
            flags, factors = _terms(self.kf, self.means, X, idx, _pdict(P))
            self._exact[key] = (idx, flags, _exact(factors))
        return self._exact[key]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _assert_chain(K, L, shape):
    """The addition chain of every shape the launch may run at stays under the bar's budget; returns the largest."""
    sms = _sms()
    shapes = [(t, 1) for t in AUTO_THREADS] if shape is None else [shape]
    n = max(_chain(K, L, t, c, sms) for t, c in shapes)
    assert n <= MAX_CHAIN, (K, L, shape, n)
    return n


def _set_shape(reg, shape):
    reg.set_gn_grid(*(shape or (0, 1)))


def _check_round(cs, oracle, out, X, P, what, flags_want=None):
    """out (the result of a registration whose last round ran at X) against the exact sums at X."""
    idx, flags, ex = cs.exact(oracle, X, P)
    got = cs.reg.search(X)
    assert (got == idx).all(), (what, int((got != idx).sum()))
    _check_exact(out["H"], out["b"], ex, what)
    want = flags if flags_want is None else flags_want
    assert (out["matched"] == want).all(), (what, int((out["matched"] != want).sum()))
    assert out["n_matched"] == int(want.sum()), (what, out["n_matched"], int(want.sum()))
    return flags


def _every_round(cs, oracle, X0, N, rounds, P, what):
    """register(X0, N) in each memo mode, then register(X0, n) for every n in `rounds`: a bit-exact prefix of the
    N-round trace, the H/b and flags of round n - 1 exact at trace[n - 1], the keyframe weight det(H^-1) bit for bit."""
    reg = cs.reg
    for mode in (0, 1, 2):
        reg.set_memo(mode)
        full = reg.register(X0, N)
        tr = reg.register_trace()
        assert tr.shape == (N + 1, 3, 4) and bits_equal(tr[0], np.asarray(X0)[:3]), (what, mode)
        assert bits_equal(tr[N], full["X"]), (what, mode)
        for n in rounds:
            out = reg.register(X0, n)
            tn = reg.register_trace()
            assert bits_equal(tn, tr[:n + 1]), (what, mode, n, "trace prefix")
            assert bits_equal(out["X"], tr[n]), (what, mode, n)
            _check_round(cs, oracle, out, tr[n - 1], P, (what, mode, n))
            reg.register_async(X0, n)
            f = reg.register_fetch(want_matched=True)
            for k in ("X", "H", "b"):
                assert bits_equal(f[k], out[k]), (what, mode, n, k)
            assert (f["matched"] == out["matched"]).all() and f["n_matched"] == out["n_matched"], (what, mode, n)
            assert bits_equal(f["weight"], reg.inv_det6(f["H"])), (what, mode, n, "weight")
    reg.set_memo(2)


# ------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def small(oracle):
    return Case(oracle, synth.registration_case(**SMALL), max_keyframes=2)


@pytest.fixture(scope="module")
def baseline(oracle):
    return Case(oracle, synth.registration_case(K=16), max_keyframes=16)


# ------------------------------------------------------------------ CPU: the exact reference itself
def test_exact_reference_equals_the_oracle_every_round(oracle):
    """fsum of _terms at the oracle's pose and indices of every round == the oracle's own H/b of that round, within
    REL * sum |terms| (its sequential sums err by far less on this case), and the flags of its last round."""
    c = synth.registration_case(**SMALL)
    _, ots, kf = _keyframes(oracle, c)
    oq = oracle.OracleTree(c["query"])
    means = oq.leaves()[0]
    ref = oracle.icp_run(ots, oq, c["T_guess"], iters=10, num_threads=2)
    for it in range(10):
        flags, factors = _terms(kf, means, ref["X_hist"][it], ref["idx_hist"][it])
        assert flags.any(), it
        _check_exact(ref["H_hist"][it], ref["b_hist"][it], _exact(factors), ("oracle", it))
    assert (flags == ref["matched"].astype(bool)).all()


# ------------------------------------------------------------------ GPU 1: every round, exactly
SHAPES = [None, (512, 2), (256, 4)]
SHAPE_IDS = ["auto", "512x2", "256x4"]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("start", ["guess", "shifted", "restart", "reweigh"])
def test_every_round_is_exact(small, oracle, start, shape):
    """lidar_small, 15 rounds, each memo mode on its own: from the guess, from 1.5 m off it (large moves, many resumed
    walks), restarted at the converged pose (nearly every walk kept: the weight comes from the ww table), and at the
    reweigh parameters after set_params on the live context."""
    reg, P = small.reg, PARAMS["default"]
    _assert_chain(small.K, small.L, shape)
    _set_shape(reg, shape)
    X0 = np.array(small.c["T_guess"], dtype=np.float64)
    try:
        if start == "shifted":
            X0[0, 3] += 1.5
        elif start == "restart":
            X0 = reg.register(X0, 15)["X"]
        elif start == "reweigh":
            reg.register(X0, 15)
            P = PARAMS["reweigh"]
            reg.set_params(*P)
        _every_round(small, oracle, X0, 15, range(1, 16), P, (start, shape))
        if start == "restart":  # the restart keeps nearly every walk from round 1 on
            reg.register(X0, 5)
            walked = reg.register_walked()
            assert walked[0] == small.K * small.L and (walked[1:] < small.K * small.L // 10).all(), walked
    finally:
        reg.set_params(*PARAMS["default"])
        _set_shape(reg, None)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_every_round_is_exact_at_16_keyframes(baseline, oracle, shape):
    """The 16-keyframe baseline (~20k moving leaves x 16): rounds 1, 2, 5 and 9 of a 9-round run."""
    _assert_chain(baseline.K, baseline.L, shape)
    _set_shape(baseline.reg, shape)
    try:
        _every_round(baseline, oracle, baseline.c["T_guess"], 9, (1, 2, 5, 9), PARAMS["default"], ("K16", shape))
    finally:
        _set_shape(baseline.reg, None)


@pytest.mark.gpu
def test_chained_launches_record_the_last_round_only(small, oracle):
    """register(X0, 100) chains a 64-round launch and a 36-round one: its H/b and flags are those of round 99 alone,
    exact at trace[35] of the last launch, whose trace[0] is the 64-round pose bit for bit.  From 1.5 m off round 0
    matches leaves the converged rounds do not, so a first launch that recorded its flags would show."""
    reg, P = small.reg, PARAMS["default"]
    X0 = np.array(small.c["T_guess"], dtype=np.float64)
    X0[0, 3] += 1.5
    at64 = reg.register(X0, 64)["X"]
    out = reg.register(X0, 100)
    tr = reg.register_trace()
    assert tr.shape == (37, 3, 4) and bits_equal(tr[0], at64) and bits_equal(tr[36], out["X"])
    assert reg.register_walked().shape == (36,)
    _check_round(small, oracle, out, tr[35], P, "round 99")
    _, first, _ = small.exact(oracle, X0, P)
    _, last, _ = small.exact(oracle, tr[35], P)
    assert (first & ~last).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4, 7])
def test_partial_registration_flags_are_the_union_of_its_rounds(small, oracle, n):
    """register_async(partial=True): the flags are the union of every round's exact gate flags, the H/b the last
    round's."""
    reg, P = small.reg, PARAMS["default"]
    X0 = np.array(small.c["T_guess"], dtype=np.float64)
    X0[0, 3] += 1.5
    reg.register_async(X0, n, partial=True)
    out = reg.register_fetch(want_matched=True)
    tr = reg.register_trace()
    assert tr.shape == (n + 1, 3, 4) and bits_equal(tr[n], out["X"])
    union = np.zeros(small.L, bool)
    for it in range(n):
        union |= small.exact(oracle, tr[it], P)[1]
    last = _check_round(small, oracle, out, tr[n - 1], P, ("partial", n), flags_want=union)
    assert (union & ~last).any(), n  # the earlier rounds do add flags here
    assert bits_equal(out["weight"], reg.inv_det6(out["H"]))


# ------------------------------------------------------------------ 2. a live context == a fresh one
MAX_KF = 8
GRID_SHAPES = [(512, 2), (256, 4), (1024, 1), (768, 1)]


def _script(seed):
    """~40 operations on one context, as tuples.  The seed draws the slot names, the shapes and every registration's
    guess offset; the order of the operations is fixed, so that each transition is reached whatever the seed.

      ("grid", (threads, ctas))  ("put", slot, tree)  ("drop", slot)  ("moving", L or "all")  ("moving_tree",)
      ("params", name)  ("memo", mode)  ("calibrate",)  ("timing", on)
      ("reg", iters, "register" | "async" | "partial", (dx, dy, dyaw), exact)
    trees 0..3 are the keyframes of a 4-keyframe case, "big" a larger scan at keyframe 1's pose."""
    rs = np.random.RandomState(seed)
    s = [int(v) for v in rs.permutation(MAX_KF)]  # slot names: s[0] .. s[7]
    g = [GRID_SHAPES[int(i)] for i in rs.permutation(len(GRID_SHAPES))]

    def reg(iters, via, exact=False):
        off = (float(rs.uniform(-0.4, 0.4)), float(rs.uniform(-0.2, 0.2)), float(rs.uniform(-0.02, 0.02)))
        return ("reg", iters, via, off, exact)

    return [
        ("grid", g[0]), ("put", s[0], 0), ("put", s[1], 1), ("moving", "all"),
        reg(7, "register", True),
        ("put", s[2], 2),
        reg(1, "async"),
        ("put", s[1], "big"),  # an overwrite with a larger tree: the pool grows
        reg(64, "register", True),
        ("moving", 17), reg(2, "partial"),
        ("moving", 16), ("timing", True), reg(7, "async"),
        ("moving", 33), ("params", "gate"), reg(65, "register", True),
        ("timing", False), ("moving", "all"), ("memo", 1), ("grid", g[1]),
        reg(100, "register"),
        ("params", "reweigh"), ("put", s[3], 3), ("calibrate",),
        reg(7, "async", True),
        ("moving_tree",), ("memo", 0),
        reg(2, "register"),
        ("drop", s[0]), ("drop", s[2]), ("drop", s[3]),  # down to the big keyframe alone
        reg(64, "partial"),
        ("params", "default"), ("grid", g[2]), ("memo", 2), ("timing", True),
        reg(1, "register", True),
        ("put", s[4], 0), ("moving", 17), ("timing", False),
        reg(7, "partial"),
        ("moving", "all"), ("grid", g[3]),
        reg(100, "register"),
    ]


def _states(script, n_all):
    """The context state after every operation (slots -> tree, L, moving kind, parameters, shape, memo, timing); raises
    on an illegal one."""
    st = dict(slots={}, L=0, moving=None, params="default", grid=None, memo=2, timing=False)
    out = []
    for op in script:
        kind = op[0]
        if kind == "grid":
            assert op[1] in GRID_SHAPES
            st["grid"] = op[1]
        elif kind == "put":
            assert 0 <= op[1] < MAX_KF and op[2] in (0, 1, 2, 3, "big"), op
            st["slots"] = {**st["slots"], op[1]: op[2]}
        elif kind == "drop":
            assert op[1] in st["slots"], op
            st["slots"] = {k: v for k, v in st["slots"].items() if k != op[1]}
        elif kind == "moving":
            L = n_all if op[1] == "all" else op[1]
            assert 1 <= L <= n_all, op
            st.update(L=L, moving="means")
        elif kind == "moving_tree":
            st.update(L=n_all, moving="tree")
        elif kind == "params":
            assert op[1] in PARAMS
            st["params"] = op[1]
        elif kind == "memo":
            assert op[1] in (0, 1, 2)
            st["memo"] = op[1]
        elif kind == "timing":
            st["timing"] = bool(op[1])
        elif kind == "calibrate":
            assert st["slots"] and st["L"] >= 1 and st["grid"] is not None
        else:
            assert kind == "reg", op
            _, iters, via, off, exact = op
            assert st["slots"] and st["L"] >= 1 and st["grid"] is not None, op
            assert iters >= 1 and via in ("register", "async", "partial") and (via == "register" or iters <= 64), op
        out.append(dict(st))
    return out


SEED = 2024


def test_script_is_deterministic_and_legal():
    a, b = _script(SEED), _script(SEED)
    assert a == b and len(a) >= 40
    states = _states(a, n_all=4000)
    regs = [op for op in a if op[0] == "reg"]
    assert {op[1] for op in regs} == {1, 2, 7, 64, 65, 100}
    assert {op[2] for op in regs} == {"register", "async", "partial"}
    assert 3 <= sum(op[4] for op in regs) <= len(regs) // 2 + 1
    assert [op[1] for op in a if op[0] == "moving"] == ["all", 17, 16, 33, "all", 17, "all"]
    assert min(len(st["slots"]) for st in states[4:]) == 1
    assert {st["params"] for st in states} == set(PARAMS) and {st["memo"] for st in states} == {0, 1, 2}
    assert len({st["grid"] for st in states if st["grid"]}) == len(GRID_SHAPES)
    assert any(op[0] == "calibrate" for op in a) and any(op[0] == "moving_tree" for op in a)
    for seed in range(20):  # every seed gives a legal script
        _states(_script(seed), n_all=4000)


SCRIPT_CASE = dict(K=4, beams=16, azimuths=512, seed=21)


@pytest.fixture(scope="module")
def script_world(oracle):
    c = synth.registration_case(**SCRIPT_CASE)
    fts, ots, kf = _keyframes(oracle, c)
    scene = synth.StreetScene(seed=7)
    big_scan = synth.lidar_scan(scene, synth.keyframe_poses(4)[1], beams=32, azimuths=1024, seed=77)
    big, obig = FlatTree(big_scan), oracle.OracleTree(big_scan)
    big.apply_transform(c["kf_poses"][1])
    obig.apply_transform(c["kf_poses"][1])
    assert big.num_nodes > max(f.num_nodes for f in fts)
    trees = {0: fts[0], 1: fts[1], 2: fts[2], 3: fts[3], "big": big}
    leaves = {0: kf[0], 1: kf[1], 2: kf[2], 3: kf[3], "big": obig.leaves()[:3]}
    return dict(c=c, trees=trees, leaves=leaves, means=FlatTree(c["query"]).leaf_means())


def _apply(reg, op, w):
    kind = op[0]
    if kind == "grid":
        reg.set_gn_grid(*op[1])
    elif kind == "put":
        reg.put_keyframe(op[1], w["trees"][op[2]])
    elif kind == "drop":
        reg.drop_keyframe(op[1])
    elif kind == "moving":
        reg.set_moving(w["means"] if op[1] == "all" else w["means"][:op[1]])
    elif kind == "moving_tree":
        reg._moving_tree = reg.build_tree(w["c"]["query"])
        reg.set_moving_tree(reg._moving_tree)
    elif kind == "params":
        reg.set_params(*PARAMS[op[1]])
    elif kind == "memo":
        reg.set_memo(op[1])
    elif kind == "timing":
        reg.debug_timing(op[1], fetch=False)
    elif kind == "calibrate":
        assert reg.calibrate(w["c"]["T_guess"]) >= 1


def _register(reg, X0, iters, via):
    if via == "register":
        r = reg.register(X0, iters)
    else:
        reg.register_async(X0, iters, partial=(via == "partial"))
        r = reg.register_fetch(want_matched=True)
    r["trace"] = reg.register_trace()
    r["walked"] = reg.register_walked()
    r["records"] = reg.register_walk_records()
    return r


def _fresh(st, w):
    reg = Registrar(device=0, max_keyframes=MAX_KF, **_pdict(PARAMS[st["params"]]))
    for slot in sorted(st["slots"]):
        reg.put_keyframe(slot, w["trees"][st["slots"][slot]])
    _apply(reg, ("moving_tree",) if st["moving"] == "tree" else ("moving", st["L"]), w)
    reg.set_gn_grid(*st["grid"])
    reg.set_memo(st["memo"])
    return reg


def _assert_same(got, want, what):
    for k in ("X", "H", "b", "trace"):
        assert bits_equal(got[k], want[k]), (what, k)
    for k in ("walked", "records"):
        assert (got[k] == want[k]).all(), (what, k, got[k], want[k])
    assert (got["matched"] == want["matched"]).all() and got["n_matched"] == want["n_matched"], what
    if "weight" in want:
        assert bits_equal(got["weight"], want["weight"]), (what, "weight")


@pytest.mark.gpu
def test_a_live_context_equals_a_fresh_one_after_any_history(script_world):
    w = script_world
    script = _script(SEED)
    states = _states(script, n_all=w["means"].shape[0])
    live = Registrar(device=0, max_keyframes=MAX_KF)
    sms = _sms()
    n_exact = 0
    for i, (op, st) in enumerate(zip(script, states)):
        if op[0] != "reg":
            _apply(live, op, w)
            continue
        _, iters, via, off, exact = op
        X0 = w["c"]["T_guess"] @ synth.pose_xyyaw(*off)
        got = _register(live, X0, iters, via)
        want = _register(_fresh(st, w), X0, iters, via)
        _assert_same(got, want, (i, op))
        assert got["n_matched"] == int(got["matched"].sum()), (i, op)
        if exact:
            slots = sorted(st["slots"])
            kf = [w["leaves"][st["slots"][s]] for s in slots]
            means = live.get_moving()
            K, L = len(slots), means.shape[0]
            assert _chain(K, L, *st["grid"], sms) <= MAX_CHAIN
            X = got["trace"][-2]  # the last round's pose
            flags, factors = _terms(kf, means, X, live.search(X), _pdict(PARAMS[st["params"]]))
            _check_exact(got["H"], got["b"], _exact(factors), (i, op))
            if via != "partial":
                assert (got["matched"] == flags).all() and got["n_matched"] == int(flags.sum()), (i, op)
            n_exact += 1
    assert n_exact >= 4


@pytest.mark.gpu
def test_two_contexts_interleaved_on_one_device(small, oracle):
    """Two contexts on the same device, enqueued A, B, A and fetched B then A: each equals its solo run."""
    a = Case(oracle, small.c, max_keyframes=2)
    b = Registrar(device=0, max_keyframes=1)
    b.put_keyframe(0, small.fts[1])
    b.set_moving(small.means[:1000])
    b.set_gn_grid(256, 4)
    XA1 = np.array(small.c["T_guess"], dtype=np.float64)
    XA2 = XA1.copy()
    XA2[0, 3] += 1.5
    XB = small.c["T_guess"] @ synth.pose_xyyaw(0.1, -0.1, 0.01)

    def fetched(reg):
        r = reg.register_fetch(want_matched=True)
        r["trace"] = reg.register_trace()
        r["walked"] = reg.register_walked()
        r["records"] = reg.register_walk_records()
        return r

    a.reg.register_async(XA1, 10)
    b.register_async(XB, 7, partial=True)
    a.reg.register_async(XA2, 15)
    got_b, got_a = fetched(b), fetched(a.reg)

    solo_a = Case(oracle, small.c, max_keyframes=2).reg
    solo_a.register_async(XA2, 15)
    _assert_same(got_a, fetched(solo_a), "A")
    solo_b = Registrar(device=0, max_keyframes=1)
    solo_b.put_keyframe(0, small.fts[1])
    solo_b.set_moving(small.means[:1000])
    solo_b.set_gn_grid(256, 4)
    solo_b.register_async(XB, 7, partial=True)
    _assert_same(got_b, fetched(solo_b), "B")
    a.reg.register_async(XA1, 10)  # A's first registration on its own, after all that
    first = fetched(a.reg)
    solo_a.register_async(XA1, 10)
    _assert_same(first, fetched(solo_a), "A first")
    _check_round(a, oracle, got_a, got_a["trace"][14], PARAMS["default"], "A exact")
