"""CPU tests (no GPU): pin the plain-C oracle (oracle/cfr_oracle.c) against
 (a) the known answers in the reference's own gtests (cited file:line, csrc/liars_dice/ of the original project), and
 (b) golden fixtures generated from the compiled reference (oracle/make_golden.py).
"""
import os

import numpy as np
import pytest

from oracle.oracle import game_dims

SHAPES = [(1, 4), (1, 6), (2, 3)]


def children(tree, i):
    return list(range(tree[i, 2], tree[i, 3]))


# ---------------------------------------------------------------- liars_dice_test.cc (2x6f)
def test_game_integers(port):
    D, F = 2, 6
    A, H, Q = game_dims(D, F)
    import ctypes as C
    q, f = C.c_int(), C.c_int()
    for a, (eq, ef) in {0: (1, 0), 1: (1, 1), 6: (2, 0)}.items():      # liars_dice_test.cc:46-62
        port.lib.orc_unpack_action(D, F, a, C.byref(q), C.byref(f))
        assert (q.value, f.value) == (eq, ef)
    lo, hi = C.c_int(), C.c_int()
    for lb, exp in {-1: (0, 24), 0: (1, 25), 11: (12, 25), 24: (25, 25)}.items():   # :64-94
        port.lib.orc_bid_range(D, F, lb, C.byref(lo), C.byref(hi))
        assert (lo.value, hi.value) == exp
    assert [port.num_matches(D, F, 0, f) for f in range(6)] == [2, 0, 0, 0, 0, 0]          # :104-108
    assert [port.num_matches(D, F, H - 1, f) for f in range(6)] == [2] * 6                  # :110-115
    assert [port.num_matches(D, F, 5, f) for f in range(6)] == [2, 1, 1, 1, 1, 1]           # :117-121
    tree = port.unroll_tree(D, F, -1, 0, 3)                                  # player alternation :96-102
    for n in range(1, len(tree)):
        assert tree[n, 1] == 1 - tree[tree[n, 4], 1]


# ---------------------------------------------------------------- tree_test.cc
def test_tree_known_answers(port):
    t = port.unroll_tree(1, 2)                                     # tree_test.cc:20-34
    assert len(t) == 31
    assert children(t, 0) == [1, 2, 3, 4] and children(t, 1) == [5, 6, 7, 8] and children(t, 2) == [9, 10, 11]
    assert children(t, 15) == [25, 26] and children(t, 16) == [27] and children(t, 25) == [30]
    t = port.unroll_tree(2, 6, 22, 0, 0)                           # :36-52
    assert len(t) == 1 and t[0, 4] == -1 and children(t, 0) == []
    t = port.unroll_tree(2, 6, 22, 0, 1)                           # :54-70
    assert len(t) == 3 and children(t, 0) == [1, 2] and t[1, 4] == 0 and t[2, 4] == 0
    t = port.unroll_tree(2, 6, 22, 0, 2)                           # :72-89
    assert len(t) == 4 and t[3, 4] == 1
    t = port.unroll_tree(2, 6, 21, 0, 2)                           # :91-105
    assert len(t) == 7 and children(t, 0) == [1, 2, 3] and children(t, 1) == [4, 5] and children(t, 2) == [6]


def test_tree_is_breadth_first_prefix(port):                       # tree_test.cc:107-125
    full = port.unroll_tree(1, 5)
    for d in range(20):
        sub = port.unroll_tree(1, 5, -1, 0, d)
        assert (full[:len(sub), :2] == sub[:, :2]).all()
        has = sub[:, 3] > sub[:, 2]
        assert (full[:len(sub)][has] == sub[has]).all()


def test_trees_match_golden(port, golden):
    g = golden("trees.npz")
    for key in g.files:
        _, D, F, lb, pl, md = key.split("_")
        t = port.unroll_tree(int(D), int(F), int(lb), int(pl), int(md))
        assert t.shape == g[key].shape and (t == g[key]).all(), key


# ---------------------------------------------------------------- subgame_solving_test.cc:48-104
@pytest.mark.parametrize("D,F", [(1, 6), (2, 3)])
def test_win_probability_one_hot(port, D, F):
    A, H, Q = game_dims(D, F)
    for op in range(H):
        b = np.zeros(H); b[op] = 1
        for bet in range(A - 1):
            quantity, face = 1 + bet // F, bet % F
            v = port.win_probability(D, F, bet, b)
            for my in range(H):
                m = port.num_matches(D, F, my, face) + port.num_matches(D, F, op, face)
                assert v[my] == (1.0 if m >= quantity else 0.0)


def test_prob_normalisation_tiny(port):                           # subgame_solving_test.cc:298-310
    probs = np.array([2.93185e-81, 3.00956e-81, 3.17805e-81, 8.80785e-81])
    q = port.query(1, 4, 0, -1, 0, probs, probs)
    assert abs(q[2 + 9:2 + 9 + 4].astype(np.float64).sum() - 1.0) < 1e-6


def test_query_layout_roundtrip(port):                            # subgame_solving_test.cc:267-296
    D, F = 1, 3
    A, H, Q = game_dims(D, F)
    b1 = np.arange(H, dtype=np.float64); b1 /= b1.sum()
    b2 = np.arange(H) + 0.5; b2 /= b2.sum()
    tree = port.unroll_tree(D, F)
    for trav in (0, 1):
        for node in tree:
            if node[0] == A - 1:
                continue
            q = port.query(D, F, trav, node[0], node[1], b1, b2)
            assert q[0] == node[1] and q[1] == trav
            onehot = q[2:2 + A]
            assert onehot.sum() == (0 if node[0] < 0 else 1) and (node[0] < 0 or onehot[node[0]] == 1)
            assert np.allclose(q[2 + A:2 + A + H], b1, atol=1e-6) and np.allclose(q[2 + A + H:], b2, atol=1e-6)


# ---------------------------------------------------------------- CFR convergence thresholds of the reference tests
def test_cfr_1x2f_linear_exploitability(port):                    # subgame_solving_test.cc:162-179
    b = np.full((2, 2), 0.5)
    s = port.cfr_solve(1, 2, b, [180], num_iters=180, max_depth=1000, want=("avg",))
    e = port.exploitability(1, 2, s["avg"][0])
    assert 0.0 <= e.mean() < 1e-3


def test_fulltree_golden(port, golden):
    g = golden("fulltree.npz")
    for (D, F) in [(1, 2), (1, 3), (1, 4)]:
        A, H, Q = game_dims(D, F)
        b = np.full((2, H), 1.0 / H)
        s = port.cfr_solve(D, F, b, [16, 1024], num_iters=1024, max_depth=100000, want=("avg",))
        assert np.array_equal(s["avg"][0], g[f"avg16_{D}x{F}"])              # bit-exact vs reference (-ffp-contract=off)
        assert np.array_equal(s["root_means"], g[f"mu_{D}x{F}"])
        e = np.stack([port.exploitability(D, F, s["avg"][c]) for c in range(2)])
        assert np.array_equal(e, g[f"expl_{D}x{F}_nofma"])
        # the reference's own two builds bracket the self-noise (SURVEY appendix B)
        assert abs(e[1].mean() - g[f"expl_{D}x{F}_fast"][1].mean()) < 5e-4


# ---------------------------------------------------------------- golden trajectories from the compiled reference
@pytest.mark.parametrize("D,F", SHAPES)
def test_cfr_zero_net_bit_exact_vs_golden(port, golden, D, F):
    g = golden(f"cfr_zero_{D}x{F}.npz")
    cps = list(g["checkpoints"])
    for i, (lb, pl) in enumerate(g["roots"]):
        s = port.cfr_solve(D, F, g[f"beliefs{i}"], cps, lb, pl, num_iters=64)
        for k in ("regrets", "last", "sum", "avg", "root_means"):
            assert np.array_equal(s[k], g[f"{k}{i}"]), (k, i)


@pytest.mark.parametrize("D,F", SHAPES)
def test_cfr_discount_variants_bit_exact_vs_golden(port, golden, D, F):
    """Vanilla CFR and DCFR (subgame_solving.cc:592-617, incl. the alpha >= 5 / beta <= -5 shortcuts): the C port follows
    the compiled reference bit for bit (both use glibc pow)."""
    from oracle.make_golden import VARIANTS
    g = golden("cfr_variants.npz")
    for name, kw in VARIANTS.items():
        s = port.cfr_solve(D, F, g[f"beliefs_{D}x{F}"], list(g["checkpoints"]), 1, 1, num_iters=8, **kw)
        for k in ("regrets", "last", "sum", "avg", "root_means"):
            assert np.array_equal(s[k], g[f"{k}_{name}_{D}x{F}"]), (name, k)


@pytest.mark.parametrize("D,F", SHAPES)
def test_fictitious_play_bit_exact_vs_golden(port, golden, D, F):
    """FP (subgame_solving.cc:364-506): linear / plain / optimistic averaging, depth 2, 3 and full depth — the C port follows
    the compiled reference bit for bit (fixture from oracle/make_golden.py)."""
    from oracle.make_golden import FP_CASES, FP_CPS, FP_ROOTS
    g = golden("fp_zero.npz")
    for (lin, opt, md) in FP_CASES:
        if md > 3 and (D, F) != (1, 4):
            continue
        for (lb, pl) in FP_ROOTS:
            s = port.fp_solve(D, F, g[f"beliefs_{D}x{F}"], FP_CPS, lb, pl, num_iters=max(FP_CPS), max_depth=md, linear_update=lin, optimistic=opt)
            for k in ("last", "sum", "avg", "root_means"):
                assert np.array_equal(s[k], g[f"{k}_{int(lin)}{int(opt)}{md}_{lb}_{D}x{F}"]), (lin, opt, md, lb, k)


@pytest.mark.parametrize("D,F", SHAPES)
def test_cfr_net_short_horizon_vs_golden(port, golden, net_weights, D, F):
    g = golden(f"cfr_net_{D}x{F}.npz")
    w = net_weights(D, F)
    assert np.allclose([w.astype(np.float64).sum(), np.abs(w).astype(np.float64).sum()], g["w_checksum"], rtol=1e-9)
    assert np.array_equal(w[:8], g["w_head"])
    cps = list(g["checkpoints"])
    for i, (lb, pl) in enumerate(g["roots"]):
        s = port.cfr_solve(D, F, g[f"beliefs{i}"], cps, lb, pl, num_iters=16, net_w=w)
        # C fp32 MLP vs ATen fp32 MLP: 1e-6-level leaf differences, amplified by regret matching over iterations
        assert np.abs(s["queries"][0] - g[f"queries{i}"][0]).max() < 1e-6
        assert np.abs(s["leaf_values"][0] - g[f"leaf_values{i}"][0]).max() < 2e-6
        for k in ("regrets", "sum", "avg", "last", "root_means"):
            assert np.abs(s[k][0] - g[f"{k}{i}"][0]).max() < 1e-5, (k, i)     # after 1 step
            assert np.abs(s[k][1] - g[f"{k}{i}"][1]).max() < 1e-4, (k, i)     # after 2 steps
        assert np.abs(s["root_means"][2] - g[f"root_means{i}"][2]).max() < 1e-3


def test_selfplay_walk_bit_exact_vs_golden(port, golden):
    g = golden("selfplay_zero.npz")
    for (D, F) in SHAPES:
        for sl in (1, 0):
            q, v = port.rl_runner(D, F, seed=7, n_games=4, num_iters=32, sample_leaf=bool(sl))
            assert np.array_equal(q, g[f"q_{D}x{F}_{sl}"]) and np.array_equal(v, g[f"v_{D}x{F}_{sl}"])


@pytest.mark.parametrize("D,F", SHAPES)
def test_selfplay_walk_fictitious_play_bit_exact_vs_golden(port, golden, D, F):
    """The port's walk with the FP solver (use_cfr = False): sampling and belief propagation with FP's average strategies, the
    examples from its best-response pass, bit-identical to the reference's RlRunner(seed = 7) stream."""
    g = golden("selfplay_zero.npz")
    q, v = port.rl_runner(D, F, seed=7, n_games=4, num_iters=32, sample_leaf=True, use_cfr=False)
    assert np.array_equal(q, g[f"q_fp_{D}x{F}"]) and np.array_equal(v, g[f"v_fp_{D}x{F}"])


def test_selfplay_walk_beyond_nine_hands_bit_exact_vs_golden(port, golden):
    """The port's walk against the compiled reference's RlRunner at 7x1f, 2x6f, 1x17f, 3x4f and 4x3f (up to 81 hands and 35
    actions): CFR linear, plain and DCFR, linear FP, sample_leaf on and off, the zero net and a constant-output Net2
    (selfplay_large.npz, oracle/make_golden_r4.py)."""
    from oracle import make_golden_r4 as r4
    g = golden("selfplay_large.npz")
    keys = set()
    for c in r4.cases():
        k = r4.case_key(*c)
        q, v = r4.stream(port, *c)
        assert len(q) >= 2 * r4.GAMES_PER_STREAM, (k, len(q))
        assert np.array_equal(q, g["q_" + k]) and np.array_equal(v, g["v_" + k]), k
        keys |= {"q_" + k, "v_" + k}
    assert keys == set(g.files)


def test_selfplay_walk_trace_and_subgame_limit(port):
    """rl_runner(trace=True): one row per solved subgame, (game, root last_bid, root player, act_iteration, br_sampler), in the
    order of the examples; max_subgames cuts the same stream short."""
    D, F, iters = 2, 3, 3
    A, H, Q = game_dims(D, F)
    for sl in (True, False):
        q, v, tr = port.rl_runner(D, F, seed=11, n_games=6, num_iters=iters, sample_leaf=sl, trace=True, cap=4096)
        assert tr.shape == (len(q) // 2, 5) and len(q) % 2 == 0
        assert np.array_equal(np.unique(tr[:, 0]), np.arange(6))
        assert np.all(np.diff(tr[:, 0]) >= 0)
        first = np.r_[True, np.diff(tr[:, 0]) > 0]                        # every game starts at the initial state
        assert np.all(tr[first, 1] == -1) and np.all(tr[first, 2] == 0)
        assert np.all((tr[:, 3] >= 0) & (tr[:, 3] <= iters)) and {0, iters} <= set(tr[:, 3].tolist())
        assert set(tr[:, 4].tolist()) <= {0, 1}
        # the trace's root is the root of the examples: player and the one-hot last bid of both queries of each subgame
        for t in range(2):
            assert np.array_equal(q[t::2, 0], tr[:, 2].astype(np.float32)) and np.all(q[t::2, 1] == t)
            onehot = q[t::2, 2:2 + A]
            assert np.array_equal(np.where(onehot.any(1), onehot.argmax(1), -1), tr[:, 1])
        if not sl:                                                         # one action per subgame: the bids rise by player
            same = ~first[1:]
            assert np.all(tr[1:, 1][same] > tr[:-1, 1][same]) and np.all(tr[1:, 2][same] != tr[:-1, 2][same])
        n = len(tr) // 2
        q2, v2, tr2 = port.rl_runner(D, F, seed=11, n_games=6, num_iters=iters, sample_leaf=sl, trace=True, max_subgames=n)
        assert np.array_equal(q2, q[:2 * n]) and np.array_equal(v2, v[:2 * n]) and np.array_equal(tr2, tr[:n])


# ---------------------------------------------------------------- cross-check with the compiled reference's stored outputs
def test_port_vs_compiled_reference_live(port, golden):
    """The port against the compiled reference (fixture reference_live.npz, oracle/make_golden.py live): synthetic beliefs,
    40-iteration CFR solves from two roots and RlRunner example streams, bit for bit."""
    P, g = port, golden("reference_live.npz")
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        assert np.array_equal(P.synthetic_beliefs(H, 11), g[f"beliefs11_{D}x{F}"])
        b = P.synthetic_beliefs(H, 5)
        for lb, pl in [(-1, 0), (4, 1)]:
            x = P.cfr_solve(D, F, b, [0, 1, 5, 40], lb, pl, num_iters=40)
            for k in ("regrets", "last", "sum", "avg", "root_means", "traverser_values"):
                assert np.array_equal(x[k], g[f"{k}_{lb}_{pl}_{D}x{F}"]), (D, F, lb, k)
        qa, va = P.rl_runner(D, F, seed=3, n_games=2, num_iters=24)
        assert np.array_equal(qa, g[f"q_{D}x{F}"]) and np.array_equal(va, g[f"v_{D}x{F}"])


@pytest.mark.parametrize("D,F", SHAPES)
def test_port_recursive_eval_bit_exact_vs_golden(port, golden, D, F):
    """BASELINE config 5 in the C port: compute_sampled_strategy_recursive_to_leaf (recursive_solving.cc:76-134,301-327) with the
    restated mt19937 / discrete_distribution, reach weights of compute_stategy_stats and the float32 accumulation loop of
    recursive_eval.cc:343-369 reproduce the fixture generated from the compiled reference bit for bit."""
    from oracle.make_golden import recursive_eval_reference
    g = golden("recursive_eval_zero.npz")
    iters, reps = (int(x) for x in g[f"cfg_{D}x{F}"])
    r = recursive_eval_reference(port, D, F, iters, reps)
    for k in ("summed_strategy", "summed_reach", "checkpoints", "exploitability"):
        assert np.array_equal(r[k], g[f"{k}_{D}x{F}"]), k
    if (D, F) == (1, 4):
        assert np.array_equal(r["first_strategies"], g["first_strategies_1x4"])


@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("netname", ["zero_out", "random"])
def test_port_evaluation_entry_points_vs_golden(port, golden, use_cfr, netname):
    """compute_strategy_recursive / _to_leaf + exploitability + eval_net (rela/pybind.cc:45-84, recursive_solving.cc:46-134,
    stats.cc:44-153) in the C port against the fixture from the compiled reference: strategies bit-identical when the net's output
    layer is zero, all four numbers within 1e-6 relative (eval_net sums float32 terms in std::sort order; the port's scalar fp32
    net differs from ATen by ~1e-7)."""
    from oracle.make_golden import eval_weights
    g = golden("net_evaluation.npz")
    D, F, iters = 1, 4, 32
    tag = f"{'cfr' if use_cfr else 'fp'}_{netname}_{D}x{F}"
    r = port.net_evaluation(D, F, eval_weights(D, F, netname), num_iters=iters, use_cfr=use_cfr)
    want = g[f"values_{tag}"]
    assert np.all(np.abs(r["values"] - want) <= 1e-6 * np.abs(want)), (r["values"], want)
    if netname == "zero_out":
        assert np.array_equal(r["strategy_recursive"], g[f"strategy_recursive_{tag}"])
        assert np.array_equal(r["strategy_to_leaf"], g[f"strategy_to_leaf_{tag}"])


def test_reference_net_in_the_kernels_arithmetic(net_weights, golden):
    """ref_set_net_emulation (oracle/ref_harness.cc) evaluates the reference's own Net2 with the arithmetic of the tensor-core
    kernels (outputs stored in reference_live.npz) —
    the model behind the P5 comparison sets m1 / m2 of datagen_stats.npz.  Pinned here against an independent numpy restatement
    (fp16 operands, fp32 accumulation and LayerNorm, GELU of model 1 / 2 with one fp16 rounding per operation), and its error level
    against the fp32 net must be the kernels' measured one (5.0e-4 / 6.3e-4 relative rms)."""
    from scipy.special import erf
    D, F = 1, 6
    A, H, Q = game_dims(D, F)
    w = net_weights(D, F)
    g = golden("reference_live.npz")
    outs = {model: g[f"emulation{model}_leaf_values"].astype(np.float64) for model in (0, 1, 2)}
    q = g["emulation_queries"].astype(np.float64)
    for model, lo, hi in ((1, 3.5e-4, 7e-4), (2, 4.5e-4, 9e-4)):
        rel = np.sqrt(((outs[model] - outs[0]) ** 2).mean() / (outs[0] ** 2).mean())
        assert lo < rel < hi, (model, rel)
    # numpy restatement of model 2 on the same query rows (leaf value = net output x the opponent's reach sum; compare the ratios)
    h16 = lambda x: np.asarray(x, np.float64).astype(np.float16).astype(np.float64)
    o, parts = 0, []
    for shp in ((256, Q), (256,), (256,), (256,), (256, 256), (256,), (256,), (256,), (H, 256), (H,)):
        n = int(np.prod(shp)); parts.append(np.asarray(w[o:o + n], np.float64).reshape(shp)); o += n
    W1, b1, g1, be1, W2, b2, g2, be2, W3, b3 = parts

    def ln(x, g, bb):
        x = np.asarray(x, np.float32)
        m = x.mean(-1, keepdims=True); v = ((x - m) ** 2).mean(-1, keepdims=True)
        return ((x - m) / np.sqrt(v + np.float32(1e-5))).astype(np.float64) * g + bb

    def gelu2(y):
        hy = h16(y / 2)
        s = np.minimum(h16(hy * hy), 13.0)
        p = h16(s * h16(s * h16(-1.124832e-2) + h16(2.960456e-1)) + h16(1.594992))
        t = h16(np.tanh(h16(hy * p)))
        return h16(hy * t + hy)
    x = gelu2(ln(h16(q) @ h16(W1).T + b1, g1, be1))
    x = gelu2(ln(x @ h16(W2).T + b2, g2, be2))
    mine = x @ h16(W3).T + b3
    # the harness multiplies the net output by the opponent's reach sum (one scalar per row): recover it from the fp32 run
    ge = lambda y: 0.5 * y * (1 + erf(y / np.sqrt(2)))
    e = ge(ln(q @ W1.T + b1, g1, be1)); e = ge(ln(e @ W2.T + b2, g2, be2)); e = e @ W3.T + b3
    scaler = (outs[0] * e).sum(1) / (e * e).sum(1)
    want = mine * scaler[:, None]
    got = outs[2]
    err = np.sqrt(((got - want) ** 2).mean() / (want ** 2).mean())
    assert err < 1e-4, err         # the two restatements differ only in fp32 summation order (and the 2.4e-4 ulp of a flipped rounding)
