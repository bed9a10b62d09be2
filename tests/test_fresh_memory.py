"""No result may depend on what fresh device memory holds.  cfrb_debug_fill_allocations(byte) fills every floating-point device
buffer the library allocates with one byte before it is used; each solve below runs with the fill off and under every pattern, and
its outputs must be bit-identical, and equal to the bit-exact reference where one exists (the C port, one-subgame wave solves, the
host's strategy_reach).  A fresh process usually gets zero pages from cudaMalloc, so a read of memory nobody wrote, a missing
memset or a copy that races a memset passes every other test here.

Patterns: 0x00; 0xFF (NaN in every type); 0x7F (~1e306 in fp64, 3.4e38 in fp32, NaN in fp16); 0xBF (finite negative: -0.12 in
fp64, -1.5 in fp32, where the solver only ever stores non-negative reach, regrets and sums); 0x47 (finite positive: 2e35 in fp64,
5e4 in fp32)."""
import contextlib

import numpy as np
import pytest

from oracle.oracle import game_dims
from test_game_matrix import CPS, CTA, FULL, ONE_PER_PATH, beliefs, case_id, compare_with_port, roots_of

PATTERNS = (0x00, 0xFF, 0x7F, 0xBF, 0x47)
_FILL = [-1]


def _set_fill(byte):
    from rebel_b200 import capi
    capi._check(capi.lib().cfrb_debug_fill_allocations(byte))
    _FILL[0] = byte


@contextlib.contextmanager
def filled(byte):
    """Fresh floating-point device buffers hold `byte` (-1: whatever cudaMalloc gives) inside the block."""
    prev = _FILL[0]
    _set_fill(byte)
    try:
        yield
    finally:
        _set_fill(prev)


@pytest.fixture
def fill():
    """`filled`, with the fill off again after the test whatever happens."""
    try:
        yield filled
    finally:
        _set_fill(-1)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _diff(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if a.shape != b.shape:
        return f"shape {a.shape} vs {b.shape}"
    bad = a.view(np.int64) != b.view(np.int64)
    return f"{int(bad.sum())} of {a.size} entries differ, {int((~np.isfinite(a)).sum())} non-finite"


def _check_records(got, want, tag):
    assert got.keys() == want.keys(), tag
    for k in want:
        assert _same(got[k], want[k]), (tag, k, _diff(got[k], want[k]))


# ------------------------------------------------------------------------------------------------------------------------ CPU
def test_fill_argument_is_checked_before_any_device_work():
    from rebel_b200 import capi
    for bad in (256, -2, 1 << 20):
        with pytest.raises(capi.CfrbError, match="cfrb_debug_fill_allocations"):
            capi._check(capi.lib().cfrb_debug_fill_allocations(bad))
    try:
        capi._check(capi.lib().cfrb_debug_fill_allocations(0x7F))
    finally:
        capi._check(capi.lib().cfrb_debug_fill_allocations(-1))


# ------------------------------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def rb():
    import rebel_b200
    assert rebel_b200.capi.lib().cfrb_device_count() > 0, "no CUDA device: the CUDA path cannot be tested"
    return rebel_b200


def _memo(solve):
    """The port's solve, computed once per subgame: the same reference serves every pattern."""
    cache = {}

    def f(D, F, b, cps, lb, pl, **kw):
        key = (D, F, b.tobytes(), tuple(cps), lb, pl, tuple(sorted(kw.items())))
        if key not in cache:
            cache[key] = solve(D, F, b, cps, lb, pl, **kw)
        return cache[key]
    return f


WAVE_CASES = ONE_PER_PATH + [(1, 5, FULL, "f64", CTA, 0)]


SOLVERS = ["linear_cfr", "linear_fp", "optimistic_fp"]


def _solver_kw(rb, port, solver):
    """(wave solver settings, the port's solve, the tables to compare)."""
    if solver == "linear_cfr":
        return {}, port.cfr_solve, ("regrets", "last", "sum", "avg")
    optimistic = solver == "optimistic_fp"

    def fp_solve(D, F, b, cps, lb, pl, num_iters, max_depth, solver, optimistic):
        return port.fp_solve(D, F, b, cps, lb, pl, num_iters=num_iters, max_depth=max_depth, optimistic=optimistic)
    return dict(solver=rb.SOLVER_FP, optimistic=optimistic), fp_solve, ("last", "sum", "avg")


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("case", WAVE_CASES, ids=case_id)
def test_wave_paths_equal_the_port_under_every_fill(rb, port, fill, case, solver):
    """Each CFR kernel path (d2, warp, CTA, and the CTA path on a full-depth tree) with fp64 tables and the zero net: root means and
    tables bit-identical to the C port with the fill off and under every pattern."""
    kw, solve, keys = _solver_kw(rb, port, solver)
    solve = _memo(solve)
    for byte in (-1,) + PATTERNS:
        with fill(byte):
            compare_with_port(rb, port, case, kw, solve, keys)


def _wave_records(rb, D, F, md, cps, keys, weights=None, **kw):
    """root means and `keys` tables of a wave of test_game_matrix.roots_of at every checkpoint of cps."""
    A, H, _ = game_dims(D, F)
    roots = roots_of(A)
    S = rb.WaveSolver(D, F, len(roots), max_depth=md, **kw)
    if weights is not None:
        S.set_weights(weights)
    S.begin([r[0] for r in roots], [r[1] for r in roots], beliefs(H, len(roots), 1000 * D + F))
    out, done = {}, 0
    for c in cps:
        S.run(c - done)
        done = c
        for k, v in S.fetch(("root_means",) + tuple(keys)).items():
            out[f"{k}@{c}"] = v
    path = S.kernel_path()
    S.close()
    return out, path


@pytest.mark.gpu
@pytest.mark.parametrize("solver", SOLVERS)
def test_fp32_tables_on_the_cta_path_under_every_fill(rb, fill, solver):
    kw = {} if solver == "linear_cfr" else dict(solver=rb.SOLVER_FP, optimistic=solver == "optimistic_fp")
    keys = ("regrets", "last", "sum", "avg") if solver == "linear_cfr" else ("last", "sum", "avg")
    run = lambda: _wave_records(rb, 2, 7, 2, CPS, keys, net_mode=rb.NET_ZERO, state_dtype=rb.STATE_F32, **kw)
    want, path = run()
    assert path == CTA
    assert all(np.isfinite(v).all() for v in want.values())
    for byte in PATTERNS:
        with fill(byte):
            got, _ = run()
        _check_records(got, want, (solver, hex(byte)))


def _tc_mode(rb, D, F):
    from rebel_b200 import capi
    if capi.tc_net_supported(D, F):
        return rb.NET_TC_F16X2
    assert capi.tc_cluster_net_supported(D, F), (D, F)
    return rb.NET_TC_CLUSTER


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,md", [(6, 2, 1), (5, 2, 2), (2, 7, 2)], ids=["6x2f-d1", "5x2f-d2", "2x7f-d2"])
@pytest.mark.parametrize("net", ["fp32", "tc"])
def test_value_net_paths_under_every_fill(rb, fill, D, F, md, net):
    """NET_FP32 and the tensor-core net that serves the game (the wide kernel at 5x2f, the cluster kernel at 6x2f and 2x7f) with
    trained weights: eight subgames leave one partial query tile, so its padding rows and columns, and at 6x2f and 5x2f the
    compacted tiles of the depth-2 kernel (row_src, dead rows), meet the fill."""
    from test_value_net_accuracy import trained_weights
    w = trained_weights(D, F)
    mode = rb.NET_FP32 if net == "fp32" else _tc_mode(rb, D, F)
    run = lambda: _wave_records(rb, D, F, md, [1, 2, 3, 17], ("regrets", "last", "sum", "avg"), weights=w, net_mode=mode)
    want, _ = run()
    assert all(np.isfinite(v).all() for v in want.values())
    for byte in PATTERNS:
        with fill(byte):
            got, _ = run()
        _check_records(got, want, (D, F, md, mode, hex(byte)))


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["cfr", "fp"])
def test_selfplay_waves_under_every_fill(rb, fill, solver):
    """Self-play waves at 2x4f with the shared initial-state solve, as test_selfplay_share runs them: every wave's tables (their
    trees' entries), root means and examples, and the exported session, bit-identical under every pattern."""
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    from test_selfplay_share import _session
    D, F, K, iters = 2, 4, 256, 48
    w = flatten_state_dict(make_selfplay_net(D, F, seed=3).state_dict())
    sv = rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP
    want, solved = _session(D, F, K, iters, sv, rb.STATE_F64, True, w)
    assert solved[0] == (1, K)
    for byte in PATTERNS:
        with fill(byte):
            got, got_solved = _session(D, F, K, iters, sv, rb.STATE_F64, True, w)
        assert got_solved == solved, hex(byte)
        assert len(got) == len(want)
        for i, (a, b) in enumerate(zip(got, want)):
            _check_records(a, b, (solver, hex(byte), f"record {i}"))


def _full_game(rb, solver):
    from rebel_b200 import capi
    g = capi.FullGame(2, 4, solver=solver)
    if solver == rb.SOLVER_CFR:
        g.track_regrets()
    out, done = {}, 0
    for c in (1, 2, 7, 16):
        g.step(c - done)
        done = c
        out[f"exploitability@{c}"] = g.exploitability()
    out["strategy"] = g.strategy()
    if solver == rb.SOLVER_CFR:
        imm, sums, node, count = g.regrets()
        out.update(immediate=imm, sums=sums, node_sums=node, count=np.int64(count))
    g.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["cfr", "fp"])
def test_full_game_under_every_fill(rb, fill, solver):
    sv = rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP
    want = _full_game(rb, sv)
    assert all(np.isfinite(v).all() for v in want.values())
    for byte in PATTERNS:
        with fill(byte):
            got = _full_game(rb, sv)
        _check_records(got, want, (solver, hex(byte)))


@pytest.mark.gpu
def test_fp_forest_under_every_fill(rb, fill):
    """FpForest.solve on test_gpu_forest_bit_exact_against_wave_subgames's roots at 2x4f against one-subgame wave solves (fill
    off), and FpForest.reach against the host's strategy_reach, under every pattern."""
    from rebel_b200 import capi
    from test_stats_to_leaf import compact_reach, full_tree, real_beliefs, wave_means
    D, F = 2, 4
    A, H = 2 * D * F + 1, F ** D
    tree = full_tree(D, F)
    cases = []
    for depth in (1, 2, 3, 4):
        cand = np.nonzero((tree[:, 5] == depth) & (tree[:, 0] != A - 1))[0]
        nodes = np.unique(cand[np.linspace(0, len(cand) - 1, min(len(cand), 12)).astype(int)])
        b = real_beliefs(D, F, tree, nodes, seed=depth)
        for iters in (1, 2, 7, 64):
            cases.append((depth, nodes, b, iters, wave_means(D, F, tree, nodes, b, iters)))
    g = capi.FullGame(D, F)
    g.step(16)
    s = g.strategy()
    g.close()
    r, node_reach = compact_reach(tree, H, s)
    rnodes = np.concatenate([[0], np.nonzero(((tree[:, 5] == 2) | (tree[:, 5] == 4)) & (tree[:, 0] != A - 1))[0]])
    for byte in (-1,) + PATTERNS:
        with fill(byte):
            f = capi.FpForest(D, F)
            for depth, nodes, b, iters, want in cases:
                got = f.solve(depth, nodes, b, iters)
                assert _same(got, want), (hex(byte), depth, iters, _diff(got, want))
            nr, rows = f.reach(s, rnodes)
            f.close()
        assert _same(nr, node_reach[rnodes]), (hex(byte), _diff(nr, node_reach[rnodes]))
        want_rows = np.transpose(r[:, rnodes], (1, 0, 2))
        assert _same(rows, want_rows), (hex(byte), _diff(rows, want_rows))


@pytest.mark.gpu
def test_two_large_fp_waves_on_the_cta_path_equal_the_forest(rb, fill):
    """2x5f: the 364 non-terminal depth-4 roots with last bid 14 (subtree depth 6), positive beliefs, 16 iterations of linear FP
    in one WaveSolver(max_depth=6) on the CTA-group path, two handles back to back (each closed before the next opens), with the
    fill off and under every pattern: every root of every handle equals FpForest.solve bit for bit.  Each handle holds four
    [364][82k nodes x 25 hands] fp64 tables (table_stride is set by the largest depth-6 template, the one at the initial state)."""
    from rebel_b200 import capi
    from test_stats_to_leaf import full_tree
    D, F = 2, 5
    A, H = 2 * D * F + 1, F ** D
    tree = full_tree(D, F)
    nodes = np.nonzero((tree[:, 5] == 4) & (tree[:, 0] == 14))[0]
    assert len(nodes) == 364
    rng = np.random.RandomState(0)
    b = rng.rand(len(nodes), 2, H) + 0.01
    b /= b.sum(-1, keepdims=True)
    f = capi.FpForest(D, F)
    want = f.solve(4, nodes, b, 16)
    f.close()
    assert np.isfinite(want).all()
    bad = []
    for byte in (-1,) + PATTERNS:
        for handle in (1, 2):
            with fill(byte):
                W = capi.WaveSolver(D, F, len(nodes), max_depth=6, num_iters=16, net_mode=capi.NET_ZERO, solver=capi.SOLVER_FP,
                                    linear_update=True)
                assert W.kernel_path() == CTA
                W.begin(tree[nodes, 0].astype(np.int32), tree[nodes, 1].astype(np.int32), b)
                W.run(16)
                mu = W.fetch(("root_means",))["root_means"]
                W.close()
            if not _same(mu, want):
                roots = (mu.reshape(len(nodes), -1).view(np.int64) != want.reshape(len(nodes), -1).view(np.int64)).any(1)
                nan = (~np.isfinite(mu.reshape(len(nodes), -1))).any(1)
                bad.append(f"fill {byte:#x} handle {handle}: {int(roots.sum())} of {len(nodes)} roots differ, {int(nan.sum())} NaN")
    assert not bad, bad


@pytest.mark.gpu
def test_compute_stats_with_net_under_every_fill(rb, fill, tmp_path):
    """compute_stats_with_net at 2x4f (mdp_depth 1, 64 iterations, seed-0 net) twice on the dense path and once with device_walk:
    three finite, equal triples, with the fill off and under every pattern."""
    import rebel_b200.rela as rela
    from test_stats_to_leaf import _save_model, stats_cfg
    path = _save_model(tmp_path, 2, 4, "random")
    cfg = stats_cfg(rela, 2, 4, 64, mdp_depth=1)
    want = None
    for byte in (-1,) + PATTERNS:
        with fill(byte):
            got = [rela.compute_stats_with_net(cfg, path, device_walk=dw) for dw in (False, False, True)]
        assert all(np.isfinite(t).all() for t in got), (hex(byte), got)
        assert got[0] == got[1] == got[2], (hex(byte), got)
        want = got[0] if want is None else want
        assert got[0] == want, (hex(byte), got[0], want)
