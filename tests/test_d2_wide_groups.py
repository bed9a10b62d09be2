"""The depth-2 CFR kernel solves a wave's costliest subgames on whole CTAs ("wide tickets", cfrb_debug_d2_wide) with every item of
every phase computed by one thread in the same order as on one warp, so results must not change by a bit: wide tickets off, the
wave's own rule and every solved subgame wide give the same examples, tables, root means, rebuilt sums and averages."""
import numpy as np
import pytest

from oracle.oracle import game_dims

ALL = 1 << 30      # more wide tickets than any wave has subgames: every solved subgame wide


def _tree_entries(S, D, F):
    """The compact tables' entries [n, table_stride] of the current wave's subgames: (N - 1) x H of each row; the rest holds whatever
    earlier waves or allocations left there."""
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    n_edges = np.array([len(capi.unroll_tree(D, F, b, 0, 2)) - 1 for b in range(-1, A - 1)])
    lb, _ = S.wave_roots()
    stride = S.fetch_compact("snapshot").shape[1]
    return np.arange(stride)[None, :] < (n_edges[lb + 1] * H)[:, None]


def _selfplay(D, F, K, iters, solver, dtype, mode, weights, wide, grid=0):
    """Every wave's examples, fetched tables and root means, the rebuilt sum and average of the last wave, and the session export of
    a self-play loop from the first wave (every game at the initial state) into stationary waves."""
    import rebel_b200 as rb
    S = rb.WaveSolver(D, F, K, num_iters=iters, net_mode=mode, solver=solver, state_dtype=dtype)
    if mode != rb.NET_ZERO:
        S.set_weights(weights)
    S.debug_d2_wide(wide)
    if grid:
        S.debug_d2_grid(grid)
    S.selfplay_create(np.uint32(7) + np.arange(K, dtype=np.uint32) * np.uint32(104729))
    out = []
    for i in range(6):
        S.selfplay_wave(keep_examples=i > 0)
        mask = _tree_entries(S, D, F)
        rec = {w: np.where(mask, S.fetch_compact(w), 0.0) for w in ("regrets", "last", "snapshot")}
        rec["mu"] = S.fetch(("root_means",))["root_means"]
        if i > 0:
            rec["q"], rec["v"] = S.selfplay_examples()
        out.append(rec)
    out.append({"sum": np.where(_tree_entries(S, D, F), S.fetch_compact("sum"), 0.0), "avg": S.fetch(("avg",))["avg"]})
    S.selfplay_wave(start_next=False, keep_examples=True)
    q, v = S.selfplay_examples()
    out.append({"q": q, "v": v, "image": np.frombuffer(S.selfplay_export(), np.uint8)})
    S.close()
    return out


def _same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys()
        for key in x:
            assert x[key].tobytes() == y[key].tobytes(), f"{what}: record {i}: {key}"


CASES = [   # (D, F, solver, state dtype, net)
    (1, 4, "cfr", "f64", "tc"), (1, 6, "cfr", "f64", "tc"), (2, 3, "cfr", "f64", "tc"),
    (1, 6, "fp", "f64", "tc"), (2, 3, "fp", "f64", "tc"),
    (1, 6, "cfr", "f32", "tc"), (1, 4, "fp", "f32", "tc"),
    (1, 6, "cfr", "f64", "zero"), (2, 3, "fp", "f32", "zero"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,solver,dtype,net", CASES)
def test_wide_tickets_selfplay_bit_identical(D, F, solver, dtype, net):
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    w = flatten_state_dict(make_selfplay_net(D, F, seed=5).state_dict())
    args = (D, F, 256, 40, rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP, rb.STATE_F64 if dtype == "f64" else rb.STATE_F32,
            rb.NET_TC_F16X2 if net == "tc" else rb.NET_ZERO, w)
    off = _selfplay(*args, wide=0)
    _same(off, _selfplay(*args, wide=-1), "rule")
    _same(off, _selfplay(*args, wide=ALL), "all wide")


@pytest.mark.gpu
def test_wide_tickets_selfplay_on_two_ctas():
    """Two CTAs take every solved subgame as a wide ticket and then draw the narrow counter dry, wave after wave: 64 iterations put
    the waves on a CUDA graph, whose replays must find both ticket counters back at zero."""
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    w = flatten_state_dict(make_selfplay_net(1, 6, seed=6).state_dict())
    args = (1, 6, 256, 64, rb.SOLVER_CFR, rb.STATE_F64, rb.NET_TC_F16X2, w)
    _same(_selfplay(*args, wide=0), _selfplay(*args, wide=ALL, grid=2), "all wide on two CTAs")


@pytest.mark.gpu
def test_wide_tickets_on_two_ctas_and_graph_replay():
    """Two CTAs take every wide ticket and then, warp by warp, every narrow one; the runs replayed from a CUDA graph on the same handle
    find both ticket counters back at zero."""
    import rebel_b200 as rb
    from oracle.oracle import Oracle
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, n, iters = 1, 6, 96, 64
    A, H, _ = game_dims(D, F)
    w = flatten_state_dict(make_selfplay_net(D, F, seed=2).state_dict())
    port = Oracle("port")
    rng = np.random.RandomState(4)
    lb = rng.randint(-1, A - 1, size=n).astype(np.int32)
    lb[:5] = -1
    pl = rng.randint(0, 2, size=n).astype(np.int32)
    b = np.stack([port.synthetic_beliefs(H, 50 + i) for i in range(n)])

    def solve(S):
        S.begin(lb, pl, b)
        S.run(iters)
        f = S.fetch(("root_means", "last", "avg", "sum", "regrets"))
        f["q"], f["v"] = S.examples()
        return f

    def handle(wide, grid):
        S = rb.WaveSolver(D, F, n, num_iters=iters, net_mode=rb.NET_TC_F16X2)
        S.set_weights(w)
        S.debug_d2_wide(wide)
        if grid:
            S.debug_d2_grid(grid)
        return S

    S = handle(0, 0)
    ref = solve(S)
    S.close()
    for wide in (ALL, n // 3):
        S = handle(wide, 2)
        for rep in range(3):     # eager, captured, replayed
            _same([ref], [solve(S)], f"wide {wide}, run {rep}")
        S.close()


@pytest.mark.gpu
def test_wide_ticket_lone_root_host_wave():
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    H = 6
    w = flatten_state_dict(make_selfplay_net(1, 6, seed=1).state_dict())
    rng = np.random.RandomState(9)
    b = rng.rand(1, 2, H)
    b /= b.sum(axis=2, keepdims=True)
    res = []
    for wide in (0, 1):
        S = rb.WaveSolver(1, 6, 1, num_iters=128, net_mode=rb.NET_TC_F16X2)
        S.set_weights(w)
        S.debug_d2_wide(wide)
        S.begin(np.array([-1], np.int32), np.array([0], np.int32), b, act_iteration=np.array([77], np.int32))
        S.run(128)
        f = S.fetch(("root_means", "snapshot", "last", "avg", "sum", "regrets"))
        f["q"], f["v"] = S.examples()
        res.append(f)
        S.close()
    _same([res[0]], [res[1]], "lone root")


@pytest.mark.gpu
def test_wide_ticket_rule_takes_them_where_they_pay():
    """The rule gives wide tickets to a self-play wave of 8192 games past its first waves and to a lone root, and none to a wave of
    8192 root subgames or of 64 root subgames on a 64-subgame handle (16 CTAs: wide roots would queue on them)."""
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, K = 1, 6, 8192
    A, H, _ = game_dims(D, F)
    w = flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())
    S = rb.WaveSolver(D, F, K, num_iters=64, net_mode=rb.NET_TC_F16X2)
    S.set_weights(w)
    S.selfplay_create(np.arange(K, dtype=np.uint32) * np.uint32(1000000))
    for _ in range(12):
        S.selfplay_wave()
    S.sync()
    m = S.wave_wide
    assert 0 < m < S.wave_solved, (m, S.wave_solved)
    S.selfplay_wave(start_next=False)
    S.sync()
    b = np.full((K, 2, H), 1.0 / H)
    S.begin(np.full(K, -1, np.int32), np.zeros(K, np.int32), b)
    assert S.wave_wide == 0
    S.close()
    for n, want in ((1, 1), (64, 0)):
        S = rb.WaveSolver(D, F, n, num_iters=64, net_mode=rb.NET_TC_F16X2)
        S.set_weights(w)
        S.begin(np.full(n, -1, np.int32), np.zeros(n, np.int32), b[:n])
        assert S.wave_wide == want, (n, S.wave_wide)
        S.close()
