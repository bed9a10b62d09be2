"""Dead value-net rows: the depth-2 CFR kernel leaves out of the tensor-core net's query tiles every pseudo-leaf whose opponent-reach
scaler s has s * B <= 2^-151, B the bound on the net's output of cfrb_set_weights.  The backward half forms (float)(net * s), which
is +-0 for such a leaf whatever the net returns, so nothing the solver computes may change.

CPU: the bound against the net on random rows, and a weight that is not finite turns it off.
GPU: every table, root value mean, leaf row, self-play example and match / local-best-response result byte for byte against the
same run with every row evaluated, on a resident-kernel game (1x6f, 2x3f) and a wide-kernel game (2x5f), in both tensor-core
modes, with fp64 and fp32 tables, and on a capped persistent grid whose warps take many subgames per launch; the wave test also
with weights away from the initialisation (the `distinct` and `trained` families of test_value_net_accuracy.py).
"""
import numpy as np
import pytest

from oracle.oracle import game_dims


def _net(D, F, seed, wide_layer2=False):
    import torch
    from rebel_b200.models import make_selfplay_net
    net = make_selfplay_net(D, F, seed=seed)
    if wide_layer2:     # LayerNorm 2 and the output layer far from their initialisation: a bound that leans on the init fails
        g = torch.Generator().manual_seed(100 + seed)
        with torch.no_grad():
            net.body[5].weight.copy_(torch.randn(256, generator=g) * 3)
            net.body[5].bias.copy_(torch.randn(256, generator=g) * 3)
            net.output.weight.copy_(torch.randn(net.output.weight.shape, generator=g) * 0.5)
            net.output.bias.copy_(torch.randn(net.output.bias.shape, generator=g))
    return net


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("D,F", [(1, 6), (2, 3), (2, 5)])
@pytest.mark.parametrize("wide_layer2", [False, True])
def test_output_bound_covers_the_net(D, F, wide_layer2):
    """B is finite and above |net(x)| for query-like rows and for rows of any scale (LayerNorm bounds the net whatever x is)."""
    import torch
    from rebel_b200 import capi
    from rebel_b200.models import flatten_state_dict
    A, H, Q = game_dims(D, F)
    worst = 0.0
    for seed in range(3):
        net = _net(D, F, seed, wide_layer2)
        B = capi.net_output_bound(D, F, flatten_state_dict(net.state_dict()))
        assert np.isfinite(B) and B > 0
        rng = np.random.RandomState(seed)
        n = 4096
        x = np.zeros((n, Q))
        x[:, 0] = rng.randint(0, 2, n); x[:, 1] = rng.randint(0, 2, n)
        x[np.arange(n), 2 + rng.randint(0, A, n)] = 1
        b = rng.rand(n, 2, H) ** 4
        x[:, 2 + A:] = (b / b.sum(-1, keepdims=True)).reshape(n, 2 * H)
        x = np.concatenate([x, rng.randn(n, Q) * 10.0 ** rng.uniform(-3, 4, (n, 1))])
        with torch.no_grad():
            out = net(torch.from_numpy(x).float()).abs().max().item()
        assert out <= B, (seed, out, B)
        worst = max(worst, out / B)
    assert worst > 1e-3        # not vacuous


def test_output_bound_off_for_non_finite_weights():
    from rebel_b200 import capi
    from rebel_b200.models import flatten_state_dict
    w = flatten_state_dict(_net(1, 6, 0).state_dict())
    assert np.isfinite(capi.net_output_bound(1, 6, w))
    for i, v in [(5, np.nan), (w.size - 1, np.inf), (w.size // 2, -np.inf)]:
        bad = w.copy()
        bad[i] = v
        assert capi.net_output_bound(1, 6, bad) == np.inf, i
    with pytest.raises(capi.CfrbError):
        capi.net_output_bound(1, 6, w[:-1])


# ---------------------------------------------------------------------------------------------- GPU
MODES = ["NET_TC_F16", "NET_TC_F16X2"]
GAMES = [(1, 6), (2, 3), (2, 5)]


def _solver(rb, D, F, K, mode, dtype, skip, w, cap=0, **kw):
    S = rb.WaveSolver(D, F, K, net_mode=getattr(rb, mode), state_dtype=dtype, **kw)
    S.debug_skip_dead_rows(skip)
    S.set_weights(w)
    if cap:
        S.debug_d2_grid(cap)
    return S


def _same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), \
        (what, int((a != b).sum()), float(np.nanmax(np.abs(a.astype(np.float64) - b.astype(np.float64)))))


# weight families of test_value_net_accuracy.py: the initialisation, every LayerNorm parameter distinct with the output layer x30,
# and the trainer's weights after 400 steps (on the games that generate training data)
GAME_FAMILIES = [(D, F, fam) for D, F in GAMES for fam in ("init", "distinct", "trained") if fam != "trained" or (D, F) != (2, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [0, 3])
@pytest.mark.parametrize("dtype", ["STATE_F64", "STATE_F32"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,F,family", GAME_FAMILIES)
def test_wave_bit_identical_without_dead_rows(D, F, family, mode, dtype, cap):
    """A wave of mixed roots, 90 iterations in two runs (the second replayed from a CUDA graph on its second call): regrets, last
    and sum strategies, snapshot, root value means and the leaf rows (queries, net outputs, scalers) byte for byte with and without
    the dead rows; the evaluated-row counter adds up."""
    import rebel_b200 as rb
    from test_value_net_accuracy import family_weights
    A, H, Q = game_dims(D, F)
    K = 600
    rng = np.random.RandomState(D * 10 + F)
    b = rng.rand(K, 2, H) ** 3
    b /= b.sum(-1, keepdims=True)
    lb = rng.randint(-1, A - 2, size=K).astype(np.int32); lb[:8] = -1
    pl = rng.randint(0, 2, size=K).astype(np.int32)
    act = rng.randint(0, 90, size=K).astype(np.int32)
    w = family_weights(family, D, F)
    got = []
    for skip in (True, False):
        S = _solver(rb, D, F, K, mode, getattr(rb, dtype), skip, w, cap)
        assert S.kernel_path() == 0
        e0 = S.net_rows_evaluated
        for _ in range(2):               # the same key twice: the second wave is captured into a graph
            S.begin(lb, pl, b, act)
            S.run(64)
            S.run(26)
        ev = S.net_rows_evaluated - e0
        rows = S.leaf_rows
        r = {k: S.fetch_compact(k) for k in ("snapshot", "last", "sum", "regrets")}
        r["mu"] = S.fetch(("root_means",))["root_means"]
        r["q"], r["out"], r["sc"] = S.leaf_io()
        S.close()
        got.append((r, ev, rows))
    (on, ev_on, rows), (off, ev_off, rows_off) = got
    assert rows == rows_off and ev_off == 2 * 90 * rows, (ev_off, rows)
    dead_frac = 1 - ev_on / ev_off
    print(f"[dead-rows] {D}x{F}f {family} {mode} {dtype} cap {cap}: {100 * dead_frac:.1f} % of the rows dead")
    assert 0 < dead_frac < 1
    for k in ("snapshot", "last", "sum", "regrets", "mu", "q", "out", "sc"):
        _same(on[k], off[k], k)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["STATE_F64", "STATE_F32"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_selfplay_examples_bit_identical_without_dead_rows(net_weights, D, F, mode, dtype):
    """The device self-play loop: every wave's training examples byte for byte, and fewer rows evaluated."""
    import rebel_b200 as rb
    K, iters, waves = 256, 64, 5
    got = []
    for skip in (True, False):
        S = _solver(rb, D, F, K, mode, getattr(rb, dtype), skip, net_weights(D, F), num_iters=iters)
        S.selfplay_create(np.uint32(17) + np.arange(K, dtype=np.uint32) * np.uint32(1000003))
        S.selfplay_wave()
        ex = []
        for _ in range(waves):
            S.selfplay_wave(keep_examples=True)
            ex.append(S.selfplay_examples())
        S.selfplay_wave(start_next=False)
        S.sync()
        got.append((ex, S.net_rows_evaluated))
        S.close()
    (ex_on, ev_on), (ex_off, ev_off) = got
    for (q0, v0), (q1, v1) in zip(ex_on, ex_off):
        _same(q0, q1, "queries"); _same(v0, v1, "values")
    print(f"[dead-rows] self-play {D}x{F}f {mode} {dtype}: {100 * (1 - ev_on / ev_off):.1f} % of the rows dead")
    assert ev_on < ev_off


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_match_and_lbr_bit_identical_without_dead_rows(net_weights, mode):
    """Head-to-head match and local best response at 1x6f: payoffs, plies and the traced probabilities byte for byte."""
    import rebel_b200 as rb
    from rebel_b200 import capi
    D, F = 1, 6
    w = net_weights(D, F)
    got = []
    for skip in (True, False):
        mk = lambda: _solver(rb, D, F, 64, mode, rb.STATE_F64, skip, w, num_iters=48)
        a, b = mk(), mk()
        M = capi.Match(a, b, 64, 128, seed=5, policy=capi.MATCH_SAMPLED)
        res = M.play()
        tr = M.trace(3)
        M.close()
        L = capi.LbrMatch(a, 32, 32, seed=9)
        lres = L.play()
        ltr = L.lbr_trace(1)
        L.close()
        a.close(); b.close()
        got.append((res, tr, lres, ltr))
    (r0, t0, l0, lt0), (r1, t1, l1, lt1) = got
    for k in ("payoff_a", "plies"):
        _same(r0[k], r1[k], k); _same(l0[k], l1[k], "lbr " + k)
    assert r0["solves"] == r1["solves"] and l0["solves"] == l1["solves"]
    _same(t0["prob"], t1["prob"], "trace prob")
    _same(lt0["values"], lt1["values"], "lbr values")
