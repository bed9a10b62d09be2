"""CFR self-play waves do not maintain the sum-strategy table S (the self-play loop reads only snapshots and root value means); a
reader of S rebuilds it by solving the wave again.  The rebuilt sum and average strategy must be the bits a host wave of the same
roots computes, reading them must not change anything the loop produces, and they are refused once the weights have changed."""
import numpy as np
import pytest

from oracle.oracle import game_dims


def _edges(tab, lb, D, F):
    """The entries of compact [n][table_stride] tables that belong to each subgame's tree."""
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    n_edges = np.array([len(capi.unroll_tree(D, F, b, 0, 2)) - 1 for b in range(-1, A - 1)])
    mask = np.arange(tab.shape[1])[None, :] < (n_edges[lb + 1] * H)[:, None]
    return np.where(mask, tab, 0.0)


def _solver(D, F, K, iters, solver, dtype, w):
    import rebel_b200 as rb
    S = rb.WaveSolver(D, F, K, num_iters=iters, net_mode=rb.NET_TC_F16X2,
                      solver=rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP,
                      state_dtype=rb.STATE_F64 if dtype == "f64" else rb.STATE_F32)
    S.set_weights(w)
    return S


def _seeds(K):
    return np.uint32(17) + np.arange(K, dtype=np.uint32) * np.uint32(1000003)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 3)])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_rebuilt_sum_matches_a_host_wave(D, F, dtype, net_weights):
    K, iters, waves = 256, 64, 3
    w = net_weights(D, F)
    S = _solver(D, F, K, iters, "cfr", dtype, w)      # reads the sum after its waves
    T = _solver(D, F, K, iters, "cfr", dtype, w)      # the same loop, never reading it
    for X in (S, T):
        X.selfplay_create(_seeds(K))
        X.selfplay_wave()
        for _ in range(waves):
            X.selfplay_wave(keep_examples=True)
    lb, pl = S.wave_roots()
    assert len(np.unique(lb)) > 3
    bel = S.selfplay_state()[2]
    mu0 = S.fetch(("root_means",))["root_means"]
    snap0 = S.fetch_compact("snapshot")
    launches = S.kernel_launches
    got_sum = S.fetch_compact("sum")
    assert S.kernel_launches > launches               # the wave was solved again
    launches = S.kernel_launches
    got_avg = S.fetch(("avg",))["avg"]
    assert S.kernel_launches == launches              # ... once
    # the rebuild rewrote the wave's other tables with the bits they held
    assert np.array_equal(S.fetch(("root_means",))["root_means"], mu0)
    assert np.array_equal(S.fetch_compact("snapshot"), snap0)
    assert np.array_equal(T.fetch(("root_means",))["root_means"], mu0)
    assert np.array_equal(T.fetch_compact("snapshot"), snap0)
    # ... and the loop goes on as if nothing had been read: the examples of that wave and of the next one
    for _ in range(2):
        S.selfplay_wave(keep_examples=True)
        T.selfplay_wave(keep_examples=True)
        for a, b in zip(S.selfplay_examples(), T.selfplay_examples()):
            assert np.array_equal(a, b)
    T.close()
    # a host wave of the same roots keeps S from the start
    Hw = _solver(D, F, K, iters, "cfr", dtype, w)
    Hw.begin(lb, pl, bel)
    Hw.run(iters)
    assert np.array_equal(Hw.fetch(("root_means",))["root_means"], mu0)
    assert np.array_equal(_edges(got_sum, lb, D, F), _edges(Hw.fetch_compact("sum"), lb, D, F))
    assert np.array_equal(got_avg, Hw.fetch(("avg",))["avg"])
    Hw.close()
    # a finished wave (no next wave started) is rebuilt the same way
    lb, pl = S.wave_roots()
    bel = S.selfplay_state()[2]
    S.selfplay_wave(start_next=False)
    got_sum = S.fetch_compact("sum")
    Hw = _solver(D, F, K, iters, "cfr", dtype, w)
    Hw.begin(lb, pl, bel)
    Hw.run(iters)
    assert np.array_equal(_edges(got_sum, lb, D, F), _edges(Hw.fetch_compact("sum"), lb, D, F))
    Hw.close()
    S.close()


@pytest.mark.gpu
def test_sum_read_after_new_weights_is_refused(net_weights):
    from rebel_b200.capi import CfrbError
    D, F, K, iters = 1, 6, 128, 64
    w = net_weights(D, F)
    S = _solver(D, F, K, iters, "cfr", "f64", w)
    S.selfplay_create(_seeds(K))
    S.selfplay_wave()
    S.selfplay_wave()
    S.sync()
    mu = S.fetch(("root_means",))["root_means"]
    S.set_weights(w, version=7)          # even the same weights: the wave cannot be proven to replay
    for read in (lambda: S.fetch_compact("sum"), lambda: S.fetch(("avg",)), lambda: S.fetch(("sum",))):
        with pytest.raises(CfrbError, match="weights"):
            read()
    # what the loop reads is still there
    assert np.array_equal(S.fetch(("root_means",))["root_means"], mu)
    # the next wave is solved with the new weights and can be rebuilt
    S.selfplay_wave()
    assert np.isfinite(S.fetch_compact("sum")).all()
    S.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_fp_selfplay_keeps_the_sum(dtype, net_weights):
    D, F, K, iters = 1, 6, 128, 64
    w = net_weights(D, F)
    S = _solver(D, F, K, iters, "fp", dtype, w)
    S.selfplay_create(_seeds(K))
    S.selfplay_wave()
    S.selfplay_wave()
    lb, pl = S.wave_roots()
    bel = S.selfplay_state()[2]
    launches = S.kernel_launches
    got_sum = S.fetch_compact("sum")
    assert S.kernel_launches == launches              # no rebuild
    Hw = _solver(D, F, K, iters, "fp", dtype, w)
    Hw.begin(lb, pl, bel)
    Hw.run(iters)
    assert np.array_equal(_edges(got_sum, lb, D, F), _edges(Hw.fetch_compact("sum"), lb, D, F))
    S.close()
    Hw.close()
