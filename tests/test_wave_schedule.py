"""The depth-2 CFR kernel's schedule: persistent warps take the wave's subgames costliest first (sg_order, a stable sort by
template cost built on the host for cfrb_begin_wave and in sp_scan_kernel for self-play waves).  Which warp solves a subgame,
and when, must not change a bit of any result."""
import numpy as np
import pytest

from oracle.oracle import game_dims


def _template_costs(D, F):
    """(N - 1) x H + L of every depth-2 template, from the tree enumeration."""
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    out = []
    for lb in range(-1, A - 1):
        t = capi.unroll_tree(D, F, lb, 0, 2)
        nchild = t[:, 3] - t[:, 2]
        L = int(((nchild == 0) & (t[:, 0] != A - 1)).sum())
        out.append((len(t) - 1) * H + L)
    return np.array(out, np.int64)


def _edges(tab, lb, D, F):
    """The entries of compact [n][table_stride] tables that belong to each subgame's tree ((N - 1) x H of them; the rest of a
    row is whatever an earlier wave left there)."""
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    n_edges = np.array([len(capi.unroll_tree(D, F, b, 0, 2)) - 1 for b in range(-1, A - 1)])
    mask = np.arange(tab.shape[1])[None, :] < (n_edges[lb + 1] * H)[:, None]
    return np.where(mask, tab, 0.0)


@pytest.mark.parametrize("D,F", [(1, 6), (2, 5), (2, 3)])
def test_host_schedule_sorts_by_template_cost(D, F):
    from rebel_b200 import capi
    A, _, _ = game_dims(D, F)
    tcost = _template_costs(D, F)
    lb = np.random.RandomState(D * 10 + F).randint(-1, A - 1, size=777).astype(np.int32)
    order, cost = capi.schedule_order(D, F, lb)
    assert np.array_equal(cost, tcost[lb + 1])
    # costliest first; equal costs by template index, then by wave position (stable)
    expect = sorted(range(lb.size), key=lambda k: (-tcost[lb[k] + 1], lb[k], k))
    assert np.array_equal(order, np.array(expect, np.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_wave_order_is_the_cost_sort(D, F):
    import rebel_b200 as rb
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    K = 1024
    S = rb.WaveSolver(D, F, K, num_iters=8, net_mode=rb.NET_ZERO)
    # a self-play wave a few steps into the games: subgames of many sizes, ordered on the device
    S.selfplay_create(np.arange(K, dtype=np.uint32) * np.uint32(7919) + np.uint32(5))
    for _ in range(6):
        S.selfplay_wave()
    lb, _ = S.wave_roots()
    assert len(np.unique(lb)) > 3
    order = S.wave_order()
    host, cost = capi.schedule_order(D, F, lb)
    assert np.array_equal(np.sort(order), np.arange(K))
    assert np.all(np.diff(cost[order]) <= 0)
    assert np.array_equal(order, host)
    S.selfplay_wave(start_next=False)
    # a host-built wave
    rng = np.random.RandomState(3)
    lb = rng.randint(-1, A - 1, size=K).astype(np.int32)
    b = rng.rand(K, 2, H) + 0.1
    S.begin(lb, rng.randint(0, 2, size=K).astype(np.int32), b / b.sum(-1, keepdims=True))
    assert np.array_equal(S.wave_order(), capi.schedule_order(D, F, lb)[0])
    S.close()


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["cfr", "fp"])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_results_do_not_depend_on_the_schedule(solver, dtype):
    """Self-play examples, root value means and sampling-strategy snapshots, bit for bit: the resident grid, a grid of two CTAs
    (every warp solves dozens of subgames per launch), and a host wave holding the same subgames at shuffled positions."""
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, K, iters, waves = 1, 6, 512, 64, 4
    A, H, _ = game_dims(D, F)
    kw = dict(num_iters=iters, net_mode=rb.NET_TC_F16X2, solver=rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP,
              state_dtype=rb.STATE_F64 if dtype == "f64" else rb.STATE_F32)
    w = flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())
    seeds = np.uint32(11) + np.arange(K, dtype=np.uint32) * np.uint32(1000000)

    def selfplay(cap):
        S = rb.WaveSolver(D, F, K, **kw)
        S.set_weights(w)
        resident = S.debug_d2_grid(cap)
        assert cap == 0 or resident > cap
        S.selfplay_create(seeds)
        S.selfplay_wave()
        q, v = [], []
        for _ in range(waves):
            S.selfplay_wave(keep_examples=True)
            a, c = S.selfplay_examples()
            q.append(a); v.append(c)
        # the wave now solved: its subgames, root value means, snapshots and sums
        out = {"q": np.concatenate(q), "v": np.concatenate(v), "mu": S.fetch(("root_means",))["root_means"],
               "snap": S.fetch_compact("snapshot"), "sum": S.fetch_compact("sum"), "roots": S.wave_roots(),
               "bel": S.selfplay_state()[2]}
        return S, out

    S, ref = selfplay(0)
    assert len(np.unique(ref["roots"][0])) > 3       # a mixed wave
    S2, capped = selfplay(2)
    S2.close()
    for key in ("q", "v", "mu", "snap", "sum"):
        assert np.array_equal(ref[key], capped[key]), key
    # the same subgames as a host wave, in wave order and at shuffled positions (same act_iteration per subgame)
    lb, pl = ref["roots"]
    bel = ref["bel"]
    act = np.random.RandomState(5).randint(0, iters + 1, size=K).astype(np.int32)
    S.begin(lb, pl, bel, act)
    S.run(iters)
    f0 = S.fetch(("root_means",))["root_means"]
    s0, m0 = _edges(S.fetch_compact("snapshot"), lb, D, F), _edges(S.fetch_compact("sum"), lb, D, F)
    assert np.array_equal(f0, ref["mu"])
    assert np.array_equal(m0, _edges(ref["sum"], lb, D, F))
    perm = np.random.RandomState(6).permutation(K)
    S.begin(lb[perm], pl[perm], bel[perm], act[perm])
    S.run(iters)
    assert np.array_equal(S.fetch(("root_means",))["root_means"], f0[perm])
    assert np.array_equal(_edges(S.fetch_compact("snapshot"), lb[perm], D, F), s0[perm])
    assert np.array_equal(_edges(S.fetch_compact("sum"), lb[perm], D, F), m0[perm])
    S.close()
