"""Head-to-head matches between two ReBeL agents (cfrb_match_*, rela.play_match, python -m rebel_b200.head_to_head): the policy
each agent plays is its recursive to-leaf strategy along the path played, bit for bit; match means agree with the exact EV of the
two full strategies; results do not depend on the number of concurrent games; games the full-tree tools refuse are played."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def make_cfg(rela, D, F, iters, use_cfr=True, net_mode=0, max_depth=2):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, max_depth, True, use_cfr
    return cfg


def net(D, F, seed):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    return flatten_state_dict(make_selfplay_net(D, F, seed=seed).state_dict())


def solver(D, F, slots, iters, use_cfr=True, net_mode=0, weights=None, **kw):
    from rebel_b200 import capi
    S = capi.WaveSolver(D, F, slots, max_depth=2, num_iters=iters, linear_update=True, net_mode=net_mode,
                        solver=capi.SOLVER_CFR if use_cfr else capi.SOLVER_FP, **kw)
    if weights is not None:
        S.set_weights(weights)
    return S


def normalize(b):
    """normalize_beliefs_inplace with the sum taken in sequential order."""
    s = 0.0
    for v in b.tolist():
        s += v + 1e-80
    return (b + 1e-80) / s


# ------------------------------------------------------------------------------------------------ CPU
def test_cli_parser():
    from rebel_b200.head_to_head import build_parser
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "5", "--net_a", "x.ckpt", "--random_net_seed_b", "1",
                                   "--games", "64", "--policy", "average", "--subgame_iters", "256", "--subgame_iters_b", "128",
                                   "--cfr", "--cfr_b", "no", "--no_linear", "--dcfr", "1.5", "0", "2", "--net_mode", "1",
                                   "--concurrent_games", "512", "--mdp_depth", "3", "--seed", "7"])
    assert (a.num_dice, a.num_faces, a.net_a, a.net_b, a.random_net_seed_b) == (2, 5, "x.ckpt", None, 1)
    assert (a.games, a.policy, a.subgame_iters, a.subgame_iters_b, a.cfr, a.cfr_b) == (64, "average", 256, 128, True, "no")
    assert a.no_linear and a.dcfr == [1.5, 0.0, 2.0] and (a.net_mode, a.concurrent_games, a.mdp_depth, a.seed) == (1, 512, 3, 7)
    d = build_parser().parse_args([])
    assert d.policy == "sampled" and d.subgame_iters_b is None and d.cfr_b is None


def test_h2h_line_round_trip():
    from rebel_b200.head_to_head import h2h_line, parse_h2h
    line = h2h_line("a.ckpt", "zero", 1024, 0.125, 0.03125, [0.25, 0.0])
    d = parse_h2h(line)
    assert line.startswith("H2H {") and d == {"net_a": "a.ckpt", "net_b": "zero", "games": 1024, "mean": 0.125, "stderr": 0.03125,
                                               "ci95": [0.125 - 1.96 * 0.03125, 0.125 + 1.96 * 0.03125], "seat0": 0.25, "seat1": 0.0}


def test_pair_statistics(rela):
    rng = np.random.RandomState(0)
    x = rng.choice([-1.0, 1.0], size=200).astype(np.float32)
    s = rela.match_stats(torch.from_numpy(x))
    pairs = (x[0::2].astype(np.float64) + x[1::2]) / 2
    assert s["mean"] == pytest.approx(pairs.mean(), abs=1e-15)
    assert s["stderr"] == pytest.approx(pairs.std(ddof=1) / np.sqrt(len(pairs)), rel=1e-12)
    assert s["seat_means"] == pytest.approx([x[0::2].mean(), x[1::2].mean()], abs=1e-12)
    # seat-swapped pairs are reduced as pairs: a seat advantage that cancels within every pair has zero spread
    y = np.tile(np.array([1.0, -1.0], np.float32), 50)
    s = rela.match_stats(torch.from_numpy(y))
    assert s["mean"] == 0.0 and s["stderr"] == 0.0 and s["seat_means"] == [1.0, -1.0]
    # ... whereas the per-game spread would be 0.1
    assert np.std(y, ddof=1) / np.sqrt(len(y)) > 0.09


# ------------------------------------------------------------------------------------------------ GPU
def check_trace(M, tree, strategies, H, games):
    """Every traced decision probability is the agent's recursive strategy at the full-tree node, hand and action; every traced
    subgame's root beliefs are the host restatement of RecursiveEvaluator::expand along the path."""
    checked = 0
    for g in range(games):
        t = M.trace(g)
        bel = [np.full((2, H), 1.0 / H) for _ in range(2)]
        node, rnd = 0, -1
        for i, (agent, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            if r != rnd:
                if rnd >= 0:
                    bel = [np.stack([normalize(b[0]), normalize(b[1])]) for b in bel]
                rnd = r
                for k in range(2):
                    assert np.array_equal(t["root_beliefs"][r, k], bel[k]), (g, r, k)
            assert tree[node, 0] == lb and tree[node, 1] == actor, (g, i)
            assert t["prob"][i] == strategies[agent][node, hand, action], (g, i)
            for k in range(2):
                bel[k][actor] = bel[k][actor] * strategies[k][node, :, action]
            lo = 0 if lb < 0 else lb + 1
            node = tree[node, 2] + action - lo
            checked += 1
        assert len(t["plies"]) and t["plies"][-1, 4] == strategies[0].shape[2] - 1   # ends with the liar call
        assert (t["plies"][:, 0] == (t["plies"][:, 2] ^ (g & 1))).all()    # agent A sits in seat 0 in even games
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("net_a", ["zero", "fp32", "tc_x2"])
def test_gpu_average_policy_is_recursive_strategy(rela, D, F, use_cfr, net_a):
    from rebel_b200 import capi
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_a]
    wa = net(D, F, 0) if mode else None
    iters_a, iters_b = 64, 32
    sa = rela.strategy_recursive_to_leaf(make_cfg(rela, D, F, iters_a, use_cfr, mode), 0,
                                         None if wa is None else torch.from_numpy(wa)).numpy()
    sb = rela.strategy_recursive_to_leaf(make_cfg(rela, D, F, iters_b, use_cfr, 0), 0).numpy()
    tree = capi.unroll_tree(D, F)
    H = sa.shape[1]
    games = 128
    A_ = solver(D, F, 64, iters_a, use_cfr, mode, wa)
    B_ = solver(D, F, 64, iters_b, use_cfr, 0)
    M = capi.Match(A_, B_, 64, games, seed=3, policy=capi.MATCH_AVERAGE)
    res = M.play()
    assert set(np.unique(res["payoff_a"]).tolist()) <= {-1.0, 1.0} and (res["plies"] >= 1).all()
    n = check_trace(M, tree, [sa, sb], H, games)
    assert n >= games
    M.close(); A_.close(); B_.close()


def even_iteration_probs(iters):
    w = np.array([0.0 if i % 2 else i / 2 + 1 for i in range(iters)])
    return w / w.sum()


@pytest.mark.gpu
def test_gpu_sampled_decisions_resolve_to_the_same_bits(rela):
    from scipy.stats import chisquare
    from rebel_b200 import capi
    D, F, iters = 1, 4, 64
    w = net(D, F, 0)
    A_ = solver(D, F, 2048, iters, True, 3, w)
    B_ = solver(D, F, 2048, iters, True, 0)
    games = 256
    M = capi.Match(A_, B_, 64, games, seed=11, policy=capi.MATCH_SAMPLED)
    M.play()
    traces = [M.trace(g) for g in range(games)]
    M.close()
    # every (game, subgame, agent) solved alone with its traced root beliefs and act_iteration
    subs = [[], []]
    for g, t in enumerate(traces):
        for r in range(len(t["act_iteration"])):
            plies = [q for q in t["plies"].tolist() if q[5] == r]
            root_lb, root_player = plies[0][1], plies[0][2]
            for k in range(2):
                subs[k].append((g, r, root_lb, root_player, t["root_beliefs"][r, k], t["act_iteration"][r, k]))
    snaps = []
    for k, S in enumerate((A_, B_)):
        lb = np.array([s[2] for s in subs[k]], np.int32)
        pl = np.array([s[3] for s in subs[k]], np.int32)
        b = np.stack([s[4] for s in subs[k]])
        act = np.array([s[5] for s in subs[k]], np.int32)
        S.begin(lb, pl, b, act)
        S.run(iters)
        snaps.append({(s[0], s[1]): (i, s[2], s[3]) for i, s in enumerate(subs[k])})
        snaps[k]["table"] = S.fetch_compact("snapshot")
    checked = 0
    for g, t in enumerate(traces):
        node, rnd = 0, -1
        for i, (agent, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            if r != rnd:
                node, rnd = 0, r
            idx, root_lb, root_player = snaps[agent][(g, r)]
            tmpl = (A_ if agent == 0 else B_).tree(root_lb, root_player)
            lo = 0 if lb < 0 else lb + 1
            child = tmpl[node, 2] + action - lo
            assert t["prob"][i] == snaps[agent]["table"][idx, (child - 1) * A_.H + hand], (g, i)
            node = child
            checked += 1
    assert checked > games
    acts = np.concatenate([t["act_iteration"].ravel() for t in traces])
    assert (acts >= 0).all() and (acts < iters).all() and (acts % 2 == 0).all()
    p = even_iteration_probs(iters)
    bins = np.arange(0, iters + 1, 16)
    obs = np.histogram(acts, bins)[0]
    exp = np.array([p[lo:hi].sum() for lo, hi in zip(bins[:-1], bins[1:])]) * len(acts)
    assert chisquare(obs, exp).pvalue > 1e-3
    A_.close(); B_.close()


@pytest.mark.gpu
@pytest.mark.parametrize("b_seed", [None, 1])
def test_gpu_match_mean_matches_exact_ev(rela, b_seed):
    D, F, iters = 1, 4, 64
    wa = torch.from_numpy(net(D, F, 0))
    wb = None if b_seed is None else torch.from_numpy(net(D, F, b_seed))
    ca, cb = make_cfg(rela, D, F, iters, True, 3), make_cfg(rela, D, F, iters, True, 0 if wb is None else 3)
    sa = rela.strategy_recursive_to_leaf(ca, 0, wa)
    sb = rela.strategy_recursive_to_leaf(cb, 0, wb)
    ev0, ev1 = rela.ev_of_strategies(D, F, sa, sb)
    r = rela.play_match(ca, cb, 0, 1 << 17, seed=5, policy="average", flat_weights_a=wa, flat_weights_b=wb)
    assert r["stderr"] <= 0.01
    assert abs(r["mean"] - (ev0 + ev1) / 2) <= 4 * r["stderr"], (r["mean"], ev0, ev1, r["stderr"])


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_gpu_results_do_not_depend_on_concurrency(rela, D, F):
    wa, wb = torch.from_numpy(net(D, F, 0)), torch.from_numpy(net(D, F, 1))
    ca, cb = make_cfg(rela, D, F, 64, True, 3), make_cfg(rela, D, F, 64, True, 3)
    r1 = rela.play_match(ca, cb, 0, 4096, seed=9, flat_weights_a=wa, flat_weights_b=wb, concurrent_games=256)
    r2 = rela.play_match(ca, cb, 0, 4096, seed=9, flat_weights_a=wa, flat_weights_b=wb, concurrent_games=4096)
    assert torch.equal(r1["payoff_a"], r2["payoff_a"]) and torch.equal(r1["plies"], r2["plies"])
    assert r1["solves"] == r2["solves"]


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_gpu_agent_against_itself_is_fair(rela, D, F):
    w = torch.from_numpy(net(D, F, 0))
    c = make_cfg(rela, D, F, 64, True, 3)
    r = rela.play_match(c, c, 0, 8192, seed=13, flat_weights_a=w, flat_weights_b=w)
    assert abs(r["mean"]) <= 4 * r["stderr"], (r["mean"], r["stderr"])


@pytest.mark.gpu
def test_gpu_plays_a_game_the_full_tree_tools_refuse(rela):
    D, F, games = 2, 5, 2048
    wa, wb = torch.from_numpy(net(D, F, 0)), torch.from_numpy(net(D, F, 1))
    ca, cb = make_cfg(rela, D, F, 128, True, 3), make_cfg(rela, D, F, 128, True, 3)
    with pytest.raises(RuntimeError, match="too large"):
        rela.strategy_recursive_to_leaf(ca, 0, wa)
    r = rela.play_match(ca, cb, 0, games, seed=1, flat_weights_a=wa, flat_weights_b=wb, concurrent_games=1024)
    assert r["payoff_a"].shape == (games,) and set(r["payoff_a"].unique().tolist()) <= {-1.0, 1.0}
    assert (r["plies"] >= 1).all() and (r["plies"] <= 21).all()
    assert np.isfinite(r["stderr"]) and r["stderr"] > 0 and r["solves"] >= 2 * games


@pytest.mark.gpu
def test_gpu_match_validation():
    from rebel_b200 import capi
    a = solver(1, 4, 64, 16)
    bad = {
        "different games": solver(1, 5, 64, 16),
        "different max_depth": capi.WaveSolver(1, 4, 64, max_depth=3, num_iters=16, net_mode=0),
        "different state dtypes": solver(1, 4, 64, 16, state_dtype=capi.STATE_F32),
        "capacity": solver(1, 4, 16, 16),
    }
    for what, b in bad.items():
        with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create: .*" + what.split()[-1]):
            capi.Match(a, b, 32, 64)
        b.close()
    sp = solver(1, 4, 64, 16)
    sp.selfplay_create(np.arange(4, dtype=np.uint32))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*self-play"):
        capi.Match(a, sp, 32, 64)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*two handles"):
        capi.Match(a, a, 32, 64)
    ok = solver(1, 4, 64, 16)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*even"):
        capi.Match(a, ok, 32, 63)
    M = capi.Match(a, ok, 32, 64)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*live match"):
        capi.Match(a, sp, 32, 64)
    assert len(M.play()["payoff_a"]) == 64
    M.close()
    a.close(); sp.close(); ok.close()


@pytest.mark.gpu
def test_gpu_cli_end_to_end(rela, tmp_path):
    from rebel_b200.head_to_head import agent_params, build_parser, parse_h2h
    from rebel_b200.models import make_selfplay_net
    from rebel_b200.recursive_eval import load_net_weights
    D, F = 1, 4
    paths = []
    for seed in (0, 1):
        p = str(tmp_path / f"net{seed}.ckpt")
        torch.jit.save(torch.jit.script(make_selfplay_net(D, F, seed=seed)), p)
        paths.append(p)
    argv = ["--num_dice", str(D), "--num_faces", str(F), "--net_a", paths[0], "--net_b", paths[1], "--games", "2048",
            "--subgame_iters", "64", "--cfr", "--seed", "4"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.head_to_head"] + argv, cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    lines = [l for l in p.stdout.split("\n") if l.startswith("H2H ")]
    assert len(lines) == 1, p.stdout
    d = parse_h2h(lines[0])
    assert d["net_a"] == paths[0] and d["net_b"] == paths[1] and d["games"] == 2048
    args = build_parser().parse_args(argv)
    wa, wb = load_net_weights(paths[0]), load_net_weights(paths[1])
    r = rela.play_match(agent_params(rela, args, wa, 64, True), agent_params(rela, args, wb, 64, True), 0, 2048, seed=4,
                        flat_weights_a=wa, flat_weights_b=wb)
    assert d["mean"] == r["mean"] and d["stderr"] == r["stderr"]
    assert d["ci95"] == [r["mean"] - 1.96 * r["stderr"], r["mean"] + 1.96 * r["stderr"]]
