"""Local best response against a ReBeL agent (cfrb_match_create_lbr, rela.play_lbr, python -m rebel_b200.local_br): LBR's beliefs,
action values and decisions are a host restatement's bit for bit; its match payoff agrees with the exact EV of its pure strategy
against the agent's full recursive strategy, which never exceeds the agent's exploitability; results do not depend on the number
of concurrent games or on the capacity per round; games the full-tree tools refuse are played."""
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


def matches_table(D, F):
    """num_matches(hand, face): dice of the hand showing the face or the wild last face; hand = D base-F digits."""
    H = F ** D
    m = np.zeros((H, F), np.int64)
    for h in range(H):
        digits = [(h // F ** i) % F for i in range(D)]
        for f in range(F):
            m[h, f] = sum(1 for d in digits if d == f or d == F - 1)
    return m


def lbr_values(beta, lb, hl, mt, F, A, child_sigma):
    """LBR's action values at a node with last bid lb, for LBR's hand hl and belief beta over the agent's hand: [A], NaN where
    illegal.  child_sigma(a) = the agent's strategy [H, A] (absolute actions) at the node reached by raise a.  Every sum is serial
    and in fp64, in the order of the definition."""
    H = len(beta)
    vals = np.full(A, np.nan)
    lo = 0 if lb < 0 else lb + 1
    true = lambda bid, h: mt[hl, bid % F] + mt[h, bid % F] >= 1 + bid // F
    for a in range(lo, A - 1):
        sg = child_sigma(a)
        v = 0.0
        for h in range(H):
            inner = 0.0
            for a2 in range(a + 1, A):
                u = (1.0 if true(a, h) else -1.0) if a2 == A - 1 else (-1.0 if true(a2, h) else 1.0)
                inner += float(sg[h, a2]) * u
            v += float(beta[h]) * inner
        vals[a] = v
    if lb >= 0:
        v = 0.0
        for h in range(H):
            v += float(beta[h]) * (-1.0 if true(lb, h) else 1.0)
        vals[A - 1] = v
    return vals


def lbr_argmax(vals):
    """The first action (smallest index) with the largest value."""
    best = -1
    for a, v in enumerate(vals.tolist()):
        if not np.isnan(v) and (best < 0 or v > vals[best]):
            best = a
    return best


def update_beta(beta, s):
    beta = beta * s
    tot = 0.0
    for v in beta.tolist():
        tot += v
    return beta / tot


# ------------------------------------------------------------------------------------------------ CPU
def test_cli_parser():
    from rebel_b200.local_br import build_parser
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "5", "--net", "x.ckpt", "--games", "64", "--subgame_iters",
                                   "256", "--cfr", "--no_linear", "--net_mode", "1", "--concurrent_games", "512", "--max_subgames",
                                   "40", "--mdp_depth", "3", "--seed", "7"])
    assert (a.num_dice, a.num_faces, a.net, a.random_net_seed, a.games, a.subgame_iters) == (2, 5, "x.ckpt", None, 64, 256)
    assert a.cfr and a.no_linear and a.dcfr is None and (a.net_mode, a.concurrent_games, a.max_subgames, a.mdp_depth, a.seed) == \
        (1, 512, 40, 3, 7)
    d = build_parser().parse_args([])
    assert d.policy == "average" and d.max_subgames == 0 and not d.cfr


def test_lbr_line_round_trip():
    from rebel_b200.local_br import lbr_line, parse_lbr
    line = lbr_line("a.ckpt", 1024, 0.125, 0.03125, [0.25, 0.0])
    assert line.startswith("LBR {") and parse_lbr(line) == {
        "net": "a.ckpt", "games": 1024, "mean": 0.125, "stderr": 0.03125, "ci95": [0.125 - 1.96 * 0.03125, 0.125 + 1.96 * 0.03125],
        "seat0": 0.25, "seat1": 0.0}


def test_sampled_policy_is_refused_by_the_cli():
    from rebel_b200.local_br import main
    with pytest.raises(SystemExit) as e:
        main(["--policy", "sampled"])
    assert e.value.code == 2


def test_lbr_rule_on_a_hand_made_1x2f_strategy():
    """1x2f: hands 0 (face 0) and 1 (the wild face 1); bids 0 = 1x0, 1 = 1x1, 2 = 2x0, 3 = 2x1, 4 = liar."""
    D, F, A = 1, 2, 5
    mt = matches_table(D, F)
    assert mt.tolist() == [[1, 0], [1, 1]]
    # LBR holds face 0 after the bid 1x1, believing the agent holds hand 1 with probability 3/4
    sig = {2: np.array([[0, 0, 0, 0.5, 0.5], [0, 0, 0, 1.0, 0.0]]), 3: np.array([[0, 0, 0, 0, 1.0], [0, 0, 0, 0, 1.0]])}
    v = lbr_values(np.array([0.25, 0.75]), 1, 0, mt, F, A, lambda a: sig[a])
    # liar on 1x1: false against hand 0 (+1), true against hand 1 (-1)
    # raise 2x0 (true against both): the agent's 2x1 is false (LBR calls and wins), its liar call loses: +1 whatever it does
    # raise 2x1 (false against both): the agent calls
    assert np.isnan(v[:2]).all() and v[2:].tolist() == [1.0, -1.0, -0.5]
    assert lbr_argmax(v) == 2
    # ties go to the smallest action: with hand 1 after 2x0 against a certain hand 0, raising to 2x1 and calling are both -1
    v = lbr_values(np.array([1.0, 0.0]), 2, 1, mt, F, A, lambda a: sig[a])
    assert v[3] == v[4] == -1.0 and lbr_argmax(v) == 3
    # belief update: the agent's action with probabilities (0.2, 0.6) over its hands
    assert update_beta(np.array([0.5, 0.5]), np.array([0.2, 0.6])).tolist() == [0.1 / 0.4, 0.3 / 0.4]


# ------------------------------------------------------------------------------------------------ GPU
def solver(D, F, cap, iters, use_cfr=True, net_mode=0, weights=None, max_depth=2, **kw):
    from rebel_b200 import capi
    S = capi.WaveSolver(D, F, cap, max_depth=max_depth, num_iters=iters, linear_update=True, net_mode=net_mode,
                        solver=capi.SOLVER_CFR if use_cfr else capi.SOLVER_FP, **kw)
    if weights is not None:
        S.set_weights(weights)
    return S


def lbr_pure_strategy(tree, sigma, mt, D, F):
    """LBR's decision at every full-tree node (as the player acting there, against the agent in the other seat) as a dense
    pure strategy [N, H, A]; beta along the path from the agent's actions on it."""
    N, H, A = sigma.shape
    out = np.zeros_like(sigma)
    for x in range(N):
        lb, actor = int(tree[x, 0]), int(tree[x, 1])
        if lb == A - 1:
            continue
        path = []
        n = x
        while n > 0:
            path.append(n)
            n = int(tree[n, 4])
        beta = np.full(H, 1.0 / H)
        for c in reversed(path):
            p = int(tree[c, 4])
            if int(tree[p, 1]) != actor:               # an agent action
                beta = update_beta(beta, sigma[p, :, int(tree[c, 0])])
        lo = 0 if lb < 0 else lb + 1
        for hl in range(H):
            v = lbr_values(beta, lb, hl, mt, F, A, lambda a: sigma[int(tree[x, 2]) + a - lo])
            out[x, hl, lbr_argmax(v)] = 1.0
    return out


def check_lbr_traces(M, tree, sigma, mt, D, F, games):
    N, H, A = sigma.shape
    lbr_plies = 0
    for g in range(games):
        t, lt = M.trace(g), M.lbr_trace(g)
        me = g & 1
        beta = np.full(H, 1.0 / H)
        node = 0
        for i, (who, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            assert tree[node, 0] == lb and tree[node, 1] == actor, (g, i)
            lo = 0 if lb < 0 else lb + 1
            if who == 0:
                assert actor == me and t["prob"][i] == sigma[node, hand, action], (g, i)
                beta = update_beta(beta, sigma[node, :, action])
            else:
                assert actor == me ^ 1 and t["prob"][i] == 1.0, (g, i)
                assert np.array_equal(lt["beliefs"][i], beta), (g, i)
                want = lbr_values(beta, lb, hand, mt, F, A, lambda a: sigma[int(tree[node, 2]) + a - lo])
                got = lt["values"][i]
                assert np.array_equal(np.isnan(got), np.isnan(want)), (g, i, got, want)
                ok = ~np.isnan(want)
                assert np.array_equal(got[ok], want[ok]), (g, i, got, want)
                assert action == lbr_argmax(want), (g, i)
                lbr_plies += 1
            node = int(tree[node, 2]) + action - lo
        assert len(t["plies"]) and t["plies"][-1, 4] == A - 1
        assert (t["act_iteration"][:, 1] == 0).all() and (t["root_beliefs"][:, 1] == 0).all()
    return lbr_plies


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,depth", [(1, 4, 2), (2, 3, 2), (1, 4, 3)])
@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("net_name", ["zero", "fp32", "tc_x2"])
def test_gpu_lbr_decisions_bit_for_bit(rela, D, F, depth, use_cfr, net_name):
    from rebel_b200 import capi
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_name]
    w = net(D, F, 0) if mode else None
    iters = 64
    sigma = rela.strategy_recursive_to_leaf(make_cfg(rela, D, F, iters, use_cfr, mode, depth), 0,
                                            None if w is None else torch.from_numpy(w)).numpy()
    tree = capi.unroll_tree(D, F)
    S = solver(D, F, 256, iters, use_cfr, mode, w, max_depth=depth)
    games = 128
    M = capi.LbrMatch(S, 64, games, seed=3)
    res = M.play()
    assert set(np.unique(res["payoff_a"]).tolist()) <= {-1.0, 1.0}
    assert res["whatif_solves"] > 0 and res["solves"] > res["whatif_solves"]
    assert check_lbr_traces(M, tree, sigma, matches_table(D, F), D, F, games) >= games
    M.close(); S.close()


def exact_lbr_ev(rela, D, F, cfg, w):
    from rebel_b200 import capi
    sigma = rela.strategy_recursive_to_leaf(cfg, 0, w).numpy()
    s_lbr = lbr_pure_strategy(capi.unroll_tree(D, F), sigma, matches_table(D, F), D, F)
    ev0, ev1 = rela.ev_of_strategies(D, F, torch.from_numpy(s_lbr), torch.from_numpy(sigma))
    br0, br1 = rela.exploitability_of_strategy(D, F, torch.from_numpy(sigma))
    return (ev0 + ev1) / 2, (br0 + br1) / 2


@pytest.mark.gpu
def test_gpu_lbr_mean_matches_exact_ev_and_bounds_exploitability(rela):
    D, F, iters = 1, 4, 64
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, iters, True, 3)
    ev, expl = exact_lbr_ev(rela, D, F, cfg, w)
    assert ev <= expl + 1e-12, (ev, expl)
    r = rela.play_lbr(cfg, 0, 1 << 16, seed=5, flat_weights=w)
    assert abs(r["mean"] - ev) <= 4 * r["stderr"], (r["mean"], ev, r["stderr"])
    assert torch.equal(r["payoff_lbr"].abs(), torch.ones(1 << 16))


@pytest.mark.gpu
def test_gpu_lbr_finds_a_weak_agents_weakness(rela):
    D, F = 1, 4
    cfg = make_cfg(rela, D, F, 8, True, 0)
    ev, expl = exact_lbr_ev(rela, D, F, cfg, None)
    assert ev > 0.01 and ev <= expl + 1e-12, (ev, expl)
    r = rela.play_lbr(cfg, 0, 1 << 14, seed=2)
    assert r["mean"] - 4 * r["stderr"] > 0, (r["mean"], r["stderr"], ev)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_gpu_lbr_results_do_not_depend_on_scheduling(rela, D, F):
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 64, True, 3)
    A = 2 * D * F + 1
    games = 1024
    runs = [rela.play_lbr(cfg, 0, games, seed=9, flat_weights=w, concurrent_games=256),
            rela.play_lbr(cfg, 0, games, seed=9, flat_weights=w, concurrent_games=4096),
            rela.play_lbr(cfg, 0, games, seed=9, flat_weights=w, concurrent_games=512, max_subgames=A - 1)]
    assert runs[2]["max_subgames"] == A - 1 and runs[2]["deferred_slot_rounds"] > 0
    for r in runs[1:]:
        assert torch.equal(runs[0]["payoff_lbr"], r["payoff_lbr"]) and torch.equal(runs[0]["plies"], r["plies"])
        assert (r["solves"], r["whatif_solves"]) == (runs[0]["solves"], runs[0]["whatif_solves"])


@pytest.mark.gpu
def test_gpu_lbr_plays_a_game_the_full_tree_tools_refuse(rela):
    D, F, games = 2, 5, 1024
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 128, True, 3)
    with pytest.raises(RuntimeError, match="too large"):
        rela.strategy_recursive_to_leaf(cfg, 0, w)
    r = rela.play_lbr(cfg, 0, games, seed=1, flat_weights=w, concurrent_games=1024)
    assert r["payoff_lbr"].shape == (games,) and set(r["payoff_lbr"].unique().tolist()) <= {-1.0, 1.0}
    assert (r["plies"] >= 1).all() and (r["plies"] <= 21).all()
    assert r["whatif_solves"] > 0 and r["solves"] > r["whatif_solves"]
    assert np.isfinite(r["stderr"]) and r["stderr"] > 0


@pytest.mark.gpu
def test_gpu_lbr_validation():
    import ctypes as C
    from rebel_b200 import capi
    m = C.c_void_p()
    with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create_lbr: null handle"):
        capi._check(capi.lib().cfrb_match_create_lbr(None, 32, 64, 0, C.byref(m)))
    a = solver(1, 4, 64, 16)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*null argument"):
        capi._check(capi.lib().cfrb_match_create_lbr(a._h, 32, 64, 0, None))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*even"):
        capi.LbrMatch(a, 32, 63)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*n_slots"):
        capi.LbrMatch(a, 0, 64)
    small = solver(1, 4, 7, 16)                      # 1x4f: A - 1 = 8 what-if subgames per decision
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*capacity"):
        capi.LbrMatch(small, 32, 64)
    small.close()
    sp = solver(1, 4, 64, 16)
    sp.selfplay_create(np.arange(4, dtype=np.uint32))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*self-play"):
        capi.LbrMatch(sp, 32, 64)
    M = capi.LbrMatch(a, 1024, 64)                   # more slots than subgames per round
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*live match"):
        capi.LbrMatch(a, 32, 64)
    b = solver(1, 4, 64, 16)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*live match"):
        capi.Match(a, b, 32, 64)
    r = M.play()
    assert len(r["payoff_a"]) == 64 and r["whatif_solves"] > 0
    M.close()
    N = capi.Match(a, b, 32, 64)                     # a two-agent match on the same handles afterwards
    with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_lbr_counts: not an LBR match"):
        capi._check(capi.lib().cfrb_match_lbr_counts(N._m, None, None))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*live match"):
        capi.LbrMatch(b, 32, 64)
    N.close()
    a.close(); b.close(); sp.close()


@pytest.mark.gpu
def test_gpu_cli_end_to_end(rela, tmp_path):
    from rebel_b200.head_to_head import agent_params
    from rebel_b200.local_br import build_parser, parse_lbr
    from rebel_b200.models import make_selfplay_net
    from rebel_b200.recursive_eval import load_net_weights
    D, F = 1, 4
    path = str(tmp_path / "net0.ckpt")
    torch.jit.save(torch.jit.script(make_selfplay_net(D, F, seed=0)), path)
    argv = ["--num_dice", str(D), "--num_faces", str(F), "--net", path, "--games", "2048", "--subgame_iters", "64", "--cfr",
            "--seed", "4"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.local_br"] + argv, cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    lines = [l for l in p.stdout.split("\n") if l.startswith("LBR ")]
    assert len(lines) == 1, p.stdout
    assert "exploitability >= mean - 1.96 stderr" in p.stdout
    d = parse_lbr(lines[0])
    assert d["net"] == path and d["games"] == 2048
    w = load_net_weights(path)
    r = rela.play_lbr(agent_params(rela, build_parser().parse_args(argv), w, 64, True), 0, 2048, seed=4, flat_weights=w)
    assert d["mean"] == r["mean"] and d["stderr"] == r["stderr"]
    assert [d["seat0"], d["seat1"]] == r["seat_means"]
    p = subprocess.run([sys.executable, "-m", "rebel_b200.local_br", "--policy", "sampled"], cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=300)
    assert p.returncode == 2 and "sampled is not supported" in p.stderr
