"""Playing ReBeL's every-node policy (compute_strategy_recursive: a subgame re-solved at every decision): per-ply head-to-head
matches (cfrb_match_create2, rela.play_match's policy / policy_b, head_to_head --policy every_node --policy_b) and the every-node
rela.Agent.  Every decision and belief of an every-node agent is the host walk's bit for bit, a to-leaf agent in the same match
plays its own to-leaf strategy, match means agree with the exact EV, and pairs of equal to-leaf policies still play the to-leaf
walk bit for bit."""
import ctypes
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


def match2(a, b, n_slots, n_games, seed, policy_a, policy_b):
    """A capi.Match made by cfrb_match_create2 whatever the pair."""
    from rebel_b200 import capi
    M = capi.Match.__new__(capi.Match)
    M.a, M.b, M.G = a, b, n_games
    M._m = ctypes.c_void_p()
    capi._check(capi.lib().cfrb_match_create2(a._h, b._h, n_slots, n_games, seed, policy_a, policy_b, ctypes.byref(M._m)))
    return M


# ------------------------------------------------------------------------------------------------ CPU
def test_cli_parsers_take_the_new_policies():
    from rebel_b200.head_to_head import build_parser
    from rebel_b200.play import build_parser as play_parser
    a = build_parser().parse_args(["--policy", "every_node", "--policy_b", "sampled"])
    assert (a.policy, a.policy_b) == ("every_node", "sampled")
    d = build_parser().parse_args([])
    assert d.policy == "sampled" and d.policy_b is None
    assert play_parser().parse_args(["--policy", "every_node"]).policy == "every_node"
    assert play_parser().parse_args([]).policy == "sampled"
    with pytest.raises(SystemExit):
        build_parser().parse_args(["--policy_b", "bogus"])


def test_match_bench_parser_defaults():
    src = open(os.path.join(ROOT, "scripts", "match_bench.py")).read()
    assert 'ap.add_argument("--policy_a", choices=tuple(POLICIES), default="sampled")' in src
    assert 'ap.add_argument("--policy_b", choices=tuple(POLICIES), default="sampled")' in src


def test_h2h_line_policy_keys():
    from rebel_b200.head_to_head import h2h_line, parse_h2h
    plain = parse_h2h(h2h_line("a", "b", 8, 0.5, 0.25, [1.0, 0.0]))
    assert "policy_a" not in plain and "policy_b" not in plain
    d = parse_h2h(h2h_line("a", "b", 8, 0.5, 0.25, [1.0, 0.0], ("every_node", "sampled")))
    assert (d["policy_a"], d["policy_b"]) == ("every_node", "sampled")
    assert {k: v for k, v in d.items() if not k.startswith("policy")} == plain


def test_cache_bytes():
    from rebel_b200 import capi
    EN, AV, SA = capi.MATCH_EVERY_NODE, capi.MATCH_AVERAGE, capi.MATCH_SAMPLED
    # 2x6f, depth 2: the root template has 1 + 24 + C(25, 2) = 325 nodes, 324 edges, 36 hands
    one = 8192 * 324 * 36 * 8
    assert capi.match_cache_bytes(2, 6, 2, 8192, EN, SA) == one
    assert 0.7e9 < one < 0.8e9
    assert capi.match_cache_bytes(2, 6, 2, 8192, AV, SA) == 2 * one
    for p in (AV, SA):
        assert capi.match_cache_bytes(2, 6, 2, 8192, p) == 0          # the to-leaf walk reads its tables in place
    assert capi.match_cache_bytes(2, 6, 2, 8192, EN, EN) == 0
    with pytest.raises(capi.CfrbError, match="bad policy"):
        capi.match_cache_bytes(1, 4, 2, 64, 3, AV)


def test_bad_policy_names_are_refused(rela):
    cfg = make_cfg(rela, 1, 4, 16)
    with pytest.raises(RuntimeError, match="policy must be 'sampled', 'average' or 'every_node'"):
        rela.Agent(cfg, device=0, tables=8, policy="to_leaf")
    with pytest.raises(RuntimeError, match="policy must be 'sampled', 'average' or 'every_node'"):
        rela.play_match(cfg, cfg, 0, 8, policy="average", policy_b="best")


# ------------------------------------------------------------------------------------------------ GPU
def check_ply_trace(M, tree, strategies, policies, H, games, max_depth=2):
    """Per-ply trace of a match: agent k plays policies[k] ('every_node' or a to-leaf policy) with dense strategy strategies[k]
    (None: not checked).  Every traced probability of a checked agent is its strategy at the full-tree node, hand and action;
    every traced belief row of a checked agent is its walk's (every-node: the mover's row times the root row, eps-normalised;
    to-leaf: unnormalised inside its subgame, both rows eps-normalised at its pseudo-leaves); act_iteration is -1 / the draw where
    the agent solved and -2 where it played on inside its subgame."""
    A = strategies[0].shape[2] if strategies[0] is not None else strategies[1].shape[2]
    checked = 0
    for g in range(games):
        t = M.trace(g)
        P = len(t["plies"])
        assert P >= 1 and len(t["act_iteration"]) == P and t["plies"][-1, 4] == A - 1, g
        bel = [np.full((2, H), 1.0 / H) for _ in range(2)]
        depth = [0, 0]
        node = 0
        for i, (agent, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            assert r == i and agent == actor ^ (g & 1), (g, i)
            assert tree[node, 0] == lb and tree[node, 1] == actor, (g, i)
            for k in range(2):
                act = int(t["act_iteration"][i, k])
                if policies[k] != "every_node" and depth[k] > 0:
                    assert act == -2, (g, i, k)
                elif policies[k] == "sampled":
                    assert act >= 0 and act % 2 == 0, (g, i, k)
                else:
                    assert act == -1, (g, i, k)
                if strategies[k] is not None:
                    assert np.array_equal(t["root_beliefs"][i, k], bel[k]), (g, i, k)
            if strategies[agent] is not None:
                assert t["prob"][i] == strategies[agent][node, hand, action], (g, i)
                checked += 1
            terminal = action == A - 1
            for k in range(2):
                if strategies[k] is None:
                    continue
                row = bel[k][actor] * strategies[k][node, :, action]
                if policies[k] == "every_node":
                    bel[k][actor] = normalize(row)
                    continue
                bel[k][actor] = row
                depth[k] += 1
                if not terminal and depth[k] == max_depth:
                    bel[k] = np.stack([normalize(bel[k][0]), normalize(bel[k][1])])
                    depth[k] = 0
            for k in range(2):
                if strategies[k] is None and policies[k] != "every_node":
                    depth[k] = 0 if (not terminal and depth[k] + 1 == max_depth) else depth[k] + 1
            lo = 0 if lb < 0 else lb + 1
            node = tree[node, 2] + action - lo
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("net_a", ["zero", "fp32", "tc_x2"])
def test_gpu_every_node_match_is_strategy_recursive(rela, D, F, use_cfr, net_a):
    from rebel_b200 import capi
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_a]
    wa = net(D, F, 0) if mode else None
    iters_a, iters_b = 64, 32
    sa = rela.strategy_recursive(make_cfg(rela, D, F, iters_a, use_cfr, mode), 0, None if wa is None else torch.from_numpy(wa)).numpy()
    sb = rela.strategy_recursive(make_cfg(rela, D, F, iters_b, use_cfr, 0), 0).numpy()
    tree = capi.unroll_tree(D, F)
    games = 128
    A_ = solver(D, F, 64, iters_a, use_cfr, mode, wa)
    B_ = solver(D, F, 64, iters_b, use_cfr, 0)
    M = capi.Match(A_, B_, 64, games, seed=3, policy=capi.MATCH_EVERY_NODE)
    res = M.play()
    assert set(np.unique(res["payoff_a"]).tolist()) <= {-1.0, 1.0} and (res["plies"] >= 1).all()
    assert res["solves_a"] == res["solves_b"] == int(res["plies"].sum()) == res["solves"] // 2
    assert res["subgame_iters"] == res["solves_a"] * (iters_a + iters_b)
    assert check_ply_trace(M, tree, [sa, sb], ["every_node"] * 2, sa.shape[1], games) >= games
    M.close(); A_.close(); B_.close()


@pytest.mark.gpu
def test_gpu_every_node_against_average_to_leaf(rela):
    from rebel_b200 import capi
    D, F, games = 1, 4, 128
    wa = net(D, F, 0)
    sa = rela.strategy_recursive(make_cfg(rela, D, F, 64, True, 3), 0, torch.from_numpy(wa)).numpy()
    sb = rela.strategy_recursive_to_leaf(make_cfg(rela, D, F, 32, True, 0), 0).numpy()
    tree = capi.unroll_tree(D, F)
    A_ = solver(D, F, 64, 64, True, 3, wa)
    B_ = solver(D, F, 64, 32, True, 0)
    M = capi.Match(A_, B_, 64, games, seed=5, policy=capi.MATCH_EVERY_NODE, policy_b=capi.MATCH_AVERAGE)
    res = M.play()
    assert check_ply_trace(M, tree, [sa, sb], ["every_node", "average"], sa.shape[1], games) >= 2 * games
    solved_b = sum(int((M.trace(g)["act_iteration"][:, 1] == -1).sum()) for g in range(games))
    assert res["solves_a"] == int(res["plies"].sum()) and res["solves_b"] == solved_b < res["solves_a"]
    M.close(); A_.close(); B_.close()


@pytest.mark.gpu
def test_gpu_every_node_against_sampled_to_leaf(rela):
    """A's decisions are strategy_recursive's; every subgame B solved resolves to the same bits alone, from its traced beliefs and
    act_iteration."""
    from rebel_b200 import capi
    D, F, iters, games = 1, 4, 64, 128
    wa = net(D, F, 0)
    sa = rela.strategy_recursive(make_cfg(rela, D, F, iters, True, 3), 0, torch.from_numpy(wa)).numpy()
    tree = capi.unroll_tree(D, F)
    A_ = solver(D, F, 2048, iters, True, 3, wa)
    B_ = solver(D, F, 2048, iters, True, 0)
    M = capi.Match(A_, B_, 64, games, seed=11, policy=capi.MATCH_EVERY_NODE, policy_b=capi.MATCH_SAMPLED)
    M.play()
    H = A_.H
    assert check_ply_trace(M, tree, [sa, None], ["every_node", "sampled"], H, games) >= games // 2
    traces = [M.trace(g) for g in range(games)]
    M.close()
    subs = []                                              # (game, ply, root last bid, root player, beliefs, act_iteration)
    for g, t in enumerate(traces):
        for i, (agent, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            if t["act_iteration"][i, 1] >= 0:
                subs.append((g, i, lb, actor, t["root_beliefs"][i, 1], t["act_iteration"][i, 1]))
    B_.begin(np.array([s[2] for s in subs], np.int32), np.array([s[3] for s in subs], np.int32), np.stack([s[4] for s in subs]),
             np.array([s[5] for s in subs], np.int32))
    B_.run(iters)
    table = B_.fetch_compact("snapshot")
    where = {(s[0], s[1]): (i, s[2], s[3]) for i, s in enumerate(subs)}
    checked = 0
    for g, t in enumerate(traces):
        cur = None
        for i, (agent, lb, actor, hand, action, r) in enumerate(t["plies"].tolist()):
            if (g, i) in where:
                idx, root_lb, root_player = where[(g, i)]
                cur, node = (idx, B_.tree(root_lb, root_player)), 0
            lo = 0 if lb < 0 else lb + 1
            child = cur[1][node, 2] + action - lo
            if agent == 1:
                assert t["prob"][i] == table[cur[0], (child - 1) * H + hand], (g, i)
                checked += 1
            node = child
    assert checked >= games // 2
    A_.close(); B_.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pair", [("every_node", "average"), ("every_node", "every_node")])
def test_gpu_match_mean_matches_exact_ev(rela, pair):
    D, F, iters = 1, 4, 64
    wa = torch.from_numpy(net(D, F, 0))
    ca, cb = make_cfg(rela, D, F, iters, True, 3), make_cfg(rela, D, F, iters, True, 0)
    sa = rela.strategy_recursive(ca, 0, wa)
    sb = rela.strategy_recursive(cb, 0) if pair[1] == "every_node" else rela.strategy_recursive_to_leaf(cb, 0)
    ev0, ev1 = rela.ev_of_strategies(D, F, sa, sb)
    r = rela.play_match(ca, cb, 0, 1 << 17, seed=5, policy=pair[0], policy_b=pair[1], flat_weights_a=wa)
    assert r["stderr"] <= 0.01
    assert abs(r["mean"] - (ev0 + ev1) / 2) <= 4 * r["stderr"], (r["mean"], ev0, ev1, r["stderr"])


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
@pytest.mark.parametrize("policy_b", ["every_node", "sampled"])
def test_gpu_results_do_not_depend_on_concurrency(rela, D, F, policy_b):
    wa, wb = torch.from_numpy(net(D, F, 0)), torch.from_numpy(net(D, F, 1))
    ca, cb = make_cfg(rela, D, F, 64, True, 3), make_cfg(rela, D, F, 64, True, 3)
    kw = dict(seed=9, policy="every_node", policy_b=policy_b, flat_weights_a=wa, flat_weights_b=wb)
    r1 = rela.play_match(ca, cb, 0, 4096, concurrent_games=256, **kw)
    r2 = rela.play_match(ca, cb, 0, 4096, concurrent_games=4096, **kw)
    assert torch.equal(r1["payoff_a"], r2["payoff_a"]) and torch.equal(r1["plies"], r2["plies"])
    assert (r1["solves_a"], r1["solves_b"]) == (r2["solves_a"], r2["solves_b"])
    assert r1["solves_a"] == int(r1["plies"].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_gpu_every_node_agent_against_itself_is_fair(rela, D, F):
    w = torch.from_numpy(net(D, F, 0))
    c = make_cfg(rela, D, F, 64, True, 3)
    r = rela.play_match(c, c, 0, 8192, seed=13, policy="every_node", flat_weights_a=w, flat_weights_b=w)
    assert abs(r["mean"]) <= 4 * r["stderr"], (r["mean"], r["stderr"])


@pytest.mark.gpu
def test_gpu_plays_a_game_the_exact_tools_refuse(rela):
    D, F, games = 2, 6, 512
    wa, wb = torch.from_numpy(net(D, F, 0)), torch.from_numpy(net(D, F, 1))
    ca, cb = make_cfg(rela, D, F, 64, True, 3), make_cfg(rela, D, F, 64, True, 3)
    with pytest.raises(RuntimeError, match="too large"):
        rela.strategy_recursive(ca, 0, wa)
    with pytest.raises(RuntimeError, match="more than 23 actions"):
        rela.exploitability_recursive(ca, 0, wa)
    r = rela.play_match(ca, cb, 0, games, seed=1, policy="every_node", flat_weights_a=wa, flat_weights_b=wb, concurrent_games=256)
    assert r["payoff_a"].shape == (games,) and set(r["payoff_a"].unique().tolist()) <= {-1.0, 1.0}
    assert (r["plies"] >= 1).all() and r["solves_a"] == r["solves_b"] == int(r["plies"].sum())
    assert np.isfinite(r["stderr"]) and r["stderr"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["average", "sampled"])
def test_gpu_create2_of_equal_to_leaf_policies_is_the_to_leaf_walk(policy):
    from rebel_b200 import capi
    D, F, games = 1, 6, 512
    p = {"average": capi.MATCH_AVERAGE, "sampled": capi.MATCH_SAMPLED}[policy]
    out = []
    for make in (lambda a, b: capi.Match(a, b, 128, games, seed=17, policy=p), lambda a, b: match2(a, b, 128, games, 17, p, p)):
        A_ = solver(D, F, 128, 64, True, 3, net(D, F, 0))
        B_ = solver(D, F, 128, 32, True, 0)
        M = make(A_, B_)
        out.append(M.play())
        out[-1]["trace"] = M.trace(3)
        M.close(); A_.close(); B_.close()
    a, b = out
    assert np.array_equal(a["payoff_a"], b["payoff_a"]) and np.array_equal(a["plies"], b["plies"])
    assert (a["solves"], a["subgame_iters"], a["solves_a"], a["solves_b"]) == (b["solves"], b["subgame_iters"], b["solves_a"], b["solves_b"])
    for k in ("plies", "prob", "act_iteration", "root_beliefs"):
        assert np.array_equal(a["trace"][k], b["trace"][k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,use_cfr", [(1, 4, True), (1, 4, False), (2, 3, True)])
def test_gpu_every_node_agent_policy_is_strategy_recursive(rela, D, F, use_cfr):
    from rebel_b200 import capi
    cfg = make_cfg(rela, D, F, 32, use_cfr, 0)
    S = rela.strategy_recursive(cfg, 0).numpy()
    tree = capi.unroll_tree(D, F)
    T, A = 256, S.shape[2]
    H = S.shape[1]
    ag = rela.Agent(cfg, 0, T, "every_node", seed=1)
    rng = np.random.RandomState(D * 10 + F + use_cfr)
    ids = np.arange(T)
    seats = (ids & 1).astype(np.int32)
    ag.new_games(ids, seats, rng.randint(0, H, size=T).astype(np.int32))
    node = np.zeros(T, np.int64)
    last = np.full(T, -1)
    player = np.zeros(T, np.int64)
    plies = np.zeros(T, np.int64)
    live = ids.copy()
    zero_prob = 0
    while len(live):
        pol = ag.policy(live).numpy()
        acts = np.zeros(len(live), np.int32)
        for i, t in enumerate(live):
            assert np.array_equal(pol[i], S[node[t]]), (t, node[t])
            if player[t] == seats[t]:
                acts[i] = -1
            else:                 # the opponent: half the time the action the agent finds least likely (probability 0 if any)
                lo = 0 if last[t] < 0 else last[t] + 1
                legal = np.arange(lo, A - 1 if last[t] < 0 else A)
                unlikely = legal[np.argmin(S[node[t]][:, legal].max(axis=0))]
                acts[i] = unlikely if rng.rand() < 0.5 else rng.choice(legal)
                zero_prob += S[node[t], :, acts[i]].max() == 0.0
        played, _, done = ag.step(live, acts)
        played, done = played.numpy(), done.numpy()
        for i, t in enumerate(live):
            lo = 0 if last[t] < 0 else last[t] + 1
            node[t] = tree[node[t], 2] + played[i] - lo
            last[t], player[t] = played[i], player[t] ^ 1
            plies[t] += 1
        live = live[~done]
    assert np.array_equal(ag.state(ids)["subgames"].numpy(), plies)   # one solve per node visited
    ag.close()


@pytest.mark.gpu
def test_gpu_every_node_agents_replay_a_match(rela):
    from rebel_b200 import capi
    D, F, games = 1, 4, 128
    wa = net(D, F, 0)
    ca, cb = make_cfg(rela, D, F, 64, True, 3), make_cfg(rela, D, F, 32, True, 0)
    A_ = solver(D, F, 64, 64, True, 3, wa)
    B_ = solver(D, F, 64, 32, True, 0)
    M = capi.Match(A_, B_, 64, games, seed=21, policy=capi.MATCH_EVERY_NODE)
    M.play()
    traces = [M.trace(g) for g in range(games)]
    M.close(); A_.close(); B_.close()
    agents = [rela.Agent(ca, 0, games, "every_node", flat_weights=torch.from_numpy(wa)), rela.Agent(cb, 0, games, "every_node")]
    ids = np.arange(games)
    for k in range(2):
        seats = (ids & 1) ^ k                                    # agent A sits in seat 0 in even games
        hands = [next(p[3] for p in traces[g]["plies"].tolist() if p[2] == seats[g]) for g in range(games)]
        agents[k].new_games(ids, seats, hands)
    checked = 0
    for ply in range(max(len(t["plies"]) for t in traces)):
        live = np.array([g for g in range(games) if ply < len(traces[g]["plies"])])
        pols = [ag.policy(live).numpy() for ag in agents]
        states = [ag.state(live) for ag in agents]
        acts = np.zeros(len(live), np.int32)
        for i, g in enumerate(live):
            agent, lb, actor, hand, action, r = traces[g]["plies"][ply].tolist()
            assert pols[agent][i, hand, action] == traces[g]["prob"][ply], (g, ply)
            for k in range(2):
                assert np.array_equal(states[k]["root_beliefs"][i].numpy(), traces[g]["root_beliefs"][ply, k]), (g, ply, k)
            acts[i] = action
            checked += 1
        for ag in agents:
            played, _, done = ag.step(live, acts)
            assert np.array_equal(played.numpy(), acts)
            assert np.array_equal(done.numpy(), np.array([ply == len(traces[g]["plies"]) - 1 for g in live]))
    assert checked >= 2 * games
    for ag in agents:
        ag.close()


@pytest.mark.gpu
def test_gpu_validation():
    from rebel_b200 import capi
    a, b = solver(1, 4, 64, 16), solver(1, 4, 64, 16)
    with pytest.raises(capi.CfrbError, match=r"cfrb error -1: cfrb_match_create: bad policy"):
        capi.Match(a, b, 32, 64, policy=3)
    with pytest.raises(capi.CfrbError, match=r"cfrb error -1: cfrb_match_create2: bad policy \(0, 9\)"):
        capi.Match(a, b, 32, 64, policy=capi.MATCH_AVERAGE, policy_b=9)
    M = capi.Match.__new__(capi.Match)
    M._m = ctypes.c_void_p()
    with pytest.raises(capi.CfrbError, match=r"cfrb error -1: cfrb_match_create2: null handle .*cfrb_match_create_lbr"):
        capi._check(capi.lib().cfrb_match_create2(a._h, None, 32, 64, 0, capi.MATCH_EVERY_NODE, capi.MATCH_AVERAGE,
                                                   ctypes.byref(M._m)))
    # the to-leaf agent's cache against a capped free-memory figure, refused before anything is allocated
    need = capi.match_cache_bytes(1, 4, 2, 64, capi.MATCH_EVERY_NODE, capi.MATCH_AVERAGE)
    assert need > 0
    b.debug_to_leaf_free_cap(need - 1)
    with pytest.raises(capi.CfrbError, match=r"cfrb error -5: cfrb_match_create2: .*need %d bytes" % need):
        capi.Match(a, b, 64, 128, policy=capi.MATCH_EVERY_NODE, policy_b=capi.MATCH_AVERAGE)
    M = capi.Match(a, b, 64, 128, policy=capi.MATCH_EVERY_NODE)     # two every-node agents need no cache
    assert len(M.play()["payoff_a"]) == 128
    M.close()
    b.debug_to_leaf_free_cap(need)
    M = capi.Match(a, b, 64, 128, policy=capi.MATCH_EVERY_NODE, policy_b=capi.MATCH_AVERAGE)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*live match"):
        capi.Match(a, b, 64, 128, policy=capi.MATCH_EVERY_NODE)
    assert len(M.play()["payoff_a"]) == 128
    M.close()
    a.close(); b.close()


@pytest.mark.gpu
def test_gpu_cli_end_to_end(rela, tmp_path):
    from rebel_b200.head_to_head import agent_params, build_parser, parse_h2h
    from rebel_b200.play import parse_play
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    argv = ["--num_dice", "1", "--num_faces", "4", "--random_net_seed_a", "0", "--games", "1024", "--subgame_iters", "64", "--cfr",
            "--seed", "4", "--policy", "every_node", "--policy_b", "sampled"]
    p = subprocess.run([sys.executable, "-m", "rebel_b200.head_to_head"] + argv, cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    lines = [l for l in p.stdout.split("\n") if l.startswith("H2H ")]
    assert len(lines) == 1, p.stdout
    d = parse_h2h(lines[0])
    assert (d["policy_a"], d["policy_b"], d["games"]) == ("every_node", "sampled", 1024)
    from rebel_b200.head_to_head import agent_weights
    args = build_parser().parse_args(argv)
    wa = agent_weights(1, 4, None, 0)
    r = rela.play_match(agent_params(rela, args, wa, 64, True), agent_params(rela, args, None, 64, True), 0, 1024, seed=4,
                        policy="every_node", policy_b="sampled", flat_weights_a=wa)
    assert d["mean"] == r["mean"] and d["stderr"] == r["stderr"]
    argv = ["--num_dice", "1", "--num_faces", "4", "--subgame_iters", "64", "--cfr", "--games", "2", "--seed", "3", "--policy",
            "every_node"]
    p = subprocess.run([sys.executable, "-m", "rebel_b200.play"] + argv, cwd=str(tmp_path), env=env, input="1 1\nliar\nliar\nliar\n",
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    out = p.stdout
    assert "every_node policy" in out and out.count("reveal:") == 2
    lines = [l for l in out.split("\n") if l.startswith("PLAY ")]
    assert len(lines) == 1, out
    d = parse_play(lines[0])
    assert d["games"] == 2 and d["agent_wins"] + d["human_wins"] == 2
