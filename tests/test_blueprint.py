"""Blueprints: fixed full-tree strategies as match players (cfrb_blueprint_*, cfrb_match_create3, capi.Blueprint).  A blueprint
built from an agent's frozen recursive policy plays that agent's games bit for bit, a blueprint built from a solver holds the bits
that solver's own fetch returns, and match means between blueprints and agents agree with the exact EV of the two tables."""
import json

import numpy as np
import pytest

from rebel_b200 import capi


def tree(D, F):
    """The full tree: (child_begin, nchild) per node, in the compact table's BFS order."""
    t = capi.unroll_tree(D, F)
    return t[:, 2], t[:, 3] - t[:, 2]


def uniform_table(D, F):
    cb, nc = tree(D, F)
    H = F ** D
    s = np.zeros((len(cb) - 1, H))
    for n in range(len(cb)):
        if nc[n]:
            s[cb[n] - 1:cb[n] - 1 + nc[n]] = 1.0 / nc[n]
    return s


def net(D, F, seed):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    return flatten_state_dict(make_selfplay_net(D, F, seed=seed).state_dict())


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("D,F", [(1, 4), (2, 5), (1, 11)])
def test_bytes_by_hand(D, F):
    A, H = 1 + 2 * D * F, F ** D
    N = 2 ** A - 1                                   # the root, each increasing bid sequence, each closed by the liar call
    assert capi.blueprint_bytes(D, F) == 8 * (N - 1) * H + 4 * N + H * F


def test_bytes_of_the_documented_games():
    mb = {g: capi.blueprint_bytes(*g) / 1e6 for g in [(2, 4), (2, 5), (5, 2), (1, 11)]}
    assert round(mb[(2, 4)]) == 17 and round(mb[(2, 5)] / 1e3, 2) == 0.43
    assert round(mb[(5, 2)] / 1e3, 2) == 0.55 and round(mb[(1, 11)] / 1e3, 2) == 0.77


def test_full_tree_size_is_two_to_the_a_minus_one():
    for D, F in [(1, 2), (1, 4), (2, 3)]:
        assert len(tree(D, F)[0]) == 2 ** (1 + 2 * D * F) - 1


def test_more_than_23_actions_is_refused_before_any_device_work():
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.blueprint_bytes(2, 6)
    import ctypes
    out = ctypes.c_void_p()
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi._check(capi.lib().cfrb_blueprint_create(0, 2, 6, capi._p(np.zeros(4), capi._dp), ctypes.byref(out)))
    assert not out.value
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.blueprint_check(2, 6, np.zeros(4))


def test_a_uniform_table_passes():
    capi.blueprint_check(1, 2, uniform_table(1, 2))
    capi.blueprint_check(1, 4, uniform_table(1, 4))


def test_wrong_shape_is_refused():
    with pytest.raises(ValueError, match=r"must be \[30, 2\]"):
        capi.blueprint_check(1, 2, np.zeros((29, 2)))
    with pytest.raises(ValueError, match=r"must be \[30, 2\]"):
        capi.Blueprint(1, 2, np.zeros((30, 3)))


def test_validation_names_the_first_bad_node_and_hand():
    D, F = 1, 2
    cb, nc = tree(D, F)
    n = next(i for i in range(len(cb)) if nc[i] >= 2 and i > 0)
    e = cb[n] - 1                                    # the node's first edge
    s = uniform_table(D, F); s[e, 1] = np.nan
    with pytest.raises(capi.CfrbError, match=f"node {n}, hand 1: non-finite entry for child 0"):
        capi.blueprint_check(D, F, s)
    s = uniform_table(D, F); s[e + 1, 0] = -0.25; s[e, 0] += 0.5
    with pytest.raises(capi.CfrbError, match=f"node {n}, hand 0: negative entry for child 1"):
        capi.blueprint_check(D, F, s)
    s = uniform_table(D, F); s[e, 1] += 2e-6
    with pytest.raises(capi.CfrbError, match=f"node {n}, hand 1: the row over the node's {nc[n]} children sums to"):
        capi.blueprint_check(D, F, s)
    s = uniform_table(D, F); s[e, 1] += 5e-7                # within 1e-6 of 1
    capi.blueprint_check(D, F, s)
    s = uniform_table(D, F); s[0, 0] = np.inf; s[e, 1] = np.nan   # the first bad row in BFS order is the root's
    with pytest.raises(capi.CfrbError, match="node 0, hand 0: non-finite"):
        capi.blueprint_check(D, F, s)


def test_create3_refuses_a_seat_without_an_agent():
    import ctypes
    out = ctypes.c_void_p()
    empty = capi.MatchAgent(None, None, 0)
    with pytest.raises(capi.CfrbError, match="needs a handle or a blueprint"):
        capi._check(capi.lib().cfrb_match_create3(ctypes.byref(empty), ctypes.byref(empty), 8, 8, 0, ctypes.byref(out)))


# ------------------------------------------------------------------------------------------------ GPU
def solver(D, F, slots, iters, use_cfr, weights, max_depth=2):
    S = capi.WaveSolver(D, F, slots, max_depth=max_depth, num_iters=iters, linear_update=True,
                        net_mode=capi.NET_ZERO if weights is None else capi.NET_FP32,
                        solver=capi.SOLVER_CFR if use_cfr else capi.SOLVER_FP)
    if weights is not None:
        S.set_weights(weights)
    return S


def frozen(S, every_node):
    """The agent's full recursive policy as a blueprint, and the table its walk filled."""
    (S.recursive_exploitability if every_node else S.to_leaf_exploitability)()
    return capi.Blueprint.from_solver(S), S.to_leaf_strategy()


def play(M, traced):
    r = M.play()
    r["traces"] = [M.trace(g) for g in range(traced)]
    M.close()
    return r


def assert_same_games(live, bp, k_live, traced):
    """Payoffs, plies, the solving agent's solves and every traced ply, probability, and the solving agent's act_iterations and
    beliefs are the same; the blueprint solves nothing and traces -2 on every ply."""
    assert np.array_equal(live["payoff_a"], bp["payoff_a"]) and np.array_equal(live["plies"], bp["plies"])
    kb = 1 - k_live                                  # the seat of the solving opponent
    key = "solves_b" if kb == 1 else "solves_a"
    assert live[key] == bp[key] > 0
    assert bp["solves_a" if k_live == 0 else "solves_b"] == 0
    for g in range(traced):
        x, y = live["traces"][g], bp["traces"][g]
        assert np.array_equal(x["plies"], y["plies"]), g
        assert np.array_equal(x["prob"].view(np.int64), y["prob"].view(np.int64)), g
        assert np.array_equal(x["act_iteration"][:, kb], y["act_iteration"][:, kb]), g
        assert (y["act_iteration"][:, k_live] == -2).all(), g
        assert np.array_equal(x["root_beliefs"][:, kb].view(np.int64), y["root_beliefs"][:, kb].view(np.int64)), g


CASES = [  # D, F, max_depth, CFR, net seed (None: the zero net)
    (1, 4, 2, True, None),
    (1, 4, 3, False, 0),
    (2, 3, 2, True, 1),
    (1, 6, 2, False, 0),
]


@pytest.mark.gpu
@pytest.mark.parametrize("every_node", [False, True], ids=["to_leaf", "every_node"])
@pytest.mark.parametrize("D,F,depth,use_cfr,seed", CASES)
def test_gpu_blueprint_plays_the_frozen_agent_bit_for_bit(D, F, depth, use_cfr, seed, every_node):
    """blueprint(S_A) against B (sampled) plays play_match(A average / every_node, B sampled)'s games, in either seat."""
    games, slots, iters = 256, 256, 32
    w = None if seed is None else net(D, F, seed)
    policy = capi.MATCH_EVERY_NODE if every_node else capi.MATCH_AVERAGE
    A_ = solver(D, F, slots, iters, use_cfr, w, depth)
    bp, table = frozen(A_, every_node)
    assert np.array_equal(bp.strategy().view(np.int64), table.view(np.int64))
    for seat in (0, 1):
        B1, B2 = solver(D, F, slots, iters, True, None, depth), solver(D, F, slots, iters, True, None, depth)
        if seat == 0:
            live = play(capi.Match(A_, B1, slots, games, seed=7, policy=policy, policy_b=capi.MATCH_SAMPLED), games)
            fixed = play(capi.Match(bp, B2, slots, games, seed=7, policy_b=capi.MATCH_SAMPLED), games)
        else:
            live = play(capi.Match(B1, A_, slots, games, seed=7, policy=capi.MATCH_SAMPLED, policy_b=policy), games)
            fixed = play(capi.Match(B2, bp, slots, games, seed=7, policy=capi.MATCH_SAMPLED), games)
        assert_same_games(live, fixed, seat, games)
        B1.close(); B2.close()
    bp.close(); A_.close()


@pytest.mark.gpu
def test_gpu_from_full_game_holds_the_solvers_bits():
    fg = capi.FullGame(1, 6)
    fg.step(64)
    bp = capi.Blueprint.from_full_game(fg)
    assert np.array_equal(bp.strategy().view(np.int64), fg.strategy().view(np.int64))
    up = capi.Blueprint(1, 6, fg.strategy())        # the host upload of the same table
    assert np.array_equal(up.strategy().view(np.int64), fg.strategy().view(np.int64))
    bp.close(); up.close(); fg.close()


@pytest.mark.gpu
def test_gpu_from_handle_needs_a_walk():
    S = solver(1, 4, 8, 8, True, None)
    with pytest.raises(capi.CfrbError, match="no full-tree strategy"):
        capi.Blueprint.from_solver(S)
    S.close()


@pytest.mark.gpu
def test_gpu_results_do_not_depend_on_n_slots():
    D, F, games = 1, 6, 4096
    fg = capi.FullGame(D, F)
    fg.step(128)
    bp = capi.Blueprint.from_full_game(fg)
    out = []
    for slots in (256, 8192):
        B = solver(D, F, slots, 32, True, net(D, F, 0))
        r = capi.Match(B, bp, slots, games, seed=3, policy=capi.MATCH_SAMPLED).play()
        out.append(r); B.close()
        bb = capi.Match(bp, bp, slots, games, seed=3).play()
        out.append(bb)
    assert np.array_equal(out[0]["payoff_a"], out[2]["payoff_a"]) and np.array_equal(out[0]["plies"], out[2]["plies"])
    assert out[0]["solves_a"] == out[2]["solves_a"] and out[0]["solves_b"] == out[2]["solves_b"] == 0
    assert np.array_equal(out[1]["payoff_a"], out[3]["payoff_a"]) and out[1]["solves"] == out[3]["solves"] == 0
    bp.close(); fg.close()


@pytest.mark.gpu
def test_gpu_refusals():
    bp4 = capi.Blueprint(1, 4, uniform_table(1, 4))
    bp2 = capi.Blueprint(1, 2, uniform_table(1, 2))
    S = solver(1, 4, 8, 8, True, None)
    with pytest.raises(capi.CfrbError, match="different games"):
        capi.Match(bp4, bp2, 8, 8)
    with pytest.raises(capi.CfrbError, match="different games"):
        capi.Match(bp2, S, 8, 8, policy=capi.MATCH_AVERAGE)
    with pytest.raises(capi.CfrbError, match="bad policy"):
        capi.Match(bp4, S, 8, 8, policy=9)
    with pytest.raises(capi.CfrbError, match="smaller than n_slots"):
        capi.Match(bp4, S, 16, 16, policy=capi.MATCH_AVERAGE)
    with pytest.raises(capi.CfrbError, match="n_games must be even"):
        capi.Match(bp4, bp4, 8, 7)
    M = capi.Match(bp4, S, 8, 8, policy=capi.MATCH_AVERAGE)
    with pytest.raises(capi.CfrbError, match="already plays in a live match"):
        capi.Match(S, bp4, 8, 8, policy=capi.MATCH_AVERAGE)
    M.close(); S.close(); bp4.close(); bp2.close()


def seat_mean_ev(S, s1, s2):
    """compute_ev2(s1, s2) = (player 0 playing s1 against s2, -(player 0 playing s2 against s1)): the EV of s1 in seat 0 and in
    seat 1, whose mean is what the payoff of agent a (s1, seat 0 in even games) averages to."""
    ev0, ev1 = S.ev2_compact(s1, s2)
    return (ev0 + ev1) / 2


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 3)])
def test_gpu_match_means_match_the_exact_ev(D, F):
    games = 1 << 17
    cfr, fp = capi.FullGame(D, F), capi.FullGame(D, F, solver=capi.SOLVER_FP)
    cfr.step(1024); fp.step(64)
    s_cfr, s_fp = cfr.strategy(), fp.strategy()
    b_cfr, b_fp = capi.Blueprint.from_full_game(cfr), capi.Blueprint.from_full_game(fp)
    A_ = solver(D, F, 8192, 64, True, net(D, F, 0))
    r = capi.Match(b_cfr, b_fp, 8192, games, seed=21).play()
    m, se = r["payoff_a"].mean(), r["payoff_a"].std() / np.sqrt(games)
    ev = seat_mean_ev(A_, s_cfr, s_fp)
    assert r["solves"] == 0 and abs(m - ev) <= 4 * se, (m, ev, se)
    _, s_a = frozen(A_, False)                       # the agent's own to-leaf average policy against the CFR blueprint
    r = capi.Match(A_, b_cfr, 8192, games, seed=22, policy=capi.MATCH_AVERAGE).play()
    m, se = r["payoff_a"].mean(), r["payoff_a"].std() / np.sqrt(games)
    ev = seat_mean_ev(A_, s_a, s_cfr)
    assert r["solves_b"] == 0 and r["solves_a"] > 0 and abs(m - ev) <= 4 * se, (m, ev, se)
    b_cfr.close(); b_fp.close(); A_.close(); cfr.close(); fp.close()


@pytest.mark.gpu
def test_gpu_blueprint_match_2x5f():
    """The largest game class: a 2x5f CFR blueprint against itself is fair, and against the uniform table wins."""
    D, F, games = 2, 5, 1 << 15
    fg = capi.FullGame(D, F)
    uni = capi.Blueprint(D, F, fg.strategy())       # before its first iteration the average is uniform
    fg.step(256)
    bp = capi.Blueprint.from_full_game(fg)
    r = capi.Match(bp, bp, 8192, games, seed=1).play()
    m, se = r["payoff_a"].mean(), r["payoff_a"].std() / np.sqrt(games)
    assert abs(m) <= 4 * se, (m, se)
    r = capi.Match(bp, uni, 8192, games, seed=2).play()
    assert r["payoff_a"].mean() > 0.2 and (r["plies"] >= 1).all()
    bp.close(); uni.close(); fg.close()


# ------------------------------------------------------------------------------------------------ LBR against a blueprint
def matches_table(D, F):
    """num_matches(hand, face): dice of the hand showing the face or the wild last face; hand = D base-F digits."""
    H = F ** D
    return np.array([[sum(1 for i in range(D) if (h // F ** i) % F in (f, F - 1)) for f in range(F)] for h in range(H)])


def lbr_values(beta, lb, hl, mt, F, A, row):
    """LBR's action values [A] (NaN where illegal) at a node with last bid lb, for LBR's hand hl and belief beta over the agent's
    hand; row(a) = the agent's compact rows [nc, H] at the node raise a reaches.  Serial fp64 sums in the rule's order."""
    H = len(beta)
    vals = np.full(A, np.nan)
    true = lambda bid, h: mt[hl, bid % F] + mt[h, bid % F] >= 1 + bid // F
    for a in range(0 if lb < 0 else lb + 1, A - 1):
        sg, v = row(a), 0.0
        for h in range(H):
            inner = 0.0
            for i, a2 in enumerate(range(a + 1, A)):
                u = (1.0 if true(a, h) else -1.0) if a2 == A - 1 else (-1.0 if true(a2, h) else 1.0)
                inner += float(sg[i, h]) * u
            v += float(beta[h]) * inner
        vals[a] = v
    if lb >= 0:
        v = 0.0
        for h in range(H):
            v += float(beta[h]) * (-1.0 if true(lb, h) else 1.0)
        vals[A - 1] = v
    return vals


def lbr_argmax(vals):
    best = -1
    for a, v in enumerate(vals.tolist()):
        if not np.isnan(v) and (best < 0 or v > vals[best]):
            best = a
    return best


def hand_made_1x2f():
    """A fixed, far-from-uniform 1x2f table: at every node the hand-0 row favours the lowest child, the hand-1 row the highest."""
    cb, nc = tree(1, 2)
    s = np.zeros((len(cb) - 1, 2))
    for n in range(len(cb)):
        k = nc[n]
        if k:
            w = np.arange(1, k + 1, dtype=np.float64)
            s[cb[n] - 1:cb[n] - 1 + k, 0] = w[::-1] / w.sum()
            s[cb[n] - 1:cb[n] - 1 + k, 1] = w / w.sum()
    return s


def test_lbr_rule_on_a_hand_made_1x2f_table():
    """1x2f: hands 0 (face 0) and 1 (the wild face 1); bids 0 = 1x0, 1 = 1x1, 2 = 2x0, 3 = 2x1, 4 = liar."""
    D, F, A = 1, 2, 5
    mt = matches_table(D, F)
    assert mt.tolist() == [[1, 0], [1, 1]]
    s = hand_made_1x2f()
    cb, nc = tree(D, F)
    x = cb[0] + 1                                     # the node after the opening bid 1x1
    assert nc[x] == 3
    row = lambda a: s[cb[cb[x] + a - 2] - 1:cb[cb[x] + a - 2] - 1 + nc[cb[x] + a - 2]]
    # LBR holds face 0 and believes the agent holds hand 1 with probability 3/4.  Raise 2x0 (true for both hands): the agent's
    # only raise 2x1 is false and called (+1), its liar call loses (+1).  Raise 2x1 (false for both): the agent can only call.
    v = lbr_values(np.array([0.25, 0.75]), 1, 0, mt, F, A, row)
    assert np.isnan(v[:2]).all() and v[2:].tolist() == [1.0, -1.0, -0.5] and lbr_argmax(v) == 2


@pytest.mark.gpu
def test_gpu_lbr_against_a_hand_made_table_follows_the_rule():
    D, F, A, H, games = 1, 2, 5, 2, 256
    s = hand_made_1x2f()
    cb, nc = tree(D, F)
    mt = matches_table(D, F)
    bp = capi.Blueprint(D, F, s)
    M = capi.LbrMatch(bp, 64, games, seed=4)
    r = M.play()
    assert r["solves"] == 0 and r["whatif_solves"] == 0 and set(np.unique(r["payoff_a"]).tolist()) <= {-1.0, 1.0}
    decisions = 0
    for g in range(games):
        t, lt = M.trace(g), M.lbr_trace(g)
        beta, node = np.full(H, 1.0 / H), 0
        for i, (who, lb, actor, hand, action, _) in enumerate(t["plies"].tolist()):
            lo = 0 if lb < 0 else lb + 1
            rows = s[cb[node] - 1:cb[node] - 1 + nc[node]]
            if who == 0:
                assert actor == g & 1 and t["prob"][i] == rows[action - lo, hand]
                beta = beta * rows[action - lo]
                beta = beta / (beta[0] + beta[1])
            else:
                assert np.array_equal(lt["beliefs"][i], beta)
                want = lbr_values(beta, lb, hand, mt, F, A, lambda a: s[cb[cb[node] + a - lo] - 1:cb[cb[node] + a - lo] - 1 + nc[cb[node] + a - lo]])
                assert np.array_equal(lt["values"][i], want, equal_nan=True) and action == lbr_argmax(want), (g, i)
                decisions += 1
            node = cb[node] + action - lo
        assert t["plies"][-1, 4] == A - 1
    assert decisions >= games
    M.close(); bp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("every_node", [False, True], ids=["to_leaf", "every_node"])
@pytest.mark.parametrize("D,F,depth,use_cfr,seed", CASES)
def test_gpu_lbr_against_the_frozen_agent_bit_for_bit(D, F, depth, use_cfr, seed, every_node):
    """LBR against blueprint(S_A) plays play_lbr(A, average / every_node)'s games: payoffs, plies, every traced ply and LBR's
    values and beliefs; the blueprint solves nothing."""
    games, iters = 256, 32
    w = None if seed is None else net(D, F, seed)
    A_ = solver(D, F, 256, iters, use_cfr, w, depth)
    bp, _ = frozen(A_, every_node)
    live = capi.LbrMatch(A_, 64, games, seed=5, policy=capi.MATCH_EVERY_NODE if every_node else capi.MATCH_AVERAGE)
    fixed = capi.LbrMatch(bp, 64, games, seed=5)
    x, y = live.play(), fixed.play()
    assert np.array_equal(x["payoff_a"], y["payoff_a"]) and np.array_equal(x["plies"], y["plies"])
    assert x["solves"] > 0 and y["solves"] == y["whatif_solves"] == 0
    for g in range(games):
        tx, ty, lx, ly = live.trace(g), fixed.trace(g), live.lbr_trace(g), fixed.lbr_trace(g)
        assert np.array_equal(tx["plies"][:, :5], ty["plies"][:, :5]), g
        assert np.array_equal(tx["prob"].view(np.int64), ty["prob"].view(np.int64)), g
        assert np.array_equal(lx["values"].view(np.int64), ly["values"].view(np.int64)), g
        assert np.array_equal(lx["beliefs"].view(np.int64), ly["beliefs"].view(np.int64)), g
    live.close(); fixed.close(); bp.close(); A_.close()


@pytest.mark.gpu
def test_gpu_lbr_bounds_the_blueprints_exact_exploitability_2x5f():
    D, F, games = 2, 5, 1 << 16
    fg = capi.FullGame(D, F)
    fg.step(256)
    expl = float(np.mean(fg.exploitability()))
    bp = capi.Blueprint.from_full_game(fg)
    r = capi.LbrMatch(bp, 8192, games, seed=6).play()
    m, se = r["payoff_a"].mean(), r["payoff_a"].std() / np.sqrt(games)
    lbr = -m                                          # payoff_a is the blueprint's; LBR's is its negative
    assert r["solves"] == 0 and lbr - 4 * se <= expl, (lbr, se, expl)
    bp.close(); fg.close()


# ------------------------------------------------------------------------------------------------ files, rela and the CLIs
def test_file_round_trip_and_refusals(tmp_path):
    from rebel_b200.blueprint import load_blueprint, save_blueprint
    s = uniform_table(1, 4)
    p = str(tmp_path / "bp.npz")
    assert save_blueprint(p, 1, 4, s, "to_leaf", {"iterations": 64, "net": "zero"}, [0.25, 0.125]) == p
    d = load_blueprint(p, 1, 4)
    assert np.array_equal(d["strategy"], s) and d["strategy"].dtype == np.float64
    assert (d["num_dice"], d["num_faces"], d["source"], d["br"], d["exploitability"]) == (1, 4, "to_leaf", [0.25, 0.125], 0.1875)
    assert d["settings"] == {"iterations": 64, "net": "zero"}
    with pytest.raises(ValueError, match="holds a 1x4f blueprint, not 1x3f"):
        load_blueprint(p, 1, 3)
    bad = str(tmp_path / "bad.npz")
    with open(bad, "wb") as f:
        np.savez(f, num_dice=1, num_faces=4, strategy=s[:-1], source="to_leaf", settings="{}", br=np.zeros(2), exploitability=0.0)
    with pytest.raises(ValueError, match=r"is \[510, 4\], the file holds \[509, 4\]"):
        load_blueprint(bad, 1, 4)
    with pytest.raises(ValueError, match="source must be one of"):
        save_blueprint(p, 1, 4, s, "sampled", {}, [0, 0])
    with pytest.raises(ValueError, match="more than 23 actions"):
        load_blueprint(p, 2, 6)


def test_cli_parsers():
    from rebel_b200.exploitability import build_parser as expl_parser
    from rebel_b200.head_to_head import blueprint_conflicts, build_parser
    from rebel_b200.local_br import build_parser as lbr_parser
    from rebel_b200.play import build_parser as play_parser
    from rebel_b200.solve_game import build_parser as solve_parser
    assert solve_parser().parse_args(["--save", "a.npz"]).save == "a.npz" and solve_parser().parse_args([]).save is None
    assert expl_parser().parse_args(["--every_node", "--save", "b.npz"]).save == "b.npz" and expl_parser().parse_args([]).save is None
    a = build_parser().parse_args(["--blueprint_a", "x.npz", "--net_b", "n.ckpt"])
    assert (a.blueprint_a, a.blueprint_b) == ("x.npz", None) and blueprint_conflicts(a) == []
    a = build_parser().parse_args(["--blueprint_b", "x.npz", "--net_b", "n.ckpt", "--random_net_seed_b", "1", "--net_a", "m"])
    assert blueprint_conflicts(a) == ["--net_b", "--random_net_seed_b"]
    assert lbr_parser().parse_args(["--blueprint", "y.npz"]).blueprint == "y.npz" and lbr_parser().parse_args([]).blueprint is None
    assert play_parser().parse_args(["--blueprint", "z.npz"]).blueprint == "z.npz"


@pytest.mark.parametrize("cli,argv", [
    ("head_to_head", ["--blueprint_a", "x.npz", "--net_a", "n.ckpt"]),
    ("head_to_head", ["--blueprint_b", "x.npz", "--random_net_seed_b", "0"]),
    ("local_br", ["--blueprint", "x.npz", "--net", "n.ckpt"]),
    ("local_br", ["--blueprint", "x.npz", "--random_net_seed", "3"]),
    ("play", ["--blueprint", "x.npz", "--net", "n.ckpt"]),
])
def test_cli_refuses_a_net_for_a_blueprint_seat(cli, argv):
    import importlib
    with pytest.raises(SystemExit) as e:
        importlib.import_module(f"rebel_b200.{cli}").main(argv)
    assert e.value.code == 2


@pytest.mark.parametrize("cli,flag", [("head_to_head", "--blueprint_a"), ("head_to_head", "--blueprint_b"), ("local_br", "--blueprint"),
                                      ("play", "--blueprint")])
def test_cli_refuses_more_than_23_actions_and_another_game(cli, flag, tmp_path):
    import importlib
    from rebel_b200.blueprint import save_blueprint
    p = str(tmp_path / "bp.npz")
    save_blueprint(p, 1, 4, uniform_table(1, 4), "solve_game", {}, [0, 0])
    main = importlib.import_module(f"rebel_b200.{cli}").main
    with pytest.raises(SystemExit, match="more than 23 actions"):
        main(["--num_dice", "2", "--num_faces", "6", flag, p])
    with pytest.raises(SystemExit, match="not 1x6f"):
        main(["--num_dice", "1", "--num_faces", "6", flag, p])


def test_cli_lines_report_blueprints():
    from rebel_b200.exploitability import expl_line, parse_expl
    from rebel_b200.head_to_head import h2h_line, parse_h2h
    from rebel_b200.local_br import lbr_line, parse_lbr
    r = {"exploitability": 0.5, "br": [0.25, 0.75], "subgames": 3, "subgame_iters": 9, "seconds": 1.0}
    assert parse_expl(expl_line("n", "1x4f", r, saved="a.npz"))["saved"] == "a.npz"
    assert "saved" not in parse_expl(expl_line("n", "1x4f", r))
    d = parse_lbr(lbr_line("blueprint:a.npz", 8, 0.1, 0.01, [0.1, 0.1], "blueprint", 0.2))
    assert (d["policy"], d["exploitability"], d["net"]) == ("blueprint", 0.2, "blueprint:a.npz")
    assert "exploitability" not in parse_lbr(lbr_line("n", 8, 0.1, 0.01, [0.1, 0.1]))
    d = parse_h2h(h2h_line("blueprint:a.npz", "zero", 8, 0.0, 0.1, [0, 0], ("blueprint", "sampled")))
    assert (d["net_a"], d["policy_a"], d["policy_b"]) == ("blueprint:a.npz", "blueprint", "sampled")


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


def test_rela_refuses_before_any_device_work(rela):
    import torch
    c = make_cfg(rela, 1, 4, 8)
    s = torch.from_numpy(uniform_table(1, 4))
    with pytest.raises(RuntimeError, match="flat_weights_a must be None"):
        rela.play_match(c, c, 0, 8, blueprint_a=s, flat_weights_a=torch.zeros(4))
    with pytest.raises(RuntimeError, match="flat_weights_b must be None"):
        rela.play_match(c, c, 0, 8, blueprint_b=s, flat_weights_b=torch.zeros(4))
    with pytest.raises(RuntimeError, match="flat_weights must be None"):
        rela.play_lbr(c, 0, 8, blueprint=s, flat_weights=torch.zeros(4))
    with pytest.raises(RuntimeError, match=r"is a \[510, 4\] table"):
        rela.play_match(c, c, 0, 8, blueprint_a=s[:-1])
    big = make_cfg(rela, 2, 6, 8)
    with pytest.raises(RuntimeError, match="more than 23 actions"):
        rela.play_lbr(big, 0, 8, blueprint=s)
    with pytest.raises(RuntimeError, match="more than 23 actions"):
        rela.Agent.from_blueprint(2, 6, s)
    with pytest.raises(RuntimeError, match=r"\[510, 4\]"):
        rela.Agent.from_blueprint(1, 4, s[:-1])


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,use_cfr", [(1, 4, True), (2, 3, False)])
def test_gpu_rela_blueprints_replay_the_frozen_agent(rela, D, F, use_cfr):
    """play_match / play_lbr with S_A = exploitability_to_leaf(return_strategy=True)['strategy'] in A's place give
    play_match(A average, B sampled)'s and play_lbr(A, average)'s results; rela.Agent.from_blueprint(S_A) answers a scripted
    batch of tables as rela.Agent(A, 'average') does."""
    import torch
    w = torch.from_numpy(net(D, F, 0))
    ca, cb = make_cfg(rela, D, F, 64, use_cfr, 1), make_cfg(rela, D, F, 32, True, 0)
    e = rela.exploitability_to_leaf(ca, 0, flat_weights=w, return_strategy=True)
    s_a = e["strategy"]
    assert s_a.dtype == torch.float64 and tuple(s_a.shape) == ((1 << (1 + 2 * D * F)) - 2, F ** D)
    live = rela.play_match(ca, cb, 0, 512, seed=3, policy="average", policy_b="sampled", flat_weights_a=w, concurrent_games=128)
    fixed = rela.play_match(ca, cb, 0, 512, seed=3, policy="average", policy_b="sampled", blueprint_a=s_a, concurrent_games=128)
    assert torch.equal(live["payoff_a"], fixed["payoff_a"]) and torch.equal(live["plies"], fixed["plies"])
    assert live["solves_b"] == fixed["solves_b"] > 0 and fixed["solves_a"] == 0
    live = rela.play_lbr(ca, 0, 512, seed=4, flat_weights=w, concurrent_games=128)
    fixed = rela.play_lbr(ca, 0, 512, seed=4, blueprint=s_a, concurrent_games=128)
    assert torch.equal(live["payoff_lbr"], fixed["payoff_lbr"]) and fixed["solves"] == 0 and fixed["policy"] == "blueprint"
    e_en = rela.exploitability_recursive(ca, 0, flat_weights=w, return_strategy=True)
    live = rela.play_lbr(ca, 0, 256, seed=5, flat_weights=w, concurrent_games=128, policy="every_node")
    fixed = rela.play_lbr(ca, 0, 256, seed=5, blueprint=e_en["strategy"], concurrent_games=128)
    assert torch.equal(live["payoff_lbr"], fixed["payoff_lbr"])
    # the agent: a scripted batch of tables, the same keys, the opponent's moves from a fixed stream
    G = 64
    ag = rela.Agent(ca, 0, G, "average", seed=9, flat_weights=w)
    bp = rela.Agent.from_blueprint(D, F, s_a, device=0, tables=G, seed=9)
    A, H = ag.num_actions, ag.num_hands
    assert (bp.num_actions, bp.num_hands) == (A, H)
    hands, seats = np.random.RandomState(1).randint(0, H, size=G), np.arange(G) % 2
    for x in (ag, bp):
        x.new_games(np.arange(G), seats, hands, keys=np.arange(G) + 100)
    opp = np.random.RandomState(2)
    lb, player, running = np.full(G, -1), np.zeros(G, np.int64), np.ones(G, bool)
    steps = 0
    while running.any():
        ids = np.flatnonzero(running)
        assert torch.equal(ag.policy(ids), bp.policy(ids))
        acts = []
        for g in ids:
            lo = 0 if lb[g] < 0 else lb[g] + 1
            hi = A - 1 if lb[g] < 0 else A
            acts.append(-1 if player[g] == seats[g] else int(opp.randint(lo, hi)))
        a1, p1, d1 = ag.step(ids, acts)
        a2, p2, d2 = bp.step(ids, acts)
        assert torch.equal(a1, a2) and torch.equal(d1, d2)
        assert np.array_equal(p1.numpy().view(np.int64), p2.numpy().view(np.int64))
        lb[ids], player[ids] = a1.numpy(), player[ids] ^ 1
        running[ids[d1.numpy()]] = False
        steps += 1
    st = bp.state(np.arange(G))
    assert (st["subgames"] == 0).all() and (st["act_iteration"] == -1).all()
    assert bp.counts()["solves"] == 0 and ag.counts()["solves"] > 0 and steps >= 2
    ag.close(); bp.close()


@pytest.mark.gpu
def test_gpu_cli_end_to_end_2x5f(tmp_path):
    """solve_game --save, then head_to_head --blueprint_b and local_br --blueprint on the saved file."""
    import os
    import subprocess
    import sys
    from rebel_b200.head_to_head import parse_h2h
    from rebel_b200.local_br import parse_lbr
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    run = lambda mod, argv: subprocess.run([sys.executable, "-m", f"rebel_b200.{mod}"] + argv, cwd=str(tmp_path), env=env,
                                           capture_output=True, text=True, timeout=900)
    game = ["--num_dice", "2", "--num_faces", "5"]
    p = run("solve_game", game + ["--subgame_iters", "256", "--cfr", "--save", "cfr.npz"])
    assert p.returncode == 0, p.stderr[-4000:]
    solve = json.loads([l for l in p.stdout.split("\n") if l.startswith("SOLVE ")][0][6:])
    assert solve["saved"] == "cfr.npz" and os.path.exists(tmp_path / "cfr.npz")
    p = run("head_to_head", game + ["--blueprint_b", "cfr.npz", "--games", "512", "--subgame_iters", "64", "--cfr",
                                    "--concurrent_games", "512", "--policy", "average"])
    assert p.returncode == 0, p.stderr[-4000:]
    d = parse_h2h([l for l in p.stdout.split("\n") if l.startswith("H2H ")][0])
    assert (d["net_b"], d["policy_a"], d["policy_b"], d["games"]) == ("blueprint:cfr.npz", "average", "blueprint", 512)
    p = run("local_br", game + ["--blueprint", "cfr.npz", "--games", "8192"])
    assert p.returncode == 0, p.stderr[-4000:]
    d = parse_lbr([l for l in p.stdout.split("\n") if l.startswith("LBR ")][0])
    assert d["policy"] == "blueprint" and d["exploitability"] == solve["exploitability"]
    assert d["mean"] - 4 * d["stderr"] <= d["exploitability"]


@pytest.mark.gpu
def test_gpu_cli_exploitability_save_then_play(tmp_path):
    """exploitability --every_node --save writes the every-node policy; play --blueprint plays a scripted human against it."""
    import os
    import subprocess
    import sys
    from rebel_b200.blueprint import load_blueprint
    from rebel_b200.exploitability import parse_expl
    from rebel_b200.play import parse_play
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root + os.pathsep + os.environ.get("PYTHONPATH", ""))
    game = ["--num_dice", "1", "--num_faces", "4"]
    p = subprocess.run([sys.executable, "-m", "rebel_b200.exploitability"] + game + ["--random_net_seed", "0", "--subgame_iters", "64",
                       "--cfr", "--every_node", "--save", "en.npz"], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    d = parse_expl([l for l in p.stdout.split("\n") if l.startswith("EXPL ")][0])
    f = load_blueprint(str(tmp_path / "en.npz"), 1, 4)
    assert d["saved"] == "en.npz" and d["policy"] == "every_node" and f["source"] == "every_node"
    assert f["br"] == d["br"] and f["settings"]["iterations"] == 64 and f["settings"]["net"] == "random_net_seed=0"
    capi.blueprint_check(1, 4, f["strategy"])
    p = subprocess.run([sys.executable, "-m", "rebel_b200.play"] + game + ["--blueprint", "en.npz", "--games", "2", "--seed", "3"],
                       cwd=str(tmp_path), env=env, input="1 1\nliar\nliar\nliar\n", capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    assert "every_node blueprint" in p.stdout and p.stdout.count("reveal:") == 2
    d = parse_play([l for l in p.stdout.split("\n") if l.startswith("PLAY ")][0])
    assert d["net"] == "blueprint:en.npz" and d["games"] == 2 and d["agent_wins"] + d["human_wins"] == 2
