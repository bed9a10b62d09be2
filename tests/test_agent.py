"""A ReBeL agent played from outside (cfrb_agent_*, rela.Agent, python -m rebel_b200.play): at every table the agent plays its
recursive to-leaf strategy along the path played, bit for bit, whichever tables a call lists and in whatever order; a replayed
match reproduces the match walk's probabilities; bad calls are refused without touching any table."""
import ctypes
import itertools
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


def normalize(b):
    """normalize_beliefs_inplace with the sum taken in sequential order."""
    s = 0.0
    for v in b.tolist():
        s += v + 1e-80
    return (b + 1e-80) / s


def legal_actions(last_bid, A):
    return np.arange(0, A - 1) if last_bid < 0 else np.arange(last_bid + 1, A)


# ------------------------------------------------------------------------------------------------ CPU
def test_cli_parser():
    from rebel_b200.play import build_parser
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "3", "--net", "x.ckpt", "--subgame_iters", "256", "--cfr",
                                   "--mdp_depth", "3", "--policy", "average", "--games", "5", "--seed", "7"])
    assert (a.num_dice, a.num_faces, a.net, a.subgame_iters, a.cfr, a.mdp_depth) == (2, 3, "x.ckpt", 256, True, 3)
    assert (a.policy, a.games, a.seed) == ("average", 5, 7)
    d = build_parser().parse_args([])
    assert (d.num_dice, d.num_faces, d.net, d.subgame_iters, d.cfr, d.mdp_depth) == (1, 6, None, 1024, False, 2)
    assert (d.policy, d.games, d.seed) == ("sampled", 1, 0)
    # the settings head_to_head.agent_params reads, at its defaults
    assert (d.net_mode, d.no_linear, d.dcfr, d.device) == (None, False, None, 0)


def test_play_line_round_trip():
    from rebel_b200.play import parse_play, play_line
    line = play_line("zero", 4, 3, 1)
    assert line.startswith("PLAY {") and parse_play(line) == {"net": "zero", "games": 4, "agent_wins": 3, "human_wins": 1,
                                                              "agent_mean": 0.5}


@pytest.mark.parametrize("D,F", [(1, 4), (2, 3), (3, 2)])
def test_hand_index_is_base_f_digits(D, F):
    from rebel_b200.play import dice_to_hand, hand_to_dice
    for hand in range(F ** D):
        dice = hand_to_dice(hand, D, F)
        assert len(dice) == D and all(0 <= f < F for f in dice)
        assert hand == sum(f * F ** i for i, f in enumerate(dice)) and dice_to_hand(dice, F) == hand
    assert hand_to_dice(F ** D - 1, D, F) == [F - 1] * D


@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_payoff_rule_with_the_wild_face(D, F):
    """bidder_wins against a brute-force count over the dealt dice of every hand pair and every bid."""
    from rebel_b200.play import bidder_wins, num_actions
    all_dice = list(itertools.product(range(F), repeat=D))        # die i = digit i of the hand index
    index = {d: sum(f * F ** i for i, f in enumerate(d)) for d in all_dice}
    wins = 0
    for d0, d1 in itertools.product(all_dice, repeat=2):
        for bid in range(num_actions(D, F) - 1):
            quantity, face = 1 + bid // F, bid % F
            count = sum(1 for f in d0 + d1 if f == face or f == F - 1)
            assert bidder_wins(bid, index[d0], index[d1], D, F) == (count >= quantity), (d0, d1, bid)
            wins += count >= quantity
    assert 0 < wins < len(all_dice) ** 2 * (num_actions(D, F) - 1)


def test_bid_parsing():
    from rebel_b200.play import bid_name, parse_bid
    D, F = 1, 4                                          # actions 0..7 = quantity 1..2 x face 1..4, 8 = liar
    assert parse_bid("1 1", -1, D, F) == 0 and parse_bid(" 2 4 \n", -1, D, F) == 7 and parse_bid("LIAR", 3, D, F) == 8
    for bad, last in [("liar", -1), ("1 1", 0), ("1 3", 4), ("3 1", -1), ("1 5", -1), ("1 0", -1), ("x", -1), ("1 2 3", -1), ("", -1)]:
        assert isinstance(parse_bid(bad, last, D, F), str), (bad, last)
    assert [bid_name(a, D, F) for a in (0, 5, 8)] == ["1 1", "2 2", "liar"]


def test_agent_needs_a_device(rela):
    from rebel_b200 import capi
    if capi.lib().cfrb_device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no CUDA device"):
        rela.Agent(make_cfg(rela, 1, 4, 16), device=0, tables=8, policy="average")


# ------------------------------------------------------------------------------------------------ GPU
AVERAGE_CASES = [(D, F, cfr, n, 2) for D, F in [(1, 4), (2, 3)] for cfr in (True, False) for n in ("zero", "fp32", "tc_x2")]
AVERAGE_CASES.append((1, 4, True, "zero", 3))


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,use_cfr,net_name,depth", AVERAGE_CASES)
def test_gpu_average_policy_is_recursive_strategy(rela, D, F, use_cfr, net_name, depth):
    """At every node of 256 random games, policy() is strategy_recursive_to_leaf at the full-tree node for every hand, the agent's
    probability rows are its hand's row, and the root beliefs of every subgame are the host restatement of expand."""
    from rebel_b200 import capi
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_name]
    w = torch.from_numpy(net(D, F, 0)) if mode else None
    cfg = make_cfg(rela, D, F, 64, use_cfr, mode, depth)
    strat = rela.strategy_recursive_to_leaf(cfg, 0, w).numpy()
    tree = capi.unroll_tree(D, F)
    N, H, A = strat.shape
    T = 256
    ag = rela.Agent(cfg, 0, T, "average", seed=1, flat_weights=w)
    rng = np.random.RandomState(7)
    seats = np.arange(T) % 2
    hands = rng.randint(0, H, size=(T, 2))                        # by seat
    ag.new_games(np.arange(T), seats, hands[np.arange(T), seats])
    node, sub = np.zeros(T, np.int64), np.zeros(T, np.int64)
    bel = np.full((T, 2, H), 1.0 / H)
    running = np.ones(T, bool)
    checked = roots = unlikely = 0
    while running.any():
        ids = np.flatnonzero(running)
        pol = ag.policy(ids).numpy()
        st = ag.state(ids)
        acts = np.full(len(ids), -1, np.int32)
        for k, t in enumerate(ids):
            assert np.array_equal(pol[k], strat[node[t]]), (t, node[t])
            if sub[t] == 0:
                assert np.array_equal(st["root_beliefs"][k].numpy(), bel[t]), (t, node[t])
                roots += 1
            lb, actor = tree[node[t], 0], tree[node[t], 1]
            assert st["last_bid"][k] == lb and st["player"][k] == actor
            if actor != seats[t]:
                legal = legal_actions(lb, A)
                # now and then the action the agent's model finds least likely for the opponent's hand
                acts[k] = legal[np.argmin(strat[node[t], hands[t, actor], legal])] if rng.rand() < 0.3 else rng.choice(legal)
        played, probs, done = ag.step(ids, acts)
        played, probs, done = played.numpy(), probs.numpy(), done.numpy()
        for k, t in enumerate(ids):
            lb, actor, a = tree[node[t], 0], tree[node[t], 1], played[k]
            if actor == seats[t]:
                assert np.array_equal(probs[k], strat[node[t], hands[t, actor]]) and strat[node[t], hands[t, actor], a] > 0
            else:
                assert a == acts[k] and np.isnan(probs[k]).all()
                unlikely += strat[node[t], hands[t, actor], a] < 1e-3
            bel[t, actor] = bel[t, actor] * strat[node[t], :, a]
            node[t] = tree[node[t], 2] + a - (0 if lb < 0 else lb + 1)
            sub[t] += 1
            assert done[k] == (a == A - 1)
            if a == A - 1:
                running[t] = False
            elif sub[t] == depth:
                bel[t] = np.stack([normalize(bel[t, 0]), normalize(bel[t, 1])])
                sub[t] = 0
            checked += 1
    assert checked > 2 * T and roots > T
    st = ag.state(np.arange(T))
    assert (st["subgames"].numpy() >= 1).all() and ag.counts()["solves"] == int(st["subgames"].sum())
    ag.close()


@pytest.mark.gpu
def test_gpu_zero_probability_actions_follow_expand(rela):
    """Opponent actions the agent's strategy gives probability 0 are applied all the same: the next root beliefs are the
    eps-normalised products, as in expand.  Regret matching floors every regret at the smoothing epsilon, so "probability 0" is
    a probability of order 1e-80 here; the sampled policy has such actions for most hands at most nodes."""
    D, F, iters, T = 1, 4, 64, 256
    cfg = make_cfg(rela, D, F, iters, True, 0)
    ag = rela.Agent(cfg, 0, T, "sampled", seed=5)
    H, A = ag.num_hands, ag.num_actions
    rng = np.random.RandomState(3)
    seats = np.arange(T) % 2
    hands = rng.randint(0, H, size=(T, 2))
    ag.new_games(np.arange(T), seats, hands[np.arange(T), seats])
    lb, player, sub = np.full(T, -1), np.zeros(T, np.int64), np.zeros(T, np.int64)
    bel = np.full((T, 2, H), 1.0 / H)
    running = np.ones(T, bool)
    zero = checked = 0
    while running.any():
        ids = np.flatnonzero(running)
        pol = ag.policy(ids).numpy()
        st = ag.state(ids)
        acts = np.full(len(ids), -1, np.int32)
        for k, t in enumerate(ids):
            if sub[t] == 0:
                assert np.array_equal(st["root_beliefs"][k].numpy(), bel[t]), t
                assert np.isfinite(bel[t]).all() and abs(bel[t].sum(1) - 1).max() < 1e-12
                checked += 1
            if player[t] != seats[t]:
                legal = legal_actions(lb[t], A)
                p = pol[k][hands[t, player[t]], legal]
                acts[k] = legal[np.argmin(p)] if p.min() < 1e-50 else rng.choice(legal)
                zero += p.min() < 1e-50
        played = ag.step(ids, acts)[0].numpy()
        for k, t in enumerate(ids):
            a = played[k]
            bel[t, player[t]] = bel[t, player[t]] * pol[k][:, a]
            lb[t], player[t], sub[t] = a, player[t] ^ 1, sub[t] + 1
            if a == A - 1:
                running[t] = False
            elif sub[t] == 2:
                bel[t] = np.stack([normalize(bel[t, 0]), normalize(bel[t, 1])])
                sub[t] = 0
    assert zero > 10 and checked > T
    ag.close()


@pytest.mark.gpu
def test_gpu_replays_a_match(rela):
    """The traced games of a capi.Match fed into two rela.Agents, one per side: every traced probability is the acting agent's
    policy at that ply, and every traced root belief is the agent's."""
    from rebel_b200 import capi
    D, F, games = 1, 4, 256
    wa = net(D, F, 0)
    ca, cb = make_cfg(rela, D, F, 64, True, 3), make_cfg(rela, D, F, 32, True, 0)
    A_ = capi.WaveSolver(D, F, 64, max_depth=2, num_iters=64, linear_update=True, net_mode=3, solver=capi.SOLVER_CFR)
    A_.set_weights(wa)
    B_ = capi.WaveSolver(D, F, 64, max_depth=2, num_iters=32, linear_update=True, net_mode=0, solver=capi.SOLVER_CFR)
    M = capi.Match(A_, B_, 64, games, seed=21, policy=capi.MATCH_AVERAGE)
    M.play()
    traces = [M.trace(g) for g in range(games)]
    M.close(); A_.close(); B_.close()
    agents = [rela.Agent(ca, 0, games, "average", flat_weights=torch.from_numpy(wa)), rela.Agent(cb, 0, games, "average")]
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
            if ply == 0 or traces[g]["plies"][ply - 1][5] != r:
                for k in range(2):
                    assert np.array_equal(states[k]["root_beliefs"][i].numpy(), traces[g]["root_beliefs"][r, k]), (g, r, k)
            acts[i] = action
            checked += 1
        for ag in agents:
            played, _, done = ag.step(live, acts)
            assert np.array_equal(played.numpy(), acts)
            assert np.array_equal(done.numpy(), np.array([ply == len(traces[g]["plies"]) - 1 for g in live]))
    assert checked >= 2 * games
    for ag in agents:
        ag.close()


def even_iteration_probs(iters):
    w = np.array([0.0 if i % 2 else i / 2 + 1 for i in range(iters)])
    return w / w.sum()


@pytest.mark.gpu
def test_gpu_sampled_policy(rela):
    """act_iterations follow i/2 + 1 on even i; a lone WaveSolver re-solve from the recorded root beliefs and act_iteration gives
    policy() bit for bit; the agent's actions at the root with a fixed hand follow its policy rows."""
    from scipy.stats import chisquare
    from rebel_b200 import capi
    D, F, iters, T = 1, 4, 64, 2048
    w = net(D, F, 0)
    cfg = make_cfg(rela, D, F, iters, True, 3)
    ag = rela.Agent(cfg, 0, T, "sampled", seed=9, flat_weights=torch.from_numpy(w))
    H, A = ag.num_hands, ag.num_actions
    rng = np.random.RandomState(4)
    seats = np.zeros(T, np.int32)                                 # the agent moves first, with hand 0, at every table
    ag.new_games(np.arange(T), seats, np.zeros(T, np.int32))
    lb, player = np.full(T, -1), np.zeros(T, np.int64)
    seen = np.zeros(T, np.int64)
    running = np.ones(T, bool)
    subs = []                                                     # (root last bid, root player, beliefs, act_iteration, policy)
    root_rows = root_actions = None
    while running.any():
        ids = np.flatnonzero(running)
        pol = ag.policy(ids).numpy()
        st = ag.state(ids)
        for k, t in enumerate(ids):
            if st["subgames"][k] > seen[t]:                       # policy() solved a new subgame at this node
                seen[t] = int(st["subgames"][k])
                subs.append((lb[t], player[t], st["root_beliefs"][k].numpy(), int(st["act_iteration"][k]), pol[k]))
        acts = np.array([-1 if player[t] == seats[t] else rng.choice(legal_actions(lb[t], A)) for t in ids], np.int32)
        played, probs, _ = ag.step(ids, acts)
        played, probs = played.numpy(), probs.numpy()
        if root_rows is None:
            root_rows, root_actions = pol[:, 0], played
            assert np.array_equal(probs, root_rows)
        for k, t in enumerate(ids):
            lb[t], player[t] = played[k], player[t] ^ 1
            running[t] = played[k] != A - 1
    assert ag.counts()["solves"] == len(subs) > T
    acts = np.array([s[3] for s in subs])
    assert (acts >= 0).all() and (acts < iters).all() and (acts % 2 == 0).all()
    p = even_iteration_probs(iters)
    bins = np.arange(0, iters + 1, 16)
    exp = np.array([p[lo:hi].sum() for lo, hi in zip(bins[:-1], bins[1:])]) * len(acts)
    assert chisquare(np.histogram(acts, bins)[0], exp).pvalue > 1e-3
    # re-solve every recorded subgame alone: the root node's snapshot is the policy at that root
    S = capi.WaveSolver(D, F, len(subs), max_depth=2, num_iters=iters, linear_update=True, net_mode=3, solver=capi.SOLVER_CFR)
    S.set_weights(w)
    S.begin(np.array([s[0] for s in subs], np.int32), np.array([s[1] for s in subs], np.int32), np.stack([s[2] for s in subs]),
            acts.astype(np.int32))
    S.run(iters)
    snap = S.fetch_compact("snapshot")
    for i, (root_lb, root_player, _, _, pol) in enumerate(subs):
        tmpl = S.tree(root_lb, root_player)
        lo = 0 if root_lb < 0 else root_lb + 1
        for child in range(tmpl[0, 2], tmpl[0, 3]):
            a = lo + child - tmpl[0, 2]
            assert np.array_equal(pol[:, a], snap[i, (child - 1) * H:child * H]), (i, a)
    S.close()
    # the agent's first actions (root, hand 0) against the mean of its tables' policy rows
    expected = root_rows.sum(0)
    obs = np.bincount(root_actions, minlength=A).astype(np.float64)
    big = expected >= 5
    e = np.append(expected[big], expected[~big].sum()) if (~big).any() else expected[big]
    o = np.append(obs[big], obs[~big].sum()) if (~big).any() else obs[big]
    assert obs[expected == 0].sum() == 0 and big.sum() >= 2
    assert chisquare(o[e > 0], e[e > 0]).pvalue > 1e-3
    ag.close()


def serve(rela, cfg, w, G, how, seed=3):
    """G keyed games (the agent in seat g % 2, opponent moves from a per-game stream) served `how`: every running table in each
    call ('all'), random subsets in shuffled order on permuted tables ('subsets'), or one table per call ('single').  Returns
    every game's log of (action, probs, root beliefs, act_iteration) after each step."""
    ag = rela.Agent(cfg, 0, G, "sampled", seed=seed, flat_weights=w)
    H, A = ag.num_hands, ag.num_actions
    deal = np.random.RandomState(100)
    hands = deal.randint(0, H, size=G)
    seats = np.arange(G) % 2
    rng = np.random.RandomState(200)
    table = rng.permutation(G) if how == "subsets" else np.arange(G)
    if how == "single":
        for g in range(G):
            ag.new_games([table[g]], [seats[g]], [hands[g]], keys=[g])
    else:
        ag.new_games(table, seats, hands, keys=np.arange(G))
    opp = [np.random.RandomState(1000 + g) for g in range(G)]
    lb, player = np.full(G, -1), np.zeros(G, np.int64)
    running = np.ones(G, bool)
    logs = [[] for _ in range(G)]
    while running.any():
        live = np.flatnonzero(running)
        if how == "all":
            batches = [live]
        elif how == "single":
            batches = [[g] for g in live]
        else:
            live = rng.permutation(live)
            batches = [live[:max(1, rng.randint(1, len(live) + 1))]]
        for games in batches:
            games = np.asarray(games)
            acts = np.array([-1 if player[g] == seats[g] else opp[g].choice(legal_actions(lb[g], A)) for g in games], np.int32)
            played, probs, done = ag.step(table[games], acts)
            st = ag.state(table[games])
            for k, g in enumerate(games):
                a = int(played[k])
                logs[g].append((a, probs[k].numpy().tobytes(), st["root_beliefs"][k].numpy().tobytes(), int(st["act_iteration"][k])))
                lb[g], player[g] = a, player[g] ^ 1
                running[g] = not bool(done[k])
    counts = ag.counts()
    ag.close()
    return logs, counts["solves"]


@pytest.mark.gpu
def test_gpu_results_do_not_depend_on_the_batch(rela):
    D, F, G = 2, 3, 96
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 64, True, 3)
    ref, solves = serve(rela, cfg, w, G, "all")
    assert sum(len(l) for l in ref) > 2 * G
    for how in ("subsets", "single"):
        logs, s = serve(rela, cfg, w, G, how)
        assert s == solves
        for g in range(G):
            assert logs[g] == ref[g], (how, g)


@pytest.mark.gpu
def test_gpu_agent_against_agent_matches_exact_ev(rela):
    """Two rela.Agents play 2^15 games through the API (seats swapped in pairs, shared deals); the mean payoff is the exact EV of
    their recursive strategies."""
    from rebel_b200.play import bidder_wins
    D, F, iters = 1, 4, 64
    wa = torch.from_numpy(net(D, F, 0))
    ca, cb = make_cfg(rela, D, F, iters, True, 3), make_cfg(rela, D, F, iters, True, 0)
    ev0, ev1 = rela.ev_of_strategies(D, F, rela.strategy_recursive_to_leaf(ca, 0, wa), rela.strategy_recursive_to_leaf(cb, 0))
    games, T = 1 << 15, 8192
    agents = [rela.Agent(ca, 0, T, "average", seed=1, flat_weights=wa), rela.Agent(cb, 0, T, "average", seed=2)]
    H, A = agents[0].num_hands, agents[0].num_actions
    deal = np.random.RandomState(17)
    payoff = np.zeros(games, np.float32)
    ids = np.arange(T)
    for base in range(0, games, T):
        g = base + ids
        hands = np.repeat(deal.randint(0, H, size=(T // 2, 2)), 2, axis=0)      # games 2i, 2i+1 share the deal
        seat_a = g & 1                                                           # agent A sits in seat 0 in even games
        agents[0].new_games(ids, seat_a, hands[ids, seat_a], keys=g)
        agents[1].new_games(ids, 1 - seat_a, hands[ids, 1 - seat_a], keys=g)
        lb, player = np.full(T, -1), np.zeros(T, np.int64)
        running = np.ones(T, bool)
        while running.any():
            live = np.flatnonzero(running)
            mover = (player[live] != seat_a[live]).astype(np.int64)             # 0: agent A moves
            acts = np.zeros(len(live), np.int32)
            for k in range(2):
                mine = live[mover == k]
                if len(mine):
                    acts[mover == k] = agents[k].step(mine, np.full(len(mine), -1, np.int32))[0].numpy()
            for k in range(2):
                theirs = mover == 1 - k
                if theirs.any():
                    agents[k].step(live[theirs], acts[theirs])
            for i, t in enumerate(live):
                if acts[i] == A - 1:
                    caller = player[t]
                    winner = caller ^ 1 if bidder_wins(lb[t], hands[t, 0], hands[t, 1], D, F) else caller
                    payoff[base + t] = 1.0 if winner == seat_a[t] else -1.0
                    running[t] = False
                lb[t], player[t] = acts[i], player[t] ^ 1
    for ag in agents:
        ag.close()
    s = rela.match_stats(torch.from_numpy(payoff))
    assert (payoff != 0).all() and s["stderr"] <= 0.01
    assert abs(s["mean"] - (ev0 + ev1) / 2) <= 4 * s["stderr"], (s["mean"], ev0, ev1, s["stderr"])


def snapshot(ag, T):
    return {k: v.clone() for k, v in ag.state(np.arange(T)).items()}


def same_state(a, b):
    return all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.gpu
def test_gpu_validation(rela):
    from rebel_b200 import capi
    T = 8
    ag = rela.Agent(make_cfg(rela, 1, 4, 16), 0, T, "sampled")
    H, A = ag.num_hands, ag.num_actions
    ag.new_games([0, 1, 2, 3], [0, 1, 0, 1], [0, 1, 2, 3])
    ag.step([0, 3], [-1, 4])                                      # table 0: the agent's bid; table 3: the opponent's bid 4
    before = snapshot(ag, T)
    bad = [
        ("new_games", ([0, T], [0, 0], [0, 0]), f"table {T}: id out of range"),
        ("new_games", ([5, 5], [0, 0], [0, 0]), "table 5: listed twice"),
        ("new_games", ([0, 6], [0, 0], [1, H]), "table 6: hand"),
        ("new_games", ([0, 6], [0, 2], [1, 1]), "table 6: seat"),
        ("step", ([2, -1], [-1, 0]), "table -1: id out of range"),
        ("step", ([2, 2], [-1, -1]), "table 2: listed twice"),
        ("step", ([2, 6], [-1, -1]), "table 6: no running game"),
        ("step", ([2, 1], [-1, A - 1]), "table 1: illegal action: liar call before any bid"),
        ("step", ([2, 1], [-1, -1]), "table 1: -1 .* opponent's turn"),
        ("step", ([2, 3], [-1, 4]), "table 3: illegal action 4: not above the last bid"),
        ("step", ([2, 3], [-1, A]), "table 3: action"),
        ("policy", ([2, 7],), "table 7: no running game"),
    ]
    for fn, args, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            getattr(ag, fn)(*args)
        assert same_state(before, snapshot(ag, T)), (fn, args)
    assert ag.counts()["solves"] == 2                            # tables 0 and 3 at the game root
    ag.close()
    # the C ABI directly, on WaveSolver handles
    L = capi.lib()
    L.cfrb_agent_create.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_uint64, ctypes.c_int32, ctypes.POINTER(ctypes.c_void_p)]
    L.cfrb_agent_destroy.argtypes = [ctypes.c_void_p]
    small = capi.WaveSolver(1, 4, 16, num_iters=16, net_mode=0)
    out = ctypes.c_void_p()
    assert L.cfrb_agent_create(small._h, 32, 0, capi.MATCH_AVERAGE, ctypes.byref(out)) == -1
    assert "capacity" in L.cfrb_last_error().decode() and not out
    a, b = capi.WaveSolver(1, 4, 64, num_iters=16, net_mode=0), capi.WaveSolver(1, 4, 64, num_iters=16, net_mode=0)
    M = capi.Match(a, b, 32, 64)
    assert L.cfrb_agent_create(a._h, 32, 0, capi.MATCH_AVERAGE, ctypes.byref(out)) == -1
    assert "live match" in L.cfrb_last_error().decode()
    M.close()
    assert L.cfrb_agent_create(a._h, 32, 0, capi.MATCH_AVERAGE, ctypes.byref(out)) == 0 and out
    with pytest.raises(capi.CfrbError, match="live match"):        # the agent's handle serves only the agent
        capi.Match(a, b, 32, 64)
    assert L.cfrb_agent_destroy(out) == 0
    capi.Match(a, b, 32, 64).close()
    small.close(); a.close(); b.close()


@pytest.mark.gpu
def test_gpu_plays_a_game_the_full_tree_tools_refuse(rela):
    D, F, T = 2, 5, 1024
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 64, True, 3)
    with pytest.raises(RuntimeError, match="too large"):
        rela.strategy_recursive_to_leaf(cfg, 0, w)
    ag = rela.Agent(cfg, 0, T, "sampled", seed=2, flat_weights=w)
    H, A = ag.num_hands, ag.num_actions
    rng = np.random.RandomState(5)
    seats = np.arange(T) % 2
    hands = rng.randint(0, H, size=T)
    ag.new_games(np.arange(T), seats, hands)
    lb, player = np.full(T, -1), np.zeros(T, np.int64)
    running = np.ones(T, bool)
    rows = 0
    while running.any():
        ids = np.flatnonzero(running)
        pol = ag.policy(ids).numpy()
        acts = np.array([-1 if player[t] == seats[t] else rng.choice(legal_actions(lb[t], A)) for t in ids], np.int32)
        played, probs, done = ag.step(ids, acts)
        for k, t in enumerate(ids):
            legal = np.zeros(A, bool)
            legal[legal_actions(lb[t], A)] = True
            assert np.isfinite(pol[k]).all() and (pol[k][:, ~legal] == 0).all() and (pol[k] >= 0).all()
            assert np.abs(pol[k][:, legal].sum(1) - 1).max() < 1e-12
            if player[t] == seats[t]:
                assert np.array_equal(probs[k].numpy(), pol[k][hands[t]])
                rows += 1
            lb[t], player[t] = int(played[k]), player[t] ^ 1
            running[t] = not bool(done[k])
    st = ag.state(np.arange(T))
    assert (st["ply"].numpy() >= 2).all() and (st["ply"].numpy() <= A).all() and rows >= T
    assert ag.counts()["solves"] == int(st["subgames"].sum()) and ag.counts()["subgame_iters"] == 64 * ag.counts()["solves"]
    ag.close()


@pytest.mark.gpu
def test_gpu_cli_end_to_end(tmp_path):
    from rebel_b200.play import parse_play
    argv = ["--num_dice", "1", "--num_faces", "4", "--subgame_iters", "64", "--cfr", "--games", "2", "--seed", "3"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    stdin = "9 9\n1 1\nliar\nliar\nliar\n"                       # an illegal face first, then a bid and liar calls
    p = subprocess.run([sys.executable, "-m", "rebel_b200.play"] + argv, cwd=str(tmp_path), env=env, input=stdin,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    out = p.stdout
    assert out.count("your dice:") == 2 and "faces are 1..4" in out and "agent: " in out and out.count("reveal:") == 2
    lines = [l for l in out.split("\n") if l.startswith("PLAY ")]
    assert len(lines) == 1, out
    d = parse_play(lines[0])
    assert d["net"] == "zero" and d["games"] == 2 and d["agent_wins"] + d["human_wins"] == 2
