"""Local best response against ReBeL's every-node agent (cfrb_match_create_lbr2 with CFRB_MATCH_EVERY_NODE, rela.play_lbr's
policy="every_node", local_br --policy every_node): with the agent's strategy taken from rela.strategy_recursive, LBR's beliefs,
action values and decisions are test_local_br's host restatement bit for bit, and so is every belief the agent solves from; the
solve counts are the ones the traces imply; the payoff agrees with the exact EV of LBR's pure strategy, which never exceeds the
agent's exploitability; results do not depend on scheduling; games beyond 23 actions are played."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_local_br import check_lbr_traces, lbr_pure_strategy, make_cfg, matches_table, net, solver

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def normalize(b):
    """normalize_beliefs_inplace with the sum taken in sequential order."""
    s = 0.0
    for v in b.tolist():
        s += v + 1e-80
    return (b + 1e-80) / s


# ------------------------------------------------------------------------------------------------ CPU
def test_cli_parser_takes_every_node():
    from rebel_b200.local_br import build_parser
    assert build_parser().parse_args(["--policy", "every_node"]).policy == "every_node"
    assert build_parser().parse_args([]).policy == "average"


def test_lbr_line_policy_key_round_trips():
    from rebel_b200.local_br import lbr_line, parse_lbr
    plain = parse_lbr(lbr_line("a.ckpt", 1024, 0.125, 0.03125, [0.25, 0.0]))
    assert "policy" not in plain
    assert parse_lbr(lbr_line("a.ckpt", 1024, 0.125, 0.03125, [0.25, 0.0], "average")) == plain
    line = lbr_line("a.ckpt", 1024, 0.125, 0.03125, [0.25, 0.0], "every_node")
    assert line.startswith("LBR {") and line.endswith('"policy": "every_node"}')
    d = parse_lbr(line)
    assert d["policy"] == "every_node" and {k: v for k, v in d.items() if k != "policy"} == plain


def test_sampled_policy_is_still_refused_by_the_cli(capsys):
    from rebel_b200.local_br import SAMPLED_REFUSED, main
    with pytest.raises(SystemExit) as e:
        main(["--policy", "sampled"])
    assert e.value.code == 2 and SAMPLED_REFUSED in capsys.readouterr().err


# ------------------------------------------------------------------------------------------------ GPU
def check_every_node_rounds(M, tree, sigma, A, H, games):
    """The every-node walk's trace rounds: one per node where the agent solved a subgame it acts or updates from (its own plies,
    LBR's plies with a legal raise), with the agent's beliefs there equal to the host walk's (the mover's row times the agent's
    root row, eps-normalised, after every action); LBR's call after bid A - 2 carries the round before it.  Returns the solves
    and what-if solves the traces imply."""
    solves = whatif = 0
    for g in range(games):
        t = M.trace(g)
        me = g & 1
        bel = np.full((2, H), 1.0 / H)
        node, r = 0, 0
        if me == 0:
            solves += 1                                # the agent moves first: a solve at the game root
        for i, (who, lb, actor, hand, action, rr) in enumerate(t["plies"].tolist()):
            lo = 0 if lb < 0 else lb + 1
            m = A - 1 - lo                             # legal raises at this node
            solved = who == 0 or m > 0
            if who == 1 and m > 0:
                solves += 1 + m
                whatif += m
            if solved:
                assert rr == r, (g, i, rr, r)
                assert np.array_equal(t["root_beliefs"][r, 0], bel), (g, i)
                assert t["act_iteration"][r, 0] == -1, (g, i)
                r += 1
            else:
                assert who == 1 and action == A - 1 and rr == r - 1, (g, i)
            bel[actor] = normalize(bel[actor] * sigma[node, :, action])
            node = int(tree[node, 2]) + action - lo
        assert len(t["act_iteration"]) == r, g
    return solves, whatif


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
@pytest.mark.parametrize("depth", [1, 2, 3])
@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("net_name", ["zero", "fp32", "tc_x2"])
def test_gpu_every_node_lbr_decisions_bit_for_bit(rela, D, F, depth, use_cfr, net_name):
    from rebel_b200 import capi
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_name]
    w = net(D, F, 0) if mode else None
    iters = 64
    sigma = rela.strategy_recursive(make_cfg(rela, D, F, iters, use_cfr, mode, depth), 0,
                                    None if w is None else torch.from_numpy(w)).numpy()
    tree = capi.unroll_tree(D, F)
    N, H, A = sigma.shape
    S = solver(D, F, 256, iters, use_cfr, mode, w, max_depth=depth)
    games = 128
    M = capi.LbrMatch(S, 64, games, seed=3, policy=capi.MATCH_EVERY_NODE)
    res = M.play()
    assert set(np.unique(res["payoff_a"]).tolist()) <= {-1.0, 1.0}
    assert check_lbr_traces(M, tree, sigma, matches_table(D, F), D, F, games) >= games
    solves, whatif = check_every_node_rounds(M, tree, sigma, A, H, games)
    assert (res["solves"], res["whatif_solves"]) == (solves, whatif)
    assert res["subgame_iters"] == solves * iters and res["solves_a"] == solves and res["solves_b"] == 0
    M.close(); S.close()


@pytest.mark.gpu
def test_gpu_every_node_lbr_mean_matches_exact_ev_and_bounds_exploitability(rela):
    from rebel_b200 import capi
    D, F, iters = 1, 4, 64
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, iters, True, 3)
    sigma = rela.strategy_recursive(cfg, 0, w).numpy()
    s_lbr = lbr_pure_strategy(capi.unroll_tree(D, F), sigma, matches_table(D, F), D, F)
    ev0, ev1 = rela.ev_of_strategies(D, F, torch.from_numpy(s_lbr), torch.from_numpy(sigma))
    br0, br1 = rela.exploitability_of_strategy(D, F, torch.from_numpy(sigma))
    ev, expl = (ev0 + ev1) / 2, (br0 + br1) / 2
    assert ev <= expl + 1e-12, (ev, expl)
    r = rela.play_lbr(cfg, 0, 1 << 16, seed=5, flat_weights=w, policy="every_node")
    assert r["policy"] == "every_node"
    assert abs(r["mean"] - ev) <= 4 * r["stderr"], (r["mean"], ev, r["stderr"])
    assert torch.equal(r["payoff_lbr"].abs(), torch.ones(1 << 16))


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_gpu_every_node_lbr_results_do_not_depend_on_scheduling(rela, D, F):
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 64, True, 3)
    A = 2 * D * F + 1
    games = 1024
    kw = dict(seed=9, flat_weights=w, policy="every_node")
    runs = [rela.play_lbr(cfg, 0, games, concurrent_games=256, **kw),
            rela.play_lbr(cfg, 0, games, concurrent_games=4096, **kw),
            rela.play_lbr(cfg, 0, games, concurrent_games=512, max_subgames=A - 1, **kw)]
    assert runs[2]["max_subgames"] == A - 1 and runs[2]["deferred_slot_rounds"] > 0
    assert runs[0]["whatif_solves"] > 0
    for r in runs[1:]:
        assert torch.equal(runs[0]["payoff_lbr"], r["payoff_lbr"]) and torch.equal(runs[0]["plies"], r["plies"])
        assert (r["solves"], r["whatif_solves"]) == (runs[0]["solves"], runs[0]["whatif_solves"])


@pytest.mark.gpu
def test_gpu_every_node_lbr_plays_beyond_23_actions(rela):
    D, F, games = 2, 6, 256
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 64, True, 3)            # 36 hands: the wide tensor-core net
    with pytest.raises(RuntimeError, match="exploitability_recursive: .*more than 23 actions"):
        rela.exploitability_recursive(cfg, 0, w)
    r = rela.play_lbr(cfg, 0, games, seed=1, flat_weights=w, concurrent_games=256, policy="every_node")
    assert r["payoff_lbr"].shape == (games,) and set(r["payoff_lbr"].unique().tolist()) <= {-1.0, 1.0}
    assert (r["plies"] >= 1).all() and (r["plies"] <= 2 * D * F + 1).all()
    assert r["solves"] > r["whatif_solves"] > 0
    assert np.isfinite(r["stderr"]) and r["stderr"] > 0


@pytest.mark.gpu
def test_gpu_lbr2_validation_and_average_policy(rela):
    from rebel_b200 import capi
    L = capi.lib()
    a = solver(1, 4, 64, 16)
    m = C.c_void_p()
    for bad, msg in [(capi.MATCH_SAMPLED, "CFRB_MATCH_SAMPLED is not supported"), (3, "bad policy"), (-1, "bad policy")]:
        with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create_lbr2: " + msg):
            capi._check(L.cfrb_match_create_lbr2(a._h, 32, 64, 0, bad, C.byref(m)))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create_lbr2: null handle"):
        capi._check(L.cfrb_match_create_lbr2(None, 32, 64, 0, capi.MATCH_EVERY_NODE, C.byref(m)))
    with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create_lbr2: null argument"):
        capi._check(L.cfrb_match_create_lbr2(a._h, 32, 64, 0, capi.MATCH_EVERY_NODE, None))
    small = solver(1, 4, 7, 16)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: cfrb_match_create_lbr2: .*capacity"):
        capi.LbrMatch(small, 32, 64, policy=capi.MATCH_EVERY_NODE)
    small.close()
    cfg = make_cfg(rela, 1, 4, 16)
    for bad in ("sampled", "bogus"):
        with pytest.raises(RuntimeError, match="play_lbr: policy must be"):
            rela.play_lbr(cfg, 0, 64, policy=bad)
    assert rela.play_lbr(cfg, 0, 64)["policy"] == "average"
    # create_lbr2 with the average policy is create_lbr
    res = []
    for use2 in (False, True):
        M = capi.LbrMatch.__new__(capi.LbrMatch)
        M.a, M.b, M.G, M._m = a, None, 64, C.c_void_p()
        if use2:
            capi._check(L.cfrb_match_create_lbr2(a._h, 32, 64, 5, capi.MATCH_AVERAGE, C.byref(M._m)))
        else:
            capi._check(L.cfrb_match_create_lbr(a._h, 32, 64, 5, C.byref(M._m)))
        res.append(M.play())
        M.close()
    assert np.array_equal(res[0]["payoff_a"], res[1]["payoff_a"]) and np.array_equal(res[0]["plies"], res[1]["plies"])
    assert [res[0][k] for k in ("solves", "whatif_solves")] == [res[1][k] for k in ("solves", "whatif_solves")]
    a.close()


@pytest.mark.gpu
def test_gpu_every_node_cli_end_to_end(rela, tmp_path):
    from rebel_b200.head_to_head import agent_params
    from rebel_b200.local_br import build_parser, parse_lbr
    D, F, games = 1, 4, 1024
    argv = ["--num_dice", str(D), "--num_faces", str(F), "--random_net_seed", "0", "--games", str(games), "--subgame_iters", "32",
            "--cfr", "--seed", "4", "--policy", "every_node"]
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.local_br"] + argv, cwd=str(tmp_path), env=env, capture_output=True,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    out = [l for l in p.stdout.split("\n") if l]
    assert out[-1].startswith("LBR ") and "(every-node policy, depth 2)" in out[0], p.stdout
    d = parse_lbr(out[-1])
    assert d["policy"] == "every_node" and d["net"] == "random_net_seed=0" and d["games"] == games
    from rebel_b200.head_to_head import agent_weights
    w = agent_weights(D, F, None, 0)
    r = rela.play_lbr(agent_params(rela, build_parser().parse_args(argv), w, 32, True), 0, games, seed=4, flat_weights=w,
                      policy="every_node")
    assert d["mean"] == r["mean"] and d["stderr"] == r["stderr"] and json.loads(json.dumps(r["seat_means"])) == [d["seat0"], d["seat1"]]
