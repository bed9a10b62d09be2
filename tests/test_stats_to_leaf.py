"""compute_stats_with_net without dense full-tree tables: the FP subtree forest (cfrb_fp_forest_*, capi.FpForest) against one-subgame
wave solves bit for bit, its reach statistics against strategy_reach, compute_stats_with_net(device_walk=True) against the dense
path (the same floats and printed lines), the games only the device path serves, and training runs that evaluate them."""
import ctypes as C
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


def full_tree(D, F):
    """unroll_tree of the whole game: rows (last_bid, player_id, children_begin, children_end, parent, depth)."""
    from rebel_b200 import capi
    N = (1 << (2 * D * F + 1)) - 1
    out = np.zeros((N, 6), np.int32)
    assert capi._check(capi.lib().cfrb_unroll_tree(D, F, -1, 0, 1 << 30, out.ctypes.data_as(C.POINTER(C.c_int32)), N)) == N
    return out


def by_hand_bytes(D, F):
    """cfrb_full_game_bytes(FP) and the roots' beliefs and means [level][2][H] of the largest depth level."""
    from math import comb
    A, H = 2 * D * F + 1, F ** D
    N, T, levels = 2 ** A - 1, 2 ** (A - 1) - 1, A + 1
    tree = (5 * N + levels + 1 + 3 * T) * 4 + (2 * (N - 1) * H + 2 * (3 * N * H + 10 * T) + 2) * 8
    tables = (2 * (N - 1) * H + 2 * N * H) * 8 + 4
    level = max([A - 1] + [comb(A, d) for d in range(2, A + 1)])
    return tree + tables + 2 * level * 2 * H * 8


def stats_cfg(rela, D, F, iters, mdp_depth=2, use_cfr=True, net_mode=1):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, mdp_depth, True, use_cfr
    return cfg


# ---------------------------------------------------------------------------------------------------------------- CPU tier
@pytest.mark.parametrize("D,F", [(1, 4), (2, 4), (3, 3), (2, 5), (5, 2), (1, 10), (1, 11)])
def test_forest_bytes_by_hand(D, F):
    from rebel_b200 import capi
    assert capi.fp_forest_bytes(D, F) == by_hand_bytes(D, F)


def test_forest_refusals_without_a_device():
    from rebel_b200 import capi
    D, F, H = 1, 4, 4
    t = full_tree(D, F)
    A = 2 * D * F + 1
    at2 = [n for n in range(len(t)) if t[n, 5] == 2 and t[n, 0] != A - 1]
    term2 = [n for n in range(len(t)) if t[n, 5] == 2 and t[n, 0] == A - 1]
    b = lambda n: np.full((n, 2, H), 1.0 / H)
    capi.fp_forest_check(D, F, 2, at2[:3], b(3), 4)   # accepted
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.fp_forest_bytes(2, 6)
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.fp_forest_check(2, 6, 2, [100], np.full((1, 2, 36), 1 / 36), 4)
    bad = [
        (dict(depth=0), "depth"), (dict(depth=A), "depth"),
        (dict(nodes=[at2[1], at2[0], at2[2]]), "ascending"), (dict(nodes=[at2[0], at2[0], at2[2]]), "ascending"),
        (dict(nodes=[1, at2[0], at2[1]]), "not at depth"), (dict(nodes=[at2[0], at2[1], term2[0]] if term2[0] > at2[1] else None), "terminal"),
        (dict(nodes=[at2[0], at2[1], len(t)]), "out of range"),
        (dict(iters=0), "iters"),
    ]
    for kw, what in bad:
        if kw.get("nodes", 0) is None:
            continue
        a = dict(depth=2, nodes=at2[:3], beliefs=b(3), iters=4)
        a.update(kw)
        with pytest.raises(capi.CfrbError, match=what):
            capi.fp_forest_check(D, F, a["depth"], a["nodes"], a["beliefs"], a["iters"])
    for poison, what in ((-1e-3, "non-negative"), (np.nan, "finite"), (np.inf, "finite")):
        x = b(3)
        x[1, 0, 2] = poison
        with pytest.raises(capi.CfrbError, match=what):
            capi.fp_forest_check(D, F, 2, at2[:3], x, 4)
    x = b(3)
    x[2, 1] = 0
    with pytest.raises(capi.CfrbError, match="sums to zero"):
        capi.fp_forest_check(D, F, 2, at2[:3], x, 4)


def test_stats_device_walk_refuses_games_above_23_actions_before_any_device_work(rela):
    with pytest.raises(RuntimeError, match="more than 23 actions"):
        rela.compute_stats_with_net(stats_cfg(rela, 2, 6, 4), "/nonexistent.torchscript", device_walk=True)


# ---------------------------------------------------------------------------------------------------------------- GPU tier
def compact_reach(tree, H, s):
    """strategy_reach (rela/evaluation.h) of a compact strategy [N - 1, H]: both players' reach [2, N, H] and node_reach [N], every
    product and every hand-order sum the host's."""
    N = len(tree)
    r = np.zeros((2, N, H))
    r[:, 0] = 1.0 / H
    par, dep = tree[:, 4], tree[:, 5]
    for d in range(1, dep.max() + 1):
        c = np.nonzero(dep == d)[0]
        actor = (d - 1) & 1
        for p in range(2):
            r[p, c] = r[p, par[c]] * s[c - 1] if p == actor else r[p, par[c]]
    s0, s1 = np.zeros(N), np.zeros(N)
    for h in range(H):
        s0 = s0 + r[0, :, h]
        s1 = s1 + r[1, :, h]
    return r, s0 * s1


def wave_means(D, F, tree, nodes, beliefs, iters, max_depth=10000):
    from rebel_b200 import capi
    W = capi.WaveSolver(D, F, len(nodes), max_depth=max_depth, num_iters=iters, net_mode=capi.NET_ZERO, solver=capi.SOLVER_FP,
                        linear_update=True)
    W.begin(tree[nodes, 0].astype(np.int32), tree[nodes, 1].astype(np.int32), beliefs)
    W.run(iters)
    mu = W.fetch(("root_means",))["root_means"]
    W.close()
    return mu


def real_beliefs(D, F, tree, nodes, seed):
    """normalised reach rows of a real strategy (a few FP iterations of the full game), with some entries set to zero."""
    from rebel_b200 import capi
    g = capi.FullGame(D, F, solver=capi.SOLVER_FP)
    g.step(3)
    s = g.strategy()
    g.close()
    r, _ = compact_reach(tree, F ** D, s)
    b = np.transpose(r[:, nodes], (1, 0, 2)).copy()
    rng = np.random.RandomState(seed)
    zero = rng.rand(*b.shape) < 0.2
    zero[..., 0] = False   # every row keeps a positive entry
    zero[1::2] = False     # every other root without zeros: a zero belief makes FP's average strategy 0 / 0 there
    b[zero] = 0
    return b / b.sum(-1, keepdims=True)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3), (2, 4)])
def test_gpu_forest_bit_exact_against_wave_subgames(D, F):
    from rebel_b200 import capi
    tree = full_tree(D, F)
    A = 2 * D * F + 1
    f = capi.FpForest(D, F)
    iters_list = [1, 2, 7, 64] + ([1024] if (D, F) == (1, 4) else [])
    for depth in (1, 2, 3, 4):
        cand = np.nonzero((tree[:, 5] == depth) & (tree[:, 0] != A - 1))[0]
        nodes = cand[np.linspace(0, len(cand) - 1, min(len(cand), 12)).astype(int)]
        nodes = np.unique(nodes)
        b = real_beliefs(D, F, tree, nodes, seed=depth)
        for iters in iters_list:
            got = f.solve(depth, nodes, b, iters)
            want = wave_means(D, F, tree, nodes, b, iters)
            assert np.array_equal(got.view(np.int64), want.view(np.int64)), (D, F, depth, iters, np.abs(got - want).max())
            assert np.isfinite(got[1::2]).all()
        # a root's result does not depend on which other roots are listed
        sub = nodes[::3]
        part = f.solve(depth, sub, b[::3], 7)
        assert np.array_equal(part.view(np.int64), f.solve(depth, nodes, b, 7)[::3].view(np.int64))
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(2, 5), (5, 2), (1, 11)])
def test_gpu_forest_large_games_exact_on_small_subtrees(port, D, F):
    """Every root at depths 2 and 4 whose subtree depth A - 1 - last_bid is at most 8 against the C port's full-depth FP solve of
    that subgame (bit-identical to a wave subgame, tests/test_game_matrix.py); every other root finite."""
    from rebel_b200 import capi
    tree = full_tree(D, F)
    A, H = 2 * D * F + 1, F ** D
    f = capi.FpForest(D, F)
    rng = np.random.RandomState(D * 100 + F)
    iters = 16
    for depth in (2, 4):
        nodes = np.nonzero((tree[:, 5] == depth) & (tree[:, 0] != A - 1))[0]
        b = rng.rand(len(nodes), 2, H) + 0.01
        b /= b.sum(-1, keepdims=True)
        got = f.solve(depth, nodes, b, iters)
        assert np.isfinite(got).all()
        small = np.nonzero(A - 1 - tree[nodes, 0] <= 8)[0]
        assert len(small) > 0
        for i in small:
            lb, pl = int(tree[nodes[i], 0]), int(tree[nodes[i], 1])
            want = port.fp_solve(D, F, b[i], [iters], lb, pl, num_iters=iters, max_depth=A - 1 - lb)["root_means"][0]
            assert np.array_equal(got[i].view(np.int64), want.view(np.int64)), (D, F, depth, int(nodes[i]))
    f.close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3), (2, 4)])
def test_gpu_reach_statistics_equal_strategy_reach(D, F):
    from rebel_b200 import capi
    tree = full_tree(D, F)
    A, H = 2 * D * F + 1, F ** D
    W = capi.WaveSolver(D, F, 256, max_depth=2, num_iters=16, net_mode=capi.NET_ZERO)
    W.to_leaf_exploitability()
    net = W.to_leaf_strategy()
    W.close()
    g = capi.FullGame(D, F)
    g.step(16)
    full = g.strategy()
    g.close()
    nodes = np.nonzero(((tree[:, 5] == 2) | (tree[:, 5] == 4)) & (tree[:, 0] != A - 1))[0]
    nodes = np.concatenate([[0], nodes])
    f = capi.FpForest(D, F)
    for s in (net, full):
        r, node_reach = compact_reach(tree, H, s)
        nr, rows = f.reach(s, nodes)
        assert np.array_equal(nr.view(np.int64), node_reach[nodes].view(np.int64))
        assert np.array_equal(rows.view(np.int64), np.transpose(r[:, nodes], (1, 0, 2)).view(np.int64))
    f.close()


def _save_model(tmp_path, D, F, netname):
    from rebel_b200.models import make_selfplay_net
    net = make_selfplay_net(D, F, seed=0)
    if netname == "zero_out":
        with torch.no_grad():
            net.output.weight.zero_()
            net.output.bias.zero_()
    elif netname == "trained":
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_value_net_accuracy import trained_weights, unpack
        names = ["body.0.weight", "body.0.bias", "body.1.weight", "body.1.bias", "body.4.weight", "body.4.bias", "body.5.weight",
                 "body.5.bias", "output.weight", "output.bias"]   # the flat layout's order (flat_weights_of)
        sd = net.state_dict()
        for name, v in zip(names, unpack(trained_weights(D, F), D, F).values()):
            sd[name] = torch.as_tensor(v.astype(np.float32)).reshape(sd[name].shape)
        net.load_state_dict(sd)
    path = str(tmp_path / f"net_{D}x{F}_{netname}.torchscript")
    torch.jit.script(net).save(path)
    return path


def _stats(rela, capfd, cfg, path, device_walk):
    libc = C.CDLL(None)
    libc.fflush(None)
    capfd.readouterr()
    out = rela.compute_stats_with_net(cfg, path, device_walk=device_walk)
    libc.fflush(None)
    text = capfd.readouterr().out
    return out, [l for l in text.splitlines() if l.startswith(("eval_net", "  node", "Final MSE"))]


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3), (2, 4)])
def test_gpu_device_walk_equals_the_dense_path(rela, tmp_path, capfd, D, F):
    iters = {(1, 4): 32, (1, 6): 16, (2, 3): 8, (2, 4): 8}[(D, F)]
    cases = [(md, cfr, net) for md in (1, 2) for cfr in (True, False) for net in ("zero_out", "random")]
    if (D, F) == (2, 4):
        cases = [(2, True, "zero_out"), (1, False, "random")]
    if (D, F) == (1, 6):
        cases.append((2, True, "trained"))
    for md, cfr, netname in cases:
        path = _save_model(tmp_path, D, F, netname)
        cfg = stats_cfg(rela, D, F, iters, mdp_depth=md, use_cfr=cfr)
        dense, dl = _stats(rela, capfd, cfg, path, False)
        dev, vl = _stats(rela, capfd, cfg, path, True)
        assert np.array_equal(np.float32(dense), np.float32(dev)), (md, cfr, netname, dense, dev)
        assert dl == vl and len(dl) > 0, (md, cfr, netname)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(2, 5), (5, 2)])
def test_gpu_large_games(rela, tmp_path, monkeypatch, D, F):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    monkeypatch.setenv("CFRB_EVAL_NET_MODE", "3")
    path = _save_model(tmp_path, D, F, "random")
    cfg = stats_cfg(rela, D, F, 8, net_mode=3)
    first = rela.compute_stats_with_net(cfg, path)
    w = torch.as_tensor(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
    want = rela.exploitability_to_leaf(cfg, 0, w, 8192)["exploitability"]
    assert first[0] == np.float32(want)
    assert np.isfinite(first[1:]).all() and min(first[1:]) >= 0
    assert rela.compute_stats_with_net(cfg, path) == first


@pytest.mark.gpu
def test_gpu_forest_refuses_above_the_free_memory():
    from rebel_b200 import capi
    import torch.cuda
    free0 = torch.cuda.mem_get_info()[0]
    capi._check(capi.lib().cfrb_debug_full_game_free_cap(capi.fp_forest_bytes(2, 5) - 1))
    try:
        with pytest.raises(capi.CfrbError, match="needs"):
            capi.FpForest(2, 5)
    finally:
        capi._check(capi.lib().cfrb_debug_full_game_free_cap(0))
    assert torch.cuda.mem_get_info()[0] == free0


@pytest.mark.gpu
def test_gpu_training_2x5f_reports_evaluation_deterministically(rela, tmp_path, monkeypatch):
    from rebel_b200.train import parse_train
    env = dict(os.environ, CFRB_EVAL_NET_MODE="3")
    runs = []
    for k in range(2):
        out = tmp_path / f"run{k}"
        cmd = [sys.executable, "-m", "rebel_b200.train", "--num_dice", "2", "--num_faces", "5", "--out", str(out), "--max_epochs", "1",
               "--deterministic", "--exploit_every", "1", "--train_epoch_size", "1024", "--val_batches", "2", "--subgame_iters", "8",
               "--concurrent_games", "256"]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1200, env=env)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        lines = [parse_train(l) for l in r.stdout.splitlines() if l.startswith("TRAIN ")]
        assert lines and all(k in lines[0] for k in ("exploitability", "mse_net_reach", "mse_fp_reach"))
        runs.append([{k: v for k, v in m.items() if k != "minutes" and not k.endswith("_per_s")} for m in lines])
    assert runs[0] == runs[1]
    m = runs[0][0]
    monkeypatch.setenv("CFRB_EVAL_NET_MODE", "3")
    got = rela.compute_stats_with_net(stats_cfg(rela, 2, 5, 8, net_mode=3), str(tmp_path / "run0" / "epoch0.torchscript"))
    assert got == (np.float32(m["exploitability"]), np.float32(m["mse_net_reach"]), np.float32(m["mse_fp_reach"]))
