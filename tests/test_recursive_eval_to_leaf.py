"""recursive_eval's sampled evaluation walked on the device (cfrb_to_leaf_sampled, rela.recursive_eval_to_leaf,
`python -m rebel_b200.recursive_eval --device_walk`): its float32 sums, checkpoint exploitabilities and iteration count equal the
host walk's (rela.recursive_eval_sampled) bit for bit; its results do not depend on the wave capacity or the repeats per batch; on
2x5f and 5x2f its sampled strategy is each subgame's own solve at its drawn act_iteration; what would not fit is refused before
anything is allocated."""
import ctypes as C
import json
import math
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


def make_cfg(rela, D, F, iters, use_cfr=True, net_mode=0, max_depth=2, linear=True):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, max_depth, linear, use_cfr
    return cfg


def net(D, F, seed):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    return flatten_state_dict(make_selfplay_net(D, F, seed=seed).state_dict())


def full_tree(D, F):
    """The full game tree, rows (last_bid, player_id, children_begin, children_end, parent, depth) in BFS order."""
    from rebel_b200 import capi
    A = 2 * D * F + 1
    out = np.zeros(((1 << A) - 1, 6), np.int32)
    n = capi._check(capi.lib().cfrb_unroll_tree(D, F, -1, 0, 1 << 30, out.ctypes.data_as(C.POINTER(C.c_int32)), out.shape[0]))
    assert n == out.shape[0]
    return out


def recursion_order(tree, A, md):
    """The subgame roots in the order RecursiveEvaluator::visit (compute_strategy_recursive_to_leaf's recursion) creates them."""
    order, stack = [], [0]
    while stack:
        root = stack.pop()
        order.append(root)
        level, kids = [root], []
        for _ in range(md):                      # BFS to depth md: the pseudo-leaves in BFS order
            level = [c for n in level for c in range(tree[n, 2], tree[n, 3])]
        kids = [c for c in level if tree[c, 0] != A - 1]
        stack.extend(reversed(kids))
    return order


def expected_bytes(D, F, md, K, B):
    """cfrb_to_leaf_sampled_bytes by hand: the average walk's full tree, best-response scratch and template map, then two levels
    of roots, fp64 beliefs and reach for B repeats, the two float32 accumulators and B repeats' draws."""
    from rebel_b200 import capi
    A, H = 2 * D * F + 1, F ** D
    N, T = 2 ** A - 1, 2 ** (A - 1) - 1
    tree = 4 * (5 * N + (A + 2) + 3 * T) + 8 * (2 * (N - 1) * H + 2 * (3 * N * H + 10 * T) + 2)
    nmax = capi.unroll_tree(D, F, -1, 0, md).shape[0]
    depths = range(0, A, md)
    level = max(math.comb(A - 1, d) for d in depths)
    roots = sum(math.comb(A - 1, d) for d in depths)
    return tree + 4 * K * nmax + 2 * level * B * (4 + 32 * H) + 4 * ((N - 1) * H + N * H) + 4 * B * roots


# ------------------------------------------------------------------------------------------------ CPU
def test_parser_accepts_device_walk():
    from rebel_b200.recursive_eval import build_parser
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "5", "--device_walk", "--batch_repeats", "2"])
    assert a.device_walk and a.batch_repeats == 2
    d = build_parser().parse_args([])
    assert not d.device_walk and d.batch_repeats is None


@pytest.mark.parametrize("argv,match", [
    (["--num_dice", "2", "--num_faces", "5", "--print_regret", "--cfr"], "dense regret sums .*8.8 GB at 2x5f"),
    (["--num_dice", "1", "--num_faces", "4", "--print_regret_summary", "--cfr", "--device_walk"], "does not track regrets"),
])
def test_cli_refuses_regrets_on_the_device_walk_before_device_work(argv, match):
    from rebel_b200.recursive_eval import main
    with pytest.raises(SystemExit, match=match):
        main(argv + ["--num_repeats", "2"])


def test_cli_refuses_several_ranks_on_the_device_walk(monkeypatch):
    from rebel_b200.recursive_eval import main
    monkeypatch.setenv("WORLD_SIZE", "2")
    for argv in (["--num_dice", "1", "--num_faces", "4", "--device_walk"], ["--num_dice", "2", "--num_faces", "5"]):
        with pytest.raises(SystemExit, match="one GPU"):
            main(argv + ["--num_repeats", "2"])


@pytest.mark.parametrize("D,F,md,K,B", [(1, 4, 2, 16384, 1), (1, 4, 3, 7, 5), (2, 3, 2, 100, 3), (2, 5, 2, 16384, 1),
                                        (2, 5, 2, 2048, 4), (5, 2, 2, 16384, 2), (1, 11, 2, 16384, 1), (2, 6, 2, 16384, 1)])
def test_sampled_bytes_by_hand(D, F, md, K, B):
    from rebel_b200 import capi
    assert capi.to_leaf_sampled_bytes(D, F, md, K, B) == expected_bytes(D, F, md, K, B)


def test_sampled_bytes_sizes():
    from rebel_b200 import capi
    assert capi.to_leaf_sampled_bytes(2, 5, 2, 16384, 1) < 5e9
    assert capi.to_leaf_sampled_bytes(2, 6, 2, 16384, 1) > 80e9        # more than an H100 holds: refused on the device
    with pytest.raises(capi.CfrbError, match="full tree too large"):
        capi.to_leaf_sampled_bytes(2, 7, 2, 16384, 1)
    with pytest.raises(capi.CfrbError, match=">= 1"):
        capi.to_leaf_sampled_bytes(2, 5, 2, 16384, 0)


def test_more_than_23_actions_is_refused_before_a_device_is_touched(rela):
    with pytest.raises(RuntimeError, match="more than 23 actions .*A = 25"):
        rela.recursive_eval_to_leaf(make_cfg(rela, 2, 6, 64), 0, 2)
    from rebel_b200 import capi
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.to_leaf_recursion_order(1, 12, 2)


@pytest.mark.parametrize("D,F,md", [(1, 4, 2), (1, 4, 3), (2, 2, 1), (2, 3, 2), (1, 6, 2), (2, 4, 2)])
def test_recursion_order_to_level_order(D, F, md):
    """The map from recursion position (the order of a repeat's draws) to level position is a permutation whose levels hold the
    C(A - 1, l * md) non-terminal nodes of depth l * md, in full-tree node order; it is the reference recursion's order."""
    from rebel_b200 import capi
    A = 2 * D * F + 1
    pos, begin = capi.to_leaf_recursion_order(D, F, md)
    sizes = [math.comb(A - 1, d) for d in range(0, A, md)]
    assert np.array_equal(np.sort(pos), np.arange(sum(sizes)))
    assert np.diff(begin[:len(sizes) + 1]).tolist() == sizes and (begin[len(sizes):] == sum(sizes)).all()
    tree = full_tree(D, F)
    order = recursion_order(tree, A, md)
    by_level = sorted(order, key=lambda n: (tree[n, 5], n))
    assert [by_level[p] for p in pos] == order


def test_recursion_order_2x5f_size():
    from rebel_b200 import capi
    pos, begin = capi.to_leaf_recursion_order(2, 5, 2)
    assert pos.size == 2 ** 19 and np.array_equal(np.bincount(pos), np.ones(2 ** 19))
    assert np.diff(begin[:12]).tolist() == [math.comb(20, d) for d in range(0, 21, 2)]


# ------------------------------------------------------------------------------------------------ GPU
def edges_of_dense(tree, dense):
    """[N, H, A] -> [N - 1, H]: row c - 1 = the parent's entry for the action leading to node c."""
    return np.ascontiguousarray(dense[tree[1:, 4], :, tree[1:, 0]])


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def assert_same(host, dev, tree):
    ss = host["summed_strategy"].numpy()
    want = edges_of_dense(tree, ss)
    legal = np.zeros(ss.shape, bool)
    legal[tree[1:, 4], :, tree[1:, 0]] = True
    assert (ss[~legal] == 0).all()
    assert np.array_equal(bits(dev["summed_strategy"].numpy()), bits(want))
    assert np.array_equal(bits(dev["summed_reach"].numpy()), bits(host["summed_reach"].numpy()[:, :, 0]))
    assert dev["checkpoints"] == host["checkpoints"]
    assert np.array_equal(bits(dev["exploitability"].numpy()), bits(host["exploitability"].numpy()))
    assert dev["subgame_iters"] == host["subgame_iters"] and dev["subgames"] == host["subgames_solved"]


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,md", [(1, 4, 2), (1, 6, 2), (2, 3, 2), (2, 4, 2), (1, 4, 3)])
@pytest.mark.parametrize("use_cfr", [True, False])
@pytest.mark.parametrize("net_name", ["zero", "fp32", "tc_x2"])
def test_gpu_bit_for_bit_against_the_host_walk(rela, D, F, md, use_cfr, net_name):
    mode = {"zero": 0, "fp32": 1, "tc_x2": 3}[net_name]
    w = torch.from_numpy(net(D, F, 0)) if mode else None
    cfg = make_cfg(rela, D, F, 64, use_cfr, mode, md)
    host = rela.recursive_eval_sampled(cfg, 0, 5, seed=3, batch_repeats=2, wave_capacity=4096, flat_weights=w)
    dev = rela.recursive_eval_to_leaf(cfg, 0, 5, seed=3, flat_weights=w, wave_capacity=512, return_sums=True)
    assert dev["checkpoints"] == [1, 2, 4, 5] and dev["num_nodes"] == 2 ** (2 * D * F + 1) - 1
    assert_same(host, dev, full_tree(D, F))


@pytest.mark.gpu
@pytest.mark.parametrize("use_cfr", [True, False])
def test_gpu_no_linear_bit_for_bit(rela, use_cfr):
    D, F = 2, 3
    w = torch.from_numpy(net(D, F, 1))
    cfg = make_cfg(rela, D, F, 48, use_cfr, 3, 2, linear=False)
    host = rela.recursive_eval_sampled(cfg, 0, 3, seed=11, batch_repeats=64, wave_capacity=8192, flat_weights=w)
    dev = rela.recursive_eval_to_leaf(cfg, 0, 3, seed=11, flat_weights=w, batch_repeats=3, return_sums=True)
    assert_same(host, dev, full_tree(D, F))


@pytest.mark.gpu
def test_gpu_ev_of_full_matches_the_host_walk(rela):
    D, F = 1, 4
    cfg = make_cfg(rela, D, F, 64)
    cfg.subgame_params.max_depth = 100000
    full = rela.solve_full_tree(cfg, 0)["strategy"]
    cfg.subgame_params.max_depth = 2
    host = rela.recursive_eval_sampled(cfg, 0, 6, seed=0, full_strategy=full)
    dev = rela.recursive_eval_to_leaf(cfg, 0, 6, full_strategy=full)
    assert np.array_equal(bits(dev["ev_of_full"].numpy()), bits(host["ev_of_full"].numpy()))


def sampled_digest(rela, cfg, w, reps, K, B):
    r = rela.recursive_eval_to_leaf(cfg, 0, reps, seed=5, flat_weights=w, wave_capacity=K, batch_repeats=B, return_sums=True)
    return (r["checkpoints"], bits(r["exploitability"].numpy()).tolist(), r["subgame_iters"], r["subgames"],
            bits(r["summed_strategy"].numpy()).tobytes(), bits(r["summed_reach"].numpy()).tobytes())


@pytest.mark.gpu
def test_gpu_results_do_not_depend_on_capacity_or_batch_small(rela):
    D, F = 2, 3
    A = 2 * D * F + 1
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 32, True, 3)
    ref = sampled_digest(rela, cfg, w, 5, A - 1, 1)
    for K, B in ((16384, 64), (100, 3), (4096, 0)):
        assert sampled_digest(rela, cfg, w, 5, K, B) == ref, (K, B)


@pytest.mark.gpu
def test_gpu_results_do_not_depend_on_capacity_or_batch_2x5f(rela):
    D, F = 2, 5
    w = torch.from_numpy(net(D, F, 0))
    cfg = make_cfg(rela, D, F, 16, True, 3)
    ref = sampled_digest(rela, cfg, w, 3, 16384, 1)
    assert sampled_digest(rela, cfg, w, 3, 2048, 2) == ref


def root_beliefs(tree, last, node, md, H):
    """Beliefs at the root of the subgame at `node` under the sampled strategy `last` (compact): from the uniform game root,
    each edge multiplies its acting player's row, and every subgame boundary eps-normalises both rows (in the host walk's order)."""
    path = [node]
    while path[-1] != 0:
        path.append(int(tree[path[-1], 4]))
    path.reverse()
    b = [[1.0 / H] * H, [1.0 / H] * H]
    for q, c in zip(path, path[1:]):
        pl = int(tree[q, 1])
        b[pl] = [x * float(s) for x, s in zip(b[pl], last[c - 1])]
        if tree[c, 5] % md == 0:
            for row in range(2):
                tot = 0.0
                for x in b[row]:
                    tot += x + 1e-80
                b[row] = [(x + 1e-80) / tot for x in b[row]]
    return np.array(b)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,iters", [(2, 5, 64), (5, 2, 16)])
def test_gpu_large_game_roots_are_their_own_solves(D, F, iters):
    from rebel_b200 import capi
    A, H, md = 2 * D * F + 1, F ** D, 2
    w = net(D, F, 0)
    S = capi.WaveSolver(D, F, 16384, max_depth=md, num_iters=iters, net_mode=3)
    S.set_weights(w)
    r = S.to_leaf_sampled(1, seed=7)
    last, act = S.to_leaf_sampled_last()
    S.close()
    assert r["checkpoints"] == [1] and r["subgames"] == 2 ** (A - 2)
    assert np.isfinite(r["br"]).all() and 0 <= r["br"].sum() / 2 <= 1
    tree = full_tree(D, F)
    roots = np.nonzero(act >= 0)[0]
    assert roots.size == 2 ** (A - 2) and (tree[roots, 5] % md == 0).all() and r["subgame_iters"] == int(act[roots].sum())
    rng = np.random.RandomState(0)
    pick = [0] + [int(x) for d in (2, 4) for x in rng.choice(roots[tree[roots, 5] == d], 3, replace=False)]
    T = capi.WaveSolver(D, F, len(pick), max_depth=md, num_iters=iters, net_mode=3)
    T.set_weights(w)
    T.begin(tree[pick, 0], tree[pick, 1], np.stack([root_beliefs(tree, last, n, md, H) for n in pick]), act_iteration=act[pick])
    T.run(int(act[pick].max()))
    snap = T.fetch_compact("snapshot")
    T.close()
    for k, n in enumerate(pick):
        t = capi.unroll_tree(D, F, int(tree[n, 0]), int(tree[n, 1]), md)
        fid = np.zeros(t.shape[0], np.int64)
        fid[0] = n
        for c in range(1, t.shape[0]):
            q = t[c, 4]
            fid[c] = tree[fid[q], 2] + (c - t[q, 2])
        got = last[fid[1:] - 1]
        want = snap[k, :(t.shape[0] - 1) * H].reshape(-1, H)
        assert np.array_equal(bits(got), bits(want)), n


@pytest.mark.gpu
def test_gpu_refusals_give_the_memory_back():
    from rebel_b200 import capi
    D, F, K, iters = 1, 4, 64, 16
    before = torch.cuda.mem_get_info(0)[0]
    S = capi.WaveSolver(D, F, K, max_depth=2, num_iters=iters, net_mode=0)
    with pytest.raises(capi.CfrbError, match="cfrb error -4: .*no sampled walk"):
        S.to_leaf_sampled_sums()
    need = capi.to_leaf_sampled_bytes(D, F, 2, K, 4)
    S.debug_to_leaf_free_cap(need - 1)
    with pytest.raises(capi.CfrbError, match=f"cfrb error -5: .*needs {need} bytes .*{need - 1} free"):
        S.to_leaf_sampled(4, batch_repeats=4)
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*batch_repeats"):
        S.to_leaf_sampled(4, batch_repeats=K + 1)
    S.debug_to_leaf_free_cap(need)
    r = S.to_leaf_sampled(4, batch_repeats=4)
    assert r["checkpoints"] == [1, 2, 4]
    S.close()
    big = capi.WaveSolver(2, 6, 1, max_depth=2, num_iters=1, net_mode=0)   # A = 25: refused whatever the free memory
    with pytest.raises(capi.CfrbError, match="cfrb error -1: .*more than 23 actions"):
        big.to_leaf_sampled(1)
    big.close()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(0)[0] >= before - (64 << 20)


def run_cli(tmp_path, argv):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.recursive_eval"] + argv, cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stderr[-4000:]
    return p.stdout


TIMING = ("wall_s", "solver_s_max_over_ranks", "repeats_per_s")


def without_timing(out):
    lines = []
    for line in out.splitlines():
        if line.startswith("{"):
            d = json.loads(line)
            line = json.dumps({k: v for k, v in d.items() if k not in TIMING})
        lines.append(line)
    return lines


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_gpu_cli_device_walk_prints_the_same_report(tmp_path, D, F):
    argv = ["--num_dice", str(D), "--num_faces", str(F), "--num_repeats", "5", "--subgame_iters", "64", "--cfr"]
    host, dev = run_cli(tmp_path, argv), run_cli(tmp_path, argv + ["--device_walk"])
    assert "XXX " in host and "YYY " in host and "EV of full" in host
    assert without_timing(dev) == without_timing(host)


@pytest.mark.gpu
def test_gpu_cli_2x5f(tmp_path):
    out = run_cli(tmp_path, ["--num_dice", "2", "--num_faces", "5", "--num_repeats", "2", "--subgame_iters", "16", "--cfr",
                             "--random_net_seed", "0"])
    assert "no full-tree solve (the full tree has 2097151 nodes, more than 2^20)" in out
    assert "EV of full" not in out and "YYY" not in out
    lines = out.splitlines()
    assert any(l.startswith("    1: ") for l in lines) and any(l.startswith("    2: ") for l in lines)
    xxx = [l for l in lines if l.startswith("XXX")]
    assert len(xxx) == 1
    d = json.loads(xxx[0].split("XXX")[1])                     # scripts/eval_all.py's parse
    assert list(d) == ["net", "repeated toleaf 1", "repeated toleaf 2"]
    assert all(0 <= float(v) <= 1 for k, v in d.items() if k != "net")
