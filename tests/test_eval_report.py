"""recursive_eval's evaluation report beyond exploitability (recursive_eval.cc:270-425): compute_ev2 against the full-tree solve,
compute_immediate_regrets of the full solve's sampling strategies and of the sampled recursive strategies, the fictitious-play
sampled evaluation, and the tagged XXX / YYY lines that scripts/eval_all.py parses.  Fixture: tests/golden/ev_regrets.npz from
the compiled reference (oracle/make_golden_r3.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.ev_regret import EvRegretOracle
from oracle.make_golden_r3 import PAIRS, cfr_sampling_strategies, random_strategy, regret_summary
from oracle.oracle import game_dims

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


@pytest.fixture(scope="module")
def evport():
    """Plain-C restatement of compute_ev2 / compute_immediate_regrets (oracle/ev_regret_oracle.c)."""
    return EvRegretOracle("port")


def make_cfg(rela, D, F, iters, use_cfr=True, max_depth=2):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, 0, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, max_depth, True, use_cfr
    return cfg


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("D,F", [(1, 3), (1, 4)])
def test_port_ev2_matches_reference(port, evport, golden, D, F):
    g = golden("ev_regrets.npz")
    A, H, Q = game_dims(D, F)
    tree = port.unroll_tree(D, F)
    got = np.stack([evport.ev2(D, F, random_strategy(tree, H, A, a), random_strategy(tree, H, A, b)) for a, b in PAIRS])
    assert np.array_equal(got, g[f"ev_{D}x{F}"])
    assert abs(got[-1].sum()) < 1e-6      # a strategy against itself: zero-sum (subgame_solving_test.cc:227-244)


@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_port_immediate_regrets_of_full_solve_match_reference(port, evport, golden, D, F):
    g = golden("ev_regrets.npz")
    iters = {(int(d), int(f)): int(it) for d, f, it in g["full_iters"]}[(D, F)]
    strategies, _ = cfr_sampling_strategies(port, D, F, iters)
    assert np.array_equal(evport.immediate_regrets(D, F, strategies), g[f"full_regrets_{D}x{F}"])


def test_port_cfr_converges_in_immediate_regret(port, evport):
    """subgame_solving_test.cc:181-208: 1x2f, 4000 CFR iterations, immediate regret <= 1e-2 at every infoset."""
    strategies, _ = cfr_sampling_strategies(port, 1, 2, 4000)
    assert evport.immediate_regrets(1, 2, strategies).max() <= 1e-2


def test_cli_accepts_the_eval_all_command_line():
    """scripts/eval_all.py builds exactly this argument list (plus --cfr for CFR checkpoints)."""
    from rebel_b200.recursive_eval import build_parser
    argv = ["--net", "x.ckpt", "--mdp_depth", "2", "--num_faces", "4", "--num_dice", "1", "--subgame_iters", "1024",
            "--num_repeats", "1024", "--num_threads", "10"]
    for extra in ([], ["--cfr"]):
        a = build_parser().parse_args(argv + extra)
        assert (a.net, a.mdp_depth, a.num_faces, a.num_dice, a.subgame_iters, a.num_repeats, a.num_threads, a.cfr) == \
            ("x.ckpt", 2, 4, 1, 1024, 1024, 10, bool(extra))
    a = build_parser().parse_args(["--print_regret", "--print_regret_summary", "--net", "zero"])
    assert a.print_regret and a.print_regret_summary and a.net == "zero"
    with pytest.raises(SystemExit):
        build_parser().parse_args(["--root_only"])


def test_tagged_lines_round_trip_through_json():
    from rebel_b200.recursive_eval import tagged_line
    pairs = [("net", "/ckpt/1x4f_cfr_1000.ckpt"), ("full_tree", 0.0012345678), ("repeated toleaf 1", -0.25), ("repeated toleaf 2", 3.5e-7)]
    line = tagged_line("XXX", pairs)
    assert line.startswith('XXX {"net":"/ckpt/1x4f_cfr_1000.ckpt", "full_tree":"0.001235"')
    d = json.loads(line.split("XXX")[1])
    assert list(d) == [k for k, _ in pairs]
    assert d == {"net": "/ckpt/1x4f_cfr_1000.ckpt", "full_tree": "0.001235", "repeated toleaf 1": "-0.250000",
                 "repeated toleaf 2": "0.000000"}


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 3), (1, 4)])
def test_gpu_ev2_bit_exact(rela, golden, D, F):
    g = golden("ev_regrets.npz")
    from oracle.oracle import Oracle
    A, H, Q = game_dims(D, F)
    tree = Oracle("port").unroll_tree(D, F)
    got = np.array([rela.ev_of_strategies(D, F, torch.from_numpy(random_strategy(tree, H, A, a)), torch.from_numpy(random_strategy(tree, H, A, b)))
                    for a, b in PAIRS])
    assert np.array_equal(got, g[f"ev_{D}x{F}"])
    assert abs(got[-1].sum()) < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_gpu_full_solve_immediate_regrets_bit_exact(rela, golden, D, F):
    g = golden("ev_regrets.npz")
    iters = {(int(d), int(f)): int(it) for d, f, it in g["full_iters"]}[(D, F)]
    f = rela.solve_full_tree(make_cfg(rela, D, F, iters, max_depth=100000), 0, track_regrets=True)
    assert f["regret_count"] == iters // 2
    assert np.array_equal(f["immediate_regrets"].numpy(), g[f"full_regrets_{D}x{F}"])


@pytest.mark.gpu
def test_gpu_full_solve_converges_in_immediate_regret(rela):
    f = rela.solve_full_tree(make_cfg(rela, 1, 2, 4000, max_depth=100000), 0, track_regrets=True)
    assert f["immediate_regrets"].max().item() <= 1e-2


@pytest.mark.gpu
def test_gpu_regret_accumulator_is_batch_invariant(rela, port, evport):
    """Any split of the strategy list into batches gives the bits of the reference's single pass over it."""
    D, F = 1, 4
    A, H, Q = game_dims(D, F)
    tree = port.unroll_tree(D, F)
    s = np.stack([random_strategy(tree, H, A, 100 + i) for i in range(70)]).astype(np.float32)
    outs = [rela.immediate_regrets(D, F, torch.from_numpy(s), batch=b).numpy() for b in (1, 7, 64)]
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])
    assert np.array_equal(outs[0], evport.immediate_regrets(D, F, s.astype(np.float64)))


@pytest.mark.gpu
def test_gpu_recursive_eval_ev_and_regrets_bit_exact(rela, golden, port):
    g = golden("ev_regrets.npz")
    D, F, iters, reps, md = (int(x) for x in g["s5_cfg"])
    full = rela.solve_full_tree(make_cfg(rela, D, F, iters, max_depth=100000), 0)["strategy"]
    cfg = make_cfg(rela, D, F, iters, max_depth=md)
    plain = rela.recursive_eval_sampled(cfg, 0, reps, seed=0, batch_repeats=64, wave_capacity=4096)
    r = rela.recursive_eval_sampled(cfg, 0, reps, seed=0, batch_repeats=7, wave_capacity=4096, full_strategy=full, track_regrets=True)
    assert list(r["checkpoints"]) == list(g["s5_checkpoints"])
    assert np.array_equal(r["ev_of_full"].numpy(), g["s5_ev_of_full"])
    assert np.array_equal(r["regret_summary"].numpy(), g["s5_regret_summary"])
    assert np.array_equal(r["immediate_regrets"].numpy(), g["s5_immediate_regrets"])
    assert r["regret_count"] == reps
    tree = port.unroll_tree(D, F)
    assert tuple(r["regret_summary"][-1].tolist()) == regret_summary(g["s5_immediate_regrets"], tree, md)
    for k in ("summed_strategy", "summed_reach", "exploitability"):
        assert np.array_equal(r[k].numpy(), plain[k].numpy()), k


@pytest.mark.gpu
def test_gpu_fictitious_play_recursive_eval_bit_exact(rela, golden):
    g = golden("ev_regrets.npz")
    D, F, iters, reps, md = (int(x) for x in g["fp_cfg"])
    r = rela.recursive_eval_sampled(make_cfg(rela, D, F, iters, use_cfr=False, max_depth=md), 0, reps, seed=0, batch_repeats=64,
                                    wave_capacity=4096, track_regrets=True)
    assert list(r["checkpoints"]) == list(g["fp_checkpoints"])
    assert np.array_equal(r["summed_reach"].numpy(), g["fp_summed_reach"])
    assert np.array_equal(r["summed_strategy"].numpy(), g["fp_summed_strategy"])
    assert np.array_equal(r["exploitability"].numpy(), g["fp_exploitability"])
    assert "immediate_regrets" not in r          # the reference tracks regrets for CFR only


def _run_cli(args, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.recursive_eval"] + args, cwd=str(tmp_path), env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-4000:]
    return p.stdout


@pytest.mark.gpu
def test_gpu_cli_end_to_end_eval_all_command_line(rela, tmp_path):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, iters, reps = 1, 4, 64, 8
    net = make_selfplay_net(D, F, seed=0)
    path = str(tmp_path / "net.ckpt")
    torch.jit.save(torch.jit.script(net), path)
    out = _run_cli(["--net", path, "--mdp_depth", "2", "--num_faces", str(F), "--num_dice", str(D), "--subgame_iters", str(iters),
                    "--num_repeats", str(reps), "--num_threads", "10", "--cfr"], tmp_path)
    xxx = [l for l in out.split("\n") if "XXX" in l]
    yyy = [l for l in out.split("\n") if "YYY" in l]
    assert len(xxx) == 1 and len(yyy) == 1, out
    ex, ev = json.loads(xxx[0].split("XXX")[1]), json.loads(yyy[0].split("YYY")[1])
    names = ["net", "full_tree"] + [f"repeated toleaf {n}" for n in (1, 2, 4, 8)]
    assert list(ex) == names and list(ev) == names and ex["net"] == path
    # the same numbers through the API
    full = rela.solve_full_tree(make_cfg(rela, D, F, iters, max_depth=100000), 0)
    fe = full["exploitability"][-1].tolist()
    assert ex["full_tree"] == f"{(fe[0] + fe[1]) / 2:f}"
    cfg = make_cfg(rela, D, F, iters)
    cfg.net_mode = 3
    r = rela.recursive_eval_sampled(cfg, 0, reps, seed=0, flat_weights=torch.from_numpy(flatten_state_dict(net.state_dict())),
                                    full_strategy=full["strategy"])
    for i, n in enumerate(r["checkpoints"]):
        e, v = r["exploitability"][i].tolist(), r["ev_of_full"][i].tolist()
        assert ex[f"repeated toleaf {n}"] == f"{(e[0] + e[1]) / 2:f}"
        assert ev[f"repeated toleaf {n}"] == f"{(v[0] + v[1]) / 2:f}"
    out = _run_cli(["--net", "zero", "--mdp_depth", "2", "--num_faces", str(F), "--num_dice", str(D), "--subgame_iters", str(iters),
                    "--num_repeats", "4", "--cfr", "--print_regret_summary"], tmp_path)
    assert "Regrets (depth<=2)/rest:" in out and sum("XXX" in l for l in out.split("\n")) == 1
    assert json.loads([l for l in out.split("\n") if "XXX" in l][0].split("XXX")[1])["net"] == "zero"
