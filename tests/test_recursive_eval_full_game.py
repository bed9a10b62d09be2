"""`recursive_eval --full_game`: the full-game solve (rela.solve_full_game), the device walk with a compact EV baseline and the
immediate regrets of its sampled strategies (cfrb_to_leaf_sampled_ev_regrets, rela.recursive_eval_to_leaf(track_regrets=True)).
Without a GPU: the flag, the plan, the refusals and the byte count.  On the GPU: the bits of the host walk
(rela.recursive_eval_sampled with a dense baseline and track_regrets), the CLI's text against the host walk's and against the
default run, and the report on 2x5f."""
import json

import numpy as np
import pytest
import torch

from test_full_game_solve import full_tree
from test_recursive_eval_to_leaf import run_cli, without_timing


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def walk_cfg(rela, D, F, iters, md, net_mode=0):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.linear_update = iters, md, True, True
    return cfg


# ------------------------------------------------------------------------------------------------------------------------ CPU
def test_parser_and_plan_take_the_flag():
    from rebel_b200.recursive_eval import build_parser, device_walk_plan
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "5", "--full_game", "--cfr", "--print_regret_summary"])
    assert a.full_game and not build_parser().parse_args([]).full_game
    assert device_walk_plan(a, 1) == (True, None)
    small = build_parser().parse_args(["--num_dice", "1", "--num_faces", "4", "--full_game", "--print_regret"])
    assert device_walk_plan(small, 1) == (True, None)


@pytest.mark.parametrize("argv,env,match", [
    (["--num_dice", "1", "--num_faces", "4", "--full_game", "--no_full_tree"], {}, "does not go with --no_full_tree"),
    (["--num_dice", "2", "--num_faces", "6", "--full_game"], {}, "up to 23 actions .*A = 25"),
    (["--num_dice", "2", "--num_faces", "5", "--full_game"], {"WORLD_SIZE": "2"}, "one GPU"),
    (["--num_dice", "2", "--num_faces", "5", "--print_regret_summary", "--cfr"], {}, "8.8 GB at 2x5f.*--full_game does"),
])
def test_cli_refuses_before_device_work(monkeypatch, argv, env, match):
    from rebel_b200.recursive_eval import main
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    with pytest.raises(SystemExit, match=match):
        main(argv + ["--num_repeats", "2"])


@pytest.mark.parametrize("D,F,B", [(1, 4, 1), (2, 3, 3), (2, 5, 1), (5, 2, 2), (1, 11, 1)])
def test_walk_regret_bytes_by_hand(D, F, B):
    from rebel_b200 import capi
    A, H = 2 * D * F + 1, F ** D
    E = (2 ** A - 2) * H
    assert capi.to_leaf_sampled_regret_bytes(D, F, B) == E * 8 + B * E * 4


def test_walk_regret_bytes_refuse_2x6f():
    from rebel_b200 import capi
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.to_leaf_sampled_regret_bytes(2, 6, 1)


# ------------------------------------------------------------------------------------------------------------------------ GPU
def compact_of(dense, t):
    return dense[t[1:, 4], :, t[1:, 0]]


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,md,net", [(1, 4, 2, "zero"), (2, 3, 2, "tc"), (2, 4, 2, "zero"), (1, 4, 3, "tc")])
def test_gpu_walk_regrets_and_compact_ev_match_the_host_walk(rela, D, F, md, net):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    iters, reps, seed = 32, 5, 3
    sp_full = walk_cfg(rela, D, F, iters, 100000)
    dense = rela.solve_full_tree(sp_full, 0)["strategy"]
    compact = torch.from_numpy(compact_of(dense.numpy(), full_tree(D, F)))
    w = None if net == "zero" else torch.from_numpy(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
    cfg = walk_cfg(rela, D, F, iters, md, 0 if net == "zero" else 3)
    host = rela.recursive_eval_sampled(cfg, 0, reps, seed=seed, batch_repeats=64, wave_capacity=4096, flat_weights=w,
                                       full_strategy=dense, track_regrets=True)
    for B in (1, 3):
        dev = rela.recursive_eval_to_leaf(cfg, 0, reps, seed=seed, flat_weights=w, wave_capacity=4096, batch_repeats=B,
                                          full_strategy=compact, track_regrets=True)
        assert dev["checkpoints"] == list(host["checkpoints"])
        for k in ("exploitability", "ev_of_full", "regret_summary", "immediate_regrets"):
            assert torch.equal(dev[k], host[k]), (k, B)
        assert dev["regret_count"] == host["regret_count"] == reps
        t = full_tree(D, F)
        assert np.array_equal(dev["regret_sums_compact"].numpy(), compact_of(host["regret_sums"].numpy(), t))


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_gpu_cli_full_game_prints_the_host_walks_text(tmp_path, D, F):
    argv = ["--num_dice", str(D), "--num_faces", str(F), "--num_repeats", "5", "--subgame_iters", "64", "--cfr"]
    reg = ["--print_regret", "--print_regret_summary"]
    host = run_cli(tmp_path, argv + reg)
    full = run_cli(tmp_path, argv + reg + ["--full_game"])
    assert "Regrets: " in host and "Regrets (depth<=2)/rest" in host and "YYY " in host
    assert without_timing(full) == without_timing(host)
    assert without_timing(run_cli(tmp_path, argv + ["--full_game"])) == without_timing(run_cli(tmp_path, argv))


@pytest.mark.gpu
def test_gpu_cli_full_game_2x5f(tmp_path):
    out = run_cli(tmp_path, ["--num_dice", "2", "--num_faces", "5", "--full_game", "--num_repeats", "2", "--subgame_iters", "16",
                             "--cfr", "--random_net_seed", "0", "--print_regret_summary"])
    lines = out.splitlines()
    assert any(l.startswith("Iter=") for l in lines) and any(l.startswith("Full CFR exploitability") for l in lines)
    for n in (1, 2):
        i = next(i for i, l in enumerate(lines) if l.startswith(f"    {n}: "))
        assert lines[i + 1].startswith("\tEV of full: ") and "\tRegrets (depth<=2)/rest: " in lines[i + 1]
    assert sum(l.startswith("\tRegrets (depth<=2)/rest: ") for l in lines) >= 1       # the full solve's own line
    yyy = [l for l in lines if l.startswith("YYY")]
    assert len(yyy) == 1
    assert list(json.loads(yyy[0][len("YYY"):])) == ["net", "full_tree", "repeated toleaf 1", "repeated toleaf 2"]
    i = next(i for i, l in enumerate(lines) if l.startswith(" full_tree "))
    assert lines[i + 1].startswith("\tEV of full: 0.000000 (")
    ev0, ev1 = (float(x) for x in lines[i + 1].split("(")[1].rstrip(")").split(","))
    assert ev1 == -ev0


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(2, 5), (5, 2)])
def test_gpu_walk_regrets_large_games(rela, D, F):
    from rebel_b200 import capi
    full = rela.solve_full_game(walk_cfg(rela, D, F, 16, 100000), 0)["strategy"]
    cfg = walk_cfg(rela, D, F, 16, 2)
    runs = [rela.recursive_eval_to_leaf(cfg, 0, 2, seed=1, wave_capacity=16384, batch_repeats=B, full_strategy=full,
                                        track_regrets=True) for B in (1, 1, 2)]
    for r in runs[1:]:
        for k in ("exploitability", "ev_of_full", "regret_summary", "immediate_regrets", "regret_sums_compact"):
            assert torch.equal(r[k], runs[0][k]), k
    imm = runs[0]["immediate_regrets"]
    assert torch.isfinite(imm).all() and (imm >= 0).all() and imm.sum().item() > 0
    # refused before anything is allocated: the memory comes back
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info(0)[0]
    S = capi.WaveSolver(D, F, 16384, max_depth=2, num_iters=16, net_mode=0)
    need = capi.to_leaf_sampled_bytes(D, F, 2, 16384, 1) + capi.to_leaf_sampled_regret_bytes(D, F, 1)
    S.debug_to_leaf_free_cap(need - 1)
    with pytest.raises(capi.CfrbError, match=f"cfrb error -5: .*needs {need} bytes"):
        S.to_leaf_sampled_regrets(1)
    S.close()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(0)[0] >= before - (64 << 20)
