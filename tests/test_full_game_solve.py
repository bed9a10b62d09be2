"""The full-game solver spread over the whole GPU (cfrb_full_game_*, capi.FullGame, rela.solve_full_game, `solve_game`): its memory
need by hand, its refusals, its CLI, and on the GPU the bits of the one-CTA full-tree solve (rela.solve_full_tree) for every
solver variant, the golden 1x4f exploitability, and determinism, normalisation and convergence on the games only it can solve."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (use_cfr, linear_update, dcfr (alpha, beta, gamma) or None, optimistic)
VARIANTS = {
    "cfr_linear": (True, True, None, False),
    "cfr_plain": (True, False, None, False),
    "dcfr": (True, False, (1.5, 0.0, 2.0), False),
    "fp_linear": (False, True, None, False),
    "fp_plain": (False, False, None, False),
    "fp_optimistic": (False, True, None, True),
}


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def make_cfg(rela, D, F, iters, variant="cfr_linear"):
    use_cfr, linear, dcfr, optimistic = VARIANTS[variant]
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, 0, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.linear_update, sp.optimistic = iters, 100000, use_cfr, linear, optimistic
    if dcfr is not None:
        sp.dcfr, (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) = True, dcfr
    return cfg


def full_tree(D, F):
    """unroll_tree of the whole game: rows (last_bid, player_id, children_begin, children_end, parent, depth)."""
    from rebel_b200 import capi
    N = (1 << (2 * D * F + 1)) - 1
    out = np.zeros((N, 6), np.int32)
    n = capi._check(capi.lib().cfrb_unroll_tree(D, F, -1, 0, 1 << 30, out.ctypes.data_as(C.POINTER(C.c_int32)), N))
    assert n == N
    return out


def by_hand_bytes(D, F, solver):
    A, H = 2 * D * F + 1, F ** D
    N, T, levels = 2 ** A - 1, 2 ** (A - 1) - 1, A + 1
    tree = (5 * N + levels + 1 + 3 * T) * 4 + (2 * (N - 1) * H + 2 * (3 * N * H + 10 * T) + 2) * 8   # full tree, BR strategies + scratch
    tables = ((3 if solver == 0 else 2) * (N - 1) * H + 2 * N * H) * 8 + 4                           # edge and node tables, counter
    return tree + tables


# ------------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3), (2, 5), (5, 2), (1, 11)])
def test_full_game_bytes_by_hand(D, F):
    from rebel_b200 import capi
    for solver in (capi.SOLVER_CFR, capi.SOLVER_FP):
        assert capi.full_game_bytes(D, F, solver) == by_hand_bytes(D, F, solver), (D, F, solver)
    # one fp64 table [N][H]: about 0.42 GB at 2x5f, 0.54 GB at 5x2f, 0.74 GB at 1x11f
    A, H = 2 * D * F + 1, F ** D
    table = (2 ** A - 1) * H * 8
    assert capi.full_game_bytes(D, F, capi.SOLVER_CFR) - capi.full_game_bytes(D, F, capi.SOLVER_FP) == table - H * 8


def test_refuses_games_above_23_actions_before_any_device_work(rela):
    from rebel_b200 import capi
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.FullGame(2, 6)                                  # A = 25: refused before the device is looked at
    with pytest.raises(RuntimeError, match="more than 23 actions"):
        rela.solve_full_game(make_cfg(rela, 2, 6, 4), 0)
    with pytest.raises(capi.CfrbError, match="A > 26"):
        capi.full_game_bytes(3, 5)
    from rebel_b200.solve_game import main
    with pytest.raises(SystemExit, match="more than 23 actions"):
        main(["--num_dice", "2", "--num_faces", "6"])


def test_cli_accepts_the_recursive_eval_solver_flags(rela):
    from rebel_b200.solve_game import build_parser, make_cfg as cli_cfg
    a = build_parser().parse_args(["--num_dice", "2", "--num_faces", "5", "--subgame_iters", "1024", "--cfr", "--no_linear",
                                   "--dcfr", "1.5", "0", "2", "--optimistic", "--device", "0"])
    assert (a.num_dice, a.num_faces, a.subgame_iters, a.cfr, a.no_linear, a.optimistic) == (2, 5, 1024, True, True, True)
    sp = cli_cfg(rela, a).subgame_params
    assert sp.use_cfr and sp.dcfr and not sp.linear_update and (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) == (1.5, 0.0, 2.0)
    sp = cli_cfg(rela, build_parser().parse_args([])).subgame_params       # the reference's defaults: linear FP
    assert not sp.use_cfr and sp.linear_update and not sp.dcfr and sp.num_iters == 1024


# ------------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3), (2, 4)])
def test_gpu_bit_exact_against_the_one_cta_solver(rela, D, F, variant):
    iters = 64
    old = rela.solve_full_tree(make_cfg(rela, D, F, iters, variant), 0)
    new = rela.solve_full_game(make_cfg(rela, D, F, iters, variant), 0)
    assert new["checkpoints"] == old["checkpoints"] == [1, 2, 4, 8, 16, 32, 64]
    assert torch.equal(new["exploitability"], old["exploitability"])
    t = full_tree(D, F)
    dense = old["strategy"].numpy()
    expect = dense[t[1:, 4], :, t[1:, 0]]                    # (parent, hand, action into child) of every edge = child - 1
    assert np.array_equal(new["strategy"].numpy(), expect)


@pytest.mark.gpu
def test_gpu_golden_full_tree_1x4f(golden):
    """1024 linear-CFR iterations of 1x4f: the golden exploitabilities at 16 and 1024 iterations (5.7674e-04) bit for bit."""
    from rebel_b200 import capi
    g = golden("fulltree.npz")
    s = capi.FullGame(1, 4)
    s.step(16)
    assert np.array_equal(s.exploitability(), g["expl_1x4_nofma"][0])
    s.step(1008)
    e = s.exploitability()
    assert s.iterations == 1024 and np.array_equal(e, g["expl_1x4_nofma"][1])
    assert abs(e.mean() - 5.7674e-04) < 5e-9
    s.close()


@pytest.mark.gpu
def test_gpu_refuses_a_request_above_the_free_memory():
    from rebel_b200 import capi
    need = capi.full_game_bytes(1, 4)
    capi._check(capi.lib().cfrb_debug_full_game_free_cap(need - 1))
    try:
        with pytest.raises(capi.CfrbError, match=f"needs {need} bytes"):
            capi.FullGame(1, 4)
    finally:
        capi._check(capi.lib().cfrb_debug_full_game_free_cap(0))
    capi.FullGame(1, 4).close()


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(2, 5), (5, 2), (1, 11)])
def test_gpu_large_games(rela, D, F):
    from rebel_b200 import capi
    iters = 64
    a = rela.solve_full_game(make_cfg(rela, D, F, iters), 0)
    b = rela.solve_full_game(make_cfg(rela, D, F, iters), 0)
    assert torch.equal(a["exploitability"], b["exploitability"]) and torch.equal(a["strategy"], b["strategy"])
    e = a["exploitability"].mean(1)
    assert a["checkpoints"][-1] == iters and e[-1] < e[0], e
    t = full_tree(D, F)
    inner = np.nonzero(t[:, 3] > t[:, 2])[0]
    sums = np.add.reduceat(a["strategy"].numpy(), t[inner, 2] - 1, axis=0)   # children of a node are contiguous edges
    assert np.abs(sums - 1).max() < 1e-12
    total, handle = a["device_bytes"], a["handle_bytes"]
    assert 0 < total - handle <= capi.full_game_bytes(D, F) + (64 << 20), (total, handle)


@pytest.mark.gpu
def test_gpu_checkpoint_matches_the_dense_best_response_2x4f(rela):
    """The solver's own best responses (br_kernel on the compact strategy) against exploitability_of_strategy of its strategy
    expanded to dense [N, H, A]."""
    D, F = 2, 4
    A, H = 2 * D * F + 1, F ** D
    r = rela.solve_full_game(make_cfg(rela, D, F, 32), 0)
    t = full_tree(D, F)
    dense = np.zeros((len(t), H, A))
    dense[t[1:, 4], :, t[1:, 0]] = r["strategy"].numpy()
    e = rela.exploitability_of_strategy(D, F, torch.from_numpy(dense))
    assert np.array_equal(np.array(e), r["exploitability"][-1].numpy())


@pytest.mark.gpu
def test_gpu_cli_end_to_end(tmp_path, golden):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.run([sys.executable, "-m", "rebel_b200.solve_game", "--num_dice", "1", "--num_faces", "4", "--subgame_iters",
                        "1024", "--cfr"], cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr
    lines = p.stdout.splitlines()
    assert sum(l.startswith("Iter=") for l in lines) == 11
    assert lines[-2].startswith("Iter=    1024 exploitabilities=(")
    s = json.loads(lines[-1][len("SOLVE "):])
    g = golden("fulltree.npz")
    assert s["br"] == g["expl_1x4_nofma"][1].tolist() and s["solver"] == "cfr" and s["linear"] and s["num_nodes"] == 511
    assert s["peak_device_bytes"] > 0 and s["seconds"] >= s["solve_seconds"] + s["br_seconds"]
