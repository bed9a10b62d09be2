"""Immediate regrets of the full-game solve on the whole GPU (cfrb_full_game_track_regrets / cfrb_full_game_regrets,
capi.FullGame.track_regrets, rela.solve_full_game(track_regrets=True)): the memory need by hand and the refusals, and on the GPU
the bits of the one-CTA full-tree solve's dense accumulator (rela.solve_full_tree(track_regrets=True)), the golden regrets of the
reference, and determinism, sign and memory on the games only the full-game solver reaches."""
import numpy as np
import pytest
import torch

from oracle.make_golden_r3 import regret_summary as reference_summary

from test_full_game_solve import full_tree, make_cfg

CFR_VARIANTS = ["cfr_linear", "cfr_plain", "dcfr"]


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def by_hand_regret_bytes(D, F):
    A, H = 2 * D * F + 1, F ** D
    return (2 ** A - 2) * H * 8            # compact fp64 sums [N - 1][H]


# ------------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3), (2, 5), (5, 2), (1, 11)])
def test_regret_bytes_by_hand(D, F):
    from rebel_b200 import capi
    assert capi.full_game_regret_bytes(D, F) == by_hand_regret_bytes(D, F)


def test_regret_bytes_refuse_games_above_23_actions():
    from rebel_b200 import capi
    with pytest.raises(capi.CfrbError, match="more than 23 actions"):
        capi.full_game_regret_bytes(2, 6)
    with pytest.raises(capi.CfrbError, match=">= 1"):
        capi.full_game_regret_bytes(0, 6)


def test_regret_bytes_at_2x5f_are_a_twentieth_of_the_dense_sums():
    from rebel_b200 import capi
    D, F = 2, 5
    A, H = 2 * D * F + 1, F ** D
    dense = (2 ** A - 1) * H * A * 8       # cfrb_regrets_reset's [N][H][A]: 8.8 GB
    compact = capi.full_game_regret_bytes(D, F)         # 419 MB
    assert 419e6 < compact < 420e6 and 20 * compact < dense


# ------------------------------------------------------------------------------------------------------------------------ GPU
def hand_order_sum(row):
    """Plain left-to-right float sum (Python's sum() compensates its float additions)."""
    s = 0.0
    for v in row.tolist():
        s += v
    return s


def gather_compact(dense_sums, t):
    """Dense [N, H, A] sums -> compact [N - 1, H]: the slot of the action into every child, edge = child - 1."""
    return dense_sums[t[1:, 4], :, t[1:, 0]]


@pytest.mark.gpu
@pytest.mark.parametrize("variant", CFR_VARIANTS)
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3), (2, 4)])
def test_gpu_bit_exact_against_the_dense_accumulator(rela, D, F, variant):
    iters, depth = 64, 2
    old = rela.solve_full_tree(make_cfg(rela, D, F, iters, variant), 0, track_regrets=True)
    new = rela.solve_full_game(make_cfg(rela, D, F, iters, variant), 0, track_regrets=True, regret_depth=depth)
    assert torch.equal(new["exploitability"], old["exploitability"])
    assert new["regret_count"] == old["regret_count"] == iters // 2
    assert torch.equal(new["immediate_regrets"], old["immediate_regrets"])
    t = full_tree(D, F)
    assert np.array_equal(new["regret_sums_compact"].numpy(), gather_compact(old["regret_sums"].numpy(), t))
    assert new["regret_summary"] == reference_summary(old["immediate_regrets"].numpy(), t, depth)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_gpu_summary_at_every_depth(rela, D, F):
    """The summary's cut between the nodes above regret_depth and the rest, from the root (nothing above) to past the leaves."""
    t = full_tree(D, F)
    for depth in range(2 * D * F + 3):
        r = rela.solve_full_game(make_cfg(rela, D, F, 8), 0, track_regrets=True, regret_depth=depth)
        assert r["regret_summary"] == reference_summary(r["immediate_regrets"].numpy(), t, depth), depth


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (2, 3)])
def test_gpu_golden_full_solve_regrets(rela, golden, D, F):
    g = golden("ev_regrets.npz")
    iters = {(int(d), int(f)): int(it) for d, f, it in g["full_iters"]}[(D, F)]
    r = rela.solve_full_game(make_cfg(rela, D, F, iters), 0, track_regrets=True)
    assert r["regret_count"] == iters // 2
    assert np.array_equal(r["immediate_regrets"].numpy(), g[f"full_regrets_{D}x{F}"])


@pytest.mark.gpu
def test_gpu_capi_matches_rela_and_refuses_what_it_cannot_track(rela):
    from rebel_b200 import capi
    D, F, iters = 2, 3, 32
    s = capi.FullGame(D, F)
    s.track_regrets()
    s.track_regrets()                                        # a second call changes nothing
    s.step(5)
    s.step(iters - 5)                                        # the even-index rule counts across calls
    imm, sums, node, count = s.regrets()
    s.close()
    r = rela.solve_full_game(make_cfg(rela, D, F, iters), 0, track_regrets=True)
    assert count == iters // 2
    assert np.array_equal(imm, r["immediate_regrets"].numpy()) and np.array_equal(sums, r["regret_sums_compact"].numpy())
    for n in range(len(node)):
        assert node[n] == hand_order_sum(imm[n]), n
    s = capi.FullGame(D, F)
    with pytest.raises(capi.CfrbError, match="cfrb_full_game_track_regrets has not been called"):
        s.regrets()
    s.step(1)
    with pytest.raises(capi.CfrbError, match="already run 1 iterations"):
        s.track_regrets()
    s.close()
    fp = capi.FullGame(D, F, solver=capi.SOLVER_FP)
    with pytest.raises(capi.CfrbError, match="CFR only"):
        fp.track_regrets()
    fp.close()
    f = rela.solve_full_game(make_cfg(rela, D, F, 8, "fp_linear"), 0, track_regrets=True)   # ignored for FP, as solve_full_tree
    assert "immediate_regrets" not in f and "regret_summary" not in f


@pytest.mark.gpu
def test_gpu_refusal_above_the_free_memory_hands_the_memory_back():
    from rebel_b200 import capi
    D, F = 2, 5
    torch.cuda.synchronize()
    before = torch.cuda.mem_get_info(0)[0]
    s = capi.FullGame(D, F)
    need = capi.full_game_regret_bytes(D, F)
    capi._check(capi.lib().cfrb_debug_full_game_free_cap(need - 1))
    try:
        with pytest.raises(capi.CfrbError, match=f"cfrb error -5: .*needs {need} bytes .*{need - 1} free"):
            s.track_regrets()
    finally:
        capi._check(capi.lib().cfrb_debug_full_game_free_cap(0))
    s.track_regrets()                                        # refused before anything was allocated: the object still works
    s.step(2)
    assert s.regrets()[3] == 1
    s.close()
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info(0)[0] >= before - (64 << 20)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(2, 5), (5, 2), (1, 11)])
def test_gpu_large_games(rela, D, F):
    iters = 16
    a = rela.solve_full_game(make_cfg(rela, D, F, iters), 0, track_regrets=True)
    b = rela.solve_full_game(make_cfg(rela, D, F, iters), 0, track_regrets=True)
    assert a["regret_count"] == iters // 2
    for k in ("immediate_regrets", "regret_sums_compact", "exploitability", "strategy"):
        assert torch.equal(a[k], b[k]), k
    assert a["regret_summary"] == b["regret_summary"]
    imm = a["immediate_regrets"]
    assert torch.isfinite(imm).all() and (imm >= 0).all()
    assert imm.sum().item() > 0
    top, rest = a["regret_summary"]
    assert abs(top + rest - imm.sum().item()) <= 1e-9 * imm.sum().item()
