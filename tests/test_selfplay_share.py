"""Self-play waves solve their initial-state games once: every game at the initial state (no bid yet, player 0, every belief
bitwise 1 / H) solves the same subgame bit for bit, so the wave solves the lowest one and gives the others its tables, root means
and the snapshot of their own act_iteration.  Everything a reader sees must be what solving every game on its own gives."""
import numpy as np
import pytest

from oracle.oracle import game_dims

HEADER = 40     # cfrb_selfplay_export: header, beliefs f64 [K][2][H], mt u32 [624][K], last_bid, player, mt_idx i32 [K]


def _initial(lb, pl, bel, H):
    uniform = np.float64(1.0) / np.float64(H)
    return (lb == -1) & (pl == 0) & np.all(bel.view(np.uint64) == uniform.view(np.uint64), axis=(1, 2))


def _no_initial_state(image, K, H):
    """The session image with every initial-state game's first belief moved by one ulp: the same games, none of them shared."""
    img = bytearray(image)
    bel = np.frombuffer(img, np.float64, K * 2 * H, HEADER).reshape(K, 2, H).copy()
    lb = np.frombuffer(img, np.int32, K, HEADER + K * 2 * H * 8 + 624 * K * 4)
    pl = np.frombuffer(img, np.int32, K, HEADER + K * 2 * H * 8 + 624 * K * 4 + 4 * K)
    init = _initial(lb, pl, bel, H)
    assert init.any()
    bel[init, 0, 0] = np.nextafter(bel[init, 0, 0], 1.0)
    img[HEADER:HEADER + bel.nbytes] = bel.tobytes()
    return bytes(img)


def _tree_entries(S, D, F):
    """The compact tables' entries [n, table_stride] that belong to the current wave's subgames: (N - 1) x H of each row, the
    rest being whatever earlier waves (or earlier allocations) left there."""
    from rebel_b200 import capi
    A, H, _ = game_dims(D, F)
    n_edges = np.array([len(capi.unroll_tree(D, F, b, 0, 2)) - 1 for b in range(-1, A - 1)])
    lb, _ = S.wave_roots()
    stride = S.fetch_compact("snapshot").shape[1]
    return np.arange(stride)[None, :] < (n_edges[lb + 1] * H)[:, None]


def _session(D, F, K, iters, solver, dtype, share, weights):
    """Every wave's examples, fetched tables and session export, and the solved counts, of a self-play loop that crosses the first
    wave (every game at the initial state), stationary waves and an imported session without an initial-state game."""
    import rebel_b200 as rb
    A, H, _ = game_dims(D, F)
    S = rb.WaveSolver(D, F, K, num_iters=iters, net_mode=rb.NET_TC_F16X2, solver=solver, state_dtype=dtype)
    S.set_weights(weights)
    S.debug_selfplay_share(share)
    S.selfplay_create(np.uint32(29) + np.arange(K, dtype=np.uint32) * np.uint32(104729))
    out, solved = [], []

    def wave(**kw):
        S.selfplay_wave(**kw)
        lb, pl, bel = S.selfplay_state()
        n_init = int(_initial(lb, pl, bel, H).sum())
        solved.append((S.wave_solved, n_init))
        mask = _tree_entries(S, D, F)
        rec = {k: np.where(mask, S.fetch_compact(w), 0.0) for k, w in (("R", "regrets"), ("Sg", "last"), ("Snap", "snapshot"))}
        rec["mu"] = S.fetch(("root_means",))["root_means"]
        if kw.get("keep_examples"):
            rec["q"], rec["v"] = S.selfplay_examples()
        out.append(rec)

    def export():
        S.selfplay_wave(start_next=False, keep_examples=True)
        q, v = S.selfplay_examples()
        image = S.selfplay_export()
        out.append({"q": q, "v": v, "image": np.frombuffer(image, np.uint8)})
        return image

    wave()                                    # the first wave: one solve for the whole wave
    for _ in range(5):
        wave(keep_examples=True)
    image = export()
    S.selfplay_import(_no_initial_state(image, K, H))
    wave()                                    # no initial-state game: every game solved on its own
    for _ in range(4):
        wave(keep_examples=True)
    out.append({"sum": np.where(_tree_entries(S, D, F), S.fetch_compact("sum"), 0.0),   # the rebuilt sum of the last wave
                "avg": S.fetch(("avg",))["avg"]})
    export()
    S.close()
    return out, solved


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["cfr", "fp"])
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3)])
def test_shared_initial_state_solve_is_bit_identical(D, F, solver):
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    K, iters = 256, 48
    w = flatten_state_dict(make_selfplay_net(D, F, seed=3).state_dict())
    sv = rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP
    on, solved_on = _session(D, F, K, iters, sv, rb.STATE_F64, True, w)
    off, solved_off = _session(D, F, K, iters, sv, rb.STATE_F64, False, w)
    assert len(on) == len(off)
    for i, (a, b) in enumerate(zip(on, off)):
        assert a.keys() == b.keys()
        for key in a:
            assert a[key].tobytes() == b[key].tobytes(), f"record {i}: {key}"
    assert all(n == K for n, _ in solved_off)
    for n, n_init in solved_on:
        assert n == K - n_init + (1 if n_init else 0)
    assert solved_on[0] == (1, K)                 # the first wave
    assert solved_on[6] == (K, 0)                 # the imported session
    assert any(0 < n_init < K for _, n_init in solved_on[1:6])   # stationary waves share part of the wave


@pytest.mark.gpu
def test_shared_solve_fp32_tables():
    """The fp32 state tables take the same path."""
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, K, iters = 1, 6, 256, 48
    w = flatten_state_dict(make_selfplay_net(D, F, seed=4).state_dict())
    on, solved_on = _session(D, F, K, iters, rb.SOLVER_CFR, rb.STATE_F32, True, w)
    off, _ = _session(D, F, K, iters, rb.SOLVER_CFR, rb.STATE_F32, False, w)
    for i, (a, b) in enumerate(zip(on, off)):
        for key in a:
            assert a[key].tobytes() == b[key].tobytes(), f"record {i}: {key}"
    assert solved_on[0] == (1, K)


@pytest.mark.gpu
@pytest.mark.parametrize("solver", ["cfr", "fp"])
def test_recreated_session_replays_shared_graphs(solver):
    """A session re-created with another number of games on the same handle, after shared waves that were captured as CUDA graphs
    (num_iters >= 64, the same run key seen twice), must solve exactly what the same handle without sharing solves."""
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, K, iters = 1, 6, 256, 64
    A, H, _ = game_dims(D, F)
    w = flatten_state_dict(make_selfplay_net(D, F, seed=5).state_dict())
    sv = rb.SOLVER_CFR if solver == "cfr" else rb.SOLVER_FP

    def run(share):
        S = rb.WaveSolver(D, F, K, num_iters=iters, net_mode=rb.NET_TC_F16X2, solver=sv)
        S.set_weights(w)
        S.debug_selfplay_share(share)
        out = []
        for n_games, seed in ((K, 7), (160, 8), (K, 9)):
            S.selfplay_create(np.uint32(seed) + np.arange(n_games, dtype=np.uint32) * np.uint32(7919))
            S.selfplay_wave()
            for _ in range(4):
                S.selfplay_wave(keep_examples=True)
                lb, pl, bel = S.selfplay_state()
                n_init = int(_initial(lb, pl, bel, H).sum())
                if share:
                    assert S.wave_solved == n_games - n_init + (1 if n_init else 0)
                mask = _tree_entries(S, D, F)
                rec = {k: np.where(mask, S.fetch_compact(t), 0.0) for k, t in (("R", "regrets"), ("Sg", "last"), ("Snap", "snapshot"))}
                rec["mu"] = S.fetch(("root_means",))["root_means"]
                rec["q"], rec["v"] = S.selfplay_examples()
                out.append(rec)
            S.selfplay_wave(start_next=False)
        S.close()
        return out

    on, off = run(True), run(False)
    assert len(on) == len(off)
    for i, (a, b) in enumerate(zip(on, off)):
        for key in a:
            assert a[key].tobytes() == b[key].tobytes(), f"wave {i}: {key}"
