"""The device self-play stream against the C port's RlRunner walk, game by game, on every CFR kernel path (pytest -m gpu).

Game g of a self-play session seeded with s replays RlRunner(seed = s + 10^6 g) (recursive_solving.cc:160-275): each wave solves
one subgame of every game and emits its two training examples, so wave w of game g must equal examples 2w and 2w + 1 of the port's
walk of that seed.  Every case compares EVERY game of its waves, row for row and bit for bit, with fp64 tables, against the port
(oracle/cfr_oracle.c), which tests/test_oracle.py pins to the compiled reference's RlRunner at up to 81 hands (selfplay_large.npz).

The matrix covers the depth-2 kernel, the warp kernel and the CTA kernel (WaveSolver.kernel_path; test_census asserts each
appears), CFR linear on every game with sample_leaf on and off, CFR plain, DCFR and fictitious play on a depth-2 game and a
warp / CTA game, random_action_prob 0 and 1, num_iters = 3 (act_iteration of 0 and of num_iters), and every value-net mode with a
constant-output Net2: output weight 0 and bias b, so that every query returns exactly b in each mode (DESIGN section 2: the
tensor-core modes keep b3 in fp32 and the SIMT kernel adds it last) while the whole net path runs (query tiles, dead-row
compaction, the net launch, the scaler multiply).  Games with more than 64 hands have no device walk: cfrb_selfplay_create and
rela.SelfPlayGenerator refuse them, and the host walk of rela.run_selfplay_waves replays the port there.
"""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from oracle.oracle import game_dims

pytestmark = pytest.mark.gpu

SEED = 5
D2, WARP, CTA = 0, 1, 2
PATHS = {D2: "d2", WARP: "warp", CTA: "CTA"}
SOLVERS = {
    "cfr": dict(use_cfr=True, linear_update=True),
    "plain": dict(use_cfr=True, linear_update=False),
    "dcfr": dict(use_cfr=True, linear_update=False, dcfr=True, dcfr_alpha=1.5, dcfr_beta=0.0, dcfr_gamma=2.0),
    "fp": dict(use_cfr=False, linear_update=True),
}
CHEAP_K, COSTLY_K = 160, 32           # 160 games: every per-game kernel runs more than one 128-thread block
COSTLY = {(1, 33)}                    # the port's walk takes ~50 ms per subgame there
HOST_WALK_GAMES = [(4, 3)]            # 81 hands
REFUSED_GAMES = [(4, 3), (1, 65)]     # 81 and 65 hands: past the device walk's per-thread belief copies (kSpMaxH = 64)


def _case(D, F, solver="cfr", sample_leaf=True, net_mode=0, rap=0.25, iters=16, waves=6, max_depth=2, driver="wave"):
    return dict(D=D, F=F, solver=solver, sample_leaf=sample_leaf, net_mode=net_mode, rap=rap, iters=iters, waves=waves,
                max_depth=max_depth, driver=driver)


def _cases():
    out = []
    for D, F in [(1, 2), (7, 1), (1, 10), (2, 5), (3, 3), (5, 2), (1, 11), (2, 6), (1, 17), (2, 7), (3, 4), (1, 33)]:
        for sl in (True, False):
            out.append(_case(D, F, sample_leaf=sl))
    for D, F in [(2, 5), (2, 6)]:                       # a depth-2 game and a warp / CTA game
        for solver in ("plain", "dcfr", "fp"):
            for sl in (True, False):
                out.append(_case(D, F, solver=solver, sample_leaf=sl))
    out += [_case(1, 6, rap=0.0), _case(1, 6, rap=1.0), _case(2, 3, iters=3, waves=12)]
    out += [_case(1, 6, max_depth=3), _case(1, 4, max_depth=3, sample_leaf=False)]
    for D, F, mode in [(2, 5, 1), (3, 4, 1), (1, 6, 2), (2, 5, 2), (1, 6, 3), (2, 5, 3), (1, 6, 4), (2, 7, 4), (3, 4, 4)]:
        out.append(_case(D, F, net_mode=mode))
    out += [_case(2, 5, driver="rela"), _case(1, 6, net_mode=3, driver="generator")]
    return out


CASES = _cases()


def case_id(c):
    s = f"{c['D']}x{c['F']}f-{c['solver']}-{'leaf' if c['sample_leaf'] else 'single'}"
    if c["net_mode"]:
        s += f"-net{c['net_mode']}"
    if c["rap"] != 0.25:
        s += f"-rap{c['rap']:g}"
    if c["iters"] != 16:
        s += f"-it{c['iters']}"
    if c["max_depth"] != 2:
        s += f"-d{c['max_depth']}"
    if c["driver"] != "wave":
        s += f"-{c['driver']}"
    return s


@pytest.fixture(scope="module")
def rb():
    import rebel_b200
    assert rebel_b200.capi.lib().cfrb_device_count() > 0, "no CUDA device: the CUDA path cannot be tested"
    return rebel_b200


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def constant_output_net(D, F):
    from oracle.make_golden_r4 import constant_output_net as net
    return net(D, F)


def n_games(c):
    return COSTLY_K if (c["D"], c["F"]) in COSTLY else CHEAP_K


def open_solver(rb, c, K):
    kw = SOLVERS[c["solver"]]
    return rb.WaveSolver(c["D"], c["F"], K, max_depth=c["max_depth"], num_iters=c["iters"], linear_update=kw["linear_update"],
                         dcfr=kw.get("dcfr", False), dcfr_alpha=kw.get("dcfr_alpha", 0.0), dcfr_beta=kw.get("dcfr_beta", 0.0),
                         dcfr_gamma=kw.get("dcfr_gamma", 0.0), net_mode=c["net_mode"], state_dtype=rb.STATE_F64,
                         solver=rb.SOLVER_CFR if kw["use_cfr"] else rb.SOLVER_FP)


def rela_cfg(rela, c, K, host_walk=0):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = c["D"], c["F"]
    cfg.random_action_prob, cfg.sample_leaf = c["rap"], c["sample_leaf"]
    cfg.concurrent_games, cfg.net_mode, cfg.state_dtype, cfg.host_walk = K, c["net_mode"], 0, host_walk
    sp = cfg.subgame_params
    kw = SOLVERS[c["solver"]]
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = c["iters"], c["max_depth"], kw["linear_update"], kw["use_cfr"]
    sp.dcfr, sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma = kw.get("dcfr", False), kw.get("dcfr_alpha", 0.0), kw.get("dcfr_beta", 0.0), \
        kw.get("dcfr_gamma", 0.0)
    return cfg


def device_stream(rb, rela, c, K, w):
    """The case's waves: q [waves, K, 2, Q], v [waves, K, 2, H] and the CFR kernel path of the handle that ran them."""
    import torch
    D, F, W = c["D"], c["F"], c["waves"]
    A, H, Q = game_dims(D, F)
    S = open_solver(rb, c, K)
    path = S.kernel_path()
    if c["driver"] == "wave":            # smoke()'s driver: WaveSolver.selfplay_*
        if w is not None:
            S.set_weights(w)
        S.selfplay_create(np.uint32(SEED) + np.arange(K, dtype=np.uint32) * np.uint32(1000000), random_action_prob=c["rap"],
                          sample_leaf=c["sample_leaf"])
        S.selfplay_wave()
        q, v = [], []
        for _ in range(W):
            S.selfplay_wave(keep_examples=True)
            a, b = S.selfplay_examples()
            q.append(a); v.append(b)
        S.selfplay_wave(start_next=False)
        S.sync()
        S.close()
        return np.stack(q), np.stack(v), path
    S.close()
    tw = None if w is None else torch.from_numpy(w)
    if c["driver"] == "rela":            # the thread loops' runner, synchronously
        q, v = rela.run_selfplay_waves(rela_cfg(rela, c, K), 0, SEED, W, tw)
        q, v = q.numpy(), v.numpy()
    else:                                # train --deterministic: a SelfPlayGenerator driven wave by wave, pipelined
        g = rela.SelfPlayGenerator(rela_cfg(rela, c, K), 0, SEED)
        if tw is not None:
            g.set_weights(tw, 1)
        out = [g.run(keep_running=i + 1 < W) for i in range(W)]
        assert g.drained
        q = np.concatenate([x[0].numpy() for x in out]); v = np.concatenate([x[1].numpy() for x in out])
    return q.reshape(W, K, 2, Q), v.reshape(W, K, 2, H), path


def port_streams(port, c, K, w):
    """Game g's first `waves` subgames of RlRunner(SEED + 10^6 g): q [K, 2 waves, Q], v [K, 2 waves, H], trace [K, waves, 5]."""
    D, F, W = c["D"], c["F"], c["waves"]

    def one(g):
        return port.rl_runner(D, F, SEED + 1000000 * g, n_games=1 << 30, num_iters=c["iters"], max_depth=c["max_depth"],
                              random_action_prob=c["rap"], sample_leaf=c["sample_leaf"], net_w=w, cap=2 * W, max_subgames=W, trace=True,
                              **SOLVERS[c["solver"]])
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:   # the port's calls release the GIL
        res = list(ex.map(one, range(K)))
    for q, v, tr in res:
        assert len(q) == 2 * W and len(tr) == W
    return np.stack([r[0] for r in res]), np.stack([r[1] for r in res]), np.stack([r[2] for r in res])


def compare(c, q, v, pq, pv, tr):
    """Every game of every wave, row for row; on a difference, the first (wave, game, row, column) and the port's trace entry."""
    W, K = q.shape[:2]
    pq = pq.reshape(K, W, 2, -1).transpose(1, 0, 2, 3)
    pv = pv.reshape(K, W, 2, -1).transpose(1, 0, 2, 3)
    for name, x, y in (("query", q, pq), ("value", v, pv)):
        bad = np.argwhere(x != y)
        if len(bad):
            w, g, r, col = (int(i) for i in bad[0])      # argwhere is in C order: the first wave, then game, row, column
            t = tr[g, w]
            pytest.fail(f"{case_id(c)}: {len(bad)} {name} entries differ; first at wave {w}, game {g}, row {r}, column {col}: "
                        f"device {x[w, g, r, col]!r} port {y[w, g, r, col]!r}; port trace: game {t[0]} of the stream, root "
                        f"(last_bid {t[1]}, player {t[2]}), act_iteration {t[3]}, br_sampler {t[4]}")


# what the cases covered, from the port's traces (test_coverage reads it; it runs after them in file order)
COVERAGE = {}


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_stream_equals_port(rb, rela, port, c):
    K = n_games(c)
    w = constant_output_net(c["D"], c["F"]) if c["net_mode"] else None
    t0 = time.time()
    pq, pv, tr = port_streams(port, c, K, w)
    t_port = time.time() - t0
    t0 = time.time()
    q, v, path = device_stream(rb, rela, c, K, w)
    t_gpu = time.time() - t0
    compare(c, q, v, pq, pv, tr)
    # after wave 0: the most restarted games at the initial state in one wave (they share one solve); per game: a game ended and
    # the next one started inside the waves
    shared = int((tr[:, 1:, 1] == -1).sum(0).max())
    restarts = int((tr[:, -1, 0] > 0).sum())
    COVERAGE[case_id(c)] = dict(path=path, shared=shared, restarts=restarts, act=set(np.unique(tr[:, :, 3]).tolist()),
                                br=set(np.unique(tr[:, :, 4]).tolist()), net_mode=c["net_mode"], iters=c["iters"])
    print(f"[selfplay] {case_id(c)}: {PATHS[path]}, {c['waves']} waves x {K} games bit-identical; up to {shared} initial-state games "
          f"in a later wave, {restarts} games restarted; port {t_port:.2f} s, GPU {t_gpu:.2f} s", flush=True)


def test_coverage():
    """The cases above saw what the matrix is for (skipped when they did not all run)."""
    missing = [case_id(c) for c in CASES if case_id(c) not in COVERAGE]
    if missing:
        pytest.skip(f"{len(missing)} cases did not run in this session")
    cov = COVERAGE.values()
    assert {x["path"] for x in cov} == {D2, WARP, CTA}
    assert {x["net_mode"] for x in cov} == {0, 1, 2, 3, 4}
    assert max(x["shared"] for x in cov) >= 8, "no later wave had several restarted games sharing the initial-state solve"
    assert all(x["restarts"] > 0 for x in cov), [k for k, x in COVERAGE.items() if not x["restarts"]]
    it3 = [x for x in cov if x["iters"] == 3]
    assert it3 and all({0, 3} <= x["act"] for x in it3), "num_iters = 3 never acted at iteration 0 and at num_iters"


def test_census(rb):
    """Which CFR kernel each case's handle runs (opened without running a wave): the matrix reaches the depth-2, warp and CTA
    kernels and every net mode, and its host-walk games are the ones the device walk refuses."""
    seen = {}
    for c in CASES:
        S = open_solver(rb, c, 1)
        seen.setdefault(PATHS[S.kernel_path()], []).append(case_id(c))
        S.close()
    for p, ids in sorted(seen.items()):
        print(f"[selfplay] census {p}: {' '.join(ids)}", flush=True)
    assert set(seen) == set(PATHS.values()), seen.keys()
    assert {c["net_mode"] for c in CASES} == {0, 1, 2, 3, 4}
    for D, F in HOST_WALK_GAMES:
        S = rb.WaveSolver(D, F, 1, num_iters=4, net_mode=rb.NET_ZERO)
        with pytest.raises(rb.CfrbError, match="num_hands <= 64"):
            S.selfplay_create(np.array([SEED], np.uint32))
        S.close()


@pytest.mark.parametrize("D,F", REFUSED_GAMES, ids=lambda x: str(x))
def test_device_walk_refuses_more_than_64_hands(rb, rela, D, F):
    S = rb.WaveSolver(D, F, 4, num_iters=4, net_mode=rb.NET_ZERO)
    assert S.H > 64
    with pytest.raises(rb.CfrbError, match="num_hands <= 64"):
        S.selfplay_create(np.arange(4, dtype=np.uint32))
    S.close()
    with pytest.raises(RuntimeError, match="num_hands <= 64"):
        rela.SelfPlayGenerator(rela_cfg(rela, _case(D, F, iters=4), 4), 0, SEED)


@pytest.mark.parametrize("sample_leaf", [True, False])
def test_host_walk_beyond_64_hands_equals_port(rb, rela, port, sample_leaf):
    """4x3f (81 hands, CTA kernel): the host walk of rela.run_selfplay_waves replays the port game by game."""
    D, F = HOST_WALK_GAMES[0]
    c = _case(D, F, sample_leaf=sample_leaf)
    K, W = 64, c["waves"]
    A, H, Q = game_dims(D, F)
    pq, pv, tr = port_streams(port, c, K, None)
    q, v = rela.run_selfplay_waves(rela_cfg(rela, c, K, host_walk=1), 0, SEED, W)
    compare(c, q.numpy().reshape(W, K, 2, Q), v.numpy().reshape(W, K, 2, H), pq, pv, tr)
