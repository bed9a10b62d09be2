"""Every CFR kernel path and hand-count specialisation against the C port (oracle/cfr_oracle.c), run on an H100 (pytest -m gpu).

cfrb_create picks one of three CFR iteration kernels from the game, the tree depth and the state dtype (WaveSolver.kernel_path):
  d2    cfr_iter_d2_kernel: templates of at most three levels, at most 255 nodes, scratch in shared memory;
  warp  cfr_iter_kernel<real, 32, HC>: a warp per subgame, scratch in shared memory;
  CTA   cfr_iter_kernel<real, 256, 0>: a CTA per subgame, scratch in global memory.
d2 and warp are also compiled for H in {4, 5, 6, 9, 16} (CFRB_DISPATCH_H in cfr_kernels.cu), every other H takes HC = 0.  CASES
fills every path x HC cell with fp64 tables (warp with HC = 16 only fits with fp32 tables) and every path with fp32 tables.  Each case
names the path the library must report, so a change to the selection rule cannot quietly empty a cell.

Every wave holds the roots -1, a middle bid, A-3 (a two-level template) and A-2 (a single child), each for both players.  Against the
port: fp64 tables with the zero net are bit-identical (linear CFR on every case, vanilla CFR and DCFR and fictitious play on one case
per path); the fp32 net and fp32 tables are checked by teacher-forced single steps with the bounds of test_gpu_parity.

More than seven dice per player is refused: the terminal payoff histogram of the kernels holds 9 bins (cfr_types.h kMaxDice).  The
8x2f and 9x1f cases expect that refusal; if the library accepts them they run the bit-exact comparison like any other case.
"""
import time

import numpy as np
import pytest

from oracle.make_golden import VARIANTS
from oracle.oracle import game_dims
from test_gpu_parity import teacher_forced_steps

pytestmark = pytest.mark.gpu

D2, WARP, CTA, REFUSED = 0, 1, 2, -1
PATHS = {D2: "d2", WARP: "warp", CTA: "CTA", REFUSED: "refused"}
SPECIALISED_H = (4, 5, 6, 9, 16)
FULL = 100            # deeper than any tree here: the full game from each root
CPS = [1, 2, 3, 17, 32]

# (num_dice, num_faces, max_depth, state dtype, expected kernel path, expected HC)
CASES = [
    (2, 2, 2, "f64", D2, 4), (1, 5, 2, "f64", D2, 5), (1, 6, 2, "f64", D2, 6), (2, 3, 2, "f64", D2, 9), (2, 4, 2, "f64", D2, 16),
    (1, 2, 2, "f64", D2, 0), (3, 2, 2, "f64", D2, 0), (7, 1, 2, "f64", D2, 0), (2, 5, 2, "f64", D2, 0), (3, 3, 2, "f64", D2, 0),
    (2, 6, 1, "f64", D2, 0), (6, 2, 1, "f64", D2, 0), (7, 2, 1, "f64", D2, 0),     # H > 32: several hands per lane
    (1, 31, 1, "f64", D2, 0),                                                          # 63 actions
    (5, 2, 2, "f32", D2, 0),
    (1, 12, 2, "f64", WARP, 0), (1, 5, 3, "f64", WARP, 5), (2, 2, FULL, "f64", WARP, 4), (1, 4, FULL, "f64", WARP, 4),
    (1, 6, 3, "f64", WARP, 6), (2, 3, 3, "f64", WARP, 9),
    (2, 6, 2, "f32", WARP, 0), (1, 16, 2, "f32", WARP, 16),
    (5, 2, 2, "f64", CTA, 0), (2, 7, 2, "f64", CTA, 0), (3, 4, 2, "f64", CTA, 0), (6, 2, 2, "f64", CTA, 0),
    (1, 5, FULL, "f64", CTA, 0),
    (2, 7, 2, "f32", CTA, 0), (1, 5, FULL, "f32", CTA, 0),
    (8, 2, 1, "f64", REFUSED, None), (9, 1, 2, "f64", REFUSED, None),
]
ACCEPTED = [c for c in CASES if c[4] != REFUSED]
ONE_PER_PATH = [(6, 2, 1, "f64", D2, 0), (1, 12, 2, "f64", WARP, 0), (5, 2, 2, "f64", CTA, 0)]


def case_id(c):
    D, F, md, state = c[:4]
    return f"{D}x{F}f-{'full' if md == FULL else f'd{md}'}-{state}"


@pytest.fixture(scope="module")
def rb():
    import rebel_b200
    assert rebel_b200.capi.lib().cfrb_device_count() > 0, "no CUDA device: the CUDA path cannot be tested"
    return rebel_b200


def _note(msg):
    print("[matrix]", msg, flush=True)


def roots_of(A):
    return [(lb, pl) for lb in (-1, (A - 1) // 2, A - 3, A - 2) for pl in (0, 1)]


def beliefs(H, n, seed):
    """Random beliefs; in every other subgame player 0 almost surely does not hold every third hand.  Not exactly zero: with a
    hand of zero reach the reference's normalize_probabilities divides 0 by 0 (it asserts sum >= kAlmostZero in debug builds),
    where the average strategy of cfrb_fetch is uniform."""
    rng = np.random.RandomState(seed)
    b = rng.rand(n, 2, H)
    if H >= 3:
        b[1::2, 0, ::3] *= 1e-9
    return b / b.sum(-1, keepdims=True)


def edges(dense, tree):
    """[N, H, A] -> [N - 1, H]: the entry of every edge (parent, hand, action leading to the child)."""
    return dense[tree[1:, 4], :, tree[1:, 0]]


def open_solver(rb, case, n, **kw):
    """The case's handle with the zero net, after checking the kernel path the library chose; None if the game is refused as
    expected."""
    D, F, md, state, path, hc = case
    A, H, Q = game_dims(D, F)
    assert hc == (H if path in (D2, WARP) and H in SPECIALISED_H else 0 if path != REFUSED else None), case
    try:
        S = rb.WaveSolver(D, F, n, max_depth=md, net_mode=rb.NET_ZERO,
                          state_dtype={"f64": rb.STATE_F64, "f32": rb.STATE_F32}[state], **kw)
    except rb.CfrbError as e:
        if path == REFUSED:
            assert "at most 7 dice per player" in str(e), str(e)
            return None
        raise
    if path != REFUSED:
        assert S.kernel_path() == path, (case_id(case), PATHS[S.kernel_path()], "expected", PATHS[path])
    return S


def compare_with_port(rb, port, case, kw, port_solve, keys, exact=True, tol=0.0):
    """One wave of every root; at each checkpoint of CPS the GPU's tables (edge entries of `keys`) and root means against the
    port's, bit for bit or within tol."""
    D, F, md = case[:3]
    A, H, Q = game_dims(D, F)
    roots = roots_of(A)
    S = open_solver(rb, case, len(roots), **kw)
    if S is None:
        return
    b = beliefs(H, len(roots), 1000 * D + F)
    t0 = time.time()
    want = []
    for i, (lb, pl) in enumerate(roots):
        o = port_solve(D, F, b[i], CPS, lb, pl, num_iters=max(CPS), max_depth=md, **kw)
        tree = port.unroll_tree(D, F, lb, pl, md)
        want.append({"tree": tree, "root_means": o["root_means"], **{k: np.stack([edges(x, tree) for x in o[k]]) for k in keys}})
        del o
    t_port = time.time() - t0
    t0 = time.time()
    S.begin([r[0] for r in roots], [r[1] for r in roots], b)
    done = 0
    worst = 0.0
    for ci, c in enumerate(CPS):
        S.run(c - done); done = c
        f = S.fetch(("root_means",) + tuple(keys))
        for i, w in enumerate(want):
            tag = (case_id(case), kw, roots[i], c)
            for k in keys:
                x, y = edges(f[k][i], w["tree"]), w[k][ci]
                d = np.abs(x - y).max() if x.size else 0.0
                worst = max(worst, d)
                if exact:
                    assert np.array_equal(x, y), (tag, k, "not bit-exact", d, np.argwhere(x != y)[:3].tolist())
                else:
                    assert d < tol, (tag, k, d)
            x, y = f["root_means"][i], w["root_means"][ci]
            if exact:
                assert np.array_equal(x, y), (tag, "root means not bit-exact", np.abs(x - y).max())
            else:
                assert np.abs(x - y).max() < tol, (tag, "root means", np.abs(x - y).max())
        del f
    path = S.kernel_path()
    S.close()
    _note(f"{case_id(case)} {PATHS[path]} {kw or 'linear CFR'}: {len(roots)} roots x {max(CPS)} iterations, worst |diff| {worst:.1e}; "
          f"port {t_port:.2f} s, GPU {time.time() - t0:.2f} s")
    assert case[4] != REFUSED, f"{case_id(case)} was accepted and matched the port: its expected outcome is out of date"


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_linear_cfr_bit_exact(rb, port, case):
    if case[3] != "f64":
        pytest.skip("fp32 tables round every update: checked by test_fp32_net_teacher_forced")
    compare_with_port(rb, port, case, {}, port.cfr_solve, ("regrets", "last", "sum", "avg"))


@pytest.mark.parametrize("case", ONE_PER_PATH, ids=case_id)
@pytest.mark.parametrize("variant", ["vanilla", "dcfr"])
def test_discount_variants(rb, port, case, variant):
    """Vanilla CFR is bit-identical; DCFR evaluates n^alpha with CUDA's pow, which may differ from glibc's by an ulp, so it is
    compared to 1e-12 as in test_gpu_parity.test_discount_variants_vs_reference."""
    compare_with_port(rb, port, case, VARIANTS[variant], port.cfr_solve, ("regrets", "last", "sum", "avg"),
                      exact=variant == "vanilla", tol=1e-12)


@pytest.mark.parametrize("case", ONE_PER_PATH, ids=case_id)
@pytest.mark.parametrize("optimistic", [False, True])
def test_fictitious_play_bit_exact(rb, port, case, optimistic):
    def fp_solve(D, F, b, cps, lb, pl, num_iters, max_depth, solver, optimistic):
        return port.fp_solve(D, F, b, cps, lb, pl, num_iters=num_iters, max_depth=max_depth, optimistic=optimistic)
    compare_with_port(rb, port, case, dict(solver=rb.SOLVER_FP, optimistic=optimistic), fp_solve, ("last", "sum", "avg"))


@pytest.mark.parametrize("case", ACCEPTED, ids=case_id)
def test_fp32_net_teacher_forced(rb, port, net_weights, case):
    """NET_FP32 with the case's tables, and the zero net with fp32 tables: from the port's state after c iterations one GPU step
    reproduces the port's next state within the bounds of test_gpu_parity.test_teacher_forced_single_step."""
    D, F, md, state = case[:4]
    A, H, Q = game_dims(D, F)
    open_solver(rb, case, 1).close()
    for net_name in ("fp32", "zero") if state == "f32" else ("fp32",):
        t0 = time.time()
        teacher_forced_steps(rb, port, net_weights, D, F, md, state, net_name, roots=roots_of(A), cps=[0, 1, 2, 3, 16, 17])
        _note(f"{case_id(case)} teacher-forced {state}/{net_name}: {time.time() - t0:.2f} s")


def test_kernel_path_census(rb):
    """Every path x HC cell holds a case with fp64 tables (warp x 16 with fp32 tables), and every path one with fp32 tables."""
    cells, moved = {}, []
    for case in ACCEPTED:
        D, F, md, state, path, hc = case
        S = rb.WaveSolver(D, F, 1, max_depth=md, net_mode=rb.NET_ZERO, state_dtype={"f64": rb.STATE_F64, "f32": rb.STATE_F32}[state])
        got = S.kernel_path()
        S.close()
        cells.setdefault((PATHS[got], hc if got != CTA else 0, state), []).append(case_id(case))
        if got != path:
            moved.append((case_id(case), PATHS[got], "expected", PATHS[path]))
    for (path, hc, state), ids in sorted(cells.items()):
        _note(f"census {path:4s} HC={hc:<2d} {state}: {' '.join(ids)}")
    assert not moved, moved
    need = [(p, h, "f64") for p in ("d2", "warp") for h in (0,) + SPECIALISED_H if (p, h) != ("warp", 16)]
    need += [("CTA", 0, "f64"), ("warp", 16, "f32"), ("d2", 0, "f32"), ("warp", 0, "f32"), ("CTA", 0, "f32")]
    assert not [c for c in need if c not in cells], [c for c in need if c not in cells]


def test_more_than_seven_dice_is_refused(rb):
    for D, F, md in [(8, 2, 1), (9, 1, 2), (12, 2, 1)]:
        for net in (rb.NET_ZERO, rb.NET_FP32):
            with pytest.raises(rb.CfrbError, match=r"holds 9 bins, so at most 7 dice per player"):
                rb.WaveSolver(D, F, 1, max_depth=md, net_mode=net)
    for D, F in [(7, 2), (7, 1)]:        # the edge: a clamped count lands on the empty top bin (their cases above are bit-exact)
        S = rb.WaveSolver(D, F, 1, max_depth=1, net_mode=rb.NET_ZERO)
        assert S.H == F ** D
        S.close()
