"""TEST INFRASTRUCTURE — generates tests/golden/*.npz from the REFERENCE itself (oracle/_ref, built from a checkout of
the original project by oracle/Makefile).  Run where that checkout exists:

    make -C oracle ref REF=<checkout> && python oracle/make_golden.py [live]

The fixtures make the tests self-contained: they run without the original project.  Net weights are NOT stored:
they are re-created from the seed with rebel_b200.models.make_selfplay_net and pinned by a checksum in the fixture.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle import Oracle, game_dims  # noqa: E402
from rebel_b200.models import flatten_state_dict, make_selfplay_net  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SHAPES = [(1, 4), (1, 6), (2, 3)]


def weights(D, F):
    return flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())


VARIANTS = {
    "vanilla": dict(linear_update=False),
    "dcfr": dict(linear_update=False, dcfr=True, dcfr_alpha=1.5, dcfr_beta=0.0, dcfr_gamma=2.0),
    "dcfr_sat": dict(linear_update=False, dcfr=True, dcfr_alpha=5.0, dcfr_beta=-5.0, dcfr_gamma=1.0),
}
VARIANT_NAMES = list(VARIANTS)
FP_CPS = [1, 2, 3, 8, 33]
FP_CASES = [(True, False, 2), (False, False, 2), (True, True, 2), (True, False, 3), (True, False, 100)]   # linear, optimistic, max_depth
FP_ROOTS = [(-1, 0), (2, 1)]


EVAL_CASES = [(1, 4, 32), (1, 6, 16), (2, 3, 8)]


def eval_weights(D, F, name):
    """Flat Net2 weights of the evaluation fixtures: seed-0 random init, optionally with the output layer zeroed."""
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    sd = make_selfplay_net(D, F, seed=0).state_dict()
    if name == "zero_out":
        sd["output.weight"] = sd["output.weight"] * 0
        sd["output.bias"] = sd["output.bias"] * 0
    return flatten_state_dict(sd)


def recursive_eval_reference(lib, D, F, num_iters, num_repeats, net_w=None, keep=2):
    """The accumulation loop of the reference's recursive_eval main (recursive_eval.cc:343-369) around its own
    compute_sampled_strategy_recursive_to_leaf and compute_stategy_stats, float32 tensors emulated with numpy."""
    tree = lib.unroll_tree(D, F)
    player = tree[:, 1]   # columns: last_bid, player_id, children_begin, children_end, parent, depth
    ss = sr = None
    expl, cps, first = [], [], []
    for sid in range(num_repeats):
        s = lib.sampled_strategy(D, F, seed=sid, num_iters=num_iters, net_w=net_w)
        reach = lib.strategy_reach(D, F, s)
        w = reach[player, np.arange(len(player))].astype(np.float32)[:, :, None]
        st = s.astype(np.float32)
        if sid < keep:
            first.append(s)
        if sid == 0:
            ss, sr = st * w, w.copy()
        else:
            ss += st * w
            sr += w
        if ((sid + 1) & sid) == 0 or sid + 1 == num_repeats:
            final = ss / (sr + np.float32(1e-6))
            cps.append(sid + 1)
            expl.append(lib.exploitability(D, F, final.astype(np.float64)))
    return {"summed_strategy": ss, "summed_reach": sr, "final_strategy": ss / (sr + np.float32(1e-6)),
            "checkpoints": np.array(cps), "exploitability": np.stack(expl), "first_strategies": np.stack(first)}


def main():
    os.makedirs(OUT, exist_ok=True)
    R = Oracle("ref_nofma")
    RF = Oracle("ref_fast")

    # ---- trees (bit-exact contract)
    trees = {}
    for (D, F, lb, pl, md) in [(1, 2, -1, 0, 1000), (2, 6, 22, 0, 0), (2, 6, 22, 0, 1), (2, 6, 22, 0, 2), (2, 6, 21, 0, 2),
                               (1, 4, -1, 0, 2), (1, 4, 3, 1, 2), (1, 6, -1, 0, 2), (1, 6, 5, 1, 2), (1, 6, 10, 0, 2),
                               (2, 3, -1, 1, 2), (2, 3, 7, 0, 2), (1, 5, -1, 0, 3), (1, 4, -1, 0, 1000)]:
        trees[f"t_{D}_{F}_{lb}_{pl}_{md}"] = R.unroll_tree(D, F, lb, pl, md)
    np.savez_compressed(os.path.join(OUT, "trees.npz"), **trees)

    # ---- zero-net depth-2 CFR trajectories (deterministic: -ffp-contract=off build)
    cps = [0, 1, 2, 3, 17, 64]
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        roots = [(-1, 0), (2, 1), (A - 3, 0)]
        out = {"checkpoints": np.array(cps), "roots": np.array(roots)}
        for i, (lb, pl) in enumerate(roots):
            b = R.synthetic_beliefs(H, 1000 + i)
            s = R.cfr_solve(D, F, b, cps, lb, pl, num_iters=64)
            out[f"beliefs{i}"] = b
            for k in ("regrets", "last", "sum", "avg", "root_means"):
                out[f"{k}{i}"] = s[k]
        np.savez_compressed(os.path.join(OUT, f"cfr_zero_{D}x{F}.npz"), **out)

    # ---- discounting variants of CFR::step (subgame_solving.cc:592-617): vanilla (no discount), DCFR(1.5, 0, 2) — the
    # recursive_eval --dcfr setting (recursive_eval.cc:250-254) — and DCFR with the alpha >= 5 / beta <= -5 shortcuts
    out = {"checkpoints": np.array([1, 2, 3, 8]), "variants": np.array(VARIANT_NAMES)}
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        b = R.synthetic_beliefs(H, 2000)
        out[f"beliefs_{D}x{F}"] = b
        for name, kw in VARIANTS.items():
            s = R.cfr_solve(D, F, b, [1, 2, 3, 8], 1, 1, num_iters=8, **kw)
            for k in ("regrets", "last", "sum", "avg", "root_means"):
                out[f"{k}_{name}_{D}x{F}"] = s[k]
    np.savez_compressed(os.path.join(OUT, "cfr_variants.npz"), **out)

    # ---- fictitious play (FP, subgame_solving.cc:364-506), zero net: linear / plain / optimistic, depth 2 and full depth
    out = {"checkpoints": np.array(FP_CPS), "cases": np.array([f"{int(l)}{int(o)}{md}" for l, o, md in FP_CASES])}
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        b = R.synthetic_beliefs(H, 3000)
        out[f"beliefs_{D}x{F}"] = b
        for (lin, opt, md) in FP_CASES:
            if md > 3 and (D, F) != (1, 4):
                continue
            for (lb, pl) in FP_ROOTS:
                s = R.fp_solve(D, F, b, FP_CPS, lb, pl, num_iters=max(FP_CPS), max_depth=md, linear_update=lin, optimistic=opt)
                for k in ("last", "sum", "avg", "root_means"):
                    out[f"{k}_{int(lin)}{int(opt)}{md}_{lb}_{D}x{F}"] = s[k]
    np.savez_compressed(os.path.join(OUT, "fp_zero.npz"), **out)

    # ---- Net2 depth-2 trajectories: short horizon states + long-horizon root means from both builds
    cps_net = [1, 2, 16]
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        w = weights(D, F)
        out = {"checkpoints": np.array(cps_net), "w_checksum": np.array([w.astype(np.float64).sum(), np.abs(w).astype(np.float64).sum()]),
               "w_head": w[:8].copy()}
        roots = [(-1, 0), (1, 1)]
        out["roots"] = np.array(roots)
        for i, (lb, pl) in enumerate(roots):
            b = R.synthetic_beliefs(H, 2000 + i)
            s = R.cfr_solve(D, F, b, cps_net, lb, pl, num_iters=16, net_w=w)
            out[f"beliefs{i}"] = b
            for k in ("regrets", "last", "sum", "avg", "root_means", "queries", "leaf_values"):
                out[f"{k}{i}"] = s[k]
            long_a = R.cfr_solve(D, F, b, [1024], lb, pl, num_iters=1024, net_w=w, want=("avg",))
            long_b = RF.cfr_solve(D, F, b, [1024], lb, pl, num_iters=1024, net_w=w, want=("avg",))
            out[f"mu1024_nofma{i}"] = long_a["root_means"][0]
            out[f"mu1024_fast{i}"] = long_b["root_means"][0]
        np.savez_compressed(os.path.join(OUT, f"cfr_net_{D}x{F}.npz"), **out)

    # ---- full-tree linear CFR (BASELINE config 0): exploitability after 1024 iterations, both builds
    out = {}
    for (D, F) in [(1, 2), (1, 3), (1, 4)]:
        A, H, Q = game_dims(D, F)
        b = np.full((2, H), 1.0 / H)
        for name, lib in (("nofma", R), ("fast", RF)):
            s = lib.cfr_solve(D, F, b, [16, 1024], num_iters=1024, max_depth=100000, want=("avg",))
            out[f"expl_{D}x{F}_{name}"] = np.stack([lib.exploitability(D, F, s["avg"][c]) for c in range(2)])
            if name == "nofma":
                out[f"avg16_{D}x{F}"] = s["avg"][0]
                out[f"mu_{D}x{F}"] = s["root_means"]
    np.savez_compressed(os.path.join(OUT, "fulltree.npz"), **out)

    # ---- self-play walk (RlRunner::step) with the zero net: exact example streams
    out = {}
    for (D, F) in SHAPES:
        for sl in (1, 0):
            q, v = R.rl_runner(D, F, seed=7, n_games=4, num_iters=32, sample_leaf=bool(sl))
            out[f"q_{D}x{F}_{sl}"] = q
            out[f"v_{D}x{F}_{sl}"] = v
    for (D, F) in SHAPES:   # the same walk with the fictitious-play solver (use_cfr = false)
        q, v = R.rl_runner(D, F, seed=7, n_games=4, num_iters=32, sample_leaf=True, use_cfr=False)
        out[f"q_fp_{D}x{F}"] = q
        out[f"v_fp_{D}x{F}"] = v
    np.savez_compressed(os.path.join(OUT, "selfplay_zero.npz"), **out)

    # ---- recursive evaluation (recursive_eval.cc:117-191,343-369) with the zero net: sampled recursive strategies of
    # seeds 0..R-1, their float32 reach-weighted sums in strategy_id order, and the exploitability at powers of two
    out = {}
    for (D, F, iters, reps) in [(1, 4, 64, 8), (1, 6, 32, 4), (2, 3, 32, 2)]:
        r = recursive_eval_reference(R, D, F, iters, reps)
        for k, v in r.items():
            if k in ("summed_strategy", "summed_reach", "checkpoints", "exploitability") or (k == "first_strategies" and (D, F) == (1, 4)):
                out[f"{k}_{D}x{F}"] = v
        out[f"cfg_{D}x{F}"] = np.array([iters, reps])
    np.savez_compressed(os.path.join(OUT, "recursive_eval_zero.npz"), **out)

    # ---- evaluation entry points of the rela module (pybind.cc:45-84): compute_strategy_recursive / _to_leaf + exploitability +
    # eval_net, with a Net2 whose output layer is zeroed (exact: the net contributes exact zeros) and with the random-init net
    out = {"cases": np.array([f"{D}x{F}:{it}" for D, F, it in EVAL_CASES])}
    for (D, F, it) in EVAL_CASES:
        for use_cfr in (True, False):
            for netname in ("zero_out", "random"):
                r = R.net_evaluation(D, F, eval_weights(D, F, netname), num_iters=it, use_cfr=use_cfr)
                tag = f"{'cfr' if use_cfr else 'fp'}_{netname}_{D}x{F}"
                out[f"values_{tag}"] = r["values"]
                if (D, F) == (1, 4):
                    out[f"strategy_recursive_{tag}"] = r["strategy_recursive"]
                    out[f"strategy_to_leaf_{tag}"] = r["strategy_to_leaf"]
    np.savez_compressed(os.path.join(OUT, "net_evaluation.npz"), **out)

    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


def reference_live():
    """tests/golden/reference_live.npz: what tests/test_oracle.py compares the C port with — the compiled reference's
    synthetic beliefs, 40-iteration CFR solves and RlRunner streams, and its Net2 evaluated in the kernels' arithmetic."""
    R = Oracle("ref_nofma")
    out = {}
    for (D, F) in SHAPES:
        A, H, Q = game_dims(D, F)
        out[f"beliefs11_{D}x{F}"] = R.synthetic_beliefs(H, 11)
        b = R.synthetic_beliefs(H, 5)
        for lb, pl in [(-1, 0), (4, 1)]:
            y = R.cfr_solve(D, F, b, [0, 1, 5, 40], lb, pl, num_iters=40)
            for k in ("regrets", "last", "sum", "avg", "root_means", "traverser_values"):
                out[f"{k}_{lb}_{pl}_{D}x{F}"] = y[k]
        out[f"q_{D}x{F}"], out[f"v_{D}x{F}"] = R.rl_runner(D, F, seed=3, n_games=2, num_iters=24)
    D, F = 1, 6
    A, H, Q = game_dims(D, F)
    b = R.synthetic_beliefs(H, 3)
    for model in (0, 1, 2):        # ref_set_net_emulation: 0 = ATen fp32, 1 / 2 = the tensor-core kernels' arithmetic models
        R.set_net_emulation(model)
        r = R.cfr_solve(D, F, b, [1], last_bid=-1, player_id=0, num_iters=1, net_w=weights(D, F), want=("avg",))
        out[f"emulation{model}_leaf_values"] = r["leaf_values"][0]
        out["emulation_queries"] = r["queries"][0]
    R.set_net_emulation(0)
    np.savez_compressed(os.path.join(OUT, "reference_live.npz"), **out)


if __name__ == "__main__":
    reference_live() if sys.argv[1:] == ["live"] else main()
