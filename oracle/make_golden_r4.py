"""TEST INFRASTRUCTURE — round-4 fixture generated from the REFERENCE itself (oracle/_ref, -ffp-contract=off build), where a
checkout of the original project exists:

    make -C oracle ref REF=<checkout> && python oracle/make_golden_r4.py

  selfplay_large.npz  RlRunner example streams (recursive_solving.cc:160-275) beyond 9 hands, so that the suite holds the C port's
                      walk to the reference at up to 81 hands and 35 actions on machines without oracle/_ref:
    q_{case} / v_{case}   the examples [n][Q] / [n][H] of RlRunner(seed = SEED) playing GAMES_PER_STREAM games, NUM_ITERS
                          iterations per subgame, max_depth 2, random_action_prob 0.25, for every case of cases():
                          {D}x{F}_{solver}_{sample_leaf}_{net}
    solvers               cfr (linear CFR), plain (CFR without discounting), dcfr (DCFR 1.5 / 0 / 2), fp (linear fictitious play)
    nets                  zero: the zero net; const: constant_output_net(D, F), a seed-0 Net2 whose output layer has weight 0 and
                          bias linspace(-0.7, 0.9, H), so every query returns that bias exactly (the test rebuilds it)
Regenerating rewrites the file byte for byte (fixed seeds, no timestamps in the archive members).
"""
import io
import os
import sys
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle import Oracle  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "selfplay_large.npz")
GAMES = [(7, 1), (2, 6), (1, 17), (3, 4), (4, 3)]
SOLVERS = {
    "cfr": dict(use_cfr=True, linear_update=True),
    "plain": dict(use_cfr=True, linear_update=False),
    "dcfr": dict(use_cfr=True, linear_update=False, dcfr=True, dcfr_alpha=1.5, dcfr_beta=0.0, dcfr_gamma=2.0),
    "fp": dict(use_cfr=False, linear_update=True),
}
NETS = ("zero", "const")
NUM_ITERS, GAMES_PER_STREAM, SEED = 16, 2, 5


def constant_output_net(D, F):
    """Flat Net2 weights: seed-0 make_selfplay_net with output.weight = 0 and output.bias = linspace(-0.7, 0.9, H) in fp32."""
    import torch
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    net = make_selfplay_net(D, F, seed=0)
    with torch.no_grad():
        net.output.weight.zero_()
        net.output.bias.copy_(torch.linspace(-0.7, 0.9, F ** D))
    return flatten_state_dict(net.state_dict())


def cases():
    for D, F in GAMES:
        for solver in SOLVERS:
            for sl in (1, 0):
                for net in NETS:
                    if net == "const" and sl == 0 and solver in ("plain", "dcfr"):
                        continue           # the net path is the same for every solver: keep the fixture small
                    yield D, F, solver, sl, net


def case_key(D, F, solver, sl, net):
    return f"{D}x{F}_{solver}_{sl}_{net}"


def stream(O, D, F, solver, sl, net):
    w = None if net == "zero" else constant_output_net(D, F)
    return O.rl_runner(D, F, SEED, n_games=GAMES_PER_STREAM, num_iters=NUM_ITERS, sample_leaf=bool(sl), net_w=w, cap=4096,
                       **SOLVERS[solver])


def save_deterministic(path, arrays):
    """np.savez_compressed with fixed member timestamps, so the same arrays give the same bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.save(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    R = Oracle("ref_nofma")
    out = {}
    for c in cases():
        q, v = stream(R, *c)
        out["q_" + case_key(*c)], out["v_" + case_key(*c)] = q, v
        print(case_key(*c), len(q), "examples", flush=True)
    save_deterministic(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
