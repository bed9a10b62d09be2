"""The two-CTA cluster value net (net mode 4) against the net each game ran before: value-net time per launch and self-play
throughput, on one GPU.

    python scripts/cluster_net_bench.py [--repeats 3] [--quick]

Per launch: a wave of mixed subgames (--wave subgames, seed-0 Net2), --iters CFR iterations with every value-net launch bracketed
by CUDA events (cfrb_set_profiling); µs per launch = the run's value-net time / iterations (one launch per iteration).  Mode 1
(fp32 SIMT) against mode 4 at 2x7f, 3x4f, 6x2f, 7x2f and 1x64f; mode 3 (wide kernel) against mode 4 at 2x5f and 2x6f.
Self-play: the device-resident loop (WaveSolver.selfplay_*) with --games games x --sp_iters CFR iterations per wave, modes 1 and 4
at 2x7f and 3x4f; subgame-iters/s = games x iterations / wave time, over --sp_waves timed waves after two warm-up waves.
The runs of the two modes alternate in one process, --repeats times; each line of output is one JSON record.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import rebel_b200 as rb
from rebel_b200.models import flatten_state_dict, make_selfplay_net

PER_LAUNCH = [((2, 7), (1, 4)), ((3, 4), (1, 4)), ((6, 2), (1, 4)), ((7, 2), (1, 4)), ((1, 64), (1, 4)),
              ((2, 5), (3, 4)), ((2, 6), (3, 4))]
SELFPLAY = [(2, 7), (3, 4)]


def weights(D, F):
    return flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict())


def per_launch(D, F, mode, K, iters):
    A, H = 1 + 2 * D * F, F ** D
    rng = np.random.RandomState(1)
    b = rng.rand(K, 2, H)
    b /= b.sum(-1, keepdims=True)
    lb = rng.randint(-1, A - 2, size=K).astype(np.int32)
    pl = rng.randint(0, 2, size=K).astype(np.int32)
    S = rb.WaveSolver(D, F, K, net_mode=mode)
    S.set_weights(weights(D, F))
    S.set_profiling(1)
    S.begin(lb, pl, b)
    S.run(4)                                  # warm-up
    S.sync()
    S.begin(lb, pl, b)
    S.run(iters)
    S.sync()
    total_ms, net_ms = S.last_run_ms()
    rows = S.leaf_rows
    S.close()
    return {"net_us_per_launch": 1e3 * net_ms / iters, "run_ms": total_ms, "rows": rows}


def selfplay(D, F, mode, games, iters, waves):
    S = rb.WaveSolver(D, F, games, num_iters=iters, net_mode=mode)
    S.set_weights(weights(D, F))
    S.selfplay_create(np.uint32(7) + np.arange(games, dtype=np.uint32) * np.uint32(1000003))
    for _ in range(2):
        S.selfplay_wave()
    S.sync()
    t0 = time.perf_counter()
    for _ in range(waves):
        S.selfplay_wave()
    S.sync()
    dt = time.perf_counter() - t0
    S.selfplay_wave(start_next=False)
    S.sync()
    S.close()
    return {"subgame_iters_per_s": games * iters * waves / dt, "seconds_per_wave": dt / waves}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--wave", type=int, default=2048, help="subgames of the per-launch wave")
    ap.add_argument("--iters", type=int, default=32)
    ap.add_argument("--games", type=int, default=2048)
    ap.add_argument("--sp_iters", type=int, default=256)
    ap.add_argument("--sp_waves", type=int, default=4)
    ap.add_argument("--quick", action="store_true", help="one repeat, fewer self-play waves")
    args = ap.parse_args()
    if args.quick:
        args.repeats, args.sp_waves = 1, 2
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"card (name, power limit, max SM clock, SM clock)": card[0] if card else None}), flush=True)
    for r in range(args.repeats):
        for (D, F), modes in PER_LAUNCH:
            for mode in modes:
                rec = {"kind": "per_launch", "game": f"{D}x{F}f", "net_mode": mode, "repeat": r}
                rec.update(per_launch(D, F, mode, args.wave, args.iters))
                print(json.dumps(rec), flush=True)
        for D, F in SELFPLAY:
            for mode in (1, 4):
                rec = {"kind": "selfplay", "game": f"{D}x{F}f", "net_mode": mode, "repeat": r, "games": args.games,
                       "iters": args.sp_iters}
                rec.update(selfplay(D, F, mode, args.games, args.sp_iters, args.sp_waves))
                print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
