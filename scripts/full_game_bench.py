"""Full-game solves on the whole GPU (rela.solve_full_game): per game the time of a --iters iteration linear-CFR solve with its
checkpoints, split between the iterations and the best responses at the powers of two, the seconds per iteration, the final
exploitability and the peak device memory (the device's free memory polled every 5 ms from a second thread, so other processes on
the device count too).  On the games the one-CTA solver runs (2x4f, 3x3f) both solvers' iterations are timed in one process,
alternated, over --cmp_iters iterations each after a warm-up run of both; the speed-up is the ratio of the best seconds per
iteration.  Prints the card, its power limit and its maximum SM clock before and after.

    python scripts/full_game_bench.py [--iters 1024] [--games 2x5,5x2,1x11] [--cmp 2x4,3x3] [--cmp_iters 64] [--out full_game.json]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def peak_bytes_during(fn):
    """fn()'s result and the largest drop of the device's free memory while it ran."""
    import torch
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    low, done = [free0], threading.Event()

    def poll():
        while not done.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.005)
    t = threading.Thread(target=poll)
    t.start()
    try:
        r = fn()
    finally:
        done.set()
        t.join()
    return r, free0 - low[0]


def cfg_of(rela, D, F, iters):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, 0, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.linear_update = iters, 100000, True, True
    return cfg


def compare(capi, D, F, iters, reps):
    """Seconds per iteration of the one-CTA solver (a one-subgame WaveSolver at the root) and of capi.FullGame, alternated."""
    H = F ** D
    one = capi.WaveSolver(D, F, 1, max_depth=100000, num_iters=iters, net_mode=capi.NET_ZERO)
    one.begin([-1], [0], np.full((1, 2, H), 1.0 / H))
    full = capi.FullGame(D, F)
    one.run(iters); one.sync()          # warm-up (module load, full.step's graph capture)
    full.step(iters)
    old, new = [], []
    for _ in range(reps):
        t0 = time.perf_counter()
        one.run(iters)
        one.sync()
        old.append((time.perf_counter() - t0) / iters)
        t0 = time.perf_counter()
        full.step(iters)
        new.append((time.perf_counter() - t0) / iters)
    one.close(); full.close()
    return old, new


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--games", type=str, default="2x4,3x3,2x5,5x2,1x11", help="games solved in full with checkpoints")
    ap.add_argument("--cmp", type=str, default="2x4,3x3", help="games on which the one-CTA solver is timed against the new one")
    ap.add_argument("--cmp_iters", type=int, default=64)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import torch
    import rebel_b200.rela as rela
    from rebel_b200 import capi
    torch.cuda.init()
    res = {"card": card(), "iters": args.iters, "runs": {}, "compare": {}}
    rela.solve_full_game(cfg_of(rela, 1, 4, 64), 0)                      # warm-up: module load
    for g in args.cmp.split(",") if args.cmp else []:
        D, F = (int(x) for x in g.split("x"))
        old, new = compare(capi, D, F, args.cmp_iters, args.reps)
        c = {"one_cta_s_per_iter": old, "full_game_s_per_iter": new, "speedup": min(old) / min(new), "iters": args.cmp_iters}
        res["compare"][f"{g}f"] = c
        print(f"{g}f compare: {json.dumps(c)}", flush=True)
    for g in args.games.split(","):
        D, F = (int(x) for x in g.split("x"))
        r, peak = peak_bytes_during(lambda: rela.solve_full_game(cfg_of(rela, D, F, args.iters), 0))
        e = r["exploitability"][-1].tolist()
        run = {"num_nodes": r["num_nodes"], "br": e, "exploitability": (e[0] + e[1]) / 2, "first_checkpoint": r["exploitability"][0].tolist(),
               "seconds": r["seconds"], "solve_seconds": r["solve_seconds"], "br_seconds": r["br_seconds"],
               "checkpoints": len(r["checkpoints"]), "s_per_iter": r["solve_seconds"] / args.iters,
               "peak_device_bytes": peak, "solver_device_bytes": r["device_bytes"], "handle_bytes": r["handle_bytes"],
               "estimated_bytes_beyond_handle": capi.full_game_bytes(D, F)}
        del r
        res["runs"][f"{g}f"] = run
        print(f"{g}f: {json.dumps(run)}", flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
