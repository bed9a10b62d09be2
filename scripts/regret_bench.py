"""Immediate regrets of full-tree CFR solves on the whole GPU (cfrb_full_game_track_regrets, capi.FullGame.track_regrets).

1. Per strategy, on the games the one-CTA solver runs (2x4f, 3x3f): the dense accumulator (cfrb_regrets_add_current after each
   even iteration of a one-subgame WaveSolver at the root, one CTA per traverser) against the grid-wide compact pass, alternated in
   one process after a warm-up of both.  The dense figure times each add_current call up to a device synchronise; the grid figure
   is the extra time of FullGame iterations with tracking over the same iterations without, per strategy added (the
   first two iterations, which capture the CUDA graphs, are not timed).  The
   immediate regrets of both paths after the same iterations are compared bit for bit.
2. Per game (2x4f, 3x3f, 2x5f, 5x2f, 1x11f): a --iters iteration linear-CFR solve with its checkpoints (rela.solve_full_game),
   without and with track_regrets, and the added time and device memory.
3. recursive_eval --full_game's device walk on 2x5f (seed-0 Net2, net mode 3, depth 2, compact EV baseline): the walk's seconds
   per repeat without and with track_regrets.

Prints the card, its power limit and its maximum SM clock before and after.

    python scripts/regret_bench.py [--iters 1024] [--games 2x4,3x3,2x5,5x2,1x11] [--cmp 2x4,3x3] [--cmp_iters 64] [--out regret.json]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from full_game_bench import card, cfg_of, peak_bytes_during  # noqa: E402


def dense_per_strategy(capi, D, F, iters):
    """(seconds of each cfrb_regrets_add_current, immediate regrets [N, H]) over `iters` iterations of the one-CTA solver."""
    H = F ** D
    L = capi.lib()
    one = capi.WaveSolver(D, F, 1, max_depth=100000, num_iters=iters, net_mode=capi.NET_ZERO)
    one.begin([-1], [0], np.full((1, 2, H), 1.0 / H))
    capi._check(L.cfrb_regrets_reset(one._h))
    times = []
    for i in range(iters):
        one.run(1)
        if i % 2 == 0:
            one.sync()
            t0 = time.perf_counter()
            capi._check(L.cfrb_regrets_add_current(one._h))
            one.sync()
            times.append(time.perf_counter() - t0)
    N = capi._check(L.cfrb_full_tree_nodes(one._h))
    imm = np.zeros((N, H))
    capi._check(L.cfrb_regrets_fetch(one._h, capi._p(imm, capi._dp), None, None))
    one.close()
    return times, imm


def grid_step_seconds(capi, D, F, iters, track):
    """(seconds of the last iters - 2 of `iters` FullGame iterations, immediate regrets or None); the first two capture the graphs."""
    g = capi.FullGame(D, F)
    if track:
        g.track_regrets()
    g.step(2)
    t0 = time.perf_counter()
    g.step(iters - 2)
    s = time.perf_counter() - t0
    imm = g.regrets()[0] if track else None
    g.close()
    return s, imm


def compare(capi, D, F, iters, reps):
    dense_per_strategy(capi, D, F, 4)                      # warm-up of both paths (module load, graph captures)
    grid_step_seconds(capi, D, F, 4, True)
    dense, grid, same = [], [], True
    for _ in range(reps):
        times, imm_dense = dense_per_strategy(capi, D, F, iters)
        dense.append(float(np.median(times)))
        plain, _ = grid_step_seconds(capi, D, F, iters, False)
        tracked, imm_grid = grid_step_seconds(capi, D, F, iters, True)
        grid.append((tracked - plain) / ((iters - 2) // 2))
        same = same and np.array_equal(imm_dense, imm_grid)
    return {"dense_s_per_strategy": dense, "grid_s_per_strategy": grid, "speedup": min(dense) / max(min(grid), 1e-9),
            "bit_identical": bool(same), "iters": iters}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--games", type=str, default="2x4,3x3,2x5,5x2,1x11", help="games solved in full without and with regrets")
    ap.add_argument("--cmp", type=str, default="2x4,3x3", help="games on which the dense accumulator is timed against the grid pass")
    ap.add_argument("--cmp_iters", type=int, default=64)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--walk", type=str, default="2x5", help="games on which recursive_eval --full_game's walk is timed")
    ap.add_argument("--walk_repeats", type=int, default=1)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import torch
    import rebel_b200.rela as rela
    from rebel_b200 import capi
    torch.cuda.init()
    res = {"card": card(), "iters": args.iters, "runs": {}, "compare": {}}
    rela.solve_full_game(cfg_of(rela, 1, 4, 64), 0, track_regrets=True)      # warm-up: module load
    for g in args.cmp.split(",") if args.cmp else []:
        D, F = (int(x) for x in g.split("x"))
        c = compare(capi, D, F, args.cmp_iters, args.reps)
        res["compare"][f"{g}f"] = c
        print(f"{g}f compare: {json.dumps(c)}", flush=True)
    for g in args.games.split(",") if args.games else []:
        D, F = (int(x) for x in g.split("x"))
        run = {}
        for track in (False, True):
            r, peak = peak_bytes_during(lambda: rela.solve_full_game(cfg_of(rela, D, F, args.iters), 0, track_regrets=track))
            e = r["exploitability"][-1].tolist()
            k = "regrets" if track else "plain"
            run[k] = {"seconds": r["seconds"], "solve_seconds": r["solve_seconds"], "br_seconds": r["br_seconds"],
                      "exploitability": (e[0] + e[1]) / 2, "peak_device_bytes": peak}
            if track:
                run[k]["regret_summary"] = list(r["regret_summary"])
                run[k]["max_immediate_regret"] = r["immediate_regrets"].max().item()
            del r
        run["added_seconds"] = run["regrets"]["solve_seconds"] - run["plain"]["solve_seconds"]
        run["added_s_per_strategy"] = run["added_seconds"] / (args.iters // 2)
        run["regret_bytes"] = capi.full_game_regret_bytes(D, F)
        res["runs"][f"{g}f"] = run
        print(f"{g}f: {json.dumps(run)}", flush=True)
    for g in args.walk.split(",") if args.walk else []:
        # recursive_eval --full_game's walk: the seed-0 Net2, net mode 3, depth 2, one repeat per batch, without and with regrets
        from rebel_b200.models import flatten_state_dict, make_selfplay_net
        import torch as _t
        D, F = (int(x) for x in g.split("x"))
        w = _t.from_numpy(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
        full = rela.solve_full_game(cfg_of(rela, D, F, args.iters), 0)["strategy"]
        cfg = cfg_of(rela, D, F, args.iters)
        cfg.net_mode, cfg.subgame_params.max_depth = 3, 2
        walk = {}
        for track in (False, True):
            r = rela.recursive_eval_to_leaf(cfg, 0, args.walk_repeats, seed=0, flat_weights=w, batch_repeats=1, full_strategy=full,
                                            track_regrets=track)
            walk["regrets" if track else "plain"] = {"s_per_repeat": r["walk_seconds"] / args.walk_repeats,
                                                     "seconds": r["seconds"], "ev_of_full": r["ev_of_full"][-1].tolist()}
        walk["added_s_per_repeat"] = walk["regrets"]["s_per_repeat"] - walk["plain"]["s_per_repeat"]
        res["walk"] = {f"{g}f": walk}
        print(f"{g}f walk: {json.dumps(walk)}", flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
