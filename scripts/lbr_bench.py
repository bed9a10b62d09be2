"""Local-best-response throughput: games/s, subgame solves/s and the what-if share of the solves of LBR against the seed-0 Net2
(CFR, 1024 iterations, depth 2, tensor-core net) at 1x6f (resident tensor-core kernel), 2x5f and optionally 2x6f (wide kernel),
each game run `--repeats` times alternately, plus the split of single rounds into the agent's wave and the walk with the wave
set-up, and the device memory of the agent's handle at the default capacity (2 subgames per slot).  The agent plays `--policy`:
the to-leaf average policy (the default) or the every-node policy; `--policy both` alternates the two in every repeat.

    python scripts/lbr_bench.py [--games_1x6 16384] [--games_2x5 2048] [--games_2x6 0] [--policy average] [--repeats 2]
                                [--out lbr_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def agent(capi, D, F, capacity, iters):
    import torch
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    S = capi.WaveSolver(D, F, capacity, max_depth=2, num_iters=iters, linear_update=True, net_mode=capi.NET_TC_F16X2,
                        solver=capi.SOLVER_CFR)
    S.set_weights(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
    S.sync()
    return S, free0 - torch.cuda.mem_get_info()[0]


POLICIES = {"average": 0, "every_node": 2}   # capi.MATCH_AVERAGE, capi.MATCH_EVERY_NODE


def timed_lbr(capi, a, slots, games, seed, policy="average"):
    a.sync()
    t0 = time.perf_counter()
    M = capi.LbrMatch(a, slots, games, seed=seed, policy=POLICIES[policy])
    r = M.play()
    dt = time.perf_counter() - t0
    M.close()
    pay = -r["payoff_a"].astype(np.float64)
    pairs = (pay[0::2] + pay[1::2]) / 2
    return {"games_per_s": games / dt, "solves_per_s": r["solves"] / dt, "whatif_share": r["whatif_solves"] / r["solves"],
            "solves_per_game": r["solves"] / games, "deferred_slot_rounds": r["deferred_slot_rounds"], "seconds": dt,
            "lbr_mean": float(pairs.mean()), "lbr_stderr": float(pairs.std(ddof=1) / np.sqrt(len(pairs))),
            "mean_plies": float(np.mean(r["plies"]))}


def round_phases(capi, a, slots, games, rounds=8, policy="average"):
    """Device time of single rounds (CUDA events on the match's stream) and of the agent's cfrb_run inside them."""
    M = capi.LbrMatch(a, slots, games, seed=99, policy=POLICIES[policy])
    out = []
    for _ in range(rounds):
        a.mark(0)
        if M.run(1) == 0:
            break
        a.mark(1)
        total = a.elapsed_ms(0, 1)
        solve = a.last_run_ms()[0]
        out.append({"round_ms": total, "solve_ms": solve, "walk_and_setup_ms": total - solve,
                    "walk_share": (total - solve) / total})
    M.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games_1x6", type=int, default=16384)
    ap.add_argument("--games_2x5", type=int, default=2048)
    ap.add_argument("--games_2x6", type=int, default=0, help="0: 2x6f is not run")
    ap.add_argument("--policy", choices=("average", "every_node", "both"), default="average")
    ap.add_argument("--slots", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    from rebel_b200 import capi
    games = {g: n for g, n in (((1, 6), args.games_1x6), ((2, 5), args.games_2x5), ((2, 6), args.games_2x6)) if n > 0}
    policies = ["every_node", "average"] if args.policy == "both" else [args.policy]
    res = {"card": card(), "iters": args.iters, "slots": args.slots, "capacity": 2 * args.slots, "policies": policies,
           "handle_bytes": {}, "runs": {}, "phases": {}}
    # keys: "1x6f" for the average policy (as before), "1x6f every_node" for the every-node one
    key = lambda g, pol: f"{g[0]}x{g[1]}f" + ("" if pol == "average" else " " + pol)
    pools = {}
    for g in games:
        pools[g], res["handle_bytes"][f"{g[0]}x{g[1]}f"] = agent(capi, g[0], g[1], 2 * args.slots, args.iters)
    for g, a in pools.items():           # warm-up: module load, CUDA graphs
        for pol in policies:
            timed_lbr(capi, a, args.slots, 1024, seed=1000, policy=pol)
    for rep in range(args.repeats):
        for g, a in pools.items():
            for pol in policies:
                r = timed_lbr(capi, a, args.slots, games[g], seed=rep, policy=pol)
                res["runs"].setdefault(key(g, pol), []).append(r)
                print(f"{key(g, pol)} run {rep}: {json.dumps(r)}", flush=True)
    for g, a in pools.items():
        for pol in policies:
            ph = round_phases(capi, a, args.slots, games[g], policy=pol)
            res["phases"][key(g, pol)] = ph
            print(f"{key(g, pol)} rounds: {json.dumps(ph)}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
