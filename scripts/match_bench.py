"""Head-to-head match throughput: games/s, subgame solves/s and subgame-iters/s of seed-0 Net2 against seed-1 Net2 (CFR, 1024
iterations, depth 2, sampled policy, tensor-core net) at 1x6f (resident tensor-core kernel) and 2x5f (wide kernel), each game run
`--repeats` times alternately, plus the phase split of one round (the two agents' waves vs the walk and wave set-up).
--policy_a / --policy_b pick the agents' policies (sampled, average, every_node); a pair other than two equal to-leaf policies
plays one ply per round (cfrb_match_create2).

    python scripts/match_bench.py [--games_1x6 16384] [--games_2x5 4096] [--repeats 2] [--policy_a sampled] [--policy_b sampled]
        [--out match_bench.json]"""
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


def agents(capi, D, F, slots, iters):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    out = []
    for seed in (0, 1):
        S = capi.WaveSolver(D, F, slots, max_depth=2, num_iters=iters, linear_update=True, net_mode=capi.NET_TC_F16X2,
                            solver=capi.SOLVER_CFR)
        S.set_weights(flatten_state_dict(make_selfplay_net(D, F, seed=seed).state_dict()))
        out.append(S)
    return out


POLICIES = {"average": 0, "sampled": 1, "every_node": 2}   # capi.MATCH_*


def timed_match(capi, a, b, slots, games, seed, policies=(1, 1)):
    a.sync()
    t0 = time.perf_counter()
    M = capi.Match(a, b, slots, games, seed=seed, policy=policies[0], policy_b=policies[1])
    r = M.play()
    dt = time.perf_counter() - t0
    M.close()
    return {"games_per_s": games / dt, "solves_per_s": r["solves"] / dt, "solves_a_per_s": r["solves_a"] / dt,
            "solves_b_per_s": r["solves_b"] / dt, "subgame_iters_per_s": r["subgame_iters"] / dt,
            "seconds": dt, "mean_payoff_a": float(np.mean(r["payoff_a"])), "mean_plies": float(np.mean(r["plies"]))}


def round_phases(capi, a, b, slots, games, rounds=6, policies=(1, 1)):
    """Device time of single rounds (CUDA events on the match's stream) and of each agent's cfrb_run inside them."""
    M = capi.Match(a, b, slots, games, seed=99, policy=policies[0], policy_b=policies[1])
    out = []
    for _ in range(rounds):
        a.mark(0)
        if M.run(1) == 0:
            break
        a.mark(1)
        total = a.elapsed_ms(0, 1)
        solve = a.last_run_ms()[0] + b.last_run_ms()[0]
        out.append({"round_ms": total, "solve_ms": solve, "walk_and_setup_ms": total - solve})
    M.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games_1x6", type=int, default=16384)
    ap.add_argument("--games_2x5", type=int, default=4096)
    ap.add_argument("--slots", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--policy_a", choices=tuple(POLICIES), default="sampled")
    ap.add_argument("--policy_b", choices=tuple(POLICIES), default="sampled")
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    pols = (POLICIES[args.policy_a], POLICIES[args.policy_b])
    from rebel_b200 import capi
    games = {(1, 6): args.games_1x6, (2, 5): args.games_2x5}
    pools = {g: agents(capi, g[0], g[1], args.slots, args.iters) for g in games}
    res = {"card": card(), "iters": args.iters, "slots": args.slots, "policy_a": args.policy_a, "policy_b": args.policy_b,
           "runs": {}, "phases": {}}
    for g, (a, b) in pools.items():      # warm-up: module load, CUDA graphs of both agents
        timed_match(capi, a, b, args.slots, 2 * args.slots, seed=1000, policies=pols)
    for rep in range(args.repeats):
        for g, (a, b) in pools.items():
            r = timed_match(capi, a, b, args.slots, games[g], seed=rep, policies=pols)
            res["runs"].setdefault(f"{g[0]}x{g[1]}f", []).append(r)
            print(f"{g[0]}x{g[1]}f run {rep}: {json.dumps(r)}", flush=True)
    for g, (a, b) in pools.items():
        ph = round_phases(capi, a, b, args.slots, games[g], policies=pols)
        res["phases"][f"{g[0]}x{g[1]}f"] = ph
        print(f"{g[0]}x{g[1]}f rounds: {json.dumps(ph)}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
