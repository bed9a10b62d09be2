"""rela.Agent throughput against a uniform-random legal opponent driven from Python: seed-0 Net2, CFR, 1024 iterations, depth 2,
sampled policy, tensor-core net (mode 3), 8192 tables, at 1x6f (resident tensor-core kernel) and 2x5f (wide kernel).  Each round
is ONE step call serving every running table: the agent's own moves and the opponent's moves it observes.  Reports decisions/s
(the agent's own moves), solves/s, the share of call time outside the solves (id / action copies, scan / begin / capture / step
kernels, the sync: host wall time of the calls minus the CUDA-event time of the solves), and the median latency of one decision
at one table at 1x6f, the case of the interactive CLI.

    python scripts/agent_bench.py [--tables 8192] [--iters 1024] [--batches 3] [--latency_decisions 200] [--out agent_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def make_agent(rela, D, F, tables, iters, seed=0):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, 3, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, 2, True, True
    w = torch.from_numpy(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
    return rela.Agent(cfg, 0, tables, "sampled", seed=seed, flat_weights=w)


def play(ag, n, rng, key0):
    """n games on tables 0..n-1 to their ends, one step call per round; the agent sits in seat g % 2."""
    A, H = ag.num_actions, ag.num_hands
    ids = np.arange(n, dtype=np.int32)
    seats = (ids % 2).astype(np.int32)
    ag.new_games(ids, seats, rng.randint(0, H, size=n).astype(np.int32), keys=np.arange(key0, key0 + n))
    lb, player = np.full(n, -1), np.zeros(n, np.int64)
    running = np.ones(n, bool)
    c0 = ag.counts()
    wall = decisions = actions = calls = 0
    while running.any():
        live = np.flatnonzero(running).astype(np.int32)
        lo = np.where(lb[live] < 0, 0, lb[live] + 1)
        hi = np.where(lb[live] < 0, A - 1, A)
        mine = player[live] == seats[live]
        acts = np.where(mine, -1, lo + (rng.rand(len(live)) * (hi - lo)).astype(np.int64)).astype(np.int32)
        t0 = time.perf_counter()
        played, _, done = ag.step(live, acts)
        wall += time.perf_counter() - t0
        played, done = played.numpy(), done.numpy()
        decisions += int(mine.sum()); actions += len(live); calls += 1
        lb[live], player[live] = played, player[live] ^ 1
        running[live[done]] = False
    c1 = ag.counts()
    solves, solve_ms = c1["solves"] - c0["solves"], c1["solve_ms"] - c0["solve_ms"]
    return {"games": n, "calls": calls, "actions": actions, "decisions": decisions, "solves": solves, "seconds": wall,
            "decisions_per_s": decisions / wall, "solves_per_s": solves / wall, "actions_per_s": actions / wall,
            "solve_ms": solve_ms, "outside_solve_share": 1 - solve_ms / (1000 * wall)}


def latency(rela, D, F, iters, decisions, rng):
    """Wall time of the step calls in which the agent decides, at one table (solve included when the table is at a root)."""
    ag = make_agent(rela, D, F, 1, iters)
    A, H = ag.num_actions, ag.num_hands
    times, g = [], 0
    while len(times) < decisions:
        ag.new_games([0], [g % 2], [int(rng.randint(H))], keys=[g])
        lb, player = -1, 0
        while True:
            if player == g % 2:
                t0 = time.perf_counter()
                a, _, done = ag.step([0], [-1])
                times.append(time.perf_counter() - t0)
            else:
                a, _, done = ag.step([0], [int(rng.randint(0 if lb < 0 else lb + 1, A - 1 if lb < 0 else A))])
            lb, player = int(a[0]), player ^ 1
            if bool(done[0]):
                break
        g += 1
    ag.close()
    t = np.array(times[:decisions]) * 1000
    return {"decisions": decisions, "median_ms": float(np.median(t)), "p90_ms": float(np.percentile(t, 90))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--batches", type=int, default=3, help="timed batches of `tables` games per game")
    ap.add_argument("--latency_decisions", type=int, default=200)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import rebel_b200.rela as rela
    rng = np.random.RandomState(0)
    res = {"card": card(), "iters": args.iters, "tables": args.tables, "runs": {}}
    key = 0
    print(f"card (name, power limit): {res['card']}", flush=True)
    for D, F in ((1, 6), (2, 5)):
        ag = make_agent(rela, D, F, args.tables, args.iters)
        play(ag, 256, rng, 1 << 40)                       # warm-up: module load, the handle's CUDA graph
        for _ in range(args.batches):
            r = play(ag, args.tables, rng, key)
            key += args.tables
            res["runs"].setdefault(f"{D}x{F}f", []).append(r)
            print(f"{D}x{F}f: {json.dumps(r)}", flush=True)
        ag.close()
    res["latency_1x6f"] = latency(rela, 1, 6, args.iters, args.latency_decisions, rng)
    print(f"1x6f one table: {json.dumps(res['latency_1x6f'])}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
