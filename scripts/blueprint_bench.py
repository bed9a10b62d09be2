"""Blueprint throughput at 1x6f and 2x5f: games/s of blueprint against blueprint, of the seed-0 Net2 agent (CFR, 1024 iterations,
depth 2, tensor-core net, `--policy`) against a blueprint (with its solves/s), and of LBR against a blueprint; plus the
blueprint's device memory, by the formula and as measured.  The blueprint is the full-game CFR solve (`solve_game`, `--solve_iters`
iterations).  Each run is repeated `--repeats` times, alternating the games; the card and its power limit are read in the same run.

    python scripts/blueprint_bench.py [--games_bp 262144] [--games_agent_1x6 16384] [--games_agent_2x5 2048] [--games_lbr 65536]
                                      [--repeats 2] [--out blueprint_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


POLICIES = {"average": 0, "sampled": 1, "every_node": 2}   # capi.MATCH_*


def timed(run):
    t0 = time.perf_counter()
    r = run()
    return r, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games_bp", type=int, default=1 << 18, help="games of blueprint against blueprint")
    ap.add_argument("--games_agent_1x6", type=int, default=16384)
    ap.add_argument("--games_agent_2x5", type=int, default=2048)
    ap.add_argument("--games_lbr", type=int, default=1 << 16)
    ap.add_argument("--policy", choices=tuple(POLICIES), default="sampled", help="the agent's policy")
    ap.add_argument("--solve_iters", type=int, default=1024)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--slots", type=int, default=8192)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import torch
    from rebel_b200 import capi
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    S_ = args.slots
    res = {"card": card(), "solve_iters": args.solve_iters, "iters": args.iters, "slots": S_, "policy": args.policy, "games": {}}
    setups = {}
    for D, F in ((1, 6), (2, 5)):
        key = f"{D}x{F}f"
        fg = capi.FullGame(D, F)
        fg.step(args.solve_iters)
        expl = float(sum(fg.exploitability()) / 2)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        bp = capi.Blueprint.from_full_game(fg)
        torch.cuda.synchronize()
        measured = free0 - torch.cuda.mem_get_info()[0]
        fg.close()
        agent = capi.WaveSolver(D, F, S_, max_depth=2, num_iters=args.iters, linear_update=True, net_mode=capi.NET_TC_F16X2,
                                solver=capi.SOLVER_CFR)
        agent.set_weights(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
        agent.sync()
        setups[key] = (bp, agent, args.games_agent_1x6 if (D, F) == (1, 6) else args.games_agent_2x5)
        res["games"][key] = {"blueprint_bytes": capi.blueprint_bytes(D, F), "blueprint_bytes_measured": int(measured),
                             "blueprint_exploitability": expl, "runs": []}
    pol = POLICIES[args.policy]

    def runs(key, bp, agent, n_agent, seed, games_bp, games_lbr):
        out = {}
        r, dt = timed(lambda: capi.Match(bp, bp, S_, games_bp, seed=seed).play())
        out["bp_vs_bp_games_per_s"] = games_bp / dt
        r, dt = timed(lambda: capi.Match(agent, bp, S_, n_agent, seed=seed, policy=pol).play())
        out["agent_vs_bp_games_per_s"], out["agent_vs_bp_solves_per_s"] = n_agent / dt, r["solves_a"] / dt
        out["agent_vs_bp_mean"] = float(r["payoff_a"].mean())
        r, dt = timed(lambda: capi.LbrMatch(bp, S_, games_lbr, seed=seed).play())
        out["lbr_vs_bp_games_per_s"], out["lbr_vs_bp_mean"] = games_lbr / dt, float(-r["payoff_a"].mean())
        assert r["solves"] == 0
        return out

    for key, (bp, agent, n) in setups.items():   # warm-up: module load, CUDA graphs
        runs(key, bp, agent, 512, 1000, 8192, 8192)
    for rep in range(args.repeats):
        for key, (bp, agent, n) in setups.items():
            r = runs(key, bp, agent, n, rep, args.games_bp, args.games_lbr)
            res["games"][key]["runs"].append(r)
            print(f"{key} run {rep}: {json.dumps(r)}", flush=True)
    for bp, agent, _ in setups.values():
        bp.close()
        agent.close()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
