"""Depth-2 CFR kernel time per launch, measured the way bench.py measures it (CUDA-event pairs around every 16th value-net launch;
the rest of a run's device time is the CFR kernel), for
  (a) host waves of 1x6f root subgames (--host-sizes, 1024 iterations, tensor-core net); one root is the length of one warp's chain,
  (b) bench.py's stationary self-play loop (8192 games, the bench's seeds, 20 warm-up waves, L2 flush before each wave).
--wide lists the wide-group settings to run (cfrb_debug_d2_wide: -1 = the wave's own rule, 0 = off, m > 0 = the m costliest
solved subgames on whole CTAs), so the script also sweeps m.  One JSON line per measurement, with the card, power limit and clocks."""
import argparse, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:   # the numbers are still worth printing without the card's description
        return f"unknown ({e})"


def set_wide(S, m):
    if hasattr(S, "debug_d2_wide"):
        S.debug_d2_wide(m)
    elif m != -1:
        raise SystemExit("this build has no wide groups (cfrb_debug_d2_wide)")


def host_wave(rb, w, iters, m, reps, n=1):
    S = rb.WaveSolver(1, 6, n, num_iters=iters, net_mode=rb.NET_TC_F16X2)
    S.set_weights(w, version=1)
    set_wide(S, m)
    H = S.H
    b = np.full((n, 2, H), 1.0 / H)
    out = []
    for r in range(reps + 1):              # the first run warms up (module load, graph capture)
        S.begin(np.full(n, -1, np.int32), np.zeros(n, np.int32), b)
        S.set_profiling(16)
        S.run(iters)
        S.sync()
        tot, net = S.last_run_ms()
        if r:
            out.append((tot, net))
    taken = S.wave_wide if hasattr(S, "wave_wide") else None
    S.close()
    tot = np.array([o[0] for o in out]); net = np.array([o[1] for o in out])
    return {"cfr_us": float(np.median((tot - net) / iters * 1e3)), "net_us": float(np.median(net / iters * 1e3)),
            "wave_ms": [round(float(x), 3) for x in tot], "wide_taken": taken}


def selfplay(rb, w, K, iters, m, warmup, waves):
    S = rb.WaveSolver(1, 6, K, num_iters=iters, net_mode=rb.NET_TC_F16X2)
    S.set_weights(w, version=1)
    set_wide(S, m)
    S.selfplay_create(np.arange(K, dtype=np.uint32) * np.uint32(1000000))
    for _ in range(warmup):
        S.l2_flush()
        S.selfplay_wave(start_next=True)
    S.selfplay_wave(start_next=False)
    S.sync()
    S.set_profiling(16)
    tot, net, solved, roots = [], [], [], 0
    for _ in range(waves):
        S.l2_flush()
        S.selfplay_wave(start_next=True)
        S.sync()
        a, b = S.last_run_ms()
        tot.append(a); net.append(b); solved.append(S.wave_solved)
        lb, _ = S.wave_roots()
        roots = roots + np.bincount(lb + 1, minlength=S.A)
    S.set_profiling(0)
    S.selfplay_wave(start_next=False)
    S.sync()
    S.close()
    tot, net = np.array(tot), np.array(net)
    return {"cfr_us": float(((tot - net).sum()) / (waves * iters) * 1e3), "net_us": float(net.sum() / (waves * iters) * 1e3),
            "wave_ms": [round(float(x), 2) for x in tot], "solved_mean": float(np.mean(solved)),
            "games_per_root_bid": (roots / waves).round(1).tolist()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--wide", default="-1", help="comma-separated cfrb_debug_d2_wide settings")
    ap.add_argument("--games", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--waves", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-host", action="store_true")
    ap.add_argument("--host-sizes", default="1", help="comma-separated root subgames of the host waves of case (a)")
    args = ap.parse_args()
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    w = flatten_state_dict(make_selfplay_net(1, 6, seed=0).state_dict())
    card = gpu_info()
    print(json.dumps({"gpu": card, "note": "name, power limit, SM clock, max SM clock"}), flush=True)
    for m in [int(x) for x in args.wide.split(",")]:
        for n in ([] if args.skip_host else [int(x) for x in args.host_sizes.split(",")]):
            r = host_wave(rb, w, args.iters, m, args.reps, n)
            print(json.dumps({"case": f"a: host wave, {n} 1x6f roots", "wide": m, **r}), flush=True)
        r = selfplay(rb, w, args.games, args.iters, m, args.warmup, args.waves)
        print(json.dumps({"case": f"b: stationary self-play, {args.games} games", "wide": m, **r}), flush=True)
    print(json.dumps({"gpu_after": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
