"""How much of a self-play wave is one shared solve: the initial-state games (no bid yet, player 0, every belief bitwise 1 / H)
of every wave of bench.py's datagen loop (same game, games per GPU, iterations, value net and seeds), after the same warm-up.
A wave solves its non-initial games and one initial-state game; the others take that solve's results.  One JSON line per wave,
then a summary line."""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dice", type=int, default=1)
    ap.add_argument("--faces", type=int, default=6)
    ap.add_argument("--games", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=20, help="waves before the counted ones (bench.py: WARMUP_WAVES)")
    ap.add_argument("--steps", type=int, default=20, help="waves counted")
    args = ap.parse_args()
    import rebel_b200 as rb
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    D, F, K = args.dice, args.faces, args.games
    H = F ** D
    S = rb.WaveSolver(D, F, K, num_iters=args.iters, net_mode=rb.NET_TC_F16X2)
    S.set_weights(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()), version=1)
    S.selfplay_create(np.arange(K, dtype=np.uint32) * np.uint32(1000000))
    uniform = np.float64(1.0) / np.float64(H)
    for _ in range(args.warmup):
        S.selfplay_wave()
    counts = []
    for i in range(args.steps):
        S.selfplay_wave()
        lb, pl, bel = S.selfplay_state()
        init = int(((lb == -1) & (pl == 0) & np.all(bel.view(np.uint64) == uniform.view(np.uint64), axis=(1, 2))).sum())
        solved = S.wave_solved
        counts.append((init, solved))
        print(json.dumps({"wave": args.warmup + i, "games": K, "initial_state": init, "solved": solved}), flush=True)
    S.selfplay_wave(start_next=False)
    S.sync()
    S.close()
    init = np.array([c[0] for c in counts]); solved = np.array([c[1] for c in counts])
    print(json.dumps({"summary": f"{D}x{F}f, {K} games, waves {args.warmup}..{args.warmup + args.steps - 1}",
                      "initial_state_mean": float(init.mean()), "initial_state_min": int(init.min()), "initial_state_max": int(init.max()),
                      "initial_share": float(init.mean() / K), "solved_mean": float(solved.mean())}), flush=True)


if __name__ == "__main__":
    main()
