"""recursive_eval's sampled evaluation on the device walk (rela.recursive_eval_to_leaf) against the seed-0 Net2 (CFR, depth 2,
tensor-core net mode 3, --iters iterations): repeats/s, subgames/s, the draws / walk / best-response split and the peak device
memory of the call (the device's free memory polled every 5 ms from a second thread, so other processes on the device count too).
On the games the host walk accepts (--host, default 2x4f) rela.recursive_eval_sampled is timed on the same repeats and its sums,
checkpoint exploitabilities and iteration count are compared bit for bit.  Prints the card, its power limit and its clocks.

    python scripts/recursive_eval_bench.py [--iters 1024] [--games 2x4:8,2x5:2,5x2:2] [--host 2x4] [--out recursive_eval_bench.json]

A game is DxF:R (R repeats)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from expl_bench import agent, peak_bytes_during  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def same_bits(host, dev, D, F):
    """The host walk's dense sums at the legal entries, its checkpoints and iteration count: the device walk's bits."""
    import ctypes as C
    import numpy as np
    from rebel_b200 import capi
    A = 2 * D * F + 1
    tree = np.zeros(((1 << A) - 1, 6), np.int32)   # the full tree: (last_bid, player, children_begin, children_end, parent, depth)
    capi._check(capi.lib().cfrb_unroll_tree(D, F, -1, 0, 1 << 30, tree.ctypes.data_as(C.POINTER(C.c_int32)), tree.shape[0]))
    ss = np.ascontiguousarray(host["summed_strategy"].numpy()[tree[1:, 4], :, tree[1:, 0]])
    return (dev["checkpoints"] == host["checkpoints"] and dev["subgame_iters"] == host["subgame_iters"]
            and np.array_equal(dev["exploitability"].numpy().view(np.uint64), host["exploitability"].numpy().view(np.uint64))
            and np.array_equal(dev["summed_reach"].numpy().view(np.uint32), host["summed_reach"].numpy()[:, :, 0].view(np.uint32))
            and np.array_equal(dev["summed_strategy"].numpy().view(np.uint32), ss.view(np.uint32)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--games", type=str, default="2x4:8,2x5:2,5x2:2")
    ap.add_argument("--host", type=str, default="2x4", help="games on which the host walk is timed and compared")
    ap.add_argument("--wave_capacity", type=int, default=16384)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import torch
    import rebel_b200.rela as rela
    from rebel_b200 import capi
    torch.cuda.init()
    res = {"card": card(), "iters": args.iters, "wave_capacity": args.wave_capacity, "runs": {}}
    host = set(args.host.split(",")) if args.host else set()
    cfg, w = agent(rela, 1, 4, 64)
    rela.recursive_eval_to_leaf(cfg, 0, 2, flat_weights=w, wave_capacity=args.wave_capacity)   # warm-up: module load
    for spec in args.games.split(","):
        g, reps = spec.split(":")
        reps = int(reps)
        D, F = (int(x) for x in g.split("x"))
        cfg, w = agent(rela, D, F, args.iters)
        cmp = g in host
        r, peak = peak_bytes_during(lambda: rela.recursive_eval_to_leaf(cfg, 0, reps, flat_weights=w, wave_capacity=args.wave_capacity,
                                                                        return_sums=cmp))
        e = r["exploitability"].tolist()
        run = {"repeats": reps, "batch_repeats": r["batch_repeats"], "checkpoints": r["checkpoints"],
               "exploitability": [(x[0] + x[1]) / 2 for x in e], "subgames": r["subgames"], "subgame_iters": r["subgame_iters"],
               "seconds": r["seconds"], "draw_seconds": r["draw_seconds"], "walk_seconds": r["walk_seconds"],
               "br_seconds": r["br_seconds"], "repeats_per_s": reps / r["seconds"], "seconds_per_repeat": r["seconds"] / reps,
               "subgames_per_s": r["subgames"] / r["walk_seconds"], "peak_device_bytes": peak,
               "estimated_bytes_beyond_handle": capi.to_leaf_sampled_bytes(D, F, 2, args.wave_capacity, r["batch_repeats"])}
        if cmp:
            import time
            t0 = time.perf_counter()
            h = rela.recursive_eval_sampled(cfg, 0, reps, seed=0, batch_repeats=64, wave_capacity=8192, flat_weights=w)
            t1 = time.perf_counter()
            run["host"] = {"seconds": t1 - t0, "repeats_per_s": reps / (t1 - t0), "bit_identical": bool(same_bits(h, r, D, F))}
            del h
        res["runs"][f"{g}f"] = run
        print(f"{g}f: {json.dumps(run)}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
