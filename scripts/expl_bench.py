"""Exact exploitability of the recursive to-leaf average policy on the device walk (rela.exploitability_to_leaf) against the seed-0
Net2 (CFR, depth 2, tensor-core net, --iters iterations): wall time, subgames/s, the walk / best-response split and the peak device
memory of the call (the device's free memory polled every 5 ms from a second thread, so other processes on the device count too)
at 2x4f, 3x3f, 2x5f and 5x2f.  On the games the dense tools accept (2x4f, 3x3f) the host walk strategy_recursive_to_leaf +
exploitability_of_strategy is timed too and its best responses are compared bit for bit.  Prints the card and its power limit.

    python scripts/expl_bench.py [--iters 1024] [--games 2x4,3x3,2x5,5x2] [--dense 2x4,3x3] [--out expl_bench.json]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip()
    except OSError:
        return "unknown"


def agent(rela, D, F, iters):
    import torch
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, 3, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, 2, True, True
    return cfg, torch.from_numpy(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1024)
    ap.add_argument("--games", type=str, default="2x4,3x3,2x5,5x2")
    ap.add_argument("--dense", type=str, default="2x4,3x3", help="games on which the dense host walk is timed and compared")
    ap.add_argument("--wave_capacity", type=int, default=16384)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    import torch
    import rebel_b200.rela as rela
    from rebel_b200 import capi
    torch.cuda.init()
    res = {"card": card(), "iters": args.iters, "wave_capacity": args.wave_capacity, "runs": {}}
    dense = set(args.dense.split(",")) if args.dense else set()
    cfg, w = agent(rela, 1, 4, 64)
    rela.exploitability_to_leaf(cfg, 0, w, wave_capacity=args.wave_capacity)   # warm-up: module load
    for g in args.games.split(","):
        D, F = (int(x) for x in g.split("x"))
        cfg, w = agent(rela, D, F, args.iters)
        e, peak = peak_bytes_during(lambda: rela.exploitability_to_leaf(cfg, 0, w, wave_capacity=args.wave_capacity))
        run = {"exploitability": e["exploitability"], "br": e["br"], "subgames": e["subgames"], "seconds": e["seconds"],
               "walk_seconds": e["walk_seconds"], "br_seconds": e["br_seconds"], "subgames_per_s": e["subgames"] / e["walk_seconds"],
               "subgame_iters_per_s": e["subgame_iters"] / e["walk_seconds"], "peak_device_bytes": peak,
               "estimated_bytes_beyond_handle": capi.to_leaf_bytes(D, F, 2, args.wave_capacity)}
        if g in dense:
            t0 = time.perf_counter()
            s = rela.strategy_recursive_to_leaf(cfg, 0, w)
            t1 = time.perf_counter()
            br = rela.exploitability_of_strategy(D, F, s)
            t2 = time.perf_counter()
            run["dense"] = {"seconds": t2 - t0, "walk_seconds": t1 - t0, "br_seconds": t2 - t1, "br": list(br),
                            "bit_identical": list(br) == e["br"]}
            del s
        res["runs"][f"{g}f"] = run
        print(f"{g}f: {json.dumps(run)}", flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
