"""Exact exploitability of the recursive to-leaf average policy on the device walk (rela.exploitability_to_leaf) against the seed-0
Net2 (CFR, depth 2, tensor-core net, --iters iterations): wall time, subgames/s, the walk / best-response split and the peak device
memory of the call (the device's free memory polled every 5 ms from a second thread, so other processes on the device count too)
at 2x4f, 3x3f, 2x5f and 5x2f.  On the games the dense tools accept (2x4f, 3x3f) the host walk strategy_recursive_to_leaf +
exploitability_of_strategy is timed too and its best responses are compared bit for bit.  Prints the card and its power limit.

With --every_node the every-node policy's walk (rela.exploitability_recursive, a subgame re-solved at every non-terminal node) is
measured the same way, by default at 2x4f, 3x3f, 2x5f, 5x2f and 1x11f, and each game's to-leaf exploitability of the same agent is
reported beside it; --mode1 adds runs with the fp32 SIMT net (net mode 1, compute_exploitability_with_net's default) at those games.

    python scripts/expl_bench.py [--iters 1024] [--games 2x4,3x3,2x5,5x2] [--dense 2x4,3x3] [--out expl_bench.json]
    python scripts/expl_bench.py --every_node [--games 2x4,3x3,2x5,5x2,1x11] [--mode1 2x5] [--out expl_every_node.json]"""
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


def agent(rela, D, F, iters, net_mode=3):
    import torch
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.net_mode, cfg.state_dtype = D, F, net_mode, 0
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
    ap.add_argument("--games", type=str, default=None, help="default 2x4,3x3,2x5,5x2 (with --every_node also 1x11)")
    ap.add_argument("--dense", type=str, default="2x4,3x3", help="games on which the dense host walk is timed and compared")
    ap.add_argument("--wave_capacity", type=int, default=16384)
    ap.add_argument("--every_node", action="store_true", help="measure the every-node walk, with the to-leaf exploitability beside it")
    ap.add_argument("--mode1", type=str, default="2x5", help="with --every_node: games also run with net mode 1")
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if args.games is None:
        args.games = "2x4,3x3,2x5,5x2,1x11" if args.every_node else "2x4,3x3,2x5,5x2"
    import torch
    import rebel_b200.rela as rela
    from rebel_b200 import capi
    torch.cuda.init()
    res = {"card": card(), "iters": args.iters, "wave_capacity": args.wave_capacity, "runs": {}}
    dense = set(args.dense.split(",")) if args.dense else set()
    cfg, w = agent(rela, 1, 4, 64)
    rela.exploitability_to_leaf(cfg, 0, w, wave_capacity=args.wave_capacity)   # warm-up: module load
    if args.every_node:
        every_node(rela, capi, args, res)
        return
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
    report(res, args.out)


def every_node(rela, capi, args, res):
    """The every-node walk per game and net mode: call, walk and best-response times, subgames/s, peak device memory, and the
    to-leaf exploitability of the same agent."""
    runs = [(g, 3) for g in args.games.split(",")] + [(g, 1) for g in (args.mode1.split(",") if args.mode1 else [])]
    for g, mode in runs:
        D, F = (int(x) for x in g.split("x"))
        cfg, w = agent(rela, D, F, args.iters, mode)
        e, peak = peak_bytes_during(lambda: rela.exploitability_recursive(cfg, 0, w, wave_capacity=args.wave_capacity))
        leaf = rela.exploitability_to_leaf(cfg, 0, w, wave_capacity=args.wave_capacity)
        run = {"net_mode": mode, "exploitability": e["exploitability"], "br": e["br"], "subgames": e["subgames"],
               "seconds": e["seconds"], "walk_seconds": e["walk_seconds"], "br_seconds": e["br_seconds"],
               "subgames_per_s": e["subgames"] / e["walk_seconds"], "subgame_iters_per_s": e["subgame_iters"] / e["walk_seconds"],
               "peak_device_bytes": peak, "estimated_bytes_beyond_handle": capi.recursive_bytes(D, F, args.wave_capacity),
               "to_leaf_exploitability": leaf["exploitability"], "to_leaf_seconds": leaf["seconds"]}
        res["runs"][f"{g}f mode {mode}"] = run
        print(f"{g}f mode {mode}: {json.dumps(run)}", flush=True)
    report(res, args.out)


def report(res, out):
    print(json.dumps(res))
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
