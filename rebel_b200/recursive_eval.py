"""`recursive_eval --cfr` of the reference (csrc/liars_dice/recursive_eval.cc:196-420) on the GPU wave solver: exploitability of
the reach-weighted average of `--num_repeats` sampled recursive strategies (BASELINE config 5).

    python -m rebel_b200.recursive_eval --num_dice 2 --num_faces 3 --subgame_iters 1024 --cfr --mdp_depth 2 --num_repeats 4097 [--net model.pt]
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 -m rebel_b200.recursive_eval ...

Flags follow the reference binary (`--num_dice --num_faces --subgame_iters --mdp_depth --num_repeats --net --cfr --no_linear`).
One process per GPU: rank r solves the contiguous strategy_ids [r*R/W, (r+1)*R/W); the float32 partial sums are reduced to
rank 0 over NCCL.  With one rank every number is bit-identical to the reference (tests/test_rela_module.py); with several the
float32 summation order differs from the reference's strict id order (recursive_eval.cc:349-355), an O(1e-7) relative effect."""
import argparse
import json
import os
import time

import numpy as np
import torch


def strategy_ids(rank, world, num_repeats):
    """Contiguous block of strategy ids (= mt19937 seeds) of `rank`: [lo, hi)."""
    lo = rank * num_repeats // world
    hi = (rank + 1) * num_repeats // world
    return lo, hi


def reduce_sums(summed_strategy, summed_reach, device, backend_device_tensors=True):
    """Sum the per-rank float32 accumulators onto rank 0 (rank order is up to the collective)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
        return summed_strategy, summed_reach
    ss, sr = summed_strategy.to(device), summed_reach.to(device)
    dist.reduce(ss, 0)
    dist.reduce(sr, 0)
    return ss.cpu(), sr.cpu()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=4)
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--mdp_depth", type=int, default=2, help="depth of the recursive subgames (reference default -1 = full-tree solve only)")
    ap.add_argument("--num_repeats", type=int, default=-1, help="sampled recursive strategies to average (<= 0: skip)")
    ap.add_argument("--net", type=str, default=None, help="TorchScript / state_dict checkpoint of Net2; omitted = zero value net")
    ap.add_argument("--cfr", action="store_true", help="CFR instead of fictitious play (the reference's default solver is FP)")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--optimistic", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--no_full_tree", action="store_true", help="skip the full-tree solve the reference binary always starts with")
    ap.add_argument("--batch_repeats", type=int, default=64)
    ap.add_argument("--wave_capacity", type=int, default=8192)
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast fp32-tanh GELU (default with --net)")
    ap.add_argument("--random_net_seed", type=int, default=None, help="use a random-init Net2 (benchmarks)")
    args = ap.parse_args(argv)

    import rebel_b200.rela as rela
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    device = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=device)

    weights = None
    if args.net:
        obj = torch.load(args.net, map_location="cpu") if not args.net.endswith(".pt_script") else torch.jit.load(args.net, map_location="cpu")
        sd = obj.state_dict() if hasattr(obj, "state_dict") else obj
        weights = torch.from_numpy(flatten_state_dict(sd))
    elif args.random_net_seed is not None:
        weights = torch.from_numpy(flatten_state_dict(make_selfplay_net(args.num_dice, args.num_faces, seed=args.random_net_seed).state_dict()))
    net_mode = args.net_mode if args.net_mode is not None else (3 if weights is not None else 0)

    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = args.num_dice, args.num_faces
    cfg.net_mode, cfg.state_dtype = net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.optimistic = args.subgame_iters, args.mdp_depth, args.cfr, args.optimistic
    sp.linear_update = not args.no_linear and args.dcfr is None                      # recursive_eval.cc:273
    if args.dcfr is not None:
        sp.dcfr, (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) = True, args.dcfr

    if rank == 0 and not args.no_full_tree:
        # "Solving the game for the full tree" (recursive_eval.cc:264-300): exploitability curve at powers of two
        sp.max_depth = 100000
        total = rela.compute_exploitability_fp(cfg)
        print(f"Full {'CFR' if args.cfr else 'FP'} exploitability: {total / 2:.6e}", flush=True)
        sp.max_depth = args.mdp_depth
    if args.num_repeats <= 0 or args.mdp_depth <= 0:
        if world > 1:
            dist.destroy_process_group()
        return

    lo, hi = strategy_ids(rank, world, args.num_repeats)
    t0 = time.time()
    r = rela.recursive_eval_sampled(cfg, local, hi - lo, seed=lo, batch_repeats=args.batch_repeats, wave_capacity=args.wave_capacity,
                                    flat_weights=weights)
    ss, sr = reduce_sums(r["summed_strategy"], r["summed_reach"], device)
    solved = torch.tensor([float(r["subgames_solved"]), float(r["gpu_seconds"])], dtype=torch.float64, device=device)
    if world > 1:
        dist.all_reduce(solved[:1])
        dist.all_reduce(solved[1:], op=dist.ReduceOp.MAX)
    wall = time.time() - t0
    if rank == 0:
        final = ss / (sr + 1e-6)
        e = rela.exploitability_of_strategy(args.num_dice, args.num_faces, final)
        if world == 1:
            for n, x in zip(r["checkpoints"], r["exploitability"].tolist()):
                print(f"{n:5d}: {(x[0] + x[1]) / 2:.6e} ({x[0]:.6e},{x[1]:.6e})")
        print(json.dumps({"game": f"{args.num_dice}x{args.num_faces}f", "num_repeats": args.num_repeats, "subgame_iters": args.subgame_iters,
                          "n_gpus": world, "net_mode": net_mode, "exploitability": (e[0] + e[1]) / 2, "exploitability_p0_p1": list(e),
                          "subgames_solved": int(solved[0].item()), "wall_s": wall, "solver_s_max_over_ranks": solved[1].item(),
                          "repeats_per_s": args.num_repeats / wall}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
