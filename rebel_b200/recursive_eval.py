"""`recursive_eval` of the reference (csrc/liars_dice/recursive_eval.cc:196-425) on the GPU wave solver: the full-tree solve, the
exploitability of the reach-weighted average of `--num_repeats` sampled recursive strategies (BASELINE config 5), the EV of every
strategy against the full-tree solve, the immediate regrets (--print_regret / --print_regret_summary) and the tagged `XXX` /
`YYY` report lines that the reference's scripts/eval_all.py parses.

    python -m rebel_b200.recursive_eval --num_dice 2 --num_faces 3 --subgame_iters 1024 --cfr --mdp_depth 2 --num_repeats 4097 [--net model.ckpt]
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 -m rebel_b200.recursive_eval ...

Flags follow the reference binary (`--num_dice --num_faces --subgame_iters --mdp_depth --num_repeats --net --cfr --no_linear
--optimistic --dcfr --num_threads --print_regret --print_regret_summary`).  One process per GPU: rank r solves the contiguous
strategy_ids [r*R/W, (r+1)*R/W); the float32 partial sums are reduced to rank 0 over NCCL.  With one rank every number is
bit-identical to the reference (tests/test_rela_module.py, tests/test_eval_report.py); with several the float32 summation order
differs from the reference's strict id order (recursive_eval.cc:349-355), an O(1e-7) relative effect, and only the final
checkpoint is reported."""
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


def reduce_regrets(regret_sums, regret_count, device):
    """Sum the per-rank fp64 regret sums and counts onto rank 0; returns (immediate regrets [N, H], sums, count) there."""
    import torch.distributed as dist
    sums = regret_sums
    count = torch.tensor([float(regret_count)], dtype=torch.float64)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        sums, count = regret_sums.to(device), count.to(device)
        dist.reduce(sums, 0)
        dist.reduce(count, 0)
        sums, count = sums.cpu(), count.cpu()
    return immediate_from_sums(sums, int(count.item())), sums, int(count.item())


def immediate_from_sums(sums, count):
    """compute_immediate_regrets' read-out (subgame_solving.cc:1035-1048): max over all actions / number of strategies (the sums
    of illegal actions and of leaves stay 0)."""
    return sums.max(dim=2).values / count


def regret_summary(depths, immediate, mdp_depth):
    """report_regrets' summary (recursive_eval.cc:41-52): summed immediate regrets above mdp_depth, and of the rest."""
    top = bottom = 0.0
    for n, d in enumerate(depths):
        s = 0.0
        for v in immediate[n].tolist():
            s += v
        if d < mdp_depth:
            top += s
        else:
            bottom += s
    return top, bottom


def regret_lines(immediate, depths, mdp_depth, print_regret, print_regret_summary):
    """The text report_regrets prints (recursive_eval.cc:33-52), numbers like std::cout in fixed mode (%f)."""
    out = ""
    if print_regret:
        out += "\tRegrets: " + "".join("".join(f"{v:f} " for v in immediate[n].tolist()) + "| " for n in range(min(20, len(depths)))) + "\n"
    if print_regret_summary:
        top, bottom = regret_summary(depths, immediate, mdp_depth)
        out += f"\tRegrets (depth<={mdp_depth})/rest: {top:f}/{bottom:f}"
    return out


def tagged_line(tag, pairs):
    """One machine-readable report line of recursive_eval.cc:410-425: `TAG {"k":"v", ...}` with the values as quoted strings in
    std::to_string's %f format; the text after the tag is JSON (scripts/eval_all.py decodes it)."""
    return f"{tag} {{" + ", ".join(f"{json.dumps(k)}:{json.dumps(v if isinstance(v, str) else f'{v:f}')}" for k, v in pairs) + "}"


def load_net_weights(path):
    """Flat Net2 weights of a checkpoint: a TorchScript module saved by torch.jit.save (the released checkpoints, whatever the file
    name) or a plain state_dict saved by torch.save."""
    from rebel_b200.models import flatten_state_dict
    try:
        obj = torch.jit.load(path, map_location="cpu")
    except (RuntimeError, ValueError):
        obj = torch.load(path, map_location="cpu")
    sd = obj.state_dict() if hasattr(obj, "state_dict") else obj
    return torch.from_numpy(flatten_state_dict(sd))


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=4)
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--mdp_depth", type=int, default=2, help="depth of the recursive subgames (reference default -1 = full-tree solve only)")
    ap.add_argument("--num_repeats", type=int, default=-1, help="sampled recursive strategies to average (<= 0: skip)")
    ap.add_argument("--net", type=str, default=None,
                    help="Net2 checkpoint: a TorchScript module (any file name) or a state_dict; 'zero' or omitted = zero value net")
    ap.add_argument("--cfr", action="store_true", help="CFR instead of fictitious play (the reference's default solver is FP)")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--optimistic", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--num_threads", type=int, default=10,
                    help="ignored: accepted for the reference's command line; the subgames are solved on the GPU, not by CPU threads")
    ap.add_argument("--print_regret", action="store_true", help="CFR: immediate regrets of the first 20 nodes at every checkpoint")
    ap.add_argument("--print_regret_summary", action="store_true",
                    help="CFR: summed immediate regrets above mdp_depth / below, at every checkpoint")
    ap.add_argument("--no_full_tree", action="store_true",
                    help="skip the full-tree solve the reference binary always starts with (and the EVs against it)")
    ap.add_argument("--batch_repeats", type=int, default=64)
    ap.add_argument("--wave_capacity", type=int, default=8192)
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast fp32-tanh GELU (default with --net)")
    ap.add_argument("--random_net_seed", type=int, default=None, help="use a random-init Net2 (benchmarks)")
    return ap


def main(argv=None):
    args = build_parser().parse_args(argv)

    import rebel_b200.rela as rela
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    device = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(device)
        dist.init_process_group("nccl", device_id=device)

    weights = None
    if args.net and args.net != "zero":
        weights = load_net_weights(args.net)
    elif args.random_net_seed is not None:
        weights = torch.from_numpy(flatten_state_dict(make_selfplay_net(args.num_dice, args.num_faces, seed=args.random_net_seed).state_dict()))
    net_mode = args.net_mode if args.net_mode is not None else (3 if weights is not None else 0)
    want_regrets = args.cfr and (args.print_regret or args.print_regret_summary)   # the reference tracks them for CFR only

    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = args.num_dice, args.num_faces
    cfg.net_mode, cfg.state_dtype = net_mode, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.optimistic = args.subgame_iters, args.mdp_depth, args.cfr, args.optimistic
    sp.linear_update = not args.no_linear and args.dcfr is None                      # recursive_eval.cc:273
    if args.dcfr is not None:
        sp.dcfr, (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) = True, args.dcfr

    depths = full_tree_depths(args.num_dice, args.num_faces) if want_regrets else None
    report = []        # (name, dense strategy, (expl0, expl1), (ev0, ev1) or None) of recursive_eval.cc:394-408
    full = None
    if rank == 0 and not args.no_full_tree:
        # "Solving the game for the full tree" (recursive_eval.cc:264-309): exploitability curve at powers of two
        sp.max_depth = 100000
        f = rela.solve_full_tree(cfg, local, track_regrets=want_regrets)
        sp.max_depth = args.mdp_depth
        full = f["strategy"]
        e = f["exploitability"][-1].tolist()
        total = float(np.float32(e[0] + e[1]))
        print(f"Full {'CFR' if args.cfr else 'FP'} exploitability: {total / 2:.6e}", flush=True)
        if want_regrets:
            print(regret_lines(f["immediate_regrets"], depths, args.mdp_depth, args.print_regret, args.print_regret_summary), flush=True)
        report.append(("full_tree", full, tuple(e), rela.ev_of_strategies(args.num_dice, args.num_faces, full, full)))
    elif rank == 0:
        print("no full-tree solve (--no_full_tree): the full_tree entry and the EVs against it are not reported", flush=True)
    if args.num_repeats > 0 and args.mdp_depth > 0:
        lo, hi = strategy_ids(rank, world, args.num_repeats)
        t0 = time.time()
        r = rela.recursive_eval_sampled(cfg, local, hi - lo, seed=lo, batch_repeats=args.batch_repeats, wave_capacity=args.wave_capacity,
                                        flat_weights=weights, full_strategy=full if world == 1 else None, track_regrets=want_regrets)
        ss, sr = reduce_sums(r["summed_strategy"], r["summed_reach"], device)
        if want_regrets:
            imm, _, _ = reduce_regrets(r["regret_sums"], r["regret_count"], device)
        solved = torch.tensor([float(r["subgames_solved"]), float(r["gpu_seconds"])], dtype=torch.float64, device=device)
        if world > 1:
            dist.all_reduce(solved[:1])
            dist.all_reduce(solved[1:], op=dist.ReduceOp.MAX)
        wall = time.time() - t0
        if rank == 0:
            final = ss / (sr + 1e-6)
            e = rela.exploitability_of_strategy(args.num_dice, args.num_faces, final)
            if world == 1:
                for i, (n, x) in enumerate(zip(r["checkpoints"], r["exploitability"].tolist())):
                    print(f"{n:5d}: {(x[0] + x[1]) / 2:.6e} ({x[0]:.6e},{x[1]:.6e})")
                    extra = ""
                    if full is not None:
                        ev = r["ev_of_full"][i].tolist()
                        extra += f"\tEV of full: {(ev[0] + ev[1]) / 2:f} ({ev[0]:f},{ev[1]:f})"
                    if want_regrets and args.print_regret_summary:
                        top, bottom = r["regret_summary"][i].tolist()
                        extra += f"\tRegrets (depth<={args.mdp_depth})/rest: {top:f}/{bottom:f}"
                    if extra:
                        print(extra)
                    report.append((f"repeated toleaf {n}", None, tuple(x), tuple(r["ev_of_full"][i].tolist()) if full is not None else None))
                if want_regrets and args.print_regret:
                    print(regret_lines(imm, depths, args.mdp_depth, True, False), end="")
            else:
                ev = rela.ev_of_strategies(args.num_dice, args.num_faces, full, final.double()) if full is not None else None
                report.append((f"repeated toleaf {args.num_repeats}", None, tuple(e), ev))
                if want_regrets:
                    print(regret_lines(imm, depths, args.mdp_depth, args.print_regret, args.print_regret_summary), flush=True)
            print(json.dumps({"game": f"{args.num_dice}x{args.num_faces}f", "num_repeats": args.num_repeats, "subgame_iters": args.subgame_iters,
                              "n_gpus": world, "net_mode": net_mode, "exploitability": (e[0] + e[1]) / 2, "exploitability_p0_p1": list(e),
                              "subgames_solved": int(solved[0].item()), "wall_s": wall, "solver_s_max_over_ranks": solved[1].item(),
                              "repeats_per_s": args.num_repeats / wall}))
    if rank == 0 and report:
        print_report(report, args.net or "", full is not None)
    if world > 1:
        dist.destroy_process_group()


def full_tree_depths(num_dice, num_faces):
    """Depth of every node of the full game tree, in the reference's node order."""
    from rebel_b200 import capi
    import ctypes as C
    L = capi.lib()
    A = 1 + 2 * num_dice * num_faces
    n = (1 << A) - 1
    out = np.zeros((n, 6), np.int32)
    got = L.cfrb_unroll_tree(num_dice, num_faces, -1, 0, 1 << 30, out.ctypes.data_as(C.POINTER(C.c_int32)), n)
    assert got == n, got
    return out[:, 5].tolist()


def print_report(report, net, with_ev):
    """The per-strategy report and the two tagged lines of recursive_eval.cc:389-425."""
    res, res_ev = [("net", net)], [("net", net)]
    for name, _s, e, ev in report:
        line = f" {name} {(e[0] + e[1]) / 2.:f} ({e[0]:f},{e[1]:f})"
        if ev is not None:
            line += f"\n\tEV of full: {(ev[0] + ev[1]) / 2.:f} ({ev[0]:f},{ev[1]:f})"
            res_ev.append((name, (ev[0] + ev[1]) / 2.))
        print(line)
        res.append((name, (e[0] + e[1]) / 2.))
    print(tagged_line("XXX", res))
    if with_ev:
        print(tagged_line("YYY", res_ev))
    print(end="", flush=True)


if __name__ == "__main__":
    main()
