"""Solve a whole Liar's Dice game with CFR or fictitious play on the GPU (rela.solve_full_game): the full-tree solve that
`recursive_eval` starts with, its (node, hand) entries spread over every SM, for games of up to 23 actions (2x5f, 5x2f, 1x10f,
1x11f besides the games `recursive_eval` solves itself).

    python -m rebel_b200.solve_game --num_dice 2 --num_faces 5 --subgame_iters 1024 --cfr [--no_linear] [--dcfr A B G] [--optimistic]

Prints the reference's `Iter=... exploitabilities=(...) sum=...` line at every power of two and at the last iteration, then one
`SOLVE {...}` JSON line: the game, the solver settings, the final best-response pair and exploitability, the time of the whole
call, of the iterations and of the best responses, and the device memory the solver took.  Flags follow `recursive_eval`; the
solver is fictitious play unless --cfr is given, linear unless --no_linear or --dcfr.  --save PATH writes the final average
strategy as a blueprint file (rebel_b200.blueprint) for `head_to_head --blueprint_a / _b`, `local_br --blueprint` and
`play --blueprint`, and the SOLVE line adds "saved": PATH."""
import argparse
import json


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=4)
    ap.add_argument("--subgame_iters", type=int, default=1024, help="iterations of the full-game solve")
    ap.add_argument("--cfr", action="store_true", help="CFR instead of fictitious play (the reference's default solver is FP)")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--optimistic", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--device", type=int, default=0, help="CUDA ordinal")
    ap.add_argument("--save", type=str, default=None, metavar="PATH", help="write the final average strategy as a blueprint file")
    return ap


def make_cfg(rela, args):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = args.num_dice, args.num_faces
    cfg.net_mode, cfg.state_dtype = 0, 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr, sp.optimistic = args.subgame_iters, 100000, args.cfr, args.optimistic
    sp.linear_update = not args.no_linear and args.dcfr is None                      # recursive_eval.cc:273
    if args.dcfr is not None:
        sp.dcfr, (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) = True, args.dcfr
    return cfg


def main(argv=None):
    args = build_parser().parse_args(argv)
    A = 2 * args.num_dice * args.num_faces + 1
    if A > 23:
        raise SystemExit(f"solve_game: games with more than 23 actions are not supported (A = {A}: the full tree has 2^A - 1 nodes)")
    import rebel_b200.rela as rela
    cfg = make_cfg(rela, args)
    r = rela.solve_full_game(cfg, args.device)
    sp = cfg.subgame_params
    br = r["exploitability"][-1].tolist() if len(r["checkpoints"]) else [float("nan")] * 2
    line = {
        "game": f"{args.num_dice}x{args.num_faces}f", "num_dice": args.num_dice, "num_faces": args.num_faces,
        "num_nodes": r["num_nodes"], "iterations": args.subgame_iters, "solver": "cfr" if args.cfr else "fp",
        "linear": bool(sp.linear_update), "dcfr": list(args.dcfr) if args.dcfr is not None else None, "optimistic": args.optimistic,
        "br": br, "exploitability": (br[0] + br[1]) / 2,
        "seconds": r["seconds"], "solve_seconds": r["solve_seconds"], "br_seconds": r["br_seconds"],
        "peak_device_bytes": r["device_bytes"],
    }
    if args.save:
        from rebel_b200.blueprint import save_blueprint
        settings = {k: line[k] for k in ("solver", "iterations", "linear", "dcfr", "optimistic")}
        line["saved"] = save_blueprint(args.save, args.num_dice, args.num_faces, r["strategy"].numpy(), "solve_game", settings, br)
    print("SOLVE " + json.dumps(line), flush=True)
    return r


if __name__ == "__main__":
    main()
