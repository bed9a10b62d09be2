"""Head-to-head evaluation of two ReBeL agents on the GPU: each agent (a value net plus a solver configuration) re-solves
subgames along the path actually played, with its recursive to-leaf policy, in seat-swapped pairs of games.  Works on every game
the wave solver supports, including those whose full game tree the exploitability tools refuse (2x5f, 5x2f, 2x6f, 1x17f, ...).

    python -m rebel_b200.head_to_head --num_dice 2 --num_faces 5 --net_a ckpt_400.torchscript --net_b ckpt_200.torchscript \
        --games 65536 --subgame_iters 1024 --cfr --mdp_depth 2

Prints a summary and one tagged line `H2H {"net_a": ..., "net_b": ..., "games": ..., "mean": ..., "stderr": ..., "ci95": [lo, hi],
"seat0": ..., "seat1": ...}` whose text after the tag is JSON.  mean is agent A's expected payoff per game (+1 win, -1 loss);
seat0 / seat1 are A's mean payoffs in seat 0 (even games) and seat 1 (odd games)."""
import argparse
import json

import torch


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=4)
    ap.add_argument("--net_a", type=str, default=None, help="agent A's Net2 checkpoint (TorchScript or state_dict), or 'zero'")
    ap.add_argument("--net_b", type=str, default=None, help="agent B's Net2 checkpoint, or 'zero'")
    ap.add_argument("--random_net_seed_a", type=int, default=None, help="agent A plays a random-init Net2 of this seed")
    ap.add_argument("--random_net_seed_b", type=int, default=None, help="agent B plays a random-init Net2 of this seed")
    ap.add_argument("--games", type=int, default=8192, help="games to play (even: seat-swapped pairs)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--policy", choices=("sampled", "average"), default="sampled",
                    help="sampled: ReBeL's random-iteration policy; average: the average strategy of all iterations")
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--subgame_iters_b", type=int, default=None, help="agent B's iterations (default: --subgame_iters)")
    ap.add_argument("--mdp_depth", type=int, default=2)
    ap.add_argument("--cfr", action="store_true", help="agent A solves with CFR instead of fictitious play")
    ap.add_argument("--cfr_b", choices=("yes", "no"), default=None, help="agent B's solver (default: as agent A)")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast GELU (default 3 with a net)")
    ap.add_argument("--concurrent_games", type=int, default=8192)
    ap.add_argument("--device", type=int, default=0)
    return ap


def agent_weights(num_dice, num_faces, net, random_seed):
    """Flat Net2 weights of an agent, or None for the zero net."""
    if net and net != "zero":
        from rebel_b200.recursive_eval import load_net_weights
        return load_net_weights(net)
    if random_seed is not None:
        from rebel_b200.models import flatten_state_dict, make_selfplay_net
        return torch.from_numpy(flatten_state_dict(make_selfplay_net(num_dice, num_faces, seed=random_seed).state_dict()))
    return None


def agent_params(rela, args, weights, iters, use_cfr):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = args.num_dice, args.num_faces
    cfg.net_mode = args.net_mode if args.net_mode is not None else (3 if weights is not None else 0)
    if weights is None:
        cfg.net_mode = 0
    cfg.state_dtype = 0
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.use_cfr = iters, args.mdp_depth, use_cfr
    sp.linear_update = not args.no_linear and args.dcfr is None
    if args.dcfr is not None:
        sp.dcfr, (sp.dcfr_alpha, sp.dcfr_beta, sp.dcfr_gamma) = True, args.dcfr
    return cfg


def agent_name(net, random_seed):
    if net:
        return net
    return f"random_net_seed={random_seed}" if random_seed is not None else "zero"


def h2h_line(name_a, name_b, games, mean, stderr, seat_means):
    """The tagged report line; ci95 = mean -/+ 1.96 stderr."""
    d = {"net_a": name_a, "net_b": name_b, "games": games, "mean": mean, "stderr": stderr,
         "ci95": [mean - 1.96 * stderr, mean + 1.96 * stderr], "seat0": seat_means[0], "seat1": seat_means[1]}
    return "H2H " + json.dumps(d)


def parse_h2h(line):
    assert line.startswith("H2H "), line
    return json.loads(line[4:])


def main(argv=None):
    args = build_parser().parse_args(argv)
    import rebel_b200.rela as rela
    wa = agent_weights(args.num_dice, args.num_faces, args.net_a, args.random_net_seed_a)
    wb = agent_weights(args.num_dice, args.num_faces, args.net_b, args.random_net_seed_b)
    cfr_b = args.cfr if args.cfr_b is None else args.cfr_b == "yes"
    cfg_a = agent_params(rela, args, wa, args.subgame_iters, args.cfr)
    cfg_b = agent_params(rela, args, wb, args.subgame_iters_b or args.subgame_iters, cfr_b)
    r = rela.play_match(cfg_a, cfg_b, args.device, args.games, seed=args.seed, policy=args.policy, flat_weights_a=wa,
                        flat_weights_b=wb, concurrent_games=args.concurrent_games)
    na, nb = agent_name(args.net_a, args.random_net_seed_a), agent_name(args.net_b, args.random_net_seed_b)
    mean, se = r["mean"], r["stderr"]
    print(f"{args.num_dice}x{args.num_faces}f, {args.games} games ({args.policy} policy, depth {args.mdp_depth}): "
          f"A = {na} vs B = {nb}", flush=True)
    print(f"  A's payoff per game {mean:+.4f} +- {se:.4f} (95% CI [{mean - 1.96 * se:+.4f}, {mean + 1.96 * se:+.4f}]); "
          f"in seat 0 {r['seat_means'][0]:+.4f}, in seat 1 {r['seat_means'][1]:+.4f}", flush=True)
    print(f"  {r['solves']} subgame solves, {r['subgame_iters']} subgame iterations, {float(r['plies'].float().mean()):.2f} plies "
          f"per game, {r['seconds']:.2f} s ({args.games / r['seconds']:.1f} games/s)", flush=True)
    print(h2h_line(na, nb, args.games, mean, se, r["seat_means"]), flush=True)
    return r


if __name__ == "__main__":
    main()
