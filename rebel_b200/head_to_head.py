"""Head-to-head evaluation of two ReBeL agents on the GPU: each agent (a value net plus a solver configuration) re-solves
subgames along the path actually played, in seat-swapped pairs of games: with its recursive to-leaf policy ('sampled' or
'average'), or ('every_node') re-solving at every decision as compute_strategy_recursive does.  Works on every game
the wave solver supports, including those whose full game tree the exploitability tools refuse (2x5f, 5x2f, 2x6f, 1x17f, ...).

    python -m rebel_b200.head_to_head --num_dice 2 --num_faces 5 --net_a ckpt_400.torchscript --net_b ckpt_200.torchscript \
        --games 65536 --subgame_iters 1024 --cfr --mdp_depth 2

Prints a summary and one tagged line `H2H {"net_a": ..., "net_b": ..., "games": ..., "mean": ..., "stderr": ..., "ci95": [lo, hi],
"seat0": ..., "seat1": ...}` whose text after the tag is JSON.  mean is agent A's expected payoff per game (+1 win, -1 loss);
seat0 / seat1 are A's mean payoffs in seat 0 (even games) and seat 1 (odd games).  When --policy_b is given or either agent plays
every_node, the line also has "policy_a" and "policy_b".

--blueprint_a PATH / --blueprint_b PATH replace that agent by a blueprint file (`solve_game --save`, `exploitability --save`): a
fixed full-tree strategy that never solves.  That agent's --net_* and --random_net_seed_* are refused with it; the line names it
"blueprint:PATH" and gives its policy as "blueprint"."""
import argparse
import json

import torch


POLICIES = ("sampled", "average", "every_node")


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
    ap.add_argument("--policy", choices=POLICIES, default="sampled",
                    help="sampled: ReBeL's random-iteration policy; average: the average strategy of all iterations (both act to "
                    "the subgame's leaves); every_node: a subgame re-solved at every decision, acting with its root's average")
    ap.add_argument("--policy_b", choices=POLICIES, default=None, help="agent B's policy (default: --policy)")
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--subgame_iters_b", type=int, default=None, help="agent B's iterations (default: --subgame_iters)")
    ap.add_argument("--mdp_depth", type=int, default=2)
    ap.add_argument("--cfr", action="store_true", help="agent A solves with CFR instead of fictitious play")
    ap.add_argument("--cfr_b", choices=("yes", "no"), default=None, help="agent B's solver (default: as agent A)")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast GELU (default 3 with a net), "
                    "4 wgmma on two-CTA clusters with mode 3's GELU (also games too large for modes 2 and 3; the fp32 net where it does not fit)")
    ap.add_argument("--concurrent_games", type=int, default=8192)
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--blueprint_a", type=str, default=None, metavar="PATH", help="agent A is this blueprint file (no net, no solves)")
    ap.add_argument("--blueprint_b", type=str, default=None, metavar="PATH", help="agent B is this blueprint file (no net, no solves)")
    return ap


def blueprint_conflicts(args):
    """The flags given together with a blueprint that would configure the agent it replaces (empty: none)."""
    bad = []
    for k in ("a", "b"):
        if getattr(args, "blueprint_" + k) is not None:
            bad += [f"--{f}_{k}" for f in ("net", "random_net_seed") if getattr(args, f"{f}_{k}") is not None]
    return bad


def load_blueprint_arg(path, args, who):
    """A blueprint file of the command's game; anything else ends the command with a message."""
    from rebel_b200.blueprint import load_blueprint
    try:
        return load_blueprint(path, args.num_dice, args.num_faces)
    except (ValueError, OSError) as e:
        raise SystemExit(f"{who}: {e}")


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


def h2h_line(name_a, name_b, games, mean, stderr, seat_means, policies=None):
    """The tagged report line; ci95 = mean -/+ 1.96 stderr.  policies: (A's, B's) policy names, reported as policy_a / policy_b."""
    d = {"net_a": name_a, "net_b": name_b, "games": games, "mean": mean, "stderr": stderr,
         "ci95": [mean - 1.96 * stderr, mean + 1.96 * stderr], "seat0": seat_means[0], "seat1": seat_means[1]}
    if policies is not None:
        d["policy_a"], d["policy_b"] = policies
    return "H2H " + json.dumps(d)


def parse_h2h(line):
    assert line.startswith("H2H "), line
    return json.loads(line[4:])


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    bad = blueprint_conflicts(args)
    if bad:
        ap.error(f"{', '.join(bad)} configure an agent that a blueprint replaces")
    bp = {k: load_blueprint_arg(getattr(args, "blueprint_" + k), args, "head_to_head")
          for k in ("a", "b") if getattr(args, "blueprint_" + k) is not None}
    import rebel_b200.rela as rela
    wa = agent_weights(args.num_dice, args.num_faces, args.net_a, args.random_net_seed_a)
    wb = agent_weights(args.num_dice, args.num_faces, args.net_b, args.random_net_seed_b)
    cfr_b = args.cfr if args.cfr_b is None else args.cfr_b == "yes"
    cfg_a = agent_params(rela, args, wa, args.subgame_iters, args.cfr)
    cfg_b = agent_params(rela, args, wb, args.subgame_iters_b or args.subgame_iters, cfr_b)
    policy_b = args.policy_b or args.policy
    kw = {f"blueprint_{k}": torch.from_numpy(v["strategy"]) for k, v in bp.items()}
    r = rela.play_match(cfg_a, cfg_b, args.device, args.games, seed=args.seed, policy=args.policy, flat_weights_a=wa,
                        flat_weights_b=wb, concurrent_games=args.concurrent_games, policy_b=policy_b, **kw)
    na, nb = agent_name(args.net_a, args.random_net_seed_a), agent_name(args.net_b, args.random_net_seed_b)
    if bp:
        from rebel_b200.blueprint import blueprint_name
        na = blueprint_name(args.blueprint_a) if "a" in bp else na
        nb = blueprint_name(args.blueprint_b) if "b" in bp else nb
    mean, se = r["mean"], r["stderr"]
    named = args.policy_b is not None or "every_node" in (args.policy, policy_b) or bool(bp)
    pol_a = "blueprint" if "a" in bp else args.policy
    pol_b = "blueprint" if "b" in bp else policy_b
    pol = f"{pol_a} policy" if pol_b == pol_a else f"A {pol_a}, B {pol_b} policy"
    print(f"{args.num_dice}x{args.num_faces}f, {args.games} games ({pol}, depth {args.mdp_depth}): "
          f"A = {na} vs B = {nb}", flush=True)
    print(f"  A's payoff per game {mean:+.4f} +- {se:.4f} (95% CI [{mean - 1.96 * se:+.4f}, {mean + 1.96 * se:+.4f}]); "
          f"in seat 0 {r['seat_means'][0]:+.4f}, in seat 1 {r['seat_means'][1]:+.4f}", flush=True)
    print(f"  {r['solves']} subgame solves (A {r['solves_a']}, B {r['solves_b']}), {r['subgame_iters']} subgame iterations, {float(r['plies'].float().mean()):.2f} plies "
          f"per game, {r['seconds']:.2f} s ({args.games / r['seconds']:.1f} games/s)", flush=True)
    print(h2h_line(na, nb, args.games, mean, se, r["seat_means"], (pol_a, pol_b) if named else None), flush=True)
    return r


if __name__ == "__main__":
    main()
