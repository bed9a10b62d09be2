"""Local best response (LBR; Lisý & Bowling, 2017) against a ReBeL agent on the GPU: a lower bound on the agent's exploitability
on every game the wave solver supports, including those whose full game tree the exploitability tools refuse (2x5f, 5x2f, 2x6f,
1x17f, ...).  The agent (a value net plus a solver configuration) plays its average recursive to-leaf policy (--policy average)
or re-solves at every decision (--policy every_node, compute_strategy_recursive) along the path played; LBR best-responds one
decision at a time to the agent's actual strategy, assuming it calls the agent's next raise.

    python -m rebel_b200.local_br --num_dice 2 --num_faces 5 --net ckpt_400.torchscript --games 65536 --subgame_iters 1024 --cfr

Prints a summary and one tagged line `LBR {"net": ..., "games": ..., "mean": ..., "stderr": ..., "ci95": [lo, hi], "seat0": ...,
"seat1": ...}` whose text after the tag is JSON; with --policy every_node it ends with `"policy": "every_node"`.  mean is LBR's expected payoff per game (+1 win, -1 loss); seat0 / seat1 are its
means in seat 0 (odd games) and seat 1 (even games).  Since no strategy earns more against the agent than a best response,
exploitability >= mean, and with 95 % confidence >= mean - 1.96 stderr.

--blueprint PATH plays LBR against a blueprint file (`solve_game --save`, `exploitability --save`) instead of an agent: no subgame
is solved.  --net and --random_net_seed are refused with it.  The LBR line adds "policy": "blueprint" and the file's exact
"exploitability" beside the bound."""
import argparse
import json
import sys

import torch

from rebel_b200.head_to_head import agent_name, agent_params, agent_weights


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=4)
    ap.add_argument("--net", type=str, default=None, help="the agent's Net2 checkpoint (TorchScript or state_dict), or 'zero'")
    ap.add_argument("--random_net_seed", type=int, default=None, help="the agent plays a random-init Net2 of this seed")
    ap.add_argument("--games", type=int, default=8192, help="games to play (even: seat-swapped pairs)")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--policy", choices=("average", "every_node", "sampled"), default="average",
                    help="the agent's policy: 'average' (recursive to-leaf) or 'every_node' (a subgame re-solved at every decision); "
                    "'sampled' has no valid LBR bound and is refused")
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--mdp_depth", type=int, default=2)
    ap.add_argument("--cfr", action="store_true", help="the agent solves with CFR instead of fictitious play")
    ap.add_argument("--no_linear", action="store_true")
    ap.add_argument("--dcfr", type=float, nargs=3, metavar=("ALPHA", "BETA", "GAMMA"), default=None)
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast GELU (default 3 with a net), "
                    "4 wgmma on two-CTA clusters with mode 3's GELU (also games too large for modes 2 and 3; the fp32 net where it does not fit)")
    ap.add_argument("--concurrent_games", type=int, default=8192)
    ap.add_argument("--max_subgames", type=int, default=0, help="subgames solved per round (0: 2 x concurrent_games, at least A - 1)")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--blueprint", type=str, default=None, metavar="PATH", help="LBR against this blueprint file (no net, no solves)")
    return ap


SAMPLED_REFUSED = ("--policy sampled is not supported: LBR would have to respond to the expectation over the agent's "
                   "act_iteration draws; responding to the drawn snapshot uses information the agent's opponent does not have, "
                   "so the payoff would not bound the exploitability")


def lbr_line(name, games, mean, stderr, seat_means, policy="average", exploitability=None):
    """The tagged report line; ci95 = mean -/+ 1.96 stderr.  A policy other than 'average' adds a "policy" key, a known exact
    exploitability (a blueprint's) an "exploitability" key."""
    d = {"net": name, "games": games, "mean": mean, "stderr": stderr, "ci95": [mean - 1.96 * stderr, mean + 1.96 * stderr],
         "seat0": seat_means[0], "seat1": seat_means[1]}
    if policy != "average":
        d["policy"] = policy
    if exploitability is not None:
        d["exploitability"] = exploitability
    return "LBR " + json.dumps(d)


def parse_lbr(line):
    assert line.startswith("LBR "), line
    return json.loads(line[4:])


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if args.policy == "sampled":
        print(SAMPLED_REFUSED, file=sys.stderr, flush=True)
        raise SystemExit(2)
    bp = None
    if args.blueprint is not None:
        bad = [f for f, v in (("--net", args.net), ("--random_net_seed", args.random_net_seed)) if v is not None]
        if bad:
            ap.error(f"{', '.join(bad)} configure the agent that --blueprint replaces")
        from rebel_b200.head_to_head import load_blueprint_arg
        bp = load_blueprint_arg(args.blueprint, args, "local_br")
    import rebel_b200.rela as rela
    w = agent_weights(args.num_dice, args.num_faces, args.net, args.random_net_seed)
    cfg = agent_params(rela, args, w, args.subgame_iters, args.cfr)
    kw = {"blueprint": torch.from_numpy(bp["strategy"])} if bp else {}
    r = rela.play_lbr(cfg, args.device, args.games, seed=args.seed, flat_weights=w, concurrent_games=args.concurrent_games,
                      max_subgames=args.max_subgames, policy=args.policy, **kw)
    name = agent_name(args.net, args.random_net_seed)
    if bp:
        from rebel_b200.blueprint import blueprint_name
        name = blueprint_name(args.blueprint)
    mean, se = r["mean"], r["stderr"]
    policy = "blueprint" if bp else args.policy.replace("_", "-")
    print(f"{args.num_dice}x{args.num_faces}f, {args.games} games ({policy} policy, depth {args.mdp_depth}): LBR vs {name}", flush=True)
    print(f"  LBR's payoff per game {mean:+.4f} +- {se:.4f} (95% CI [{mean - 1.96 * se:+.4f}, {mean + 1.96 * se:+.4f}]); "
          f"in seat 0 {r['seat_means'][0]:+.4f}, in seat 1 {r['seat_means'][1]:+.4f}", flush=True)
    print(f"  exploitability >= mean - 1.96 stderr = {mean - 1.96 * se:+.4f}"
          + (f" (the blueprint's exact exploitability: {bp['exploitability']:.6f})" if bp else ""), flush=True)
    print(f"  {r['solves']} subgame solves ({r['whatif_solves']} what-if), {r['subgame_iters']} subgame iterations, "
          f"{float(r['plies'].float().mean()):.2f} plies per game, {r['seconds']:.2f} s ({args.games / r['seconds']:.1f} games/s)",
          flush=True)
    print(lbr_line(name, args.games, mean, se, r["seat_means"], "blueprint" if bp else args.policy,
                   bp["exploitability"] if bp else None), flush=True)
    return r


if __name__ == "__main__":
    main()
