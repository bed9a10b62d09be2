"""Play Liar's Dice against a ReBeL agent in the terminal.  The agent (a value net plus a solver configuration) re-solves subgames
on the GPU along the path played, exactly as in head-to-head matches (rela.Agent): with its recursive to-leaf policy ('sampled' or
'average'), or ('every_node') re-solving at every decision.

    python -m rebel_b200.play --num_dice 1 --num_faces 6 --net ckpt.torchscript --subgame_iters 1024 --cfr --mdp_depth 2 \
        --policy sampled --games 5 --seed 0

Both hands are dealt on the host from --seed; seats alternate between games (you move first in game 0).  Dice show faces 1..F, and
face F is wild: it counts for every face.  Enter a bid as `<quantity> <face>` (a bid must beat the last one: a higher quantity, or
the same quantity of a higher face) or `liar` to call the last bid.  At the liar call the bidder wins if both hands together hold
at least `quantity` dice showing `face` or the wild face.  The session ends with one tagged line `PLAY {"net": ..., "games": ...,
"agent_wins": ..., "human_wins": ..., "agent_mean": ...}` whose text after the tag is JSON.  --blueprint PATH plays against a
blueprint file (`solve_game --save`, `exploitability --save`) instead: a fixed full-tree strategy that never solves (--net is
refused with it), named "blueprint:PATH"."""
import argparse
import json
import sys

import numpy as np

from rebel_b200.head_to_head import POLICIES, agent_name, agent_params, agent_weights


def build_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_dice", type=int, default=1)
    ap.add_argument("--num_faces", type=int, default=6)
    ap.add_argument("--net", type=str, default=None, help="the agent's Net2 checkpoint (TorchScript or state_dict), or 'zero'")
    ap.add_argument("--subgame_iters", type=int, default=1024)
    ap.add_argument("--cfr", action="store_true", help="the agent solves with CFR instead of fictitious play")
    ap.add_argument("--mdp_depth", type=int, default=2)
    ap.add_argument("--policy", choices=POLICIES, default="sampled",
                    help="sampled: ReBeL's random-iteration policy; average: the average strategy of all iterations (both act to "
                    "the subgame's leaves); every_node: a subgame re-solved at every decision, acting with its root's average")
    ap.add_argument("--games", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0, help="seeds the deals and the agent's draws")
    ap.add_argument("--net_mode", type=int, default=None, help="0 zero, 1 fp32 SIMT, 2 wgmma fp16, 3 wgmma fp16 + fast GELU (default 3 with a "
                    "net), 4 wgmma on two-CTA clusters with mode 3's GELU (also games too large for modes 2 and 3; the fp32 net where it does "
                    "not fit)")
    ap.add_argument("--blueprint", type=str, default=None, metavar="PATH", help="play against this blueprint file (no net, no solves)")
    # agent_params' other settings, at head_to_head's defaults
    ap.set_defaults(no_linear=False, dcfr=None, device=0)
    return ap


def num_actions(num_dice, num_faces):
    """Bids (quantity 1..2D of each face, in the order quantity-major) and the liar call, which is the last action."""
    return 1 + 2 * num_dice * num_faces


def hand_to_dice(hand, num_dice, num_faces):
    """0-based faces of a hand index: die i is base-F digit i (least significant first), num_hands = F^D."""
    return [(hand // num_faces ** i) % num_faces for i in range(num_dice)]


def dice_to_hand(dice, num_faces):
    return sum(int(f) * num_faces ** i for i, f in enumerate(dice))


def num_matches(hand, face, num_dice, num_faces):
    """Dice of the hand that show `face` or the wild (last) face."""
    return sum(1 for d in hand_to_dice(hand, num_dice, num_faces) if d == face or d == num_faces - 1)


def bidder_wins(bid, hand0, hand1, num_dice, num_faces):
    """At the liar call on `bid`: both hands together hold at least its quantity of its face."""
    quantity, face = 1 + bid // num_faces, bid % num_faces
    return num_matches(hand0, face, num_dice, num_faces) + num_matches(hand1, face, num_dice, num_faces) >= quantity


def bid_name(action, num_dice, num_faces):
    if action == num_actions(num_dice, num_faces) - 1:
        return "liar"
    return f"{1 + action // num_faces} {1 + action % num_faces}"


def parse_bid(text, last_bid, num_dice, num_faces):
    """The action of an input line, or a string saying why it is not a legal move after last_bid (-1: no bid yet)."""
    liar = num_actions(num_dice, num_faces) - 1
    words = text.split()
    if len(words) == 1 and words[0].lower() == "liar":
        return liar if last_bid >= 0 else "there is no bid to call yet"
    if len(words) != 2 or not all(w.isdigit() for w in words):
        return "enter `<quantity> <face>` or `liar`"
    quantity, face = int(words[0]), int(words[1])
    if not 1 <= face <= num_faces:
        return f"faces are 1..{num_faces}"
    if not 1 <= quantity <= 2 * num_dice:
        return f"quantities are 1..{2 * num_dice}"
    action = (quantity - 1) * num_faces + face - 1
    if action <= last_bid:
        return f"a bid must beat {bid_name(last_bid, num_dice, num_faces)}"
    return action


def play_line(name, games, agent_wins, human_wins):
    d = {"net": name, "games": games, "agent_wins": agent_wins, "human_wins": human_wins,
         "agent_mean": (agent_wins - human_wins) / games if games else 0.0}
    return "PLAY " + json.dumps(d)


def parse_play(line):
    assert line.startswith("PLAY "), line
    return json.loads(line[5:])


def show(dice):
    return " ".join(str(d + 1) for d in dice)


def main(argv=None, stdin=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    stdin = stdin or sys.stdin
    D, F = args.num_dice, args.num_faces
    if args.blueprint is not None:
        if args.net is not None:
            ap.error("--net configures the agent that --blueprint replaces")
        from rebel_b200.blueprint import blueprint_name
        from rebel_b200.head_to_head import load_blueprint_arg
        bp = load_blueprint_arg(args.blueprint, args, "play")
    import rebel_b200.rela as rela
    if args.blueprint is not None:
        agent = rela.Agent.from_blueprint(D, F, bp["strategy"], device=args.device, tables=1, seed=args.seed)
        name = blueprint_name(args.blueprint)
        print(f"{D}x{F}f against {name} ({bp['source']} blueprint, exploitability {bp['exploitability']:.6f}); face {F} is wild",
              flush=True)
    else:
        w = agent_weights(D, F, args.net, None)
        cfg = agent_params(rela, args, w, args.subgame_iters, args.cfr)
        agent = rela.Agent(cfg, device=args.device, tables=1, policy=args.policy, seed=args.seed, flat_weights=w)
        name = agent_name(args.net, None)
        print(f"{D}x{F}f against {name} ({args.policy} policy, {args.subgame_iters} iterations, depth {args.mdp_depth}); "
              f"face {F} is wild", flush=True)
    H, A = agent.num_hands, agent.num_actions
    rng = np.random.RandomState(args.seed)
    wins = [0, 0]                                     # agent, human
    played = 0
    for g in range(args.games):
        human = g % 2
        hands = rng.randint(0, H, size=2)             # by seat
        agent.new_games([0], [1 - human], [int(hands[1 - human])], keys=[g])
        print(f"\ngame {g + 1}: you are player {human + 1}; your dice: {show(hand_to_dice(hands[human], D, F))}", flush=True)
        last, player = -1, 0
        while True:
            if player == human:
                line = None
                while True:
                    print("your bid> ", end="", flush=True)
                    line = stdin.readline()
                    if not line:
                        break
                    action = parse_bid(line, last, D, F)
                    if not isinstance(action, str):
                        break
                    print(f"  {action}", flush=True)
                if not line:
                    print("\ninput ended", flush=True)
                    print(play_line(name, played, wins[0], wins[1]), flush=True)
                    agent.close()
                    return wins
                agent.step([0], [action])
            else:
                actions, probs, _ = agent.step([0], [-1])
                action = int(actions[0])
                print(f"agent: {bid_name(action, D, F)}  (probability {float(probs[0, action]):.3f})", flush=True)
            if action == A - 1:
                caller = player
                bidder_won = bidder_wins(last, int(hands[0]), int(hands[1]), D, F)
                winner = caller ^ 1 if bidder_won else caller
                print(f"reveal: your dice {show(hand_to_dice(hands[human], D, F))}, the agent's dice "
                      f"{show(hand_to_dice(hands[1 - human], D, F))}; the bid {bid_name(last, D, F)} is "
                      f"{'true' if bidder_won else 'false'}: {'you win' if winner == human else 'the agent wins'}", flush=True)
                wins[0 if winner != human else 1] += 1
                played += 1
                print(f"score: agent {wins[0]}, you {wins[1]}", flush=True)
                break
            last, player = action, player ^ 1
    print(play_line(name, played, wins[0], wins[1]), flush=True)
    agent.close()
    return wins


if __name__ == "__main__":
    main()
