"""Time one rela.compute_stats_with_net call (the evaluation `rebel_b200.train --exploit_every` runs) by phase, and its peak device
memory, on the games and value-net modes given.  Each case runs in a process of its own with CFRB_EVAL_TIMING=1 (the phase laps on
stderr) while a thread samples the device's free memory every 10 ms; the peak is the largest drop below the free memory at the
start.  The net is the seed-0 initialisation (its cost does not depend on its weights).  Prints one JSON line per case and one
with the card's name and power limit.

    python scripts/stats_bench.py [--games 2x4f 3x3f 2x5f 5x2f 1x11f] [--net_modes 1 3] [--iters 1024] [--mdp_depth 2]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys, threading, time
import torch
sys.path.insert(0, sys.argv[1])
import rebel_b200.rela as rela
D, F, iters, md, path, walk = int(sys.argv[2]), int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), sys.argv[6], sys.argv[7]
cfg = rela.RecursiveSolvingParams()
cfg.num_dice, cfg.num_faces = D, F
sp = cfg.subgame_params
sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = iters, md, True, True
free0 = torch.cuda.mem_get_info()[0]
low, done = [free0], [False]
def poll():
    while not done[0]:
        low[0] = min(low[0], torch.cuda.mem_get_info()[0])
        time.sleep(0.01)
t = threading.Thread(target=poll)
t.start()
t0 = time.time()
out = rela.compute_stats_with_net(cfg, path, device_walk={"auto": None, "dense": False, "device": True}[walk])
sec = time.time() - t0
done[0] = True
t.join()
print("RESULT " + json.dumps({"stats": list(out), "seconds": sec, "peak_bytes": free0 - low[0]}), flush=True)
"""


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--games", nargs="+", default=["2x4f", "3x3f", "2x5f", "5x2f", "1x11f"])
    ap.add_argument("--net_modes", nargs="+", type=int, default=[1, 3])
    ap.add_argument("--iters", type=int, default=1024, help="subgame_params.num_iters (rebel_b200.train --subgame_iters)")
    ap.add_argument("--mdp_depth", type=int, default=2)
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    from rebel_b200.models import make_selfplay_net
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        for game in args.games:
            D, F = int(game.split("x")[0]), int(game.split("x")[1].rstrip("f"))
            path = os.path.join(tmp, f"net_{D}x{F}.torchscript")
            torch.jit.script(make_selfplay_net(D, F, seed=0)).save(path)
            walks = ["dense", "device"] if 2 * D * F + 1 <= 20 and game == "2x4f" else ["auto"]
            for mode in args.net_modes:
                for walk in walks:
                    env = dict(os.environ, CFRB_EVAL_TIMING="1", CFRB_EVAL_NET_MODE=str(mode))
                    r = subprocess.run([sys.executable, "-c", CHILD, ROOT, str(D), str(F), str(args.iters), str(args.mdp_depth), path, walk],
                                       capture_output=True, text=True, env=env)
                    rec = {"game": game, "net_mode": mode, "path": walk, "iters": args.iters, "mdp_depth": args.mdp_depth}
                    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
                    if r.returncode or not res:
                        rec["error"] = (r.stderr or r.stdout)[-800:]
                    else:
                        rec.update(json.loads(res[-1][7:]))
                        laps = [l[13:].rsplit(" ", 2) for l in r.stderr.splitlines() if l.startswith("[rebel_b200] ")]
                        rec["phases"] = {name.strip(): float(sec) for name, sec, _ in laps}
                    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
