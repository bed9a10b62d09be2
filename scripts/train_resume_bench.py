"""What reproducibility costs a training run: `python -m rebel_b200.train` in its threaded mode against --deterministic (the runs
alternate in one call), and the time and size of one state save and one resume, at 1x6f and 2x5f with the default sizes (epochs
of 25 600 examples in batches of 512, train_gen_ratio 4, 1 024 games per generator loop).

    python scripts/train_resume_bench.py [--epochs 15] [--reps 2] [--games 1x6 2x5] [--out DIR]

For every run, between the TRAIN lines of its first and last epoch without evaluation: epochs/s, generated examples/s (the
growth of buffer_added; a threaded run generates all the time, a deterministic one only what the throttle asks for), trained
examples/s (epochs x epoch size), the median rate of the training-step loop alone (train_examples_per_s of the TRAIN lines) and, for
deterministic runs, the median rate of the generators while they run (wave_examples_per_s).  After each
deterministic run the same run is resumed with nothing left to do, which times the loading of its state.  Exploitability is off
(--exploit_every 0).  Prints one `TRAIN_RESUME_BENCH {...}` JSON line per game with the card's name and power limit."""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rebel_b200.train import parse_train  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def run(out, D, F, epochs, *extra):
    cmd = [sys.executable, "-m", "rebel_b200.train", "--num_dice", str(D), "--num_faces", str(F), "--out", out, "--max_epochs",
           str(epochs), "--exploit_every", "0", "--max_minutes", "10"] + list(extra)
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    if r.returncode:
        raise SystemExit(f"{' '.join(cmd)} failed:\n{r.stdout[-2000:]}\n{r.stderr[-2000:]}")
    return r.stdout


def throughput(stdout, epoch_size=25600, eval_every=10):
    """Between the first and the last TRAIN line of an epoch without evaluation (buffer_added is read before an evaluation epoch's
    checkpoints and validation, minutes after them, so an evaluation epoch's line pairs an early count with a late clock)."""
    lines = [parse_train(l) for l in stdout.splitlines() if l.startswith("TRAIN ")]
    quiet = [m for m in lines if m["epoch"] % eval_every]
    a, b = quiet[0], quiet[-1]
    span, epochs = (b["minutes"] - a["minutes"]) * 60, b["epoch"] - a["epoch"]
    r = {"epochs": len(lines), "window": [a["epoch"], b["epoch"]], "epochs_per_s": epochs / span,
         "gen_examples_per_s": (b["buffer_added"] - a["buffer_added"]) / span,
         "trained_examples_per_s": epochs * epoch_size / span,
         "train_loop_examples_per_s": statistics.median(m["train_examples_per_s"] for m in lines[1:])}
    waves = [m["wave_examples_per_s"] for m in lines[1:] if "wave_examples_per_s" in m]
    if waves:   # deterministic runs: the generators' rate while they run
        r["wave_examples_per_s"] = statistics.median(waves)
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--epochs", type=int, default=15)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--games", nargs="+", default=["1x6", "2x5"])
    ap.add_argument("--out", default=None, help="directory for the runs (default: a temporary directory)")
    a = ap.parse_args()
    name, power = card()
    base = a.out or tempfile.mkdtemp(prefix="train_resume_bench_")
    for game in a.games:
        D, F = (int(x) for x in game.split("x"))
        res = {"game": f"{D}x{F}f", "card": name, "power_limit": power, "epochs_per_run": a.epochs,
               "threaded": [], "deterministic": [], "state_save": [], "resume": []}
        for rep in range(a.reps):
            for mode in ("threaded", "deterministic"):
                out = os.path.join(base, f"{D}x{F}_{mode}_{rep}")
                extra = ["--deterministic", "--state_every", "0"] if mode == "deterministic" else []
                stdout = run(out, D, F, a.epochs, *extra)
                res[mode].append(throughput(stdout))
                if mode == "deterministic":
                    m = re.search(r"state saved at epoch \d+: (\d+) bytes in ([0-9.]+) s", stdout)
                    res["state_save"].append({"bytes": int(m.group(1)), "seconds": float(m.group(2))})
                    m = re.search(r"resumed in ([0-9.]+) s", run(out, D, F, a.epochs, *extra, "--resume"))
                    res["resume"].append({"seconds": float(m.group(1))})
                print(f"[bench] {game} {mode} rep {rep}: {res[mode][-1]}", flush=True)
        for key in ("epochs_per_s", "gen_examples_per_s", "trained_examples_per_s", "train_loop_examples_per_s"):
            t = statistics.median(r[key] for r in res["threaded"])
            d = statistics.median(r[key] for r in res["deterministic"])
            res[f"deterministic_over_threaded_{key}"] = d / t
        print("TRAIN_RESUME_BENCH " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
