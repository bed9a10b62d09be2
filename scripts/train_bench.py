"""Value-net training on one GPU: the CUDA training step (rebel_b200.trainer.Net2Trainer) against the reference trainer's step
written in PyTorch (forward, huber loss, backward, clip_grad_norm_, Adam; fp32, TF32 off), and self-play throughput with and
without a concurrent training loop, at 1x6f and 2x5f with batch 512.

    python scripts/train_bench.py [--steps 200] [--rounds 5] [--gen_seconds 20]

Step times are CUDA-event times per step after warm-up; the two steps alternate in the same process, `rounds` windows of `steps`
steps each, and the median window is reported.  Torch's kernel launches per step are counted with torch.profiler.  Prints one
`TRAIN_BENCH {...}` JSON line per game, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rebel_b200.models import input_size, make_selfplay_net, output_size  # noqa: E402
from rebel_b200.trainer import Net2Trainer  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def torch_stepper(D, F):
    net = make_selfplay_net(D, F, seed=0).cuda().train()
    opt = torch.optim.Adam(net.parameters(), lr=3e-4)
    params = list(net.parameters())

    def step(q, v):
        x = v - net(q)
        loss = ((x.abs() > 1).float() * (x.abs() * 2 - 1) + (x.abs() <= 1).float() * x.pow(2)).mean(-1).mean()
        opt.zero_grad()
        loss.backward()
        total = torch.norm(torch.stack([torch.norm(p.grad.detach(), 2) for p in params]), 2)   # selfplay.py:636-651
        coef = 5.0 / (total + 1e-6)
        if coef < 1:
            for p in params:
                p.grad.detach().mul_(coef)
        opt.step()
        return loss, total
    return step


def time_window(fn, batches, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        fn(*batches[i % len(batches)])
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def launches_per_step(fn, batches, steps=10):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            fn(*batches[i % len(batches)])
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
               and "Memset" not in e.name]
    return len(kernels) / steps


def selfplay_rates(D, F, seconds, train):
    """Examples/s added by one generator loop (1024 CFR iterations, depth 2) alone or beside a training loop that keeps
    trained examples <= 4 x generated ones (train_gen_ratio 4)."""
    import rebel_b200.rela as rela
    tr = Net2Trainer(D, F, "cuda:0")
    locker = rela.ModelLocker([torch.jit.script(tr.net())], "cuda:0")
    replay = rela.ValuePrioritizedReplay(capacity=1 << 21, seed=10001, alpha=1.0, beta=1.0, prefetch=8, use_priority=False,
                                         compressed_values=False)
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.random_action_prob, cfg.sample_leaf = D, F, 0.25, True
    cfg.subgame_params.num_iters, cfg.subgame_params.max_depth = 1024, 2
    cfg.subgame_params.linear_update, cfg.subgame_params.use_cfr = True, True
    ctx = rela.Context()
    ctx.push_env_thread(rela.create_cfr_thread(locker, replay, cfg, 0))
    ctx.start()
    stream = torch.cuda.Stream()
    trained = 0
    try:
        while replay.size() < 1024:
            time.sleep(0.01)
        n0, t0 = replay.num_add(), time.time()
        while time.time() - t0 < seconds:
            if train and trained + 512 <= 4 * (replay.num_add() - n0):
                with torch.cuda.stream(stream):
                    batch, _ = replay.sample(512, "cuda:0")
                    tr.step(batch.query, batch.values)
                trained += 512
                if trained % (512 * 16) == 0:
                    stream.synchronize()
            else:
                stream.synchronize()
                time.sleep(0.002)
        stream.synchronize()
        dt = time.time() - t0
        return (replay.num_add() - n0) / dt, trained / dt
    finally:
        ctx.terminate()
        while not ctx.terminated():
            time.sleep(0.01)
        tr.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--gen_seconds", type=float, default=20)
    ap.add_argument("--games", type=str, nargs="+", default=["1x6", "2x5"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_bench needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    name, power = card()
    for game in args.games:
        D, F = map(int, game.split("x"))
        Q, H = input_size(F, D), output_size(F, D)
        g = torch.Generator().manual_seed(0)
        batches = [((torch.rand(512, Q, generator=g) * 2 - 1).cuda(), torch.randn(512, H, generator=g).cuda()) for _ in range(16)]
        tr = Net2Trainer(D, F, "cuda:0")
        ours, ref = tr.step, torch_stepper(D, F)
        for fn in (ours, ref):
            time_window(fn, batches, 20)
        t_ours, t_ref = [], []
        for _ in range(args.rounds):
            t_ours.append(time_window(ours, batches, args.steps))
            t_ref.append(time_window(ref, batches, args.steps))
        med = lambda xs: sorted(xs)[len(xs) // 2]
        res = {"game": f"{D}x{F}f", "batch": 512, "cuda_step_ms": med(t_ours), "torch_step_ms": med(t_ref),
               "cuda_step_ms_all": t_ours, "torch_step_ms_all": t_ref,
               "torch_kernels_per_step": launches_per_step(ref, batches), "cuda_kernels_per_step": launches_per_step(ours, batches)}
        tr.close()
        res["selfplay_examples_per_s"], _ = selfplay_rates(D, F, args.gen_seconds, train=False)
        res["selfplay_examples_per_s_training"], res["train_examples_per_s"] = selfplay_rates(D, F, args.gen_seconds, train=True)
        res["card"], res["power_limit"] = name, power
        print("TRAIN_BENCH " + json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
