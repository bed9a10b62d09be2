"""TEST INFRASTRUCTURE — round-2 fixtures generated from the REFERENCE itself (oracle/_ref), where a checkout of the
original project exists:

    make -C oracle ref REF=<checkout> && python oracle/make_golden_r2.py [datagen] [config5] [band]

  datagen_stats.npz   P5 (SURVEY appendix B): the statistic cfvpy/selfplay.py:158-169 logs — per last action (and "initial")
                      the example count, the sum of the targets and the sum of the per-example MSE of the seed-0 Net2 — over
                      >= 50 k training examples of the reference's RlRunner loops (recursive_solving.cc:160-182) with the seed-0
                      Net2 as value net, for TWO disjoint seed sets per shape (their difference is the band the GPU must meet).
  config5_net.npz     BASELINE config 5 with the value net: recursive_eval's sampled recursive strategies (seeds 0..R-1,
                      recursive_eval.cc:117-191,343-369) with the seed-0 Net2 evaluated in fp32 by ATen, 1x4f, 1024 iterations:
                      exploitability at powers of two.
  net_band.npz        derived tolerance of the tensor-core value nets: root value means after 1024 iterations when the
                      REFERENCE's own net is perturbed the way the tensor-core kernels perturb it — weights rounded to fp16 (fixed),
                      and on top of that outputs multiplied by 1 + sigma N(0,1), sigma = the measured relative output noise of the
                      kernels (5.4e-4 fp32-GELU, 7.7e-4 packed-half GELU), 8 noise seeds per root.
"""
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle import Oracle, game_dims  # noqa: E402
from oracle.make_golden import recursive_eval_reference, weights  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def last_action_stats(q, v, A, net=None):
    """selfplay.py:158-169: bucket = index of the one-hot last bid in the query (A = "initial": all zeros)."""
    onehot = q[:, 2:2 + A]
    aid = np.where(onehot.sum(1) > 0, onehot.argmax(1), A)
    cnt = np.bincount(aid, minlength=A + 1).astype(np.int64)
    vsum = np.zeros(A + 1); vsq = np.zeros(A + 1); lsum = np.zeros(A + 1)
    np.add.at(vsum, aid, v.astype(np.float64).sum(1))
    np.add.at(vsq, aid, (v.astype(np.float64) ** 2).sum(1))
    if net is not None:
        import torch
        with torch.no_grad():
            pred = net(torch.from_numpy(q)).numpy()
        np.add.at(lsum, aid, ((v - pred).astype(np.float64) ** 2).mean(1))
    return cnt, vsum, vsq, lsum


def datagen(R, threads=8):
    import torch
    torch.set_num_threads(1)          # one RlRunner per thread, like DataThreadLoop; no intra-op oversubscription
    from rebel_b200.models import make_selfplay_net
    out = {}
    for (D, F, games_per_thread) in [(1, 4, 1500), (1, 6, 1300)]:
        A, H, Q = game_dims(D, F)
        w = weights(D, F)
        net = make_selfplay_net(D, F, seed=0)
        for name, seed0 in (("a", 0), ("b", 5000)):
            res = [None] * threads
            t0 = time.time()

            def work(i):
                res[i] = R.rl_runner(D, F, seed0 + i, n_games=games_per_thread, num_iters=1024, net_w=w, cap=games_per_thread * 16)
            th = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
            [t.start() for t in th]; [t.join() for t in th]
            q = np.concatenate([r[0] for r in res]); v = np.concatenate([r[1] for r in res])
            cnt, vsum, vsq, lsum = last_action_stats(q, v, A, net)
            out[f"count_{name}_{D}x{F}"] = cnt; out[f"val_sum_{name}_{D}x{F}"] = vsum
            out[f"val_sq_{name}_{D}x{F}"] = vsq; out[f"loss_sum_{name}_{D}x{F}"] = lsum
            print(f"datagen {D}x{F} set {name}: {len(q)} examples in {time.time() - t0:.0f} s", flush=True)
        out[f"cfg_{D}x{F}"] = np.array([1024, 2, threads, games_per_thread])
    np.savez_compressed(os.path.join(OUT, "datagen_stats.npz"), **out)


def datagen_models(R, threads=8):
    """The reference's RlRunner loops with the ARITHMETIC MODEL of the tensor-core value-net kernels inside the reference's own net
    (ref_set_net_emulation: fp16 operands, and for model 2 the packed-half GELU) — what the reference itself generates when its
    net is evaluated the way the tensor-core kernels evaluate it.  Added to datagen_stats.npz as count_m{1,2}_* etc."""
    import torch
    torch.set_num_threads(1)
    from rebel_b200.models import make_selfplay_net
    path = os.path.join(OUT, "datagen_stats.npz")
    out = dict(np.load(path))
    for (D, F, games_per_thread) in [(1, 6, 1300), (1, 4, 1500)]:
        A, H, Q = game_dims(D, F)
        w = weights(D, F)
        net = make_selfplay_net(D, F, seed=0)
        for model in (2, 1):
            res = [None] * threads
            t0 = time.time()

            def work(i):
                R.set_net_emulation(model)          # thread-local
                res[i] = R.rl_runner(D, F, 9000 + i, n_games=games_per_thread, num_iters=1024, net_w=w, cap=games_per_thread * 16)
                R.set_net_emulation(0)
            th = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
            [t.start() for t in th]; [t.join() for t in th]
            q = np.concatenate([r[0] for r in res]); v = np.concatenate([r[1] for r in res])
            cnt, vsum, vsq, lsum = last_action_stats(q, v, A, net)
            out[f"count_m{model}_{D}x{F}"] = cnt; out[f"val_sum_m{model}_{D}x{F}"] = vsum
            out[f"val_sq_m{model}_{D}x{F}"] = vsq; out[f"loss_sum_m{model}_{D}x{F}"] = lsum
            print(f"datagen {D}x{F} kernel model {model}: {len(q)} examples in {time.time() - t0:.0f} s; counts {cnt / cnt.sum()}", flush=True)
            np.savez_compressed(path, **out)


def config5(R, RF=None):
    D, F, iters, reps = 1, 4, 1024, 64
    t0 = time.time()
    r = recursive_eval_reference(R, D, F, iters, reps, net_w=weights(D, F))
    out = {"cfg": np.array([D, F, iters, reps]), "checkpoints": r["checkpoints"], "exploitability": r["exploitability"]}
    r0 = recursive_eval_reference(R, D, F, iters, reps)
    out["exploitability_zero_net"] = r0["exploitability"]
    if RF is not None:      # the reference's own self-noise on this quantity: the -O3 build (FMA contraction) of the same sources
        rf = recursive_eval_reference(RF, D, F, iters, reps, net_w=weights(D, F))
        out["exploitability_fast_build"] = rf["exploitability"]
        print("config5 fast build", rf["exploitability"].mean(1), flush=True)
    np.savez_compressed(os.path.join(OUT, "config5_net.npz"), **out)
    print("config5", r["checkpoints"], r["exploitability"].mean(1), r0["exploitability"].mean(1), f"{time.time() - t0:.0f} s", flush=True)


def band(R):
    """Three perturbations of the reference's own value net, each a model of what the tensor-core kernels do to it:
    w16       the weights of the three Linear layers rounded to fp16 (a FIXED perturbation, identical on every iteration — the
              dominant, systematic part of the tensor-core kernels' error),
    pert{0,1} w16 plus independent relative gaussian noise of sigma = 5.4e-4 / 7.7e-4 on every output (the per-call part:
              fp16 activations, approximate GELU), 8 noise seeds."""
    out = {"sigmas": np.array([5.4e-4, 7.7e-4]), "seeds": np.arange(8)}
    for (D, F) in [(1, 4), (1, 6), (2, 3)]:
        A, H, Q = game_dims(D, F)
        w = weights(D, F)
        w16 = w.copy()
        o = 0
        for n in (256 * Q, 256, 256, 256, 256 * 256, 256, 256, 256, H * 256, H):      # state_dict order; only the weight matrices
            if n in (256 * Q, 256 * 256, H * 256):
                w16[o:o + n] = w16[o:o + n].astype(np.float16).astype(np.float32)
            o += n
        g = np.load(os.path.join(OUT, f"cfr_net_{D}x{F}.npz"))
        for i, (lb, pl) in enumerate(g["roots"]):
            b = g[f"beliefs{i}"]
            ref = g[f"mu1024_nofma{i}"]
            R.set_net_noise(0.0, 0)
            m16 = R.cfr_solve(D, F, b, [1024], int(lb), int(pl), num_iters=1024, net_w=w16, want=("avg",))["root_means"][0]
            out[f"mu_w16_{D}x{F}_{i}"] = m16
            print(f"band {D}x{F} root{i} fp16 weights: mean|dmu| {np.abs(m16 - ref).mean():.2e} max {np.abs(m16 - ref).max():.2e}", flush=True)
            for si, sigma in enumerate(out["sigmas"]):
                mus = []
                for seed in out["seeds"]:
                    R.set_net_noise(sigma, 1 + int(seed))
                    mus.append(R.cfr_solve(D, F, b, [1024], int(lb), int(pl), num_iters=1024, net_w=w16, want=("avg",))["root_means"][0])
                R.set_net_noise(0.0, 0)
                mus = np.stack(mus)
                out[f"mu_pert{si}_{D}x{F}_{i}"] = mus
                d = np.abs(mus - ref)
                print(f"band {D}x{F} root{i} fp16 weights + sigma={sigma:g}: mean|dmu| {d.mean():.2e} (per seed max {d.mean((1, 2)).max():.2e}), max {d.max():.2e}", flush=True)
    np.savez_compressed(os.path.join(OUT, "net_band.npz"), **out)


if __name__ == "__main__":
    what = sys.argv[1:] or ["band", "config5", "datagen"]
    R = Oracle("ref_nofma")      # deterministic build: band + config 5
    RF = Oracle("ref_fast")      # -O3 build for the statistical fixture (>= 100 k examples per shape)
    for k in what:
        if k == "config5":
            config5(R, RF)
        else:
            {"datagen": datagen, "datagen_models": datagen_models, "band": band}[k](RF if k.startswith("datagen") else R)
