"""Train the ReBeL value net on one GPU beside self-play: the loop of the reference's run_trainer (cfvpy/selfplay.py:262-584) with
the defaults of conf/c02_selfplay/liars_sp.yaml and conf/common/optimizer/adam.yaml, the optimisation steps on the CUDA trainer
(rebel_b200.trainer.Net2Trainer) and no dependency beyond torch.

    python -m rebel_b200.train --num_dice 1 --num_faces 4 --out runs/1x4f [--max_epochs N] [--max_minutes M]

Generator loops (rela.create_cfr_thread: CFR, 1024 iterations, depth 2, random_action_prob 0.25, sample_leaf) fill a uniform
replay buffer (rela.ValuePrioritizedReplay, use_priority=False) and follow the trainer's weights through a rela.ModelLocker that
is updated every epoch.  An epoch waits until num_add * train_gen_ratio >= train_epoch_size * (epoch + 1), then runs
train_epoch_size / batch steps on a stream of its own while generation continues; the learning rate halves every 400 epochs, at
most twice.  Every 10 epochs the run writes epoch{N}.ckpt (state_dict), epoch{N}.torchscript and epoch{N}.optim (the
torch.optim.Adam state_dict layout) under --out and evaluates the validation snapshots (one every 100 epochs, from epoch 0); every
--exploit_every epochs it runs rela.compute_stats_with_net on games whose full tree that accepts.

Prints one tagged line per epoch, `TRAIN {...}`, whose text after the tag is JSON (see train_line)."""
import argparse
import json
import os
import sys
import time

import torch

# conf/c02_selfplay/liars_sp.yaml and conf/common/optimizer/adam.yaml
DEFAULTS = dict(num_dice=1, num_faces=4, seed=0, lr=3e-4, decrease_lr_every=400, decrease_lr_times=2, grad_clip=5.0, loss="huber",
                max_epochs=10000, train_epoch_size=25600, batch=512, train_gen_ratio=4.0, replay_capacity=2000000,
                create_validation_set_every=100, subgame_iters=1024, mdp_depth=2, random_action_prob=0.25, sample_leaf=1,
                linear_update=1)


def build_parser():
    d = DEFAULTS
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--num_dice", type=int, default=d["num_dice"])
    ap.add_argument("--num_faces", type=int, default=d["num_faces"])
    ap.add_argument("--out", type=str, required=True, help="directory for checkpoints")
    ap.add_argument("--seed", type=int, default=d["seed"], help="seed of the initial net")
    ap.add_argument("--init_checkpoint", type=str, default=None, help="initial net: a Net2 state_dict (.ckpt) or TorchScript file")
    ap.add_argument("--lr", type=float, default=d["lr"])
    ap.add_argument("--decrease_lr_every", type=int, default=d["decrease_lr_every"])
    ap.add_argument("--decrease_lr_times", type=int, default=d["decrease_lr_times"], help="0 = no limit")
    ap.add_argument("--grad_clip", type=float, default=d["grad_clip"], help="0 = no clipping")
    ap.add_argument("--loss", choices=("huber", "mse"), default=d["loss"])
    ap.add_argument("--max_epochs", type=int, default=d["max_epochs"])
    ap.add_argument("--max_minutes", type=float, default=None, help="wall-clock limit of the run")
    ap.add_argument("--train_epoch_size", type=int, default=d["train_epoch_size"], help="examples trained on per epoch")
    ap.add_argument("--batch", type=int, default=d["batch"])
    ap.add_argument("--train_gen_ratio", type=float, default=d["train_gen_ratio"], help="0 = no throttling")
    ap.add_argument("--replay_capacity", type=int, default=d["replay_capacity"])
    ap.add_argument("--create_validation_set_every", type=int, default=d["create_validation_set_every"])
    ap.add_argument("--val_batches", type=int, default=None, help="batches per validation snapshot (default 51200 / batch)")
    ap.add_argument("--eval_every", type=int, default=10, help="epochs between checkpoints and validation")
    ap.add_argument("--exploit_every", type=int, default=20, help="epochs between exploitability evaluations (0 = never)")
    ap.add_argument("--subgame_iters", type=int, default=d["subgame_iters"])
    ap.add_argument("--mdp_depth", type=int, default=d["mdp_depth"])
    ap.add_argument("--random_action_prob", type=float, default=d["random_action_prob"])
    ap.add_argument("--sample_leaf", type=int, default=d["sample_leaf"])
    ap.add_argument("--linear_update", type=int, default=d["linear_update"])
    ap.add_argument("--concurrent_games", type=int, default=None, help="games per generator loop (default: the rela default)")
    ap.add_argument("--device", type=int, default=0, help="CUDA ordinal of the trainer")
    ap.add_argument("--gen_devices", type=int, nargs="+", default=None, help="CUDA ordinals of the generator loops (default: --device)")
    ap.add_argument("--threads_per_device", type=int, default=1, help="generator loops per generator device")
    return ap


def decayed_lr(lr, epoch, num_decays, every, times):
    """The lr-halving schedule of run_trainer (selfplay.py:341-351), applied at the start of `epoch`: (lr, num_decays)."""
    if epoch % every == every - 1 and (not times or num_decays < times):
        return lr / 2, num_decays + 1
    return lr, num_decays


def throttle_passed(num_add, train_gen_ratio, train_size, epoch):
    """selfplay.py:391-405: epoch may start once num_add * train_gen_ratio >= train_size * (epoch + 1)."""
    return not train_gen_ratio or num_add * train_gen_ratio >= train_size * (epoch + 1)


def last_action_index(query, num_actions):
    """get_last_action_index (selfplay.py:624-633): the last bid of each query row, num_actions for the initial state."""
    with torch.no_grad():
        one_hot = torch.cat([query[:, 2:2 + num_actions], torch.full((len(query), 1), 0.1, device=query.device)], -1)
        return one_hot.max(-1).indices


def train_line(metrics):
    return "TRAIN " + json.dumps(metrics)


def parse_train(line):
    assert line.startswith("TRAIN "), line
    return json.loads(line[6:])


def load_initial_state_dict(path):
    try:
        return torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        return torch.load(path, map_location="cpu")


def make_params(rela, args):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = args.num_dice, args.num_faces
    cfg.random_action_prob, cfg.sample_leaf = args.random_action_prob, bool(args.sample_leaf)
    sp = cfg.subgame_params
    sp.num_iters, sp.max_depth, sp.linear_update, sp.use_cfr = args.subgame_iters, args.mdp_depth, bool(args.linear_update), True
    if args.concurrent_games:
        cfg.concurrent_games = args.concurrent_games
    return cfg


def main(argv=None):
    args = build_parser().parse_args(argv)
    import rebel_b200.rela as rela
    from rebel_b200.models import make_selfplay_net
    from rebel_b200.trainer import Net2Trainer

    t_start = time.time()
    deadline = t_start + 60 * args.max_minutes if args.max_minutes else None
    os.makedirs(args.out, exist_ok=True)
    D, F, B = args.num_dice, args.num_faces, args.batch
    A = 1 + 2 * D * F
    dev = torch.device("cuda", args.device)
    sd = load_initial_state_dict(args.init_checkpoint) if args.init_checkpoint else make_selfplay_net(D, F, args.seed).state_dict()
    trainer = Net2Trainer(D, F, dev, max_batch=B, lr=args.lr, grad_clip=args.grad_clip, loss=args.loss, state_dict=sd)
    gen_devices = args.gen_devices if args.gen_devices else [args.device]
    lockers = [rela.ModelLocker([torch.jit.script(trainer.net())], f"cuda:{d}") for d in gen_devices]
    replay = rela.ValuePrioritizedReplay(capacity=args.replay_capacity, seed=10001, alpha=1.0, beta=1.0, prefetch=8,
                                         use_priority=False, compressed_values=False)
    cfg = make_params(rela, args)
    ctx = rela.Context()
    loops = []
    for i in range(len(gen_devices) * args.threads_per_device):
        loops.append(rela.create_cfr_thread(lockers[i % len(lockers)], replay, cfg, i))
        ctx.push_env_thread(loops[-1])
    train_stream = torch.cuda.Stream(dev)
    epoch_size = args.train_epoch_size // B
    val_batches = args.val_batches or max(1, 512 * 100 // B)
    val_sets, exploit_ok = [], args.exploit_every > 0
    lr, num_decays = args.lr, 0
    print(f"[train] {D}x{F}f: {len(loops)} generator loop(s) on cuda:{gen_devices}, trainer on {dev}, {epoch_size} steps of "
          f"{B} per epoch, out {args.out}", flush=True)

    def wait_for(cond):
        while not cond():
            if ctx.error():
                raise RuntimeError(f"generator loop failed: {ctx.error()}")
            if deadline and time.time() > deadline:
                return False
            time.sleep(0.02)
        return True

    ctx.start()
    t_gen = time.time()
    try:
        if not wait_for(lambda: replay.size() >= 2 * B):           # burn-in (selfplay.py:314-327)
            return
        for epoch in range(args.max_epochs):
            lr, num_decays = decayed_lr(lr, epoch, num_decays, args.decrease_lr_every, args.decrease_lr_times)
            trainer.lr = lr
            m = {"epoch": epoch, "lr": lr}
            if args.create_validation_set_every and epoch % args.create_validation_set_every == 0:
                # host memory, like the reference (selfplay.py:357-362): the snapshots accumulate over the run
                val_sets.append((f"valid_snapshot_{epoch:04d}", [replay.sample(B, "cpu")[0] for _ in range(val_batches)]))
            if not wait_for(lambda: throttle_passed(replay.num_add(), args.train_gen_ratio, args.train_epoch_size, epoch)):
                break
            t0 = time.time()
            losses, norms = [], []
            with torch.cuda.stream(train_stream):
                loss_sum = torch.zeros(A + 1, device=dev, dtype=torch.float64)
                count = torch.zeros(A + 1, device=dev, dtype=torch.float64)
                for _ in range(epoch_size):
                    batch, _ = replay.sample(B, f"cuda:{args.device}")
                    loss, gnorm = trainer.step(batch.query, batch.values)
                    losses.append(loss)
                    norms.append(gnorm)
                    idx = last_action_index(batch.query, A)
                    loss_sum += torch.bincount(idx, weights=trainer.last_row_loss.double(), minlength=A + 1)
                    count += torch.bincount(idx, minlength=A + 1).double()
                train_stream.synchronize()
            t_train = time.time() - t0
            if losses:
                L, G = torch.stack(losses).double(), torch.stack(norms).double()
                m["loss"] = float(L.mean())
                m["grad_mean"], m["grad_max"] = float(G.mean()), float(G.max())
                m["grad_clip_ratio"] = float((G >= args.grad_clip - 1e-5).double().mean()) if args.grad_clip else 0.0
                names = [str(a) for a in range(A)] + ["initial"]
                ls, cs = loss_sum.cpu().tolist(), count.cpu().tolist()
                m["loss_by_last_action"] = {k: (s / c if c else None) for k, s, c in zip(names, ls, cs)}
                m["share_by_last_action"] = {k: c / (epoch_size * B) for k, c in zip(names, cs)}
                m["train_examples_per_s"] = epoch_size * B / t_train
            m["buffer_size"], m["buffer_added"] = replay.size(), replay.num_add()
            m["gen_examples_per_s"] = replay.num_add() / (time.time() - t_gen)
            net = trainer.net()
            for lk in lockers:
                lk.update_model(net)
            m["weights_version"] = min(lp.weights_version for lp in loops)
            if epoch % args.eval_every == 0:
                val = {}
                with torch.cuda.stream(train_stream):
                    for name, batches in val_sets:
                        val[name] = float(torch.stack([trainer.loss(b.query.to(dev), b.values.to(dev))
                                                       for b in batches]).double().mean())
                m["val"] = val
                stem = os.path.join(args.out, f"epoch{epoch}")
                torch.save(net.state_dict(), stem + ".ckpt")
                torch.jit.save(torch.jit.script(net), stem + ".torchscript")
                torch.save(trainer.optimizer_state(), stem + ".optim")
                if exploit_ok and epoch % args.exploit_every == 0:
                    try:
                        e, mse_net, mse_fp = rela.compute_stats_with_net(cfg, stem + ".torchscript")
                        m["exploitability"], m["mse_net_reach"], m["mse_fp_reach"] = e, mse_net, mse_fp
                    except RuntimeError as err:
                        exploit_ok = False
                        print(f"[train] no exploitability for {D}x{F}f: {err}", file=sys.stderr, flush=True)
            m["minutes"] = (time.time() - t_start) / 60
            print(train_line(m), flush=True)
            if deadline and time.time() > deadline:
                break
    finally:
        ctx.terminate()
        while not ctx.terminated():
            time.sleep(0.01)
    if ctx.error():
        raise RuntimeError(f"generator loop failed: {ctx.error()}")


if __name__ == "__main__":
    main()
