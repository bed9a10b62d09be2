"""Train the ReBeL value net on one GPU beside self-play: the loop of the reference's run_trainer (cfvpy/selfplay.py:262-584) with
the defaults of conf/c02_selfplay/liars_sp.yaml and conf/common/optimizer/adam.yaml, the optimisation steps on the CUDA trainer
(rebel_b200.trainer.Net2Trainer) and no dependency beyond torch.

    python -m rebel_b200.train --num_dice 1 --num_faces 4 --out runs/1x4f [--max_epochs N] [--max_minutes M]
    python -m rebel_b200.train --num_dice 1 --num_faces 4 --out runs/1x4f --deterministic [--state_every S] [--resume]

Generator loops (rela.create_cfr_thread: CFR, 1024 iterations, depth 2, random_action_prob 0.25, sample_leaf) fill a uniform
replay buffer (rela.ValuePrioritizedReplay, use_priority=False) and follow the trainer's weights through a rela.ModelLocker that
is updated every epoch.  An epoch waits until num_add * train_gen_ratio >= train_epoch_size * (epoch + 1), then runs
train_epoch_size / batch steps on a stream of its own while generation continues; the learning rate halves every 400 epochs, at
most twice.  Every 10 epochs the run writes epoch{N}.ckpt (state_dict), epoch{N}.torchscript and epoch{N}.optim (the
torch.optim.Adam state_dict layout) under --out and evaluates the validation snapshots (one every 100 epochs, from epoch 0); every
--exploit_every epochs it runs rela.compute_stats_with_net (exploitability, mse_net_reach, mse_fp_reach): on games of up to 23
actions (2x5f, 5x2f, 1x10f and 1x11f included, whose evaluation runs without dense full-tree tables); above that the run says
so once and stops evaluating.

--deterministic replaces the threads by a fixed schedule, so that two runs with the same arguments print the same TRAIN lines
(but for the wall-clock fields minutes and *_per_s) and write the same checkpoints.  There is one rela.SelfPlayGenerator per
generator loop, seeded like the loop.  A round is one wave of every generator, whose examples go to the replay in generator order;
burn-in runs rounds until the buffer holds 2 * batch rows, and before epoch e rounds run until the throttle above passes.  No wave
runs during an epoch, and every generator takes the trainer's weights after it.  Such a run saves its state under --out
(state.pt, one replay.e{N}.state file, and one file per validation snapshot, written once) every --state_every epochs and when
it ends: at --max_epochs, at the --max_minutes deadline (checked between epochs) or on SIGINT / SIGTERM (the epoch in progress is
finished first).  --resume continues from that
state exactly as if the run had never stopped; it refuses a state whose run-defining arguments differ from the command line's.
Since nothing samples the replay while a deterministic run generates, the buffer's slack above --replay_capacity (a quarter of it)
must hold one epoch's generation plus one round; other arguments are refused.

Prints one tagged line per epoch, `TRAIN {...}`, whose text after the tag is JSON (see train_line)."""
import argparse
import glob
import json
import math
import os
import signal
import sys
import time

import numpy as np
import torch

# conf/c02_selfplay/liars_sp.yaml and conf/common/optimizer/adam.yaml
DEFAULTS = dict(num_dice=1, num_faces=4, seed=0, lr=3e-4, decrease_lr_every=400, decrease_lr_times=2, grad_clip=5.0, loss="huber",
                max_epochs=10000, train_epoch_size=25600, batch=512, train_gen_ratio=4.0, replay_capacity=2000000,
                create_validation_set_every=100, subgame_iters=1024, mdp_depth=2, random_action_prob=0.25, sample_leaf=1,
                linear_update=1)
STATE_EVERY = 100          # default --state_every of a deterministic run
STATE_FORMAT = 1
STATE_FILE = "state.pt"
# Arguments that define the data or the optimisation of a run: a resumed run must agree with the saved one on every one of them
# (run_definition adds the generator count and the settings the generators take from the environment).
DEFINING = ("num_dice", "num_faces", "seed", "init_checkpoint", "lr", "decrease_lr_every", "decrease_lr_times", "grad_clip", "loss",
            "train_epoch_size", "batch", "train_gen_ratio", "replay_capacity", "create_validation_set_every", "val_batches",
            "eval_every", "exploit_every", "subgame_iters", "mdp_depth", "random_action_prob", "sample_leaf", "linear_update")


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
    ap.add_argument("--deterministic", action="store_true",
                    help="fixed generation schedule: the run is reproducible and its state can be saved and resumed")
    ap.add_argument("--state_every", type=int, default=None,
                    help=f"deterministic runs: epochs between state saves (default {STATE_EVERY}; 0 = only when the run ends)")
    ap.add_argument("--resume", action="store_true", help="deterministic runs: continue from the state saved under --out")
    return ap


def parse_args(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if not args.deterministic:
        if args.resume:
            ap.error("--resume continues a --deterministic run only (a threaded run's generation depends on timing)")
        if args.state_every is not None:
            ap.error("--state_every applies to --deterministic runs only")
    elif not args.train_gen_ratio:
        ap.error("--deterministic needs --train_gen_ratio > 0: the ratio defines how much is generated before each epoch")
    if args.state_every is not None and args.state_every < 0:
        ap.error("--state_every must be >= 0")
    return args


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


def sums_by_last_action(indices, row_losses, num_actions):
    """(loss sum, row count) per last action [A + 1] of an epoch's rows, summed on the host in row order: the same bits on every
    run, unlike an atomic device sum."""
    idx = torch.cat(indices).cpu().numpy()
    loss = torch.cat(row_losses).double().cpu().numpy()
    return np.bincount(idx, weights=loss, minlength=num_actions + 1), np.bincount(idx, minlength=num_actions + 1)


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


def gen_devices_of(args):
    return args.gen_devices if args.gen_devices else [args.device]


def val_batches_of(args):
    return args.val_batches or max(1, 512 * 100 // args.batch)


def run_definition(args, cfg):
    """What a resumed run must share with the saved one: the DEFINING arguments (val_batches as used), the number of generator
    loops, and the generators' games per loop, net mode and table dtype (cfg, which takes them from the environment by default)."""
    d = {k: getattr(args, k) for k in DEFINING}
    d["val_batches"] = val_batches_of(args)
    d["generators"] = len(gen_devices_of(args)) * args.threads_per_device
    d["concurrent_games"], d["net_mode"], d["state_dtype"] = cfg.concurrent_games, cfg.net_mode, cfg.state_dtype
    return d


def load_run_state(args, cfg):
    """The state saved under --out, checked against this command line; refusals happen before any device is touched."""
    path = os.path.join(args.out, STATE_FILE)
    if not os.path.exists(path):
        raise SystemExit(f"--resume: no saved state at {path}")
    st = torch.load(path, map_location="cpu", weights_only=True)
    if st.get("format") != STATE_FORMAT:
        raise SystemExit(f"--resume: {path} has state format {st.get('format')!r}, this version reads {STATE_FORMAT}")
    now = run_definition(args, cfg)
    for k, v in now.items():
        if st["definition"].get(k) != v:
            raise SystemExit(f"--resume: {k} was {st['definition'].get(k)!r} in the saved run and is {v!r} now; a resumed run must "
                             f"keep every argument that defines its data or optimisation")
    for name in [st["replay_file"]] + [val_file(n) for n in st["val_names"]]:
        if not os.path.exists(os.path.join(args.out, name)):
            raise SystemExit(f"--resume: {os.path.join(args.out, name)}, named by {path}, is missing")
    return st


def val_file(name):
    return f"{name}.pt"


def check_replay_room(args, cfg):
    """A deterministic run samples nothing while it generates, so the ring's slack above replay_capacity (ValuePrioritizedReplay
    keeps 1.25 x capacity rows) must take the rows of the longest generation phase: one epoch's share, or the burn-in, plus at most
    one round of overshoot.  A threaded run would block there until the trainer samples; this schedule would never go on."""
    per_round = 2 * cfg.concurrent_games * len(gen_devices_of(args)) * args.threads_per_device
    slack = int(1.25 * args.replay_capacity) - args.replay_capacity
    need = math.ceil(max(args.train_epoch_size / args.train_gen_ratio, 2 * args.batch) / per_round) * per_round
    if need > slack:
        raise SystemExit(f"--deterministic: a generation phase adds up to {need} rows ({per_round} per round), more than the "
                         f"{slack} rows the replay holds beyond --replay_capacity {args.replay_capacity}; raise --replay_capacity to "
                         f"at least {4 * need}")


def _fsync(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _write_atomic(path, write):
    """write(tmp_path), then fsync and os.replace: a crash leaves either the previous file or the new one."""
    write(path + ".tmp")
    _fsync(path + ".tmp")
    os.replace(path + ".tmp", path)
    return os.path.getsize(path)


def save_run_state(out, st, replay):
    """Writes the validation snapshots not saved before (one file each: they never change), the replay's state and then state.pt,
    each under a temporary name first, so that a crash in the middle leaves the previous state intact.  Returns (bytes written,
    seconds)."""
    t0, nbytes = time.time(), 0
    for name, q, v in st["val_sets"]:
        path = os.path.join(out, val_file(name))
        if not os.path.exists(path):
            nbytes += _write_atomic(path, lambda p: torch.save({"query": q, "values": v}, p))
    replay_file = f"replay.e{st['next_epoch']}.state"
    nbytes += _write_atomic(os.path.join(out, replay_file), replay.save_state)
    names = [name for name, _, _ in st["val_sets"]]
    st = {k: v for k, v in st.items() if k != "val_sets"}
    st.update(replay_file=replay_file, val_names=names)
    nbytes += _write_atomic(os.path.join(out, STATE_FILE), lambda p: torch.save(st, p))
    for old in glob.glob(os.path.join(out, "replay.e*.state")):
        if os.path.basename(old) != replay_file:
            os.remove(old)
    return nbytes, time.time() - t0


def load_val_sets(out, names):
    sets = []
    for name in names:
        d = torch.load(os.path.join(out, val_file(name)), map_location="cpu", weights_only=True)
        sets.append((name, d["query"], d["values"]))
    return sets


def generate(gens, replay, enough):
    """Rounds of one wave per generator, the examples appended in generator order, until enough(size, num_add) holds.  Every round
    adds the same number of rows and nothing is sampled meanwhile, so the number of rounds is known up front: all but the last
    round leave each generator's next wave running, and the last one drains them.  Generators on different devices overlap."""
    per_round = sum(2 * g.concurrent_games for g in gens)
    size, added, rounds = replay.size(), replay.num_add(), 0
    while not enough(size, added):
        size, added, rounds = size + per_round, added + per_round, rounds + 1
    for r in range(rounds):
        for g in gens:
            g.run(replay, keep_running=r + 1 < rounds)
    assert enough(replay.size(), replay.num_add())


class StopRequest:
    """SIGINT / SIGTERM during a deterministic run: the epoch in progress is finished, the state saved, and the run ends.  A second
    signal interrupts at once."""

    def __init__(self):
        self.requested = False
        self._old = {s: signal.signal(s, self._handle) for s in (signal.SIGINT, signal.SIGTERM)}

    def _handle(self, signum, frame):
        if self.requested:
            raise KeyboardInterrupt
        self.requested = True
        print(f"[train] signal {signum}: stopping after the current epoch", file=sys.stderr, flush=True)

    def restore(self):
        for s, h in self._old.items():
            signal.signal(s, h)


def main(argv=None):
    args = parse_args(argv)
    import rebel_b200.rela as rela
    from rebel_b200.models import make_selfplay_net
    from rebel_b200.trainer import Net2Trainer

    t_start = time.time()
    cfg = make_params(rela, args)
    if args.deterministic:
        check_replay_room(args, cfg)
    resumed = load_run_state(args, cfg) if args.resume else None
    deadline = t_start + 60 * args.max_minutes if args.max_minutes else None
    os.makedirs(args.out, exist_ok=True)
    D, F, B = args.num_dice, args.num_faces, args.batch
    A = 1 + 2 * D * F
    dev = torch.device("cuda", args.device)
    if args.init_checkpoint and not resumed:
        sd = load_initial_state_dict(args.init_checkpoint)
    else:
        sd = make_selfplay_net(D, F, args.seed).state_dict()
    trainer = Net2Trainer(D, F, dev, max_batch=B, lr=args.lr, grad_clip=args.grad_clip, loss=args.loss, state_dict=sd)
    gen_devices = gen_devices_of(args)
    n_gen = len(gen_devices) * args.threads_per_device
    replay = rela.ValuePrioritizedReplay(capacity=args.replay_capacity, seed=10001, alpha=1.0, beta=1.0, prefetch=8,
                                         use_priority=False, compressed_values=False)
    train_stream = torch.cuda.Stream(dev)
    epoch_size = args.train_epoch_size // B
    val_batches = val_batches_of(args)
    val_sets, exploit_ok = [], args.exploit_every > 0
    lr, num_decays, start_epoch = args.lr, 0, 0
    if args.deterministic:
        ctx, loops, lockers = None, [], []
        gens = [rela.SelfPlayGenerator(cfg, gen_devices[i % len(gen_devices)], i) for i in range(n_gen)]
        if resumed:
            st = resumed
            trainer.set_state(st["params"].numpy(), st["exp_avg"].numpy(), st["exp_avg_sq"].numpy(), st["step"])
            replay.load_state(os.path.join(args.out, st["replay_file"]), gen_devices[0])
            for g, image in zip(gens, st["sessions"]):
                g.load_state(image.numpy().tobytes())
            val_sets = load_val_sets(args.out, st["val_names"])
            exploit_ok, lr, num_decays, start_epoch = st["exploit_ok"], st["lr"], st["num_decays"], st["next_epoch"]
        # the version a ModelLocker would have: 1 for the initial net, + 1 per epoch
        flat = torch.from_numpy(trainer.get_state()[0])
        for g in gens:
            g.set_weights(flat, start_epoch + 1)
        stop = StopRequest()
        state_every = STATE_EVERY if args.state_every is None else args.state_every
    else:
        lockers = [rela.ModelLocker([torch.jit.script(trainer.net())], f"cuda:{d}") for d in gen_devices]
        ctx, loops, gens = rela.Context(), [], []
        for i in range(n_gen):
            loops.append(rela.create_cfr_thread(lockers[i % len(lockers)], replay, cfg, i))
            ctx.push_env_thread(loops[-1])
    mode = "deterministic" if args.deterministic else "threaded"
    print(f"[train] {D}x{F}f: {n_gen} generator loop(s) on cuda:{gen_devices} ({mode}), trainer on {dev}, {epoch_size} steps of "
          f"{B} per epoch, out {args.out}" + (f", resumed at epoch {start_epoch}" if resumed else ""), flush=True)

    def wait_for(cond):
        while not cond():
            if ctx.error():
                raise RuntimeError(f"generator loop failed: {ctx.error()}")
            if deadline and time.time() > deadline:
                return False
            time.sleep(0.02)
        return True

    def run_state(next_epoch):
        p, m, v, step = trainer.get_state()
        return {"format": STATE_FORMAT, "definition": run_definition(args, cfg), "next_epoch": next_epoch, "lr": lr,
                "num_decays": num_decays, "params": torch.from_numpy(p), "exp_avg": torch.from_numpy(m),
                "exp_avg_sq": torch.from_numpy(v), "step": step, "val_sets": val_sets, "exploit_ok": exploit_ok,
                "sessions": [torch.frombuffer(bytearray(g.state()), dtype=torch.uint8) for g in gens]}

    def save(next_epoch):
        nbytes, secs = save_run_state(args.out, run_state(next_epoch), replay)
        print(f"[train] state saved at epoch {next_epoch}: {nbytes} bytes in {secs:.3f} s", flush=True)

    if ctx is not None:
        ctx.start()
    t_gen = time.time()
    if resumed:
        print(f"[train] resumed in {t_gen - t_start:.3f} s", flush=True)
    next_epoch = start_epoch
    try:
        if args.deterministic:
            if not resumed:
                generate(gens, replay, lambda size, added: size >= 2 * B)                    # burn-in (selfplay.py:314-327)
        elif not wait_for(lambda: replay.size() >= 2 * B):
            return
        for epoch in range(start_epoch, args.max_epochs):
            lr, num_decays = decayed_lr(lr, epoch, num_decays, args.decrease_lr_every, args.decrease_lr_times)
            trainer.lr = lr
            m = {"epoch": epoch, "lr": lr}
            if args.create_validation_set_every and epoch % args.create_validation_set_every == 0:
                # host memory, like the reference (selfplay.py:357-362): the snapshots accumulate over the run
                batches = [replay.sample(B, "cpu")[0] for _ in range(val_batches)]
                val_sets.append((f"valid_snapshot_{epoch:04d}", torch.stack([b.query for b in batches]),
                                 torch.stack([b.values for b in batches])))
            passed = lambda added: throttle_passed(added, args.train_gen_ratio, args.train_epoch_size, epoch)
            if args.deterministic:
                t0, added0 = time.time(), replay.num_add()
                generate(gens, replay, lambda size, added: passed(added))
                if replay.num_add() > added0:   # the generators' own rate, while they run
                    m["wave_examples_per_s"] = (replay.num_add() - added0) / (time.time() - t0)
            elif not wait_for(lambda: passed(replay.num_add())):
                break
            t0 = time.time()
            losses, norms, indices, row_losses = [], [], [], []
            with torch.cuda.stream(train_stream):
                for _ in range(epoch_size):
                    batch, _ = replay.sample(B, f"cuda:{args.device}")
                    loss, gnorm = trainer.step(batch.query, batch.values)
                    losses.append(loss)
                    norms.append(gnorm)
                    indices.append(last_action_index(batch.query, A))
                    row_losses.append(trainer.last_row_loss)
                train_stream.synchronize()
            t_train = time.time() - t0
            if losses:
                L, G = torch.stack(losses).double(), torch.stack(norms).double()
                m["loss"] = float(L.mean())
                m["grad_mean"], m["grad_max"] = float(G.mean()), float(G.max())
                m["grad_clip_ratio"] = float((G >= args.grad_clip - 1e-5).double().mean()) if args.grad_clip else 0.0
                names = [str(a) for a in range(A)] + ["initial"]
                ls, cs = sums_by_last_action(indices, row_losses, A)
                m["loss_by_last_action"] = {k: (float(s) / int(c) if c else None) for k, s, c in zip(names, ls, cs)}
                m["share_by_last_action"] = {k: int(c) / (epoch_size * B) for k, c in zip(names, cs)}
                m["train_examples_per_s"] = epoch_size * B / t_train
            m["buffer_size"], m["buffer_added"] = replay.size(), replay.num_add()
            m["gen_examples_per_s"] = replay.num_add() / (time.time() - t_gen)
            net = trainer.net()
            if args.deterministic:
                flat = torch.from_numpy(trainer.get_state()[0])
                for g in gens:
                    g.set_weights(flat, epoch + 2)
                m["weights_version"] = min(g.weights_version for g in gens)
            else:
                for lk in lockers:
                    lk.update_model(net)
                m["weights_version"] = min(lp.weights_version for lp in loops)
            if epoch % args.eval_every == 0:
                val = {}
                with torch.cuda.stream(train_stream):
                    for name, qs, vs in val_sets:
                        val[name] = float(torch.stack([trainer.loss(q.to(dev), v.to(dev)) for q, v in zip(qs, vs)]).double().mean())
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
            next_epoch = epoch + 1
            if args.deterministic and stop.requested:
                break
            if deadline and time.time() > deadline:
                break
            if args.deterministic and state_every and next_epoch % state_every == 0 and next_epoch < args.max_epochs:
                save(next_epoch)
        if args.deterministic:
            save(next_epoch)                 # the end of the run: max_epochs, the deadline or a signal
    finally:
        if ctx is not None:
            ctx.terminate()
            while not ctx.terminated():
                time.sleep(0.01)
        if args.deterministic:
            stop.restore()
    if ctx is not None and ctx.error():
        raise RuntimeError(f"generator loop failed: {ctx.error()}")


if __name__ == "__main__":
    main()
