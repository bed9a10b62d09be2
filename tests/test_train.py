"""The value-net trainer (cfrb_trainer_*, rebel_b200.trainer.Net2Trainer) and the training CLI (rebel_b200.train).

The CUDA step is checked against the reference trainer's step written in PyTorch (cfvpy/selfplay.py:135-152, 409-438, 636-651):
for every quantity, max |ours - fp64| <= max(4 max |torch fp32 - fp64|, 2^-20 max |fp64|), i.e. within four times the error
PyTorch's own fp32 step makes on the same inputs."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from rebel_b200.models import FLAT_ORDER, Net2, input_size, make_selfplay_net, output_size

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ the reference step in torch
def loss_func(x, kind):
    if kind == "huber":
        return (x.abs() > 1).to(x.dtype) * (x.abs() * 2 - 1) + (x.abs() <= 1).to(x.dtype) * x.pow(2)
    return x.pow(2)


def clip_grad_norm_(parameters, max_norm):
    parameters = [p for p in parameters if p.grad is not None]
    total = torch.norm(torch.stack([torch.norm(p.grad.detach(), 2) for p in parameters]), 2)
    coef = max_norm / (total + 1e-6)
    if coef < 1:
        for p in parameters:
            p.grad.detach().mul_(coef)
    return total


def torch_step(sd, osd, q, v, dtype, lr, max_norm, kind="huber"):
    """One step of the reference trainer in `dtype` on q's device from state_dict sd and Adam state osd (None = fresh)."""
    H, Q = v.shape[1], q.shape[1]
    net = _net_for(Q, H).to(device=q.device, dtype=dtype)
    net.load_state_dict({k: t.to(dtype) for k, t in sd.items()})
    net.train()
    opt = torch.optim.Adam(net.parameters(), lr=lr)
    if osd is not None:
        opt.load_state_dict(copy.deepcopy(osd))
        for s in opt.state.values():
            for k in ("exp_avg", "exp_avg_sq"):
                s[k] = s[k].to(dtype)
        for g in opt.param_groups:
            g["lr"] = lr
    opt.zero_grad()
    loss = loss_func(v.to(dtype) - net(q.to(dtype)), kind).mean(-1).mean()
    loss.backward()
    gn = clip_grad_norm_(list(net.parameters()), max_norm)
    grads = {k: p.grad.detach().clone() for k, p in zip(FLAT_ORDER, net.parameters())}
    opt.step()
    st = [opt.state[p] for p in net.parameters()]
    return dict(loss=loss.detach(), gnorm=gn.detach(), grads=grads,
                m={k: s["exp_avg"].clone() for k, s in zip(FLAT_ORDER, st)},
                v={k: s["exp_avg_sq"].clone() for k, s in zip(FLAT_ORDER, st)},
                params={k: t.detach().clone() for k, t in net.state_dict().items()}), opt


_GAMES = {}


def _net_for(Q, H):
    for (D, F) in [(1, 4), (1, 6), (2, 5), (2, 7), (2, 3)]:
        if input_size(F, D) == Q and output_size(F, D) == H:
            return Net2(num_faces=F, num_dice=D, n_hidden=256, n_layers=2, use_layer_norm=True)
    raise AssertionError((Q, H))


def ours_after(tr):
    p, m, v, _ = tr.get_state()
    sp, sm, sv = tr._split(p), tr._split(m), tr._split(v)
    return dict(grads=tr.grads(), m=sm, v=sv, params=sp)


def check_band(ours, r64, r32, what):
    """max |ours - fp64| <= max(4 max |fp32 - fp64|, 2^-20 max |fp64|)."""
    o = torch.as_tensor(ours).double().cpu()
    a = r64.double().cpu()
    b = r32.double().cpu()
    err, ref = float((o - a).abs().max()), float((b - a).abs().max())
    bound = max(4 * ref, 2.0 ** -20 * float(a.abs().max()))
    assert err <= bound, f"{what}: max|ours - fp64| = {err:.3e} > bound {bound:.3e} (torch fp32 error {ref:.3e})"
    return err, ref


def compare_step(tr, sd, osd, q, v, lr, max_norm, tag):
    loss, gn = tr.step(q, v)
    r64, _ = torch_step(sd, osd, q, v, torch.float64, lr, max_norm)
    r32, _ = torch_step(sd, osd, q, v, torch.float32, lr, max_norm)
    check_band(loss, r64["loss"], r32["loss"], f"{tag} loss")
    check_band(gn, r64["gnorm"], r32["gnorm"], f"{tag} grad norm")
    got = ours_after(tr)
    for what in ("grads", "m", "v", "params"):
        for k in FLAT_ORDER:
            check_band(got[what][k], r64[what][k], r32[what][k], f"{tag} {what} {k}")
    return r32


@pytest.fixture(scope="module")
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def selfplay_examples(D, F, rows):
    """Real training examples of the device self-play loop (random-init net, 64 CFR iterations per subgame)."""
    if (D, F) not in _GAMES:
        import rebel_b200.rela as rela
        from rebel_b200.models import flatten_state_dict
        cfg = rela.RecursiveSolvingParams()
        cfg.num_dice, cfg.num_faces, cfg.random_action_prob, cfg.sample_leaf = D, F, 0.25, True
        cfg.subgame_params.num_iters, cfg.subgame_params.max_depth = 64, 2
        cfg.subgame_params.linear_update, cfg.subgame_params.use_cfr = True, True
        cfg.concurrent_games = 256
        w = torch.from_numpy(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()))
        q, v = rela.run_selfplay_waves(cfg, 0, 5, 3, w)
        _GAMES[(D, F)] = (q.float().cuda(), v.float().cuda())
    q, v = _GAMES[(D, F)]
    assert q.shape[0] >= rows
    return q[:rows].contiguous(), v[:rows].contiguous()


def random_batch(D, F, n, seed):
    g = torch.Generator().manual_seed(seed)
    Q, H = input_size(F, D), output_size(F, D)
    return (torch.rand(n, Q, generator=g) * 2 - 1).cuda(), (torch.randn(n, H, generator=g) * 1.5).cuda()


# ------------------------------------------------------------------------------------------------------------- CPU tests
def test_cli_defaults_equal_reference_config():
    from rebel_b200 import train
    a = train.build_parser().parse_args(["--out", "x"])
    # conf/c02_selfplay/liars_sp.yaml, conf/common/optimizer/adam.yaml
    assert (a.num_dice, a.num_faces, a.seed) == (1, 4, 0)
    assert (a.decrease_lr_every, a.decrease_lr_times, a.grad_clip, a.loss) == (400, 2, 5.0, "huber")
    assert (a.max_epochs, a.train_epoch_size, a.batch, a.train_gen_ratio) == (10000, 25600, 512, 4)
    assert (a.replay_capacity, a.create_validation_set_every, a.lr) == (2000000, 100, 3e-4)
    assert (a.subgame_iters, a.mdp_depth, a.random_action_prob, a.sample_leaf, a.linear_update) == (1024, 2, 0.25, 1, 1)
    assert a.eval_every == 10


def test_lr_schedule_and_throttle_match_run_trainer():
    from rebel_b200.train import decayed_lr, throttle_passed
    lr, nd, seen = 3e-4, 0, []
    for epoch in range(2000):
        lr, nd = decayed_lr(lr, epoch, nd, 400, 2)
        seen.append(lr)
    assert seen[398] == 3e-4 and seen[399] == 1.5e-4 and seen[798] == 1.5e-4 and seen[799] == 7.5e-5 and seen[-1] == 7.5e-5
    lr, nd = 1.0, 0
    for epoch in range(1600):
        lr, nd = decayed_lr(lr, epoch, nd, 400, 0)             # decrease_lr_times 0: no limit
    assert lr == 1 / 16 and nd == 4
    assert throttle_passed(6400, 4, 25600, 0) and not throttle_passed(6399, 4, 25600, 0)
    assert throttle_passed(12800, 4, 25600, 1) and not throttle_passed(12799, 4, 25600, 1)
    assert throttle_passed(0, 0, 25600, 5)


def test_last_action_index_matches_reference():
    from rebel_b200.train import last_action_index
    A = 9
    q = torch.zeros(4, 2 + A + 8)
    q[1, 2 + 3] = 1
    q[2, 2 + A - 1] = 1
    q[3, 2 + 0] = 1
    assert last_action_index(q, A).tolist() == [A, 3, A - 1, 0]


@pytest.mark.parametrize("kw", [dict(n_layers=3, n_hidden=256), dict(n_layers=2, n_hidden=128)])
def test_trainer_refuses_other_net2_before_touching_a_device(kw):
    from rebel_b200.trainer import Net2Trainer
    sd = Net2(num_faces=4, num_dice=1, use_layer_norm=True, **kw).state_dict()
    with pytest.raises(ValueError):
        Net2Trainer(1, 4, "cuda:0", state_dict=sd)


def test_trainer_refuses_missing_keys_and_wrong_game_before_touching_a_device():
    from rebel_b200.trainer import Net2Trainer
    sd = make_selfplay_net(1, 4).state_dict()
    del sd["body.5.bias"]
    with pytest.raises(ValueError, match="missing"):
        Net2Trainer(1, 4, "cuda:0", state_dict=sd)
    with pytest.raises(ValueError, match="body.0.weight"):
        Net2Trainer(1, 6, "cuda:0", state_dict=make_selfplay_net(1, 4).state_dict())
    with pytest.raises(ValueError, match="loss"):
        Net2Trainer(1, 4, "cuda:0", loss="l1")


# ------------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 5), (2, 7)])
def test_one_step_against_torch_fp64(no_tf32, D, F):
    from rebel_b200.trainer import Net2Trainer
    sd = make_selfplay_net(D, F, seed=3).state_dict()
    for n in (1, 37, 512):
        for source in ("random", "selfplay"):
            q, v = random_batch(D, F, n, 10 * n + D + F) if source == "random" else selfplay_examples(D, F, n)
            for max_norm in (1e-3, 1e6):
                tr = Net2Trainer(D, F, "cuda:0", lr=3e-4, grad_clip=max_norm, state_dict=sd)
                compare_step(tr, sd, None, q, v, 3e-4, max_norm, f"{D}x{F}f n={n} {source} max_norm={max_norm}")
                if max_norm == 1e-3:
                    assert float(tr.last()[1]) > 1e-3          # clipping was active
                tr.close()


@pytest.mark.gpu
def test_mse_loss_step_against_torch_fp64(no_tf32):
    from rebel_b200.trainer import Net2Trainer
    D, F = 1, 6
    sd = make_selfplay_net(D, F, seed=4).state_dict()
    q, v = random_batch(D, F, 200, 77)
    tr = Net2Trainer(D, F, "cuda:0", grad_clip=5.0, loss="mse", state_dict=sd)
    loss, _ = tr.step(q, v)
    r64, _ = torch_step(sd, None, q, v, torch.float64, 3e-4, 5.0, "mse")
    r32, _ = torch_step(sd, None, q, v, torch.float32, 3e-4, 5.0, "mse")
    check_band(loss, r64["loss"], r32["loss"], "mse loss")
    got = ours_after(tr)
    for k in FLAT_ORDER:
        check_band(got["params"][k], r64["params"][k], r32["params"][k], f"mse params {k}")
    check_band(tr.loss(q, v), *(torch_eval_loss(r["params"], q, v, dt, "mse") for r, dt in ((r64, torch.float64), (r32, torch.float32))),
               "mse forward-only loss")


def torch_eval_loss(params, q, v, dtype, kind):
    net = _net_for(q.shape[1], v.shape[1]).to(device=q.device, dtype=dtype)
    net.load_state_dict(params)
    with torch.no_grad():
        return loss_func(v.to(dtype) - net(q.to(dtype)), kind).mean(-1).mean()


def fixed_dataset(steps, seed=0):
    q, v = selfplay_examples(1, 6, 512 * 3)
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, q.shape[0], (512,), generator=g).cuda() for _ in range(steps)], q, v


@pytest.mark.gpu
def test_teacher_forced_steps_along_a_torch_trajectory(no_tf32):
    """At steps 1, 10 and 200 of a torch fp32 run on 1x6f self-play examples, the trainer takes torch's parameters and Adam state
    (load_state_dict / load_optimizer_state) and one step from there stays in the band."""
    from rebel_b200.trainer import Net2Trainer
    ids, Qs, Vs = fixed_dataset(201)
    net = make_selfplay_net(1, 6, seed=5).cuda().train()
    opt = torch.optim.Adam(net.parameters(), lr=3e-4)
    tr = Net2Trainer(1, 6, "cuda:0", grad_clip=5.0)
    for t in range(201):
        if t in (1, 10, 200):
            sd = {k: x.detach().cpu().clone() for k, x in net.state_dict().items()}
            osd = opt.state_dict()
            tr.load_state_dict(sd)
            tr.load_optimizer_state(osd)
            assert tr.steps == t
            compare_step(tr, sd, osd, Qs[ids[t]], Vs[ids[t]], 3e-4, 5.0, f"step {t}")
        opt.zero_grad()
        loss_func(Vs[ids[t]] - net(Qs[ids[t]]), "huber").mean(-1).mean().backward()
        clip_grad_norm_(list(net.parameters()), 5.0)
        opt.step()


@pytest.mark.gpu
def test_optimizer_state_round_trips_through_torch():
    from rebel_b200.trainer import Net2Trainer
    q, v = random_batch(1, 4, 64, 1)
    tr = Net2Trainer(1, 4, "cuda:0")
    for _ in range(3):
        tr.step(q, v)
    osd = tr.optimizer_state()
    net = tr.net()
    opt = torch.optim.Adam(net.parameters(), lr=3e-4)
    opt.load_state_dict(osd)                                   # torch accepts it
    tr2 = Net2Trainer(1, 4, "cuda:0", state_dict=net.state_dict())
    tr2.load_optimizer_state(opt.state_dict())
    a, b = tr.get_state(), tr2.get_state()
    assert all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3])) and a[3] == b[3] == 3


def run_steps(tr, batches):
    out = []
    for q, v in batches:
        loss, gn = tr.step(q, v)
        out.append(torch.stack([loss, gn]))
    return torch.stack(out).cpu().numpy()


@pytest.mark.gpu
def test_steps_are_bit_identical_run_to_run_and_under_cuda_graph():
    from rebel_b200.trainer import Net2Trainer
    ids, Qs, Vs = fixed_dataset(50, seed=1)
    batches = [(Qs[i], Vs[i]) for i in ids]
    sd = make_selfplay_net(1, 6, seed=6).state_dict()
    states = []
    for _ in range(2):
        tr = Net2Trainer(1, 6, "cuda:0", grad_clip=0.5, state_dict=sd)
        lg = run_steps(tr, batches)
        states.append((lg,) + tr.get_state()[:3])
        tr.close()
    for a, b in zip(states[0], states[1]):
        assert np.array_equal(a, b)
    # the same 50 steps replayed from one captured step
    tr = Net2Trainer(1, 6, "cuda:0", grad_clip=0.5, state_dict=sd)
    sq, sv = batches[0][0].clone(), batches[0][1].clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):      # warm-up (nothing to initialise, but the graph pool wants it): undone below
        tr.step(sq, sv)
    torch.cuda.current_stream().wait_stream(s)
    tr.set_state(sd_flat(sd), step=0)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        loss, gn = tr.step(sq, sv)
    out = []
    for q, v in batches:
        sq.copy_(q)
        sv.copy_(v)
        g.replay()
        out.append(torch.stack([loss, gn]).clone())
    lg = torch.stack(out).cpu().numpy()
    got = (lg,) + tr.get_state()[:3]
    for a, b in zip(states[0], got):
        assert np.array_equal(a, b)


def sd_flat(sd):
    from rebel_b200.models import flatten_state_dict
    return flatten_state_dict(sd)


@pytest.mark.gpu
def test_loss_trajectory_stays_near_torch_fp32(no_tf32):
    """300 steps on a fixed 1x6f self-play dataset from the same initial net: the CUDA trainer's loss curve against torch fp32's
    (and torch fp64's as the scale of fp32 rounding along a trajectory).  Measured on an H100 (700 W power limit): max relative
    |ours - torch fp32| = 9.1e-7, |torch fp32 - fp64| = 1.6e-6 over the 300 steps (loss 0.290 -> 0.0018); the band is ten
    times the measured deviation."""
    from rebel_b200.trainer import Net2Trainer
    ids, Qs, Vs = fixed_dataset(300, seed=2)
    sd = make_selfplay_net(1, 6, seed=7).state_dict()
    tr = Net2Trainer(1, 6, "cuda:0", grad_clip=5.0, state_dict=sd)
    ours = run_steps(tr, [(Qs[i], Vs[i]) for i in ids])[:, 0]
    curves = {}
    for dt in (torch.float32, torch.float64):
        net = make_selfplay_net(1, 6, seed=7).to(device="cuda", dtype=dt).train()
        opt = torch.optim.Adam(net.parameters(), lr=3e-4)
        c = []
        for i in ids:
            opt.zero_grad()
            loss = loss_func(Vs[i].to(dt) - net(Qs[i].to(dt)), "huber").mean(-1).mean()
            loss.backward()
            clip_grad_norm_(list(net.parameters()), 5.0)
            opt.step()
            c.append(loss.detach())
        curves[dt] = torch.stack(c).double().cpu().numpy()
    rel = lambda a, b: float(np.max(np.abs(a - b) / np.abs(b)))
    d_ours, d_32 = rel(ours, curves[torch.float32]), rel(curves[torch.float32], curves[torch.float64])
    print(f"[trajectory] max relative |ours - torch fp32| = {d_ours:.3e}, |torch fp32 - fp64| = {d_32:.3e}, "
          f"loss {curves[torch.float32][0]:.4f} -> {curves[torch.float32][-1]:.4f}")
    assert ours[-1] < 0.8 * ours[0]
    assert d_ours <= TRAJECTORY_BAND, d_ours


TRAJECTORY_BAND = 1e-5


@pytest.mark.gpu
def test_invalid_batches_are_refused_and_leave_the_state_unchanged():
    from rebel_b200.trainer import Net2Trainer
    tr = Net2Trainer(1, 4, "cuda:0", max_batch=64)
    q, v = random_batch(1, 4, 65, 0)
    tr.step(q[:8], v[:8])
    before = tr.get_state()
    with pytest.raises(ValueError, match="max_batch"):
        tr.step(q, v)
    with pytest.raises(ValueError, match="shape"):
        tr.step(q[:8, :-1].contiguous(), v[:8])
    with pytest.raises(ValueError, match="shape"):
        tr.step(q[:8], torch.zeros(8, 5, device="cuda"))
    with pytest.raises(ValueError, match="device"):
        tr.step(q[:8].cpu(), v[:8].cpu())
    with pytest.raises(ValueError, match="rows"):
        tr.step(q[:8], v[:7])
    # the C ABI refuses what the wrapper would not pass: too many rows, host memory
    from rebel_b200 import capi
    import ctypes as C
    out = torch.empty(80, device="cuda")
    rc = capi.lib().cfrb_trainer_step(tr._t, C.c_void_p(q.data_ptr()), C.c_void_p(v.data_ptr()), 65, 3e-4, 5.0, 0, None,
                                      C.c_void_p(out.data_ptr()))
    assert rc < 0 and "max_batch" in capi.lib().cfrb_last_error().decode()
    hq, hv = q[:8].cpu(), v[:8].cpu()
    rc = capi.lib().cfrb_trainer_step(tr._t, C.c_void_p(hq.data_ptr()), C.c_void_p(hv.data_ptr()), 8, 3e-4, 5.0, 0, None, None)
    assert rc < 0 and "device memory" in capi.lib().cfrb_last_error().decode()
    rc = capi.lib().cfrb_trainer_step(tr._t, None, C.c_void_p(v.data_ptr()), 8, 3e-4, 5.0, 0, None, None)
    assert rc < 0 and "NULL" in capi.lib().cfrb_last_error().decode()
    after = tr.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(before[:3], after[:3])) and before[3] == after[3] == 1


@pytest.mark.gpu
def test_a_later_handle_leaves_earlier_handles_running():
    """The dynamic shared-memory limit is a process-wide attribute of each kernel: a handle created beside running ones (the
    training loop's exploitability evaluation next to its generator loops, another game's agent) must not lower it under their
    launches.  Handles of other tree depths (CFR kernels) and of a smaller game (tensor-core value net) are created after the
    first one, which must keep running."""
    from rebel_b200 import capi
    from rebel_b200.models import flatten_state_dict
    first = capi.WaveSolver(1, 6, 64, max_depth=2, num_iters=8, net_mode=capi.NET_TC_F16X2)
    first.set_weights(flatten_state_dict(make_selfplay_net(1, 6).state_dict()))
    lb = np.full(64, -1, np.int32)
    pl = np.zeros(64, np.int32)
    b = np.full((64, 2, 6), 1 / 6)
    first.begin(lb, pl, b)
    first.run(2)
    first.sync()
    for D, F, depth in ((1, 6, 1), (1, 6, 3), (1, 4, 100), (1, 4, 2)):
        other = capi.WaveSolver(D, F, 4, max_depth=depth, num_iters=8, net_mode=capi.NET_TC_F16X2)
        other.set_weights(flatten_state_dict(make_selfplay_net(D, F).state_dict()))
        H = F ** D
        other.begin(np.full(4, -1, np.int32), np.zeros(4, np.int32), np.full((4, 2, H), 1 / H))
        other.run(2)
        other.sync()
        first.run(2)
        first.sync()
        other.close()
    assert np.isfinite(first.fetch(("root_means",))["root_means"]).all()
    first.close()


@pytest.mark.gpu
def test_cli_end_to_end_1x4f(tmp_path):
    out = tmp_path / "run"
    cmd = [sys.executable, "-m", "rebel_b200.train", "--num_dice", "1", "--num_faces", "4", "--out", str(out), "--max_epochs", "21",
           "--train_epoch_size", "2048", "--val_batches", "8", "--exploit_every", "20", "--subgame_iters", "256",
           "--concurrent_games", "256", "--max_minutes", "8"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    from rebel_b200.train import parse_train
    lines = [parse_train(l) for l in r.stdout.splitlines() if l.startswith("TRAIN ")]
    assert [m["epoch"] for m in lines] == list(range(21))
    assert lines[-1]["weights_version"] > lines[0]["weights_version"]
    v0, v20 = lines[0]["val"]["valid_snapshot_0000"], lines[20]["val"]["valid_snapshot_0000"]
    assert v20 < v0, (v0, v20)
    assert "exploitability" in lines[0] and "exploitability" in lines[20]
    for e in (0, 10, 20):
        sd = torch.load(out / f"epoch{e}.ckpt")
        net = Net2(num_faces=4, num_dice=1, n_layers=2, use_layer_norm=True)
        net.load_state_dict(sd)
        torch.optim.Adam(net.parameters()).load_state_dict(torch.load(out / f"epoch{e}.optim"))
    import rebel_b200.rela as rela
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces = 1, 4
    cfg.subgame_params.num_iters, cfg.subgame_params.max_depth = 64, 2
    cfg.subgame_params.linear_update, cfg.subgame_params.use_cfr = True, True
    e = rela.compute_exploitability_with_net(cfg, str(out / "epoch20.torchscript"))
    assert np.isfinite(e) and e >= 0
    r2 = subprocess.run([sys.executable, "-m", "rebel_b200.recursive_eval", "--num_dice", "1", "--num_faces", "4", "--subgame_iters", "64",
                         "--cfr", "--net", str(out / "epoch20.torchscript")], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r2.returncode == 0, r2.stdout[-2000:] + r2.stderr[-2000:]
    print(r.stdout[-1500:])
