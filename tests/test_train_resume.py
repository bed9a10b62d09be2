"""Reproducible and resumable training runs: the self-play session image (cfrb_selfplay_export / _import), rela.SelfPlayGenerator,
the replay's save_state / load_state, and `python -m rebel_b200.train --deterministic / --resume / --state_every`."""
import os
import signal
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def make_replay(rela, capacity=40, use_priority=False, seed=7, alpha=None):
    alpha = (0.6 if use_priority else 1.0) if alpha is None else alpha
    return rela.ValuePrioritizedReplay(capacity=capacity, seed=seed, alpha=alpha, beta=0.4, prefetch=8, use_priority=use_priority,
                                       compressed_values=False)


def fill_and_sample(rela, r, use_priority, rounds=9):
    """Appends blocks of rows and samples after each, so that the ring wraps and rows get evicted."""
    g = torch.Generator().manual_seed(0)
    for _ in range(rounds):
        q, v = torch.rand(7, 5, generator=g), torch.rand(7, 3, generator=g)
        r.push([q, v, torch.rand(7, generator=g) + 0.1])
        r.sample(6, "cpu")
        if use_priority:
            r.update_priority(torch.rand(6, generator=g) + 0.1)
    return g


def replay_round_trip(tmp_path, use_priority):
    import rebel_b200.rela as rela
    r = make_replay(rela, use_priority=use_priority)
    g = fill_and_sample(rela, r, use_priority)
    assert r.num_add() > 1.25 * 40            # the ring has wrapped
    path = str(tmp_path / "replay.state")
    r.save_state(path)
    r2 = make_replay(rela, use_priority=use_priority)
    r2.load_state(path)
    assert (r2.size(), r2.num_add()) == (r.size(), r.num_add())
    for k in range(6):
        (b1, w1), (b2, w2) = r.sample(11, "cpu"), r2.sample(11, "cpu")
        assert torch.equal(b1.query, b2.query) and torch.equal(b1.values, b2.values) and torch.equal(w1, w2), k
        if use_priority:
            p = torch.rand(11, generator=g) + 0.05
            r.update_priority(p)
            r2.update_priority(p)
        if k == 2:                            # appends after the load evict and wrap alike
            q, v = torch.rand(9, 5, generator=g), torch.rand(9, 3, generator=g)
            r.push([q, v, torch.ones(9)])
            r2.push([q, v, torch.ones(9)])
        assert (r2.size(), r2.num_add()) == (r.size(), r.num_add())
    return r2


# ------------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("use_priority", [False, True])
def test_replay_state_round_trip(tmp_path, use_priority):
    replay_round_trip(tmp_path, use_priority)


def test_replay_state_refusals(tmp_path):
    import rebel_b200.rela as rela
    r = make_replay(rela, use_priority=True)
    fill_and_sample(rela, r, True)
    r.sample(4, "cpu")
    with pytest.raises(RuntimeError, match="priorities"):
        r.save_state(str(tmp_path / "pending.state"))
    r.update_priority(torch.ones(4))
    path = str(tmp_path / "replay.state")
    r.save_state(path)
    busy = make_replay(rela, use_priority=True)
    busy.push([torch.rand(2, 5), torch.rand(2, 3), torch.ones(2)])
    with pytest.raises(RuntimeError, match="not empty"):
        busy.load_state(path)
    for kw, field in ((dict(capacity=41), "capacity"), (dict(seed=8), "seed"), (dict(alpha=0.5), "alpha"),
                      (dict(use_priority=False, alpha=0.6), "use_priority")):
        other = make_replay(rela, **dict(dict(use_priority=True), **kw))
        with pytest.raises(RuntimeError, match=field):
            other.load_state(path)
        assert other.size() == 0 and other.num_add() == 0
    blob = open(path, "rb").read()
    for cut in (10, len(blob) // 2, len(blob) - 1):
        short = str(tmp_path / f"short{cut}.state")
        open(short, "wb").write(blob[:cut])
        fresh = make_replay(rela, use_priority=True)
        with pytest.raises(RuntimeError, match="truncated"):
            fresh.load_state(short)
        assert fresh.size() == 0 and fresh.num_add() == 0
    fresh.load_state(path)                     # a refused load leaves the buffer usable
    assert fresh.size() == r.size()


def test_parser_flags_and_refusals(capsys):
    from rebel_b200 import train
    a = train.parse_args(["--out", "x", "--deterministic", "--state_every", "5", "--resume"])
    assert a.deterministic and a.resume and a.state_every == 5
    a = train.parse_args(["--out", "x"])
    assert not a.deterministic and not a.resume and a.state_every is None
    for argv, msg in ((["--resume"], "--resume"), (["--deterministic", "--train_gen_ratio", "0"], "train_gen_ratio"),
                      (["--state_every", "3"], "--state_every")):
        with pytest.raises(SystemExit):
            train.parse_args(["--out", "x"] + argv)
        assert msg in capsys.readouterr().err


def write_state(out, argv):
    """A state file as a deterministic run saves it, for the arguments argv (no device involved)."""
    import rebel_b200.rela as rela
    from rebel_b200 import train
    args = train.parse_args(argv)
    st = {"format": train.STATE_FORMAT, "definition": train.run_definition(args, train.make_params(rela, args)), "next_epoch": 3,
          "replay_file": "replay.e3.state", "val_names": []}
    os.makedirs(out, exist_ok=True)
    torch.save(st, os.path.join(out, train.STATE_FILE))
    open(os.path.join(out, "replay.e3.state"), "wb").close()


@pytest.mark.parametrize("change,field", [(["--lr", "1e-3"], "lr"), (["--num_faces", "5"], "num_faces"),
                                          (["--concurrent_games", "128"], "concurrent_games"), (["--batch", "256"], "batch"),
                                          (["--gen_devices", "0", "1"], "generators"), (["--seed", "1"], "seed"),
                                          (["--exploit_every", "5"], "exploit_every")])
def test_resume_refuses_a_changed_defining_argument(tmp_path, change, field):
    import rebel_b200.rela as rela
    from rebel_b200 import train
    base = ["--out", str(tmp_path), "--deterministic", "--concurrent_games", "256"]
    write_state(str(tmp_path), base)
    # the arguments that may change do not matter
    args = train.parse_args(base + ["--resume", "--max_epochs", "9", "--state_every", "2", "--max_minutes", "3", "--gen_devices", "1"])
    st = train.load_run_state(args, train.make_params(rela, args))
    assert st["next_epoch"] == 3
    with pytest.raises(SystemExit, match=field):
        train.main(base + change + ["--resume"])


def test_deterministic_run_refuses_a_replay_too_small_for_one_epoch(tmp_path):
    from rebel_b200 import train
    with pytest.raises(SystemExit, match="replay_capacity"):
        train.main(["--out", str(tmp_path), "--deterministic", "--replay_capacity", "20000"])
    with pytest.raises(SystemExit, match="no saved state"):     # 8192 rows per phase fit the 10000-row slack
        train.main(["--out", str(tmp_path), "--deterministic", "--replay_capacity", "40000", "--resume"])


def test_resume_without_a_state_is_refused(tmp_path):
    from rebel_b200 import train
    with pytest.raises(SystemExit, match="no saved state"):
        train.main(["--out", str(tmp_path), "--deterministic", "--resume"])


# ------------------------------------------------------------------------------------------------------------- GPU tests
def run_waves(S, weights, drained):
    """One wave per entry of weights (set before the wave starts); examples and game states after each."""
    qs, vs = [], []
    for w in weights:
        S.set_weights(w)
        if drained:
            S.selfplay_wave(start_next=True)
            S.selfplay_wave(start_next=False, keep_examples=True)
        else:
            S.selfplay_wave(start_next=True, keep_examples=True)
        q, v = S.selfplay_examples()
        qs.append(q)
        vs.append(v)
    return qs, vs


def solver(D, F, K, solver_kind, dtype):
    import rebel_b200 as rb
    from rebel_b200 import capi
    return rb.WaveSolver(D, F, K, num_iters=48, net_mode=capi.NET_FP32, solver=solver_kind, state_dtype=dtype)


def seeds(K, s=5):
    return np.uint32(s) + np.arange(K, dtype=np.uint32) * np.uint32(1000000)


@pytest.mark.gpu
@pytest.mark.parametrize("D,F", [(1, 6), (2, 3)])
@pytest.mark.parametrize("solver_kind", ["cfr", "fp"])
@pytest.mark.parametrize("dtype", ["f64", "f32"])
def test_session_export_import_continues_bit_for_bit(net_weights, D, F, solver_kind, dtype):
    from rebel_b200 import capi
    sk = capi.SOLVER_CFR if solver_kind == "cfr" else capi.SOLVER_FP
    dt = capi.STATE_F64 if dtype == "f64" else capi.STATE_F32
    K, W1, W2 = 96, 3, 3
    w0 = net_weights(D, F)
    rng = np.random.RandomState(1)
    weights = [w0 * np.float32(1 + 0.05 * rng.randn()) for _ in range(W1 + W2)]   # new weights for every wave
    A = solver(D, F, K, sk, dt)
    A.selfplay_create(seeds(K))
    run_waves(A, weights[:W1], drained=True)
    image = A.selfplay_export()
    qa, va = run_waves(A, weights[W1:], drained=True)
    state_a = A.selfplay_state()
    B = solver(D, F, K, sk, dt)
    B.selfplay_create(seeds(K, 99))          # other streams, replaced by the image
    B.selfplay_import(image)
    qb, vb = run_waves(B, weights[W1:], drained=True)
    state_b = B.selfplay_state()
    for x, y in zip(qa + va + list(state_a), qb + vb + list(state_b)):
        assert np.array_equal(x, y)
    # one uninterrupted, pipelined run: draining after W1 waves did not change the streams
    C = solver(D, F, K, sk, dt)
    C.selfplay_create(seeds(K))
    qc, vc = run_pipelined(C, weights)
    for x, y in zip(qc[W1:] + vc[W1:] + list(C.selfplay_state()), qa + va + list(state_a)):
        assert np.array_equal(x, y)
    for S in (A, B, C):
        S.close()


def run_pipelined(S, weights):
    """The self-play loop's pipeline: the call that starts wave i (with weights[i]) hands over wave i - 1."""
    qs, vs = [], []
    for i, w in enumerate(weights):
        S.set_weights(w)
        S.selfplay_wave(start_next=True, keep_examples=True)
        if i:
            q, v = S.selfplay_examples()
            qs.append(q)
            vs.append(v)
    S.selfplay_wave(start_next=False, keep_examples=True)
    q, v = S.selfplay_examples()
    return qs + [q], vs + [v]


@pytest.mark.gpu
def test_session_export_import_refusals(net_weights):
    from rebel_b200 import capi
    D, F, K = 1, 6, 32
    S = solver(D, F, K, capi.SOLVER_CFR, capi.STATE_F64)
    S.selfplay_create(seeds(K))
    S.set_weights(net_weights(D, F))
    S.selfplay_wave(start_next=True)
    with pytest.raises(capi.CfrbError, match="pending"):
        S.selfplay_export()
    with pytest.raises(capi.CfrbError, match="pending"):
        S.selfplay_import(b"\0" * 64)
    S.selfplay_wave(start_next=False)
    image = S.selfplay_export()
    H = S.H
    off_player, off_mt_idx = len(image) - 8 * K, len(image) - 4 * K
    assert len(image) == 40 + K * 2 * H * 8 + 624 * K * 4 + 3 * K * 4

    def patched(offset, value, dtype=np.int32):
        b = bytearray(image)
        b[offset:offset + np.dtype(dtype).itemsize] = np.array([value], dtype).tobytes()
        return bytes(b)

    bad = [(image[:-1], "bytes"), (image + b"\0", "bytes"), (image[:20], "header"),
           (patched(off_mt_idx + 4 * 3, 625), "mt_idx"), (patched(off_mt_idx, -1), "mt_idx"),
           (patched(off_player + 4 * 5, 2), "player"), (patched(off_mt_idx - 8 * K, 9999), "last_bid"),
           (patched(40 + 8 * 7, -0.5, np.float64), "belief"), (patched(40, np.nan, np.float64), "belief")]
    others = [(solver(D, F, K + 1, capi.SOLVER_CFR, capi.STATE_F64), dict(), "n_games"),
              (solver(1, 5, K, capi.SOLVER_CFR, capi.STATE_F64), dict(), "num_faces"),
              (solver(D, F, K, capi.SOLVER_CFR, capi.STATE_F64), dict(sample_leaf=False), "sample_leaf"),
              (solver(D, F, K, capi.SOLVER_CFR, capi.STATE_F64), dict(random_action_prob=0.5), "random_action_prob")]
    S.selfplay_wave(start_next=True)
    S.selfplay_wave(start_next=False)            # the session moves on: its image differs from `image`
    before = S.selfplay_export()
    assert before != image
    for blob, what in bad:
        with pytest.raises(capi.CfrbError, match=what):
            S.selfplay_import(blob)
        assert S.selfplay_export() == before
    for T, kw, what in others:
        T.selfplay_create(seeds(T.cfg.max_subgames), **kw)
        own = T.selfplay_export()
        with pytest.raises(capi.CfrbError, match=what):
            T.selfplay_import(image)
        assert T.selfplay_export() == own
        T.close()
    S.selfplay_import(image)
    assert S.selfplay_export() == image
    S.close()


def gen_params(rela, D=1, F=4, K=128, iters=64):
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.random_action_prob, cfg.sample_leaf = D, F, 0.25, True
    cfg.subgame_params.num_iters, cfg.subgame_params.max_depth = iters, 2
    cfg.subgame_params.linear_update, cfg.subgame_params.use_cfr = True, True
    cfg.concurrent_games = K
    return cfg


@pytest.mark.gpu
def test_generator_state_round_trip(net_weights):
    import rebel_b200.rela as rela
    cfg = gen_params(rela)
    w = torch.from_numpy(net_weights(1, 4))
    w2 = w * 1.03

    def waves(g, n, keep_last=False):
        out = []
        for i in range(n):
            out.append(g.run(keep_running=keep_last or i + 1 < n))
        return out

    a = rela.SelfPlayGenerator(cfg, 0, 3)
    a.set_weights(w, 1)
    waves(a, 2, keep_last=True)
    assert not a.drained
    for call in (lambda: a.state(), lambda: a.set_weights(w, 2), lambda: a.load_state(b"")):
        with pytest.raises(RuntimeError, match="in flight"):
            call()
    a.run()
    image = a.state()
    a.set_weights(w2, 2)
    ea = waves(a, 3)
    b = rela.SelfPlayGenerator(cfg, 0, 77)
    b.load_state(image)
    b.set_weights(w2, 2)
    eb = waves(b, 3)
    for (qa, va), (qb, vb) in zip(ea, eb):
        assert torch.equal(qa, qb) and torch.equal(va, vb)
    c = rela.SelfPlayGenerator(cfg, 0, 3)        # uninterrupted
    c.set_weights(w, 1)
    waves(c, 3)
    c.set_weights(w2, 2)
    ec = waves(c, 3)
    for (qa, va), (qc, vc) in zip(ea, ec):
        assert torch.equal(qa, qc) and torch.equal(va, vc)
    # examples appended to a replay are the rows run() returns
    r = make_replay(rela, capacity=4096)
    d = rela.SelfPlayGenerator(cfg, 0, 77)
    d.load_state(image)
    d.set_weights(w2, 2)
    assert d.run(r) == 2 * 128 and r.size() == 2 * 128 and r.storage_device() == 0
    q, v, _ = r.extract()
    assert torch.equal(q, ea[0][0]) and torch.equal(v, ea[0][1])


@pytest.mark.gpu
@pytest.mark.parametrize("use_priority", [False, True])
def test_replay_state_round_trip_device_rows(tmp_path, use_priority):
    import rebel_b200.rela as rela
    r2 = replay_round_trip(tmp_path, use_priority)
    assert r2.storage_device() == 0


# ---- the CLI at 1x4f
CLI = ["--num_dice", "1", "--num_faces", "4", "--train_epoch_size", "2048", "--val_batches", "4", "--eval_every", "2",
       "--exploit_every", "4", "--create_validation_set_every", "3", "--subgame_iters", "64", "--concurrent_games", "256",
       "--replay_capacity", "100000", "--deterministic", "--state_every", "3"]
EPOCHS = 8


def cli(out, *extra):
    return [sys.executable, "-m", "rebel_b200.train", "--out", str(out)] + CLI + list(extra)


def train_lines(stdout):
    from rebel_b200.train import parse_train
    lines = [parse_train(l) for l in stdout.splitlines() if l.startswith("TRAIN ")]
    return [{k: v for k, v in m.items() if k != "minutes" and not k.endswith("_per_s")} for m in lines]


def run_cli(out, *extra):
    r = subprocess.run(cli(out, *extra), cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return train_lines(r.stdout), r.stdout


def same_tree(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(same_tree(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return isinstance(b, (list, tuple)) and len(a) == len(b) and all(same_tree(x, y) for x, y in zip(a, b))
    return a == b


def assert_same_checkpoints(da, db):
    names = sorted(n for n in os.listdir(da) if n.endswith((".ckpt", ".optim")))
    assert names and names == sorted(n for n in os.listdir(db) if n.endswith((".ckpt", ".optim")))
    for n in names:
        assert same_tree(torch.load(os.path.join(da, n)), torch.load(os.path.join(db, n))), n


@pytest.fixture(scope="module")
def reference_run(tmp_path_factory):
    out = tmp_path_factory.mktemp("uninterrupted")
    lines, stdout = run_cli(out, "--max_epochs", str(EPOCHS))
    assert [m["epoch"] for m in lines] == list(range(EPOCHS))
    assert "exploitability" in lines[0] and "exploitability" in lines[4]
    assert lines[-1]["weights_version"] == EPOCHS + 1
    assert os.path.exists(out / "state.pt") and len(list(out.glob("replay.e*.state"))) == 1
    assert sorted(p.name for p in out.glob("valid_snapshot_*.pt")) == ["valid_snapshot_0000.pt", "valid_snapshot_0003.pt",
                                                                        "valid_snapshot_0006.pt"]
    return out, lines


@pytest.mark.gpu
def test_cli_deterministic_runs_are_reproducible(tmp_path, reference_run):
    out, lines = reference_run
    again, _ = run_cli(tmp_path, "--max_epochs", str(EPOCHS))
    assert again == lines
    assert_same_checkpoints(out, tmp_path)


@pytest.mark.gpu
def test_cli_stopped_and_resumed_run_matches(tmp_path, reference_run):
    out, lines = reference_run
    first, _ = run_cli(tmp_path, "--max_epochs", "5")
    assert [m["epoch"] for m in first] == list(range(5))
    rest, stdout = run_cli(tmp_path, "--max_epochs", str(EPOCHS), "--resume")
    assert "resumed at epoch 5" in stdout
    assert first + rest == lines
    assert_same_checkpoints(out, tmp_path)


@pytest.mark.gpu
def test_cli_run_stopped_by_sigterm_resumes_to_the_same_bits(tmp_path, reference_run):
    out, lines = reference_run
    run_dir = tmp_path / "run"
    with open(tmp_path / "stderr.txt", "w") as err:
        p = subprocess.Popen(cli(run_dir, "--max_epochs", str(EPOCHS)), cwd=ROOT, stdout=subprocess.PIPE, stderr=err, text=True)
        seen = []
        try:
            for line in p.stdout:
                seen.append(line)
                if line.startswith("TRAIN "):
                    p.send_signal(signal.SIGTERM)
                    break
            rest_out, _ = p.communicate(timeout=600)
        finally:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert p.returncode == 0, (tmp_path / "stderr.txt").read_text()[-3000:]
    assert "signal" in (tmp_path / "stderr.txt").read_text()
    first = train_lines("".join(seen) + rest_out)
    assert 1 <= len(first) < EPOCHS - 1, len(first)      # stopped early, after the epoch in progress
    rest, _ = run_cli(run_dir, "--max_epochs", str(EPOCHS), "--resume")
    assert first + rest == lines
    assert_same_checkpoints(out, run_dir)
