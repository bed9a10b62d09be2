"""The tensor-core value net on games with more than 16 hands (leaf_mlp_tc_wide.cuh): 2x5f, 3x3f, 5x2f, 2x6f, 1x17f .. 1x32f.

CPU: which games have a tensor-core net (cfrb_tc_net_supported, the rule cfrb_create and `rela` share).
GPU: rows independent of their tile, the wide kernel bit-identical to the resident
kernel where both apply (CFRB_TC_WIDE=1), layer taps against a host computation, one teacher-forced CFR step, and the `rela`
data-generation loop running the tensor-core net at 2x5f with the example distribution of the fp32 net.
"""
import numpy as np
import pytest

from oracle.oracle import game_dims

SUPPORTED = [(1, 4), (1, 6), (2, 3), (2, 4), (2, 5), (3, 3), (5, 2), (2, 6), (1, 17), (1, 32)]
UNSUPPORTED = [(2, 7), (3, 4), (6, 2), (2, 8)]
WIDE = [(2, 5), (3, 3), (2, 6)]


@pytest.fixture(scope="module")
def rb():
    import rebel_b200
    assert rebel_b200.capi.lib().cfrb_device_count() > 0, "no CUDA device: the CUDA path cannot be tested"
    return rebel_b200


@pytest.fixture(scope="module")
def rela():
    import rebel_b200.rela as m
    return m


def _note(msg):
    print("[wide-net]", msg, flush=True)


def _cfg(rela, D, F, **kw):
    cfg = rela.RecursiveSolvingParams()
    sp = dict(num_iters=16, max_depth=2, linear_update=True, use_cfr=True)
    sp.update(kw.pop("subgame_params", {}))
    for k, v in dict(num_dice=D, num_faces=F, random_action_prob=0.25, sample_leaf=True, **kw).items():
        setattr(cfg, k, v)
    for k, v in sp.items():
        setattr(cfg.subgame_params, k, v)
    return cfg


# ---------------------------------------------------------------------------------------------- CPU
def test_tc_net_supported():
    """Host-only rule: a tensor-core net exists where Net2's fp16 weights (and, for the resident kernel, two query tiles) fit the
    227 KB of shared memory of an sm_90 block; no device is needed to ask."""
    from rebel_b200 import capi
    for D, F in SUPPORTED:
        assert capi.tc_net_supported(D, F), (D, F)
    for D, F in UNSUPPORTED:
        assert not capi.tc_net_supported(D, F), (D, F)
    assert not capi.tc_net_supported(2, 5, hidden=128)          # only n_hidden = 256 is built
    assert not capi.tc_net_supported(0, 5) and not capi.tc_net_supported(2, 0)
    for D, F in [(8, 1), (9, 1), (8, 2)]:                       # more than 7 dice: cfrb_create refuses the game itself
        assert not capi.tc_net_supported(D, F), (D, F)


# ---------------------------------------------------------------------------------------------- GPU
def _beliefs(rng, n, H):
    b = rng.rand(n, 2, H)
    return b / b.sum(-1, keepdims=True)


@pytest.mark.gpu
@pytest.mark.parametrize("net_name", ["tc_f16x2", "tc_f16"])
@pytest.mark.parametrize("D,F", WIDE)
def test_wide_net_rows_do_not_depend_on_their_tile(rb, net_weights, D, F, net_name):
    """Every query row is evaluated on its own: bit-identical outputs whether the wave has 1, 2, 3, 149 or 1300 subgames (one
    tile, odd / even tile counts per CTA, both warpgroups, partial last tile).  Their accuracy is checked in
    test_value_net_accuracy.py."""
    A, H, Q = game_dims(D, F)
    Kmax = 1300
    rng = np.random.RandomState(5)
    b = _beliefs(rng, Kmax, H)
    lb = rng.randint(-1, A - 2, size=Kmax).astype(np.int32); lb[:4] = -1
    pl = rng.randint(0, 2, size=Kmax).astype(np.int32)
    w = net_weights(D, F)
    mode = getattr(rb, "NET_" + net_name.upper())
    ref = None
    for K in (Kmax, 1, 2, 3, 149):
        S = rb.WaveSolver(D, F, K, net_mode=mode)
        S.set_weights(w)
        S.begin(lb[:K], pl[:K], b[:K])
        S.run(2)
        q, o, sc = S.leaf_io()
        mu = S.fetch(("root_means",))["root_means"]
        S.close()
        if ref is None:
            ref = (q, o, mu)
        else:
            n = len(q)
            assert np.array_equal(q, ref[0][:n]) and np.array_equal(o, ref[1][:n]) and np.array_equal(mu, ref[2][:K]), K


GELUS = [("kGelu0", "NET_TC_F16", None), ("kGelu1", "NET_TC_F16X2", "half"), ("kGelu2", "NET_TC_F16X2", None)]


@pytest.mark.gpu
@pytest.mark.parametrize("gelu,mode_name,x2_gelu", GELUS)
@pytest.mark.parametrize("D,F", [(1, 4), (1, 6), (2, 3), (2, 4)])
def test_wide_kernel_equals_resident_kernel(rb, net_weights, monkeypatch, D, F, gelu, mode_name, x2_gelu):
    """CFRB_TC_WIDE=1 runs the wide kernel on games the resident kernel serves.  Layer 1 from registers accumulates over K in the
    order of the shared-memory form, and layers 2 and 3 are the same instructions, so net outputs and root value means are
    bit-identical for each GELU variant."""
    A, H, Q = game_dims(D, F)
    K = 700
    rng = np.random.RandomState(7)
    b = _beliefs(rng, K, H)
    lb = rng.randint(-1, A - 2, size=K).astype(np.int32); lb[:4] = -1
    pl = rng.randint(0, 2, size=K).astype(np.int32)
    if x2_gelu:
        monkeypatch.setenv("CFRB_X2_GELU", x2_gelu)
    else:
        monkeypatch.delenv("CFRB_X2_GELU", raising=False)
    out = []
    for wide in (False, True):
        if wide:
            monkeypatch.setenv("CFRB_TC_WIDE", "1")
        else:
            monkeypatch.delenv("CFRB_TC_WIDE", raising=False)
        S = rb.WaveSolver(D, F, K, net_mode=getattr(rb, mode_name))
        S.set_weights(net_weights(D, F))
        S.begin(lb, pl, b)
        S.run(2)
        q, o, _ = S.leaf_io()
        mu = S.fetch(("root_means",))["root_means"]
        S.close()
        out.append((q, o, mu))
    (q0, o0, m0), (q1, o1, m1) = out
    assert np.array_equal(q0, q1)
    assert np.array_equal(o0, o1), (gelu, int((o0 != o1).sum()), np.abs(o0 - o1).max())
    assert np.array_equal(m0, m1), gelu


def _centred_fp16(w, Q, H, hid=256):
    """The weights as cfrb_set_weights hands them to the tensor cores: W1 / W2 and the biases centred over the 256 features,
    rounded to fp16 (bias 1 as an extra column of W1, bias 2 rounded the same way)."""
    o = 0
    def take(n):
        nonlocal o
        a = np.asarray(w[o:o + n], np.float64); o += n
        return a
    w1 = take(hid * Q).reshape(hid, Q); b1 = take(hid); g1 = take(hid); be1 = take(hid)
    w2 = take(hid * hid).reshape(hid, hid); b2 = take(hid); g2 = take(hid); be2 = take(hid)
    r = lambda x: x.astype(np.float32).astype(np.float16).astype(np.float64)
    W1 = r(np.concatenate([w1 - w1.mean(0), (b1 - b1.mean())[:, None]], 1))
    W2 = r(w2 - w2.mean(0))
    return W1, W2, r(b2 - b2.mean()), (g1, be1), (g2, be2)


@pytest.mark.gpu
def test_wide_net_layer_taps(rb, net_weights):
    """2x5f, NET_TC_F16: the raw layer-1 accumulators of the first 128 rows equal X W1'^T computed on the host in fp64 from the
    fp16 query rows and the centred fp16 weights, to fp32-accumulation tolerance (2e-5 of sum |x w|).  Layer 2 is checked from
    the kernel's own layer-1 taps: host LayerNorm + exact GELU rounded to fp16, times the centred fp16 W2, plus bias 2; the
    bound adds what one fp16 rounding of each activation (2^-10 relative, covering a rounding that lands on the other side) and
    the GELU approximation (5e-5 absolute) may move a product."""
    from scipy.special import erf
    D, F = 2, 5
    A, H, Q = game_dims(D, F)
    w = net_weights(D, F)
    rng = np.random.RandomState(3)
    K = 8
    b = _beliefs(rng, K, H)
    S = rb.WaveSolver(D, F, K, net_mode=rb.NET_TC_F16)
    S.set_weights(w)
    S.begin(np.full(K, -1, np.int32), np.arange(K, dtype=np.int32) % 2, b)
    S.run(2)
    q, _, _ = S.leaf_io()
    d1, d2 = S.net_taps()
    S.close()
    n = min(128, len(q))
    assert n >= 100
    W1, W2, b2c, (g1, be1), _ = _centred_fp16(w, Q, H)
    x = np.concatenate([q[:n].astype(np.float64), np.ones((n, 1))], 1)
    ref1 = x @ W1.T
    tol1 = 2e-5 * (np.abs(x) @ np.abs(W1).T) + 1e-7
    err1 = np.abs(d1[:n] - ref1)
    assert (err1 <= tol1).all(), (err1.max(), (err1 / tol1).max())
    y = d1[:n].astype(np.float64)
    rstd = 1.0 / np.sqrt((y * y).mean(1, keepdims=True) + 1e-5)
    z = y * rstd * g1 + be1
    act = (0.5 * z * (1 + erf(z / np.sqrt(2)))).astype(np.float16).astype(np.float64)
    ref2 = b2c + act @ W2.T
    tol2 = (np.abs(act) * 2.0 ** -10 + 5e-5) @ np.abs(W2).T + 2e-5 * (np.abs(act) @ np.abs(W2).T) + 1e-6
    err2 = np.abs(d2[:n] - ref2)
    _note(f"taps 2x5f: layer 1 max err {err1.max():.2e} ({(err1 / tol1).max():.2f} of the bound), layer 2 max err "
          f"{err2.max():.2e} ({(err2 / tol2).max():.2f} of the bound)")
    assert (err2 <= tol2).all(), (err2.max(), (err2 / tol2).max())


NOISE_TC_F16X2 = 1.5e-5     # value-noise level of NET_TC_F16X2 against the fp64 oracle (test_gpu_parity.noise_level)


@pytest.mark.gpu
def test_wide_net_teacher_forced_step(rb, port, net_weights):
    """2x5f, NET_TC_F16X2: from the C port's state after c iterations (fp32 net), one GPU step reproduces the port's next root
    value means, regrets and leaf values within 10x the tensor-core noise level of test_gpu_parity (1.5e-5)."""
    D, F = 2, 5
    A, H, Q = game_dims(D, F)
    w = net_weights(D, F)
    noise = NOISE_TC_F16X2
    cps = [0, 1, 2, 3, 4]
    S = rb.WaveSolver(D, F, 1, net_mode=rb.NET_TC_F16X2)
    S.set_weights(w)
    worst = {"mu": 0.0, "regrets": 0.0, "leaf": 0.0}
    for ri, (lb, pl) in enumerate([(-1, 0), (-1, 1), (3, 1), (A - 6, 0)]):
        b = port.synthetic_beliefs(H, 300 + ri)
        o = port.cfr_solve(D, F, b, cps, lb, pl, num_iters=max(cps), net_w=w)
        N = o["tree"].shape[0]
        pad = lambda x: np.concatenate([x, np.zeros((S.Nmax - N,) + x.shape[1:])])[None]
        for ci, c in enumerate(cps[:-1]):
            S.begin([lb], [pl], b[None])
            S.load_state(regrets=pad(o["regrets"][ci]), last=pad(o["last"][ci]), sum=pad(o["sum"][ci]),
                         root_means=o["root_means"][ci][None], num_steps=np.array([[(c + 1) // 2, c // 2]], np.int32),
                         iterations_done=c)
            S.run(1)
            g = S.fetch(("root_means", "regrets"))
            tag = (lb, pl, c)
            dmu = np.abs(g["root_means"][0] - o["root_means"][ci + 1]).max()
            Rn = o["regrets"][ci + 1]
            dR = np.abs(g["regrets"][0, :N] - Rn)
            assert dmu < 10 * noise, (tag, dmu)
            assert (dR <= 10 * noise * (1 + np.abs(Rn))).all(), (tag, dR.max())
            worst["mu"] = max(worst["mu"], dmu); worst["regrets"] = max(worst["regrets"], dR.max())
            if o["queries"].shape[1]:
                q, out, sc = S.leaf_io()
                assert np.abs(q - o["queries"][ci + 1]).max() < 1e-3, tag
                lv = np.abs(out * sc[:, None] - o["leaf_values"][ci + 1]).max()
                assert lv < 10 * noise, (tag, lv)
                worst["leaf"] = max(worst["leaf"], lv)
    S.close()
    _note("teacher-forced 2x5f tcx2: worst " + " ".join(f"{k}={v:.2e}" for k, v in worst.items()))


@pytest.mark.gpu
def test_rela_loop_uses_the_tensor_cores_at_2x5f(rela, rb, net_weights, monkeypatch):
    """The data-generation loop of `rela` (BatchedRlRunner, behind create_cfr_thread) at 2x5f with the default net mode emits,
    bit for bit, the example stream of the C-ABI device walk in NET_TC_F16X2 with the same seeds, and a different stream with
    net_mode = 1 (the fp32 net it used to fall back to)."""
    import torch
    monkeypatch.delenv("CFRB_NET_MODE", raising=False)
    monkeypatch.delenv("CFRB_X2_GELU", raising=False)
    D, F = 2, 5
    A, H, Q = game_dims(D, F)
    K, waves, iters, seed = 16, 4, 16, 9
    w = net_weights(D, F)
    cfg = _cfg(rela, D, F, concurrent_games=K, state_dtype=0, subgame_params=dict(num_iters=iters))
    assert cfg.net_mode == rb.NET_TC_F16X2
    q, v = rela.run_selfplay_waves(cfg, 0, seed, waves, torch.from_numpy(w))
    S = rb.WaveSolver(D, F, K, num_iters=iters, net_mode=rb.NET_TC_F16X2)
    S.set_weights(w)
    S.selfplay_create(np.uint32(seed) + np.arange(K, dtype=np.uint32) * np.uint32(1000000))
    S.selfplay_wave()
    got_q, got_v = [], []
    for _ in range(waves):
        S.selfplay_wave(keep_examples=True)
        a, c = S.selfplay_examples()
        got_q.append(a.reshape(-1, Q)); got_v.append(c.reshape(-1, H))
    S.selfplay_wave(start_next=False)
    S.sync()
    S.close()
    assert np.array_equal(q.numpy(), np.concatenate(got_q)) and np.array_equal(v.numpy(), np.concatenate(got_v))
    cfg1 = _cfg(rela, D, F, concurrent_games=K, state_dtype=0, net_mode=rb.NET_FP32, subgame_params=dict(num_iters=iters))
    q1, v1 = rela.run_selfplay_waves(cfg1, 0, seed, waves, torch.from_numpy(w))
    assert q1.shape == q.shape and not torch.equal(v1, v)


@pytest.mark.gpu
def test_wide_net_example_distribution_matches_fp32(rela, rb, monkeypatch):
    """P5-style check at 2x5f: the examples of the `rela` loop with NET_TC_F16X2 against two disjoint seed sets of the fp32 net.
    Per-last-action counts (chi-square), mean targets and mean losses of the seed-0 Net2 may differ from the fp32 sets by at
    most 3x the distance between the two fp32 sets (plus the floors of test_datagen_distribution_matches_reference).  Size:
    256 games x 32 waves x 16 CFR iterations per set (16 384 examples; complete games only)."""
    import torch
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    from test_rela_module import _chi2, _last_action_stats
    monkeypatch.delenv("CFRB_X2_GELU", raising=False)
    D, F = 2, 5
    A, H, Q = game_dims(D, F)
    net = make_selfplay_net(D, F, seed=0)
    w = torch.from_numpy(flatten_state_dict(net.state_dict()))
    K, waves, iters = 256, 32, 16

    def stats(net_mode, seed):
        cfg = _cfg(rela, D, F, concurrent_games=K, state_dtype=0, net_mode=net_mode, subgame_params=dict(num_iters=iters))
        q, v = rela.run_selfplay_waves(cfg, 0, seed, waves, w)
        q = q.numpy().reshape(waves, K, 2, Q); v = v.numpy().reshape(waves, K, 2, H)
        starts = q[:, :, 0, 2:2 + A].sum(-1) == 0
        last_start = waves - 1 - np.argmax(starts[::-1], axis=0)
        keep = np.arange(waves)[:, None] < last_start[None, :]
        return _last_action_stats(q[keep].reshape(-1, Q), v[keep].reshape(-1, H), A, net)

    tc = stats(rb.NET_TC_F16X2, 101)
    a = stats(rb.NET_FP32, 202)
    b = stats(rb.NET_FP32, 303)
    big = (tc[0] >= 100) & (a[0] >= 100) & (b[0] >= 100)
    mean = lambda s, c: s[big] / (c[big] * H)
    loss = lambda s, c: s[big] / c[big]

    def dist(x, y):
        return (_chi2(x[0], y[0]), np.abs(mean(x[1], x[0]) - mean(y[1], y[0])).max(),
                (np.abs(loss(x[2], x[0]) - loss(y[2], y[0])) / loss(y[2], y[0])).max())
    band = dist(a, b)
    got = [max(dist(tc, s)[k] for s in (a, b)) for k in range(3)]
    _note(f"2x5f examples tcx2 {int(tc[0].sum())}, fp32 {int(a[0].sum())} / {int(b[0].sum())}; chi2 tc-fp32 {got[0]:.1f} "
          f"(fp32 seed-to-seed {band[0]:.1f}); mean target {got[1]:.2e} ({band[1]:.2e}); relative loss {got[2]:.2e} ({band[2]:.2e})")
    assert got[0] <= 3 * max(band[0], A + 1), (got[0], band[0])
    assert got[1] <= 3 * band[1] + 1e-4, (got[1], band[1])
    assert got[2] <= 3 * band[2] + 0.02, (got[2], band[2])
