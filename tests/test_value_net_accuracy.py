"""Accuracy of the value-net kernels (leaf_mlp_tc_kernel, leaf_mlp_tc_wide_kernel, leaf_mlp_fp32_kernel) against an fp64 Net2,
with weights that reach what a freshly initialised net does not, on every game each kernel serves.

Two references, both defined here:
  * fp64 Net2: the same parameters in float64, LayerNorm with eps 1e-5, exact erf GELU, on the query rows the kernel saw
    (WaveSolver.leaf_io(); in the tensor-core modes these rows are already fp16).
  * the kernels' arithmetic model, in numpy: W1 / W2 and biases 1 / 2 centred over the 256 features and rounded to fp16 (bias 1
    as an extra column of W1), fp16 W3, fp32 b3, mean-free fp32 LayerNorm, then the GELU of the mode and one fp16 rounding of
    each activation.  GELU variants (leaf_mlp_tc.cuh kGelu): 0 the logistic fit of gelu_tc (NET_TC_F16), 1 the packed-half chain
    of gelu_hy_x2 (NET_TC_F16X2 with CFRB_X2_GELU=half; tanh.approx.f16x2 truncates towards zero), 2 fp32 gelu_hy_f32 rounded
    once (NET_TC_F16X2, the default).  The model says how far a kernel should be from fp64; it restates the arithmetic and never
    calls the library.

Weight families: `init` (make_selfplay_net), `distinct` (every LayerNorm parameter different, output layer x30), `trained`
(Net2Trainer after 400 steps on device self-play examples), `saturating` (|z| up to ~100 in both LayerNorms: the GELU tails),
`offset` (common components the host-side centring has to remove) and `offset_tight` (layer-1 variance comparable to eps).

Criteria, s = rms of the fp64 outputs:
  * tensor-core modes: rms(ours - fp64) / s <= 1.25 x the model's + 1e-6; max |ours - fp64| <= 2 x the model's + 2^-11 max |fp64|;
    rms(ours - model) / s <= RHO x the model's relative rms (the kernel is its own model, not just an error of the right size);
    per output column |mean(ours - fp64)| <= |mean(model - fp64)| + 4 standard errors (no coherent bias);
    net_output_bound >= max |ours| (the dead-row skip is sound for the kernel's own arithmetic);
  * NET_FP32: max |ours - fp64| <= 4 x max |torch fp32 - fp64| + 2^-20 max |fp64|;
  * every mode: every output finite.
"""
import hashlib

import numpy as np
import pytest
from scipy.special import erf

from oracle.oracle import game_dims

HID = 256
RESIDENT = [(1, 4), (1, 6), (2, 3), (2, 4)]
WIDE = [(2, 5), (3, 3), (5, 2), (2, 6), (1, 17), (1, 32)]
FP32_ONLY = [(2, 7), (3, 4)]
FAMILIES = ["init", "distinct", "saturating", "offset", "offset_tight"]
TRAINED_GAMES = [(1, 6), (2, 5)]
# mode name -> (net mode, CFRB_X2_GELU, GELU variant of the model; None: the fp32 SIMT kernel)
MODES = {"fp32": ("NET_FP32", None, None), "tc_f16": ("NET_TC_F16", None, 0), "tc_f16x2": ("NET_TC_F16X2", None, 2),
         "tc_f16x2_half": ("NET_TC_F16X2", "half", 1)}
ROWS_MAX = 16384        # query rows the host references evaluate per case
WAVE_ROWS = 20000       # target rows of the mixed wave
# bound on rms(ours - model) / s over the model's relative rms, per GELU variant.  Measured on an H100 80GB HBM3 (700 W power
# limit) over every game and family: at most 0.062 (variant 0), 0.061 (1), 0.23 (2, whose tanh.approx.f32 the model takes as
# exact); see DESIGN.md "Numerical contract"
RHO = {0: 0.15, 1: 0.15, 2: 0.4}
KEYS = ("w1", "b1", "g1", "be1", "w2", "b2", "g2", "be2", "w3", "b3")


def _note(msg):
    print("[net-accuracy]", msg, flush=True)


# ---------------------------------------------------------------------------------------------- parameters and families
def unpack(flat, D, F):
    """The flat cfrb_set_weights layout (state_dict order) -> dict of float64 arrays."""
    A, H, Q = game_dims(D, F)
    out, o = {}, 0
    for k, shp in zip(KEYS, [(HID, Q), (HID,), (HID,), (HID,), (HID, HID), (HID,), (HID,), (HID,), (H, HID), (H,)]):
        n = int(np.prod(shp))
        out[k] = np.asarray(flat[o:o + n], np.float64).reshape(shp).copy()
        o += n
    assert o == len(flat)
    return out


def pack(p):
    return np.concatenate([p[k].ravel() for k in KEYS]).astype(np.float32)


def _perm(a, b):
    """j -> (a j + b) mod 256 with a odd: a permutation whose neighbours are far apart."""
    return (a * np.arange(HID) + b) % HID


def _init(D, F):
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    return unpack(flatten_state_dict(make_selfplay_net(D, F, seed=0).state_dict()), D, F)


def family_weights(name, D, F):
    """Flat fp32 weights of a family (deterministic).  `trained` needs a GPU (trained_weights)."""
    if name == "trained":
        return trained_weights(D, F)
    A, H, Q = game_dims(D, F)
    p = _init(D, F)
    if name == "distinct":
        # gamma 1 in [0.5, 2], beta 1 in [0.05, 0.4], gamma 2 in [0.45, 1.95] on a grid offset by half a step from gamma 1's,
        # beta 2 negative; each in its own order, so a swapped pair or a parameter of the other LayerNorm is an O(1) change
        p["g1"] = 0.5 + 1.5 * _perm(97, 0) / 255
        p["be1"] = 0.05 + 0.35 * _perm(57, 11) / 255
        p["g2"] = 0.45 + 1.5 * _perm(151, 29) / 255
        p["be2"] = -0.05 - 0.45 * _perm(37, 101) / 255
        p["w3"] *= 30
        p["b3"] *= 30
    elif name == "saturating":
        rng = np.random.RandomState(100 * D + F)
        for lay, (a, b) in ((1, (97, 5)), (2, (151, 3))):
            p[f"g{lay}"] = 3 + 3 * _perm(a, b) / 255
            p[f"be{lay}"] = 2 * rng.randn(HID)
            # two features dominate the variance (rows x60 and x40), so that |y rstd| reaches ~13 and ~9 on them: |z| ~ 80 and ~45
            # of either sign; the others sit near their beta
            p[f"g{lay}"][:2] = (6.0, 5.0)
            for j, s in ((0, 60.0), (1, 40.0)):
                p[f"w{lay}"][j] *= s
                p[f"b{lay}"][j] *= s
    elif name in ("offset", "offset_tight"):
        rng = np.random.RandomState(200 * D + F)
        w1 = p["w1"]
        if name == "offset_tight":
            # per-feature deviations scaled to a layer-1 spread of ~3e-3 on query rows: variance ~1e-5, comparable to eps
            k = 3e-3 * np.sqrt(Q)
            w1 = w1.mean(0) + k * (w1 - w1.mean(0))
            p["b1"] = p["b1"].mean() + k * (p["b1"] - p["b1"].mean())
        # a component common to all 256 features, 10x the spread of each column, and an offset of ~20 on both biases: LayerNorm
        # removes all of it, and so must the host-side centring of cfrb_set_weights
        p["w1"] = w1 + 10 * w1.std(0) * np.where(rng.rand(Q) < 0.5, -1.0, 1.0)
        p["b1"] = p["b1"] + 20 + rng.rand()
        p["b2"] = p["b2"] + 20 + rng.rand()
    else:
        assert name == "init", name
    return pack(p)


_TRAINED = {}


def _train(D, F):
    """Net2Trainer from the seed-0 net, 400 steps at lr 1e-3 on device self-play examples (built like test_train.py's)."""
    import torch
    import rebel_b200.rela as rela
    from rebel_b200.models import flatten_state_dict, make_selfplay_net
    from rebel_b200.trainer import Net2Trainer
    cfg = rela.RecursiveSolvingParams()
    cfg.num_dice, cfg.num_faces, cfg.random_action_prob, cfg.sample_leaf = D, F, 0.25, True
    cfg.subgame_params.num_iters, cfg.subgame_params.max_depth = 64, 2
    cfg.subgame_params.linear_update, cfg.subgame_params.use_cfr = True, True
    cfg.concurrent_games = 256
    net = make_selfplay_net(D, F, seed=0)
    q, v = rela.run_selfplay_waves(cfg, 0, 5, 3, torch.from_numpy(flatten_state_dict(net.state_dict())))
    q, v = q.float().cuda(), v.float().cuda()
    tr = Net2Trainer(D, F, "cuda:0", lr=1e-3, grad_clip=5.0, state_dict=net.state_dict())
    rng = np.random.RandomState(11)
    for _ in range(400):
        idx = torch.from_numpy(rng.randint(0, q.shape[0], 512)).cuda()
        tr.step(q[idx], v[idx])
    flat = tr.get_state()[0]
    tr.close()
    return flat


def trained_weights(D, F):
    if (D, F) not in _TRAINED:
        _TRAINED[(D, F)] = _train(D, F)
    return _TRAINED[(D, F)]


# ---------------------------------------------------------------------------------------------- the references
def fp64_net(p, x):
    """Net2 in float64: Linear -> LayerNorm(eps 1e-5) -> exact GELU, twice, -> Linear."""
    def ln(y, g, b):
        m = y.mean(1, keepdims=True)
        v = ((y - m) ** 2).mean(1, keepdims=True)
        return (y - m) / np.sqrt(v + 1e-5) * g + b
    gelu = lambda z: 0.5 * z * (1 + erf(z / np.sqrt(2)))
    a = gelu(ln(np.asarray(x, np.float64) @ p["w1"].T + p["b1"], p["g1"], p["be1"]))
    a = gelu(ln(a @ p["w2"].T + p["b2"], p["g2"], p["be2"]))
    return a @ p["w3"].T + p["b3"]


def torch_net(flat, D, F, x, dtype):
    import torch
    from rebel_b200.models import make_selfplay_net
    net = make_selfplay_net(D, F, seed=0).to(dtype)
    p = unpack(flat, D, F)
    names = ("body.0.weight", "body.0.bias", "body.1.weight", "body.1.bias", "body.4.weight", "body.4.bias", "body.5.weight",
             "body.5.bias", "output.weight", "output.bias")
    net.load_state_dict({n: torch.from_numpy(p[k]).to(dtype) for n, k in zip(names, KEYS)})
    with torch.no_grad():
        return net(torch.from_numpy(np.asarray(x, np.float64)).to(dtype)).double().numpy()


f32 = lambda x: np.asarray(x, np.float64).astype(np.float32).astype(np.float64)
h16 = lambda x: np.asarray(x, np.float64).astype(np.float32).astype(np.float16).astype(np.float64)


def h16_toward_zero(x):
    """fp16 rounding towards zero (tanh.approx.f16x2, DESIGN.md 'What P5 found')."""
    r = np.asarray(x, np.float64).astype(np.float16)
    over = np.abs(r.astype(np.float64)) > np.abs(x)
    r[over] = np.nextafter(r[over], np.float16(0))
    return r.astype(np.float64)


def kernel_blob(p, variant):
    """The parameters as cfrb_set_weights hands them to the tensor-core kernels."""
    lnscale = 1.0 if variant == 0 else 0.5        # NET_TC_F16X2 stores gamma / 2, beta / 2: the affine yields y / 2
    m1, m2 = p["w1"].mean(0), p["w2"].mean(0)
    return dict(W1=h16(np.concatenate([p["w1"] - m1, (p["b1"] - p["b1"].mean())[:, None]], 1)),
                W2=h16(p["w2"] - m2), b2=h16(p["b2"] - p["b2"].mean()),
                ln1=(f32(lnscale * p["g1"]), f32(lnscale * p["be1"])), ln2=(f32(lnscale * p["g2"]), f32(lnscale * p["be2"])),
                W3=h16(p["w3"]), b3=f32(p["b3"]))


def tanh_f16x2_truncating(u):
    return h16_toward_zero(np.tanh(u))


def gelu_model(z, variant, tanh16=tanh_f16x2_truncating):
    """z: the fp32 LayerNorm affine (y, or y / 2 for variants 1 and 2) -> the fp16 activation.  tanh16: tanh.approx.f16x2 of fp16
    values (variant 1)."""
    if variant == 0:            # gelu_tc: y / (1 + 2^(y p(y^2))), fp32 with FMAs (ex2 / rcp.approx: ~2^-22 relative)
        y2 = np.minimum(f32(z * z), 52.0)
        pp = f32(y2 * f32(y2 * np.float32(1.014244e-3) + np.float32(-1.0677588e-1)) + np.float32(-2.3011216))
        with np.errstate(over="ignore"):
            return h16(f32(z * f32(1.0 / f32(np.exp2(f32(z * pp)) + 1.0))))
    c2, c1, c0 = np.float32(-1.124832e-2), np.float32(2.960456e-1), np.float32(1.594992)
    if variant == 1:            # gelu_hy_x2: HMUL2 / HFMA2 with one rounding each, tanh.approx.f16x2
        hy = h16(z)
        s = np.minimum(h16(hy * hy), 13.0)
        pp = h16(s * h16(s * h16(c2) + h16(c1)) + h16(c0))
        t = tanh16(h16(hy * pp))
        return h16(hy * t + hy)
    s = np.minimum(f32(z * z), 13.0)   # gelu_hy_f32 (tanh.approx.f32 taken as exact), one rounding to fp16
    pp = f32(s * f32(s * c2 + c1) + c0)
    return h16(f32(z * np.tanh(f32(z * pp)) + z))


def _ln_model(y, g, be, mean_free=True):
    y = f32(y)
    if not mean_free:           # the layout of the reference harness's model (uncentred weights)
        y = f32(y - f32(y.mean(1, keepdims=True)))
    rstd = f32(1.0 / np.sqrt(f32(f32((y * y).sum(1, keepdims=True)) / HID + 1e-5)))
    return f32(f32(y * rstd) * g + be)


def model_net(B, x, variant, mean_free=True, **kw):
    """The kernels' arithmetic on query rows x with parameters B (kernel_blob)."""
    xa = np.concatenate([np.asarray(x, np.float64), np.ones((len(x), 1))], 1)
    a = gelu_model(_ln_model(xa @ B["W1"].T, *B["ln1"], mean_free), variant, **kw)
    a = gelu_model(_ln_model(B["b2"] + a @ B["W2"].T, *B["ln2"], mean_free), variant, **kw)
    return f32(a @ B["W3"].T + B["b3"])


def tc_criteria(ours, ref, model, rho):
    """(measured numbers, list of failed criteria) for outputs of a tensor-core mode against fp64 and the model."""
    rms = lambda e: float(np.sqrt(np.mean(np.square(e))))
    s = rms(ref)
    eo, em = ours - ref, model - ref
    st = dict(rel_rms=rms(eo) / s, model_rel_rms=rms(em) / s, max=float(np.abs(eo).max()), model_max=float(np.abs(em).max()),
              max_ref=float(np.abs(ref).max()), rms_ref=s)
    st["rho"] = rms(ours - model) / s / st["model_rel_rms"]
    se = eo.std(0) / np.sqrt(len(eo))
    excess = np.abs(eo.mean(0)) - np.abs(em.mean(0)) - 4 * se
    st["bias_excess"] = float((excess / np.maximum(se, 1e-300)).max())      # in standard errors above the allowance
    bad = []
    if not st["rel_rms"] <= 1.25 * st["model_rel_rms"] + 1e-6:
        bad.append(f"rms error {st['rel_rms']:.3e} > 1.25 x model {st['model_rel_rms']:.3e}")
    if not st["max"] <= 2 * st["model_max"] + 2.0 ** -11 * st["max_ref"]:
        bad.append(f"max error {st['max']:.3e} > 2 x model {st['model_max']:.3e} + 2^-11 x {st['max_ref']:.3e}")
    if not st["rho"] <= rho:
        bad.append(f"rms(ours - model) / s = {st['rho']:.3f} x the model's error > {rho}")
    if (excess > 0).any():
        c = int(np.argmax(excess))
        bad.append(f"coherent bias in column {c}: mean error {eo[:, c].mean():.3e}, model {em[:, c].mean():.3e}, se {se[c]:.2e}")
    return st, bad


# ---------------------------------------------------------------------------------------------- CPU tier
def query_rows(D, F, n, seed):
    """Query-like rows (player, traverser, one-hot last bid, two belief vectors), rounded to fp16 like the tensor-core tiles."""
    A, H, Q = game_dims(D, F)
    rng = np.random.RandomState(seed)
    x = np.zeros((n, Q))
    x[:, 0] = rng.randint(0, 2, n); x[:, 1] = rng.randint(0, 2, n)
    x[np.arange(n), 2 + rng.randint(0, A, n)] = 1
    b = rng.rand(n, 2, H) ** 3
    x[:, 2 + A:] = (b / b.sum(-1, keepdims=True)).reshape(n, 2 * H)
    return h16(x)


@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_fp64_reference_is_net2_in_float64(D, F, family):
    import torch
    w = family_weights(family, D, F)
    x = query_rows(D, F, 512, 1)
    want = torch_net(w, D, F, x, torch.float64)
    got = fp64_net(unpack(w, D, F), x)
    # (offset_tight cancels ~20 down to a spread of 3e-3 in layer 1: both sides lose four digits there)
    assert np.abs(got - want).max() <= 1e-10 * np.abs(want).max(), np.abs(got - want).max()


def test_families_are_deterministic_and_distinct_has_no_equal_layernorm_parameters():
    for D, F in [(1, 4), (2, 5), (1, 32), (3, 4)]:
        for fam in FAMILIES:
            assert np.array_equal(family_weights(fam, D, F), family_weights(fam, D, F)), (fam, D, F)
        p = unpack(family_weights("distinct", D, F), D, F)
        ln = np.concatenate([p["g1"], p["be1"], p["g2"], p["be2"]]).astype(np.float32)
        assert np.unique(ln).size == ln.size == 4 * HID
        assert (p["be2"] < 0).all()
        # the families differ from init where they claim to
        i = unpack(family_weights("init", D, F), D, F)
        assert (i["g1"] == 1).all() and (i["be2"] == 0).all()
        s = unpack(family_weights("saturating", D, F), D, F)
        assert 3 <= s["g1"].min() and s["g2"].max() <= 6


@pytest.mark.parametrize("D,F", [(1, 6), (2, 5), (1, 32)])
def test_families_reach_what_they_claim(D, F):
    """saturating: |z| of 60 .. 100 in both LayerNorms, both signs; offset_tight: layer-1 variance within 10x of eps."""
    x = query_rows(D, F, 2048, 2)

    def zs(p):
        def ln(y):
            m = y.mean(1, keepdims=True)
            v = ((y - m) ** 2).mean(1, keepdims=True)
            return (y - m) / np.sqrt(v + 1e-5), v
        y1 = x @ p["w1"].T + p["b1"]
        n1, v1 = ln(y1)
        z1 = n1 * p["g1"] + p["be1"]
        a = 0.5 * z1 * (1 + erf(z1 / np.sqrt(2)))
        n2, _ = ln(a @ p["w2"].T + p["b2"])
        return z1, n2 * p["g2"] + p["be2"], v1
    z1, z2, _ = zs(unpack(family_weights("saturating", D, F), D, F))
    for z in (z1, z2):
        assert 60 <= np.abs(z).max() <= 100 and z.min() < -40 and z.max() > 40, (z.min(), z.max())
    _, _, v1 = zs(unpack(family_weights("offset_tight", D, F), D, F))
    med = float(np.median(v1))
    assert 1e-6 <= med <= 1e-4, med


def test_model_matches_the_reference_harness_emulation(net_weights, golden):
    """The GELU variants of the model inside the reference harness's layout (ref_set_net_emulation: uncentred fp16 weights, fp32
    biases, LayerNorm with the mean, fp16 activations) reproduce its stored outputs (reference_live.npz): variant 0 its model 1,
    variant 1 with a correctly rounded tanh its model 2.  Variant 2, the default, is not one of the harness's models; it is pinned
    to the harness's fp32 net at the fp16 level of the other two."""
    D, F = 1, 6
    p = unpack(net_weights(D, F), D, F)
    g = golden("reference_live.npz")
    outs = {m: g[f"emulation{m}_leaf_values"].astype(np.float64) for m in (0, 1, 2)}
    q = g["emulation_queries"].astype(np.float64)
    e = fp64_net(p, q)
    scaler = (outs[0] * e).sum(1) / (e * e).sum(1)     # the harness stores net output x the opponent's reach sum per row
    relrms = lambda a, b: float(np.sqrt(((a - b) ** 2).mean() / (b ** 2).mean()))
    got = {}
    for variant in (0, 1, 2):
        s = 1.0 if variant == 0 else 0.5
        B = dict(W1=np.concatenate([h16(p["w1"]), f32(p["b1"])[:, None]], 1), W2=h16(p["w2"]), b2=f32(p["b2"]),
                 ln1=(f32(s * p["g1"]), f32(s * p["be1"])), ln2=(f32(s * p["g2"]), f32(s * p["be2"])), W3=h16(p["w3"]), b3=f32(p["b3"]))
        got[variant] = model_net(B, h16(q), variant, mean_free=False, tanh16=lambda u: h16(np.tanh(u))) * scaler[:, None]
    assert relrms(got[0], outs[1]) < 1e-4, relrms(got[0], outs[1])
    assert relrms(got[1], outs[2]) < 1e-4, relrms(got[1], outs[2])
    r2 = relrms(got[2], outs[0])
    assert 2e-4 < r2 < 9e-4, r2


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("D,F", [(1, 6), (2, 5)])
def test_criteria_have_teeth(D, F, variant):
    """Without a device: the model with the right blob passes the criteria for `distinct`; fed a blob with one swapped gamma
    pair, with LayerNorm 1's parameters in layer 2, with beta left unscaled (lnscale on gamma only), or without b3, it fails them.
    And the bias criterion catches the truncating tanh.approx.f16x2 against a correctly rounded packed-half model (P5)."""
    p = unpack(family_weights("distinct", D, F), D, F)
    x = query_rows(D, F, 4096, 3)
    ref = fp64_net(p, x)
    B = kernel_blob(p, variant)
    model = model_net(B, x, variant)
    st, bad = tc_criteria(model, ref, model, RHO[variant])
    assert not bad, bad
    assert 1e-4 < st["model_rel_rms"] < 3e-3, st
    swapped = dict(B)
    g = B["ln1"][0].copy()
    g[[10, 11]] = g[[11, 10]]
    swapped["ln1"] = (g, B["ln1"][1])
    ln1_for_2 = dict(B, ln2=B["ln1"])
    no_b3 = dict(B, b3=0 * B["b3"])
    mutants = {"swapped gamma pair": swapped, "LN1 in layer 2": ln1_for_2, "no b3": no_b3}
    if variant:
        mutants["beta not halved"] = dict(B, ln1=(B["ln1"][0], 2 * B["ln1"][1]), ln2=(B["ln2"][0], 2 * B["ln2"][1]))
    for what, M in mutants.items():
        _, bad = tc_criteria(model_net(M, x, variant), ref, model, RHO[variant])
        assert bad, what
    if variant == 1:
        nearest = model_net(B, x, 1, tanh16=lambda u: h16(np.tanh(u)))
        _, bad = tc_criteria(model, ref, nearest, rho=np.inf)
        assert any("coherent bias" in b for b in bad), bad


# ---------------------------------------------------------------------------------------------- GPU tier
@pytest.fixture(scope="module")
def rb():
    import rebel_b200
    assert rebel_b200.capi.lib().cfrb_device_count() > 0, "no CUDA device: the CUDA path cannot be tested"
    return rebel_b200


_WAVE = {}
_TANH16 = []


def tanh_f16x2_device(rb):
    """tanh.approx.f16x2 on every fp16 input, read from the device (cfrb_debug_gelu_table): the instruction has no published
    rounding rule, and truncation towards zero (tanh_f16x2_truncating) leaves a bias of a few 1e-6 in the outputs of the
    saturating and distinct families that the bias criterion sees.  The rest of the packed-half chain is restated here."""
    if not _TANH16:
        S = rb.WaveSolver(1, 4, 1, net_mode=rb.NET_ZERO)
        _, t = S.gelu_table(0)
        S.close()
        tab = t.astype(np.float64)
        _TANH16.append(lambda u: tab[np.asarray(u, np.float64).astype(np.float16).view(np.uint16)])
    return _TANH16[0]


def _wave(rb, D, F):
    """A wave of mixed roots with ~WAVE_ROWS query rows; subgame 0 (root bid A - 6) alone gives one partial tile."""
    if (D, F) not in _WAVE:
        A, H, Q = game_dims(D, F)
        Kmax = 4096
        rng = np.random.RandomState(10 * D + F)
        b = rng.rand(Kmax, 2, H) ** 2
        b /= b.sum(-1, keepdims=True)
        lb = rng.randint(-1, A - 2, size=Kmax).astype(np.int32); lb[1:5] = -1; lb[0] = A - 6
        pl = rng.randint(0, 2, size=Kmax).astype(np.int32)
        S = rb.WaveSolver(D, F, 64, net_mode=rb.NET_FP32)
        S.set_weights(family_weights("init", D, F))
        S.begin(lb[:64], pl[:64], b[:64])
        S.run(1)
        rows = len(S.leaf_io()[0])
        S.close()
        K = int(np.clip(np.ceil(WAVE_ROWS * 64 / rows), 1, Kmax))
        _WAVE[(D, F)] = (lb[:K], pl[:K], b[:K])
    return _WAVE[(D, F)]


def _run(rb, D, F, mode, w, lb, pl, b):
    S = rb.WaveSolver(D, F, len(lb), net_mode=mode)
    S.set_weights(w)
    S.begin(lb, pl, b)
    S.run(1)
    q, o, _ = S.leaf_io()
    S.close()
    return q, o


def _pick(rows):
    """Up to ROWS_MAX rows spread over all tiles, the whole partial last tile included."""
    if rows <= ROWS_MAX:
        return np.arange(rows)
    last = np.arange((rows - 1) // 128 * 128, rows)
    return np.unique(np.concatenate([np.linspace(0, last[0] - 1, ROWS_MAX - len(last)).astype(np.int64), last]))


_REF = {}


def _fp64(p, x, key):
    k = key + (hashlib.sha1(x.tobytes()).hexdigest(),)
    if k not in _REF:
        _REF.clear()            # one case's rows at a time: the tensor-core modes of a (game, family) share them
        _REF[k] = fp64_net(p, x)
    return _REF[k]


def _cases():
    out = []
    for D, F in RESIDENT + WIDE + FP32_ONLY:
        for mode in MODES:
            if (D, F) in FP32_ONLY and mode != "fp32":
                continue
            fams = FAMILIES + (["trained"] if (D, F) in TRAINED_GAMES else [])
            out += [pytest.param(D, F, mode, fam, id=f"{D}x{F}f-{mode}-{fam}") for fam in fams]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("D,F,mode,family", _cases())
def test_value_net_against_fp64(rb, monkeypatch, D, F, mode, family):
    from rebel_b200 import capi
    mode_name, x2_gelu, variant = MODES[mode]
    for k in ("CFRB_X2_GELU", "CFRB_TC_WIDE", "CFRB_NET_MODE"):
        monkeypatch.delenv(k, raising=False)
    if x2_gelu:
        monkeypatch.setenv("CFRB_X2_GELU", x2_gelu)
    w = family_weights(family, D, F)
    p = unpack(w, D, F)
    lb, pl, b = _wave(rb, D, F)
    net_mode = getattr(rb, mode_name)
    q, o = _run(rb, D, F, net_mode, w, lb, pl, b)
    rows = len(q)
    assert rows >= min(10000, 64 * len(lb)) and rows % 128, rows
    assert np.isfinite(o).all(), (int((~np.isfinite(o)).sum()), rows)
    # the first subgame alone: one partial tile, the same rows and bit-identical outputs
    q1, o1 = _run(rb, D, F, net_mode, w, lb[:1], pl[:1], b[:1])
    n1 = len(q1)
    assert 0 < n1 and n1 % 128 and np.array_equal(q1, q[:n1]) and np.array_equal(o1, o[:n1]), n1
    idx = _pick(rows)
    x = q[idx].astype(np.float64)
    ours = o[idx].astype(np.float64)
    ref = _fp64(p, x, (D, F, family))
    tag = f"{D}x{F}f {mode} {family}: {rows} rows ({len(idx)} checked), single subgame {n1}"
    if variant is None:
        import torch
        e32 = np.abs(torch_net(w, D, F, x, torch.float32) - ref).max()
        err = np.abs(ours - ref).max()
        bound = 4 * e32 + 2.0 ** -20 * np.abs(ref).max()
        _note(f"{tag}: max |ours - fp64| {err:.3e}, torch fp32 {e32:.3e}, bound {bound:.3e}, max |fp64| {np.abs(ref).max():.3e}")
        assert err <= bound, (err, e32)
        return
    kw = dict(tanh16=tanh_f16x2_device(rb)) if variant == 1 else {}
    model = model_net(kernel_blob(p, variant), x, variant, **kw)
    st, bad = tc_criteria(ours, ref, model, RHO[variant])
    B = capi.net_output_bound(D, F, w)
    top = float(np.abs(o).max())
    _note(f"{tag}: rel rms {st['rel_rms']:.3e} (model {st['model_rel_rms']:.3e}), max {st['max']:.3e} (model {st['model_max']:.3e}), "
          f"rho {st['rho']:.3f}, bias excess {st['bias_excess']:.1f} se, max |out| {top:.3e} / bound {B:.3e}, "
          f"rms fp64 {st['rms_ref']:.3e}")
    assert top <= B, (top, B)
    assert not bad, bad


@pytest.mark.gpu
def test_trained_family_is_reproducible(rb):
    """The trained weights are a deterministic function of the game: the trainer and the self-play loop are bit-reproducible."""
    D, F = 1, 6
    w = trained_weights(D, F)
    assert np.array_equal(w, _train(D, F))
    p, i = unpack(w, D, F), unpack(family_weights("init", D, F), D, F)
    assert np.abs(p["g1"] - i["g1"]).max() > 1e-3 and np.abs(p["be2"] - i["be2"]).max() > 1e-3    # away from the initialisation
