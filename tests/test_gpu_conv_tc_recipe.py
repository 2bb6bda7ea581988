"""GPU tier: the tensor-core convs (csrc/conv_tc.cu) against the recipe-exact reference (oracle/tc_recipes.py) instead of
fp64 alone.  The reference reproduces each recipe's operand rounding bit for bit and sums the plane products in float64,
so what is left is the kernel's own fp32 accumulation: |y - y_ref| <= c * 2^-20 * sum|w||z| per output element, with c
(tc_recipes.KERNEL_BOUND_C) ten times below what a lost correction term on one tap of one 16-channel block produces
(tests/test_cpu_tc_recipe_envelope.py).  Also: operand magnitudes (the FAST recipe's e4m3 envelope), the fp16 range guard,
and the decoder's shortcut convs on Hz-scale F0 input."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import cases
import styletts2_oracle as O
import tc_recipes as R
from test_gpu_conv_tc import CONVT_TC, TC_CASES, TOL
from test_gpu_conv_tct import TCT_CASES, TOL_FAST
from util import maxdiff, oracle_sds, record

D = "cuda:0"
PROLOGUES = ["none", "lrelu"]       # both with the AdaIN affine; Snake's __sinf has no bit-exact CPU counterpart


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.fixture()
def tc_ops(monkeypatch):
    from styletts2_b200 import ops
    monkeypatch.setattr(ops, "TC_MIN_WORK", 0)          # small cases stay on the tensor-core kernels
    return ops


def _kernel_name(ops, fn):
    ops.PROFILE = []
    try:
        out = fn()
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    return out, names


def _conv(ops, x, w, mode, K, dil, pad, pre=None, act="none", slope=0.2, max_ctas=0):
    """kernel result of a bias-free conv1d on the tensor cores + the name of the launch"""
    from styletts2_b200.lib import ACT_LRELU, ACT_NONE
    wd = w.to(D)
    kw = dict(K=K, dil=dil, pad=pad, pre_act=ACT_LRELU if act == "lrelu" else ACT_NONE, slope=slope, wtc=ops.conv_tc_weight_layout(wd, mode),
              tc_max_ctas=max_ctas)
    if pre is not None:
        kw["pre"] = (pre[0].to(D).contiguous(), pre[1].to(D).contiguous())
    (y, _), names = _kernel_name(ops, lambda: ops.conv1d(x.to(D), ops.conv_weight_layout(wd), None, **kw))
    assert names and names[0].startswith("conv1d_tc"), names
    return y.cpu().double(), names[0]


def _bound_err(y, ref, scale):
    """max |y - y_ref| in units of 2^-20 sum|w||z| (the bound an fp32 accumulation obeys)"""
    return float(((y - ref).abs() / (scale * 2.0 ** -20)).max())


def _rel64(y, z, w, **kw):
    r = F.conv1d(z.double(), w.double(), None, **kw)
    return float((y - r).abs().max() / r.abs().max())


def _check_recipe(y, z, w, mode, what, **kw):
    ref = R.conv1d(z, w, mode, **kw)
    e = _bound_err(y, ref, R.sum_abs(F.conv1d, z, w, **kw))
    record("conv_tc_recipe", case=what, mode=mode, bound_err=e)
    assert math.isfinite(e) and e <= R.KERNEL_BOUND_C[mode], (what, e)
    return e


# ------------------------------------------------------------------ 1. kernel == recipe-exact reference
@pytest.mark.parametrize("act", PROLOGUES)
@pytest.mark.parametrize("kernel", ["fast_cm", "fast_tm", "accurate", "f16x3"])
@pytest.mark.parametrize("cfg", TC_CASES + [c for c in TCT_CASES if c not in TC_CASES])
def test_conv1d_tc_matches_recipe_exact_reference(cfg, kernel, act, tc_ops, monkeypatch):
    ops = tc_ops
    B, Cin, Cout, K, d, L, max_ctas = cfg
    if kernel == "fast_tm" and Cout > 128:
        pytest.skip("time-major kernel: Cout <= 128")
    mode = {"fast_cm": R.FAST, "fast_tm": R.FAST, "accurate": R.ACCURATE, "f16x3": R.F16X3}[kernel]
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128 if kernel == "fast_tm" else 0)
    x, w = rnd(B, Cin, L, seed=1), rnd(Cout, Cin, K, seed=2, scale=1 / math.sqrt(Cin * K))
    a, b = 1 + 0.3 * rnd(B, Cin, seed=4), 0.2 * rnd(B, Cin, seed=5)
    pad = O.get_padding(K, d)
    y, name = _conv(ops, x, w, mode, K, d, pad, pre=(a, b), act=act, max_ctas=max_ctas)
    assert name.startswith(f"conv1d_tc m{mode | (16 if kernel == 'fast_tm' else 0)} "), name
    _check_recipe(y, R.prologue(x, a, b, act, 0.2), w, mode, f"{kernel} {act} {cfg}", padding=pad, dilation=d)


@pytest.mark.parametrize("act", PROLOGUES)
@pytest.mark.parametrize("kernel", ["fast_cm", "fast_tm", "accurate"])
@pytest.mark.parametrize("cfg", CONVT_TC)
def test_conv_transpose1d_tc_matches_recipe_exact_reference(cfg, kernel, act, tc_ops, monkeypatch):
    ops = tc_ops
    from styletts2_b200.lib import ACT_LRELU, ACT_NONE
    Cin, Cout, K, S, P, OP, L, reflect = cfg
    mode = R.ACCURATE if kernel == "accurate" else R.FAST
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128 if kernel == "fast_tm" else 0)
    x, w = rnd(2, Cin, L, seed=1), rnd(Cin, Cout, K, seed=2, scale=1 / math.sqrt(Cin * 2))
    wd = w.to(D)
    y, _ = ops.conv_transpose1d(x.to(D), ops.convT_weight_layout(wd, S, P), None, K=K, stride=S, padding=P,
                                pre_act=ACT_LRELU if act == "lrelu" else ACT_NONE, slope=0.1, reflect_left1=reflect,
                                wtc=ops.convT_tc_weight_layout(wd, S, P, mode))
    z = R.prologue(x, act=act, slope=0.1)
    kw = dict(stride=S, padding=P, output_padding=OP)
    ref, scale = R.conv_transpose1d(z, w, mode, **kw), R.sum_abs(F.conv_transpose1d, z, w, **kw)
    if reflect:
        ref, scale = F.pad(ref, (1, 0), mode="reflect"), F.pad(scale, (1, 0), mode="reflect")
    e = _bound_err(y.cpu().double(), ref, scale)
    record("convT_tc_recipe", case=f"{kernel} {act} {cfg}", mode=mode, bound_err=e)
    assert math.isfinite(e) and e <= R.KERNEL_BOUND_C[mode], e


# ------------------------------------------------------------------ 2./3. operand magnitudes
SWEEP_KERNELS = [("fast", 256), ("fast", 64), ("accurate", 256), ("f16x3", 256)]   # Cout 64: time-major kernel
FAST_ENVELOPE = 64.0     # |z| below which FAST's e4m3 corrections are exact (DESIGN.md "Precision recipes")


def _sweep_operands(peak, target, via, Cin=96, B=2, L=300):
    x = rnd(B, Cin, L, seed=11)
    a, b = 1 + 0.2 * rnd(B, Cin, seed=12), 0.1 * rnd(B, Cin, seed=13)
    ch = slice(Cin - 7, Cin - 6) if target == "channel" else slice(None)      # a channel inside the last 16-channel block
    if via == "x":
        x[:, ch] *= peak / float(x[:, ch].abs().max())
        a[:, ch], b[:, ch] = 1.0, 0.0
    else:                                                      # a large AdaIN scale on an O(1) input
        a[:, ch] = peak / float(x[:, ch].abs().max())
        b[:, ch] = 0.0
    return x, a, b


@pytest.mark.parametrize("via", ["x", "pre_a"])
@pytest.mark.parametrize("target", ["channel", "tensor"])
@pytest.mark.parametrize("peak", [1.0, 30.0, 100.0, 300.0, 1000.0])
@pytest.mark.parametrize("recipe,Cout", SWEEP_KERNELS)
def test_activation_magnitude_sweep(recipe, Cout, peak, target, via, tc_ops, monkeypatch):
    ops = tc_ops
    mode = {"fast": R.FAST, "accurate": R.ACCURATE, "f16x3": R.F16X3}[recipe]
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128)
    K, d = 3, 1
    x, a, b = _sweep_operands(peak, target, via)
    w = rnd(Cout, x.shape[1], K, seed=14, scale=1 / math.sqrt(x.shape[1] * K))
    y, name = _conv(ops, x, w, mode, K, d, 1, pre=(a, b), act="lrelu")
    assert ("m16 " in name) == (Cout <= 128 and mode == R.FAST), name
    z = R.prologue(x, a, b, "lrelu", 0.2)
    assert float(z.abs().max()) < 1023.5
    what = f"{recipe} co{Cout} peak{peak} {target} via {via}"
    _check_recipe(y, z, w, mode, what, padding=1)
    e64 = _rel64(y, z, w, padding=1)
    record("conv_tc_sweep", case=what, rel_err_fp64=e64)
    if mode != R.FAST:
        assert e64 < TOL[mode], (what, e64)
    elif peak < FAST_ENVELOPE:
        assert e64 < TOL_FAST, (what, e64)


@pytest.mark.parametrize("wmax", [1e-3, 1e-2, 1.0, 8.0])
@pytest.mark.parametrize("recipe,Cout", SWEEP_KERNELS)
def test_weight_magnitude_sweep(recipe, Cout, wmax, tc_ops, monkeypatch):
    ops = tc_ops
    mode = {"fast": R.FAST, "accurate": R.ACCURATE, "f16x3": R.F16X3}[recipe]
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128)
    B, Cin, K, L = 2, 96, 3, 300
    x, a, b = rnd(B, Cin, L, seed=21), 1 + 0.2 * rnd(B, Cin, seed=22), 0.1 * rnd(B, Cin, seed=23)
    w = rnd(Cout, Cin, K, seed=24)
    w = w * (wmax / float(w.abs().max()))
    y, _ = _conv(ops, x, w, mode, K, 1, 1, pre=(a, b), act="lrelu")
    z = R.prologue(x, a, b, "lrelu", 0.2)
    what = f"{recipe} co{Cout} max|w| {wmax}"
    _check_recipe(y, z, w, mode, what, padding=1)
    e64 = _rel64(y, z, w, padding=1)
    record("conv_tc_weight_sweep", case=what, rel_err_fp64=e64)
    assert e64 < (TOL_FAST if mode == R.FAST else TOL[mode]), (what, e64)


# ------------------------------------------------------------------ 4. range guard
def _guard_launch(ops, kind, x, w, pre=None):
    wd = w.to(D)
    if kind == "convT":
        wtc = ops.convT_tc_weight_layout(wd, 2, 1, R.FAST)
        run = lambda: ops.conv_transpose1d(x.to(D), ops.convT_weight_layout(wd, 2, 1), None, K=4, stride=2, padding=1, wtc=wtc)
    else:
        wtc = ops.conv_tc_weight_layout(wd, R.FAST)
        kw = dict(pre=(pre[0].to(D), pre[1].to(D))) if pre is not None else {}
        run = lambda: ops.conv1d(x.to(D), ops.conv_weight_layout(wd), None, K=3, pad=1, wtc=wtc, **kw)
    return wtc, run


@pytest.mark.parametrize("kind,Cout", [("channel_major", 256), ("time_major", 64), ("convT", 256)])
def test_conv_tc_range_guard(kind, Cout, tc_ops, monkeypatch):
    """|z| >= 1024 (64 z overflows fp16) reached through x or the AdaIN scale, a NaN input, and |w| >= 16 (4096 w
    overflows) make ops.check_range() raise; clean runs do not, and a fetch clears the flag.  Finite values only."""
    ops = tc_ops
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128)
    B, Cin, L = 2, 64, 200
    x = rnd(B, Cin, L, seed=31)
    w = rnd(Cin, Cout, 4, seed=32, scale=0.05) if kind == "convT" else rnd(Cout, Cin, 3, seed=32, scale=0.05)
    ones, zeros = torch.ones(B, Cin), torch.zeros(B, Cin)
    ops.check_range()                                             # start clean
    wtc, run = _guard_launch(ops, kind, x, w, None if kind == "convT" else (ones, zeros))
    assert (wtc.mode & 16) == (16 if kind == "time_major" else 0)
    run()
    ops.check_range()                                             # clean operands: no raise
    bad_x = x.clone()
    bad_x[1, Cin - 3, 77] = 1100.0
    nan_x = x.clone()
    nan_x[0, 5, 3] = float("nan")
    cases_ = [("x", bad_x, None), ("nan", nan_x, None)]
    if kind != "convT":
        big_a = ones.clone()
        big_a[1, 9] = 2000.0 / float(x[1, 9].abs().max())
        cases_.append(("pre_a", x, (big_a, zeros)))
    for what, xi, pre in cases_:
        _, run = _guard_launch(ops, kind, xi, w, pre if pre is not None else (None if kind == "convT" else (ones, zeros)))
        y = run()[0]
        assert not torch.isfinite(y).all(), what
        with pytest.raises(FloatingPointError):
            ops.check_range()
        ops.check_range()                                         # the fetch cleared the flag
    bad_w = w.clone()
    bad_w.view(-1)[123] = 20.0
    _guard_launch(ops, kind, x, bad_w, None if kind == "convT" else (ones, zeros))      # caught by the weight layout alone
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()


# ------------------------------------------------------------------ 5. decoder shortcut convs at Hz-scale F0
@pytest.fixture(scope="module")
def private_lj():
    """a model of its own (util.gpu_model is shared): these tests change recipes and weights"""
    from styletts2_b200.models import build_model, load_keyed_weights, recursive_munch
    m = build_model(recursive_munch(cases.MODEL_CFGS["ljspeech"]))
    for k in m:
        m[k].to(D).eval()
    load_keyed_weights(m)
    return m


UNIT_F0 = torch.tensor([0.25, 0.5, 0.25])       # unit DC gain: F0 in Hz passes through


def _f0_channel(B, T, seed):
    f0 = cases.synthetic_f0(B, 2 * T, seed=seed)
    return F.conv1d(f0.unsqueeze(1), UNIT_F0.view(1, 1, 3), stride=2, padding=1)[:, 0], f0


@pytest.mark.parametrize("name,cin", [("encode", 514), ("decode.0", 1090), ("decode.3", 1090)])
def test_decoder_shortcut_conv_at_hz_scale_f0(name, cin, private_lj):
    """cat-buffer input whose F0 channel is F0 in Hz (60..400): the learned 1x1 shortcut sees it raw and must run the
    ACCURATE recipe (FAST clips its corrections there)"""
    from styletts2_b200 import modules, ops
    from styletts2_b200.lib import TC_ACCURATE, TC_FAST
    sd = oracle_sds("ljspeech", ("decoder",))["decoder"]
    blk = dict(private_lj.decoder.named_modules())[name]
    B, T = 2, 40
    x, s = rnd(B, cin, T, seed=41), rnd(B, 128, seed=42, scale=0.5)
    x[:, cin - 2] = _f0_channel(B, T, seed=43)[0]
    x[:, cin - 1] = F.conv1d(torch.rand(B, 1, 2 * T, generator=torch.Generator().manual_seed(44)) * 5, UNIT_F0.view(1, 1, 3), stride=2, padding=1)[:, 0]
    with torch.no_grad():
        ref = O.adain_resblk1d(x, s, sd, name)
    with torch.no_grad():
        y, names = _kernel_name(ops, lambda: blk(x.to(D), s.to(D)))
    sc = [n for n in names if n.startswith("conv1d_tc") and f" ci{cin} " in n and " k1 " in n]
    assert len(sc) == 1 and sc[0].startswith(f"conv1d_tc m{TC_ACCURATE} "), names
    err = maxdiff(y, ref) / float(ref.abs().max())
    try:                                                          # the same block with the shortcut on FAST, for the record
        modules.set_tc_mode(blk.conv1x1, TC_FAST)
        with torch.no_grad():
            err_fast = maxdiff(blk(x.to(D), s.to(D)), ref) / float(ref.abs().max())
    finally:
        modules.set_tc_mode(blk.conv1x1, TC_ACCURATE)
    record("decoder_shortcut_hz_f0", block=name, rel_err=err, rel_err_if_fast=err_fast, f0_peak=float(x[:, cin - 2].abs().max()))
    assert y.shape == ref.shape and err < 1e-4, (err, err_fast)


def test_decoder_with_unit_gain_f0_conv(private_lj):
    """whole decoder (lj_dec case, har teacher-forced) with a unit-gain F0_conv in both the model and the oracle's state
    dict: the cat buffers then carry F0 in Hz into every shortcut conv"""
    from styletts2_b200 import modules
    from styletts2_b200.lib import TC_ACCURATE, TC_FAST
    case = cases.DECODER_CASES["lj_dec"]
    mcfg = cases.MODEL_CFGS["ljspeech"]["decoder"]
    sd = dict(oracle_sds("ljspeech", ("decoder",))["decoder"])
    sd["F0_conv.weight_v"] = UNIT_F0.view(1, 1, 3).clone()
    sd["F0_conv.weight_g"] = UNIT_F0.norm().view(1, 1, 1).clone()
    sd["F0_conv.bias"] = torch.zeros(1)
    dec = private_lj.decoder
    with torch.no_grad():
        for k in ("weight_v", "weight_g", "bias"):
            getattr(dec.F0_conv, k).copy_(sd["F0_conv." + k])
    asr, f0, n, s = cases.decoder_inputs(case)
    rng = cases.ReplayRNG(case["seed"])
    L = 600 * case["T"]
    ri, sn = rng.rand_ini((case["B"], 9)), rng.sine_noise((case["B"], L, 9))
    with torch.no_grad():
        har = O.istftnet_har(f0, O.sub(sd, "generator"), mcfg, ri, sn)
        ref = O.decoder(asr, f0, n, s, sd, mcfg, rand_ini=ri, sine_noise=sn, har=har).squeeze(1)
        run = lambda: dec(asr.to(D), f0.to(D), n.to(D), s.to(D), sine_noise=sn.to(D), har=har.to(D)).squeeze(1)
        d = maxdiff(run(), ref)
        shortcuts = [b.conv1x1 for b in [dec.encode, *dec.decode]]
        try:
            for c in shortcuts:
                modules.set_tc_mode(c, TC_FAST)
            d_fast = maxdiff(run(), ref)
        finally:
            for c in shortcuts:
                modules.set_tc_mode(c, TC_ACCURATE)
    record("decoder_unit_gain_f0_conv", wav_maxabs=d, wav_maxabs_if_fast=d_fast, wav_scale=float(ref.abs().max()))
    assert d <= 1e-3, (d, d_fast)
