"""GPU tier: the TIME-MAJOR tensor-core Conv1d (csrc/conv_tc.cu conv1d_tct_kernel: frames on the MMA's M axis, output
channels on N = Cout rounded up; narrow HiFi-GAN stages, conv_post) against fp64 torch and against the channel-major
kernel: every epilogue variant (residual, MRF accumulate, tanh, statistics), channel counts that are not multiples of 32,
odd row lengths, tail tiles, the persistent loop on a few CTAs."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import styletts2_oracle as O
from util import maxdiff, record

D = "cuda:0"
TOL_FAST = 6e-5


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.fixture()
def tmajor_all(monkeypatch):
    from styletts2_b200 import ops
    monkeypatch.setattr(ops, "TC_TMAJOR_MAX_COUT", 128)
    monkeypatch.setattr(ops, "TC_MIN_WORK", 0)      # the tiny cases must not fall back to the FP32-pipe kernel
    return ops


TCT_CASES = [
    # B, Cin, Cout, K, dil, L, max_ctas
    (1, 32, 32, 1, 1, 256, 0),       # one MMA per M block, no taps
    (1, 32, 32, 3, 1, 256, 0),
    (2, 32, 32, 11, 1, 2000, 0),     # HiFi-GAN C=32 stage
    (2, 32, 32, 11, 5, 1531, 0),     # max window, odd length
    (3, 64, 64, 7, 3, 2000, 0),      # HiFi-GAN C=64 stage
    (2, 64, 64, 3, 1, 4099, 4),      # persistent loop on 4 CTAs (barrier phase wrap), odd length
    (2, 128, 22, 7, 1, 1201, 0),     # conv_post of iSTFTNet (Cout 22 -> 32 rows)
    (2, 32, 1, 7, 1, 3000, 0),       # conv_post of HiFi-GAN (Cout 1 -> 16 rows)
    (2, 48, 16, 3, 1, 700, 0),       # N = 16
    (2, 80, 96, 3, 5, 515, 3),       # N = 96 (3 channel groups), tail tile
    (2, 128, 128, 3, 1, 1500, 0),    # N = 128: widest accumulator (two warpgroups x 64 channels)
    (3, 128, 128, 7, 1, 1201, 5),
    (2, 22, 128, 1, 1, 2403, 0),
    (1, 64, 64, 7, 1, 100, 0),       # single partial tile: M block 1 entirely beyond the row
    (2, 64, 40, 3, 1, 129, 0),       # Cout not a multiple of 8; one frame in M block 1
]


@pytest.mark.parametrize("cfg", TCT_CASES)
def test_conv1d_tct_matches_fp64(cfg, tmajor_all):
    ops = tmajor_all
    from styletts2_b200.lib import ACT_SNAKE, TC_TMAJOR
    B, Cin, Cout, K, d, L, max_ctas = cfg
    x, w, bias = rnd(B, Cin, L, seed=1), rnd(Cout, Cin, K, seed=2, scale=1 / math.sqrt(Cin * K)), rnd(Cout, seed=3)
    a, b = 1 + 0.3 * rnd(B, Cin, seed=4), 0.2 * rnd(B, Cin, seed=5)
    alpha = 1 + 0.3 * torch.rand(1, Cin, 1, generator=torch.Generator().manual_seed(6))
    res = rnd(B, Cout, L, seed=7)
    z = a[:, :, None] * x + b[:, :, None]
    z = z + (1 / alpha) * torch.sin(alpha * z) ** 2
    pad = O.get_padding(K, d)
    ref = (F.conv1d(z.double(), w.double(), bias.double(), 1, pad, d) + res.double()).float()
    wd = w.to(D)
    wtc = ops.conv_tc_weight_layout(wd, 0)
    assert wtc.mode & TC_TMAJOR
    try:
        ops.PROFILE = []
        y, st = ops.conv1d(x.to(D), ops.conv_weight_layout(wd), bias.to(D), K=K, dil=d, pad=pad, pre=(a.to(D).contiguous(), b.to(D).contiguous()),
                           pre_act=ACT_SNAKE, alpha=alpha.to(D), res=res.to(D), want_stats=True, wtc=wtc, tc_max_ctas=max_ctas)
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert names and names[0].startswith("conv1d_tc m16"), names
    r = maxdiff(y, ref) / float(ref.abs().max())
    record("conv1d_tct", cfg=str(cfg), rel_err=r)
    assert r < TOL_FAST, r
    gb = torch.zeros(B, 2 * Cout, device=D)
    ca, cb = ops.adain_coef(st, gb)
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4 and maxdiff(cb, -ref.mean(-1) * ea) < 1e-3


def test_conv1d_tct_statistics_with_large_mean(tmajor_all):
    """Rows whose mean is 1000x their spread: the pilot-shifted one-pass partials must keep the variance (a raw sum of
    squares in fp32 would lose it)."""
    ops = tmajor_all
    B, Cin, Cout, K, L = 2, 32, 32, 3, 3001
    x, w = rnd(B, Cin, L, seed=1), rnd(Cout, Cin, K, seed=2, scale=0.01 / math.sqrt(Cin * K))
    bias = 10.0 + rnd(Cout, seed=3)
    ref = F.conv1d(x.double(), w.double(), bias.double(), 1, 1).float()
    wd = w.to(D)
    y, st = ops.conv1d(x.to(D), ops.conv_weight_layout(wd), bias.to(D), K=K, pad=1, want_stats=True, wtc=ops.conv_tc_weight_layout(wd, 0))
    ca, cb = ops.adain_coef(st, torch.zeros(B, 2 * Cout, device=D))
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False).double() + 1e-5)
    assert maxdiff(ca, ea.float()) / float(ea.abs().max()) < 2e-3      # var ~ 1e-4 of mean^2 = 100: fp32 output rounding itself is ~1e-3 of the spread
    assert maxdiff(y, ref) / float(ref.abs().max()) < TOL_FAST


def test_conv1d_tct_epilogue_variants_match_channel_major(tmajor_all):
    """No bias / no residual / out_div / MRF accumulate (modes 1, 2) / tanh: time-major == channel-major to the recipe's
    accuracy (same products, different accumulation order), and == fp32 torch."""
    ops = tmajor_all
    from styletts2_b200.lib import ACT_LRELU, ACT_TANH
    B, C, K, L = 2, 64, 7, 1777
    x = rnd(B, C, L, seed=1)
    ws = [rnd(C, C, K, seed=10 + i, scale=1 / math.sqrt(C * K)) for i in range(3)]
    res = rnd(B, C, L, seed=5)
    xa = F.leaky_relu(x, 0.1)
    parts = [(F.conv1d(xa, ws[i], None, 1, 3) + res) / math.sqrt(2) for i in range(3)]
    ref = (parts[0] + parts[1] + parts[2]) / 3
    for tmax in (128, 0):
        ops.TC_TMAJOR_MAX_COUT = tmax
        acc = torch.empty(B, C, L, device=D)
        for i in range(3):
            wd = ws[i].to(D)
            ops.conv1d(x.to(D), ops.conv_weight_layout(wd), None, K=K, pad=3, pre_act=ACT_LRELU, slope=0.1, res=res.to(D), out_div=math.sqrt(2), out=acc,
                       accum_mode=0 if i == 0 else (2 if i == 2 else 1), accum_div=3.0, wtc=ops.conv_tc_weight_layout(wd))
        r = maxdiff(acc, ref) / float(ref.abs().max())
        assert r < 1e-4, (tmax, r)
    ops.TC_TMAJOR_MAX_COUT = 128
    # tanh output activation, single output channel (HiFi-GAN conv_post, hifigan.py:344-345)
    w1, b1 = rnd(1, 32, 7, seed=20, scale=0.1), rnd(1, seed=21)
    x1 = rnd(B, 32, 5000, seed=22)
    ref1 = torch.tanh(F.conv1d(F.leaky_relu(x1, 0.01), w1, b1, 1, 3))
    wd = w1.to(D)
    y1, _ = ops.conv1d(x1.to(D), ops.conv_weight_layout(wd), b1.to(D), K=7, pad=3, pre_act=ACT_LRELU, slope=0.01, out_act=ACT_TANH,
                       wtc=ops.conv_tc_weight_layout(wd))
    assert maxdiff(y1, ref1) < 1e-4


@pytest.mark.parametrize("cfg", [(128, 64, 6, 3, 2, 1, 1000, False), (64, 32, 4, 2, 1, 0, 2000, False), (256, 128, 12, 6, 3, 0, 700, True)])
def test_conv_transpose1d_tct_matches_fp32(cfg, tmajor_all):
    ops = tmajor_all
    from styletts2_b200.lib import ACT_LRELU, TC_TMAJOR
    Cin, Cout, K, S, P, OP, L, reflect = cfg
    x, w, b = rnd(2, Cin, L, seed=1), rnd(Cin, Cout, K, seed=2, scale=1 / math.sqrt(Cin * 2)), rnd(Cout, seed=3)
    ref = F.conv_transpose1d(F.leaky_relu(x, 0.1), w, b, stride=S, padding=P, output_padding=OP)
    if reflect:
        ref = F.pad(ref, (1, 0), mode="reflect")
    res = rnd(2, Cout, ref.shape[-1], seed=4)
    ref = ref + res
    wd = w.to(D)
    wtc = ops.convT_tc_weight_layout(wd, S, P, 0)
    assert wtc.mode & TC_TMAJOR
    y, st = ops.conv_transpose1d(x.to(D), ops.convT_weight_layout(wd, S, P), b.to(D), K=K, stride=S, padding=P, pre_act=ACT_LRELU,
                                 slope=0.1, res=res.to(D), reflect_left1=reflect, want_stats=True, wtc=wtc)
    assert y.shape == ref.shape
    r = maxdiff(y, ref) / float(ref.abs().max())
    record("convT_tct", cfg=str(cfg), rel_err=r)
    assert r < 2 * TOL_FAST, r
    ca, cb = ops.adain_coef(st, torch.zeros(2, 2 * Cout, device=D))
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4 and maxdiff(cb, -ref.mean(-1) * ea) < 1e-3


@pytest.mark.parametrize("C,K,L", [(32, 3, 3000), (128, 7, 1300), (64, 11, 2048)])
def test_conv1d_tct_mrf_accumulate_plain_epilogue(C, K, L, tmajor_all):
    """MRF mean through the accumulate modes with the plain epilogue (the full-step path that loads y one step ahead):
    xs = (r0 + r1 + r2) / 3 with r_i = conv_i(x) + res (istftnet.py:369-375), statistics of the final sum."""
    ops = tmajor_all
    B = 2
    x, res = rnd(B, C, L, seed=1), rnd(B, C, L, seed=5)
    ws = [rnd(C, C, K, seed=10 + i, scale=1 / math.sqrt(C * K)) for i in range(3)]
    pad = (K - 1) // 2
    ref = sum(F.conv1d(x.double(), w.double(), None, 1, pad) + res.double() for w in ws) / 3
    acc = torch.empty(B, C, L, device=D)
    st = None
    for i in range(3):
        wd = ws[i].to(D)
        _, st = ops.conv1d(x.to(D), ops.conv_weight_layout(wd), None, K=K, pad=pad, res=res.to(D), out=acc, accum_mode=0 if i == 0 else (2 if i == 2 else 1),
                           accum_div=3.0, want_stats=(i == 2), wtc=ops.conv_tc_weight_layout(wd))
    r = maxdiff(acc, ref.float()) / float(ref.abs().max())
    assert r < 1e-4, r
    ca, cb = ops.adain_coef(st, torch.zeros(B, 2 * C, device=D))
    ea = 1 / torch.sqrt(ref.float().var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4 and maxdiff(cb, -ref.float().mean(-1) * ea) < 1e-3
