"""GPU tier: the wgmma tensor-core Conv1d against fp32 torch, for each precision recipe (csrc/conv_tc.cu):
FAST (fp16 high planes + one e4m3 K=32 correction MMA; ~2^-16 per product), ACCURATE (two fp16 planes, separate
correction accumulator; fp32-SIMT level) and F16X3 (the accurate planes in one accumulator).  Tolerances relative to the
output scale; a single 16-bit pass would be ~1e-3."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import styletts2_oracle as O
from util import maxdiff, record

D = "cuda:0"


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


TC_CASES = [
    # B, Cin, Cout, K, dil, L, max_ctas
    (1, 32, 128, 1, 1, 256, 0),      # single MMA group, no taps, no tail
    (1, 32, 128, 3, 1, 256, 0),      # taps (descriptor row shifts)
    (2, 128, 128, 3, 1, 700, 0),     # several ci blocks, tail tile
    (2, 128, 128, 7, 3, 1000, 0),
    (2, 256, 256, 11, 5, 1300, 0),   # two co blocks, max window
    (3, 64, 64, 7, 5, 2000, 0),      # Cout padded to 128
    (2, 48, 32, 11, 1, 900, 0),      # Cin, Cout padded
    (4, 128, 128, 3, 1, 3000, 5),    # persistent loop on 5 CTAs (stage ring phase wrap)
    (3, 128, 128, 7, 1, 1201, 0),    # odd row length: every channel row starts at a different 4-byte phase (16-byte cp.async windows)
    (2, 22, 128, 1, 1, 2403, 0),     # Cin not a multiple of 16 (zero-filled channels), odd length
    (2, 80, 256, 3, 5, 515, 3),      # odd length, tail tile, few CTAs
]
TOL = {0: 6e-5, 1: 3e-6, 2: 2e-5}   # FAST, ACCURATE, F16X3 (measured: the conv1d_tc / convT_tc records of ST2_PARITY_REPORT)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("cfg", TC_CASES)
def test_conv1d_tc_matches_fp32(cfg, mode):
    from styletts2_b200 import ops
    from styletts2_b200.lib import ACT_SNAKE
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
    y, st = ops.conv1d(x.to(D), ops.conv_weight_layout(wd), bias.to(D), K=K, dil=d, pad=pad, pre=(a.to(D).contiguous(), b.to(D).contiguous()),
                       pre_act=ACT_SNAKE, alpha=alpha.to(D), res=res.to(D), want_stats=True, wtc=ops.conv_tc_weight_layout(wd, mode),
                       tc_max_ctas=max_ctas)
    torch.cuda.synchronize()
    r = maxdiff(y, ref) / float(ref.abs().max())
    record("conv1d_tc", cfg=str(cfg), mode=mode, rel_err=r)
    assert r < TOL[mode], r
    gb = torch.zeros(B, 2 * Cout, device=D)
    ca, cb = ops.adain_coef(st, gb)
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4 and maxdiff(cb, -ref.mean(-1) * ea) < 1e-3


def test_conv1d_tc_channel_slice_view_input():
    """x is a channel slice of a wider buffer starting at an odd element offset (the decoder's cat buffers): the
    aligned-window copies must neither read the neighbouring channels' data into the result nor misplace rows."""
    from styletts2_b200 import ops
    from styletts2_b200.lib import ACT_LRELU
    B, Cw, Cin, Cout, K, L = 2, 70, 64, 128, 3, 777
    full = rnd(B, Cw, L, seed=1)
    x = full[:, 3:3 + Cin]
    w, bias = rnd(Cout, Cin, K, seed=2, scale=1 / math.sqrt(Cin * K)), rnd(Cout, seed=3)
    ref = F.conv1d(F.leaky_relu(x, 0.2).double(), w.double(), bias.double(), 1, 1).float()
    wd = w.to(D)
    fd = full.to(D)
    for mode in (0, 1):
        y, _ = ops.conv1d(fd[:, 3:3 + Cin], ops.conv_weight_layout(wd), bias.to(D), K=K, pad=1, pre_act=ACT_LRELU, slope=0.2,
                          wtc=ops.conv_tc_weight_layout(wd, mode))
        r = maxdiff(y, ref) / float(ref.abs().max())
        assert r < TOL[mode], (mode, r)


def test_conv1d_tc_mrf_accumulate_matches_simt():
    from styletts2_b200 import ops
    B, C, K, L = 2, 128, 3, 1500
    x = rnd(B, C, L, seed=1)
    ws = [rnd(C, C, K, seed=10 + i, scale=0.1) for i in range(3)]
    ref = (F.conv1d(x, ws[0], None, 1, 1) + F.conv1d(x, ws[1], None, 1, 1) + F.conv1d(x, ws[2], None, 1, 1)) / 3
    acc = torch.empty(B, C, L, device=D)
    for i in range(3):
        wd = ws[i].to(D)
        ops.conv1d(x.to(D), ops.conv_weight_layout(wd), None, K=K, pad=1, out=acc, accum_mode=0 if i == 0 else (2 if i == 2 else 1),
                   accum_div=3.0, wtc=ops.conv_tc_weight_layout(wd))
    assert maxdiff(acc, ref) / float(ref.abs().max()) < 1e-4


CONVT_TC = [  # Cin, Cout, K, S, P, OP, L, reflect
    (256, 128, 12, 6, 3, 0, 700, True),
    (512, 256, 20, 10, 5, 0, 300, False),
    (128, 64, 6, 3, 2, 1, 1000, False),
    (64, 32, 4, 2, 1, 0, 2000, False),
]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("cfg", CONVT_TC)
def test_conv_transpose1d_tc_matches_fp32(cfg, mode):
    from styletts2_b200 import ops
    from styletts2_b200.lib import ACT_LRELU
    Cin, Cout, K, S, P, OP, L, reflect = cfg
    x, w, b = rnd(2, Cin, L, seed=1), rnd(Cin, Cout, K, seed=2, scale=1 / math.sqrt(Cin * 2)), rnd(Cout, seed=3)
    ref = F.conv_transpose1d(F.leaky_relu(x, 0.1), w, b, stride=S, padding=P, output_padding=OP)
    if reflect:
        ref = F.pad(ref, (1, 0), mode="reflect")
    res = rnd(2, Cout, ref.shape[-1], seed=4)
    ref = ref + res
    wd = w.to(D)
    y, st = ops.conv_transpose1d(x.to(D), ops.convT_weight_layout(wd, S, P), b.to(D), K=K, stride=S, padding=P, pre_act=ACT_LRELU,
                                 slope=0.1, res=res.to(D), reflect_left1=reflect, want_stats=True,
                                 wtc=ops.convT_tc_weight_layout(wd, S, P, mode))
    assert y.shape == ref.shape
    r = maxdiff(y, ref) / float(ref.abs().max())
    record("convT_tc", cfg=str(cfg), mode=mode, rel_err=r)
    assert r < 2 * TOL[mode], r
    ca, cb = ops.adain_coef(st, torch.zeros(2, 2 * Cout, device=D))
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4 and maxdiff(cb, -ref.mean(-1) * ea) < 1e-3


@pytest.mark.parametrize("shape", [(300, 1024, 512), (4096, 1024, 2048), (1000, 257, 1024), (260, 2048, 1024), (512, 512, 50)])
def test_linear_tc_fp32_accurate(shape):
    """fp16 two-plane split (low plane pre-scaled by 2^11), 3 MMAs: must be at fp32 accuracy (duration boundary
    downstream): 2e-6 relative to the output peak, like the fp32 SIMT GEMM."""
    from styletts2_b200 import ops
    from styletts2_b200.lib import ACT_GELU
    M, K, Nf = shape
    A, W, b, R = rnd(M, K, seed=1), rnd(Nf, K, seed=2, scale=1 / math.sqrt(K)), rnd(Nf, seed=3), rnd(M, Nf, seed=4)
    ref = (F.gelu(F.linear(A.double(), W.double(), b.double())) + R.double()).float()
    Wd = W.to(D)
    y = ops.linear(A.to(D), Wd, b.to(D), act=ACT_GELU, R=R.to(D), wtc=ops.linear_tc_weight_layout(Wd))
    y32 = ops.linear(A.to(D), Wd, b.to(D), act=ACT_GELU, R=R.to(D))
    ops.LINEAR_TC_PRESPLIT = False           # on-the-fly splitting inside the GEMM must give the same bits
    try:
        y_fly = ops.linear(A.to(D), Wd, b.to(D), act=ACT_GELU, R=R.to(D), wtc=ops.linear_tc_weight_layout(Wd))
    finally:
        ops.LINEAR_TC_PRESPLIT = True
    assert torch.equal(y, y_fly)
    e_tc = maxdiff(y, ref) / float(ref.abs().max())
    e_32 = maxdiff(y32, ref) / float(ref.abs().max())
    record("linear_tc", shape=str(shape), rel_err_tc=e_tc, rel_err_fp32_simt=e_32)
    assert e_tc < 2.5e-6, (e_tc, e_32)       # measured 3e-7 .. 2.1e-6 (K=2048); the fp32 SIMT GEMM: 4e-7 .. 1e-6


def test_linear_tc_wide_dynamic_range():
    """Operand magnitudes spread over 1e-4 .. 1e2 (per input feature) and 1e-3 .. 1 (weights): the scaled low plane must
    keep every product at ~2^-22 relative accuracy, so the error of each output stays within a small multiple of
    eps_fp32 * sum_k |a_k w_k| (the bound an fp32 dot product itself obeys)."""
    from styletts2_b200 import ops
    M, K, Nf = 512, 768, 384
    g = torch.Generator().manual_seed(9)
    A = torch.randn(M, K, generator=g) * (10.0 ** (torch.rand(1, K, generator=g) * 6 - 4))
    W = torch.randn(Nf, K, generator=g) * (10.0 ** (torch.rand(Nf, 1, generator=g) * 3 - 3))
    ref = F.linear(A.double(), W.double())
    bound = F.linear(A.abs().double(), W.abs().double())          # sum_k |a_k||w_k|
    Wd = W.to(D)
    y = ops.linear(A.to(D), Wd, None, wtc=ops.linear_tc_weight_layout(Wd)).cpu().double()
    y32 = ops.linear(A.to(D), Wd, None).cpu().double()
    e_tc = float(((y - ref).abs() / bound).max())
    e_32 = float(((y32 - ref).abs() / bound).max())
    record("linear_tc_dynamic_range", err_over_sum_abs_tc=e_tc, err_over_sum_abs_fp32_simt=e_32)
    assert e_tc < 1.5e-6, (e_tc, e_32)       # fp32 SIMT lands at ~1e-7..1e-6 on the same data


def test_linear_tc_range_guard_reports_fp16_plane_overflow():
    """|x| >= 65504 cannot be held by the fp16 planes: the GEMM output turns inf/NaN (loud) AND the library's range flag is
    raised, which ops.check_range() turns into an exception (Synthesizer.synthesize checks it after every non-graph pass)."""
    from styletts2_b200 import ops
    M, K, Nf = 300, 256, 128
    A, W = rnd(M, K, seed=1), rnd(Nf, K, seed=2, scale=1 / math.sqrt(K))
    Wd = W.to(D)
    wtc = ops.linear_tc_weight_layout(Wd)
    ops.check_range()                                   # clean so far (also clears)
    ops.linear(A.to(D), Wd, None, wtc=wtc)
    ops.check_range()
    A[7, 3] = 1.0e5
    y = ops.linear(A.to(D), Wd, None, wtc=wtc)
    assert not torch.isfinite(y[7]).all()
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()                                   # the fetch cleared the flag


@pytest.mark.parametrize("cin,cout,k,s,L", [(22, 256, 12, 6, 6001), (1, 128, 60, 30, 45030), (22, 64, 12, 6, 6005)])
def test_strided_noise_conv_polyphase_route_matches_fp32(cin, cout, k, s, L):
    """noise_convs of the generators (kernel 2*stride): the polyphase rewrite onto the tensor-core kernel == F.conv1d."""
    from styletts2_b200 import ops
    from styletts2_b200.modules import Conv1d
    m = Conv1d(cin, cout, k, stride=s, padding=(s + 1) // 2).to(D)
    x = rnd(2, cin, L, seed=1)
    ref = F.conv1d(x.double(), m.weight.detach().cpu().double(), m.bias.detach().cpu().double(), stride=s, padding=(s + 1) // 2).float()
    ops.PROFILE = []
    try:
        y, st = m.run(x.to(D), want_stats=True)
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert y.shape == ref.shape
    assert any(n.startswith("polyphase_gather") for n in names) and any(n.startswith("conv1d_tc") for n in names), names
    r = maxdiff(y, ref) / float(ref.abs().max())
    assert r < TOL[0], r
    ca, cb = ops.adain_coef(st, torch.zeros(2, 2 * cout, device=D))
    ea = 1 / torch.sqrt(ref.var(-1, unbiased=False) + 1e-5)
    assert maxdiff(ca, ea) / float(ea.abs().max()) < 1e-4
