"""GPU tier: the 128-frame tiles of the tensor-core convs (csrc/conv_tc.cu) at their edges.

A tile covers 128 frames, but the InstanceNorm statistics stay one (count, mean, M2) partial per 64 frames: each 64-frame
half of a tile writes partial 2 tq + half, and a half with no valid frame writes nothing.  Both kernels -- time-major at
every N (Cout 16 / 32 / 64 / 96 / 128) and channel-major with each recipe -- run at every row length class Lq mod 128
that moves the tile edges, on one tile, and on a persistent loop of 3 CTAs.  Outputs are checked per element against the
recipe-exact reference (oracle/tc_recipes.py), every partial against float64 statistics of its 64-frame slice, and the
statistics buffer carries a NaN-filled guard channel after the last real one: a partial written past ceil(Lq / 64) or
never written shows up there or as a NaN."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import styletts2_oracle as O
import tc_recipes as R

D = "cuda:0"

# (name, recipe, Cout, time-major)
KERNELS = [(f"tct nc{c}", R.FAST, c, True) for c in (16, 32, 64, 96, 128)] + [
    ("tc fast", R.FAST, 128, False), ("tc accurate", R.ACCURATE, 128, False), ("tc f16x3", R.F16X3, 96, False)]
# (B, Cin, K, dil, L, max_ctas): L mod 128 in {0, 1, 63, 64, 65, 127}, one partial tile, a persistent loop on 3 CTAs
SHAPES = [
    (2, 32, 3, 1, 512, 0),
    (2, 32, 3, 1, 385, 0),
    (1, 48, 7, 1, 319, 0),
    (2, 32, 3, 1, 320, 0),
    (1, 32, 11, 5, 321, 0),
    (2, 32, 3, 1, 383, 0),
    (2, 32, 3, 1, 40, 0),
    (3, 64, 7, 3, 1001, 3),
]


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _run(ops, x, w, pre, mode, tmajor, K, dil, pad, max_ctas):
    """st2_conv1d_tc into a statistics buffer [B, Cout, nparts, 3] followed by one NaN-filled guard channel"""
    from styletts2_b200 import lib as L
    from styletts2_b200.lib import ACT_LRELU, TC_TMAJOR
    B, Cin, Lin = x.shape
    Cout = w.shape[0]
    Lq = Lin + 2 * pad - dil * (K - 1)
    nparts = ops.tc_stats_parts(Lq)
    wd = w.to(D)
    wtc = ops.conv_tc_weight_layout(wd, mode)
    assert bool(wtc.mode & TC_TMAJOR) == tmajor, wtc.mode
    y = torch.empty(B, Cout, Lq, device=D)
    stats = torch.full((B * Cout + 1, nparts, 3), float("nan"), device=D)
    a = L.ConvArgs()
    ops._fill_conv_args(a, x.to(D).contiguous(), ops.conv_weight_layout(wd), None, y, K=K, stride=1, dil=dil, pad=pad, Lq=Lq, y_len=Lq,
                        pre=(pre[0].to(D).contiguous(), pre[1].to(D).contiguous()), pre_act=ACT_LRELU, slope=0.2, alpha=None, res=None,
                        res_shift=0, out_div=1.0, accum_mode=0, accum_div=1.0, out_act=0, stats=stats, nparts=nparts)
    L.call("st2_conv1d_tc", C.byref(a), L.ptr(wtc.buf), wtc.mode, max_ctas, L.stream_ptr())
    torch.cuda.synchronize()
    ops.check_range()
    return y.cpu().double(), stats.cpu().double()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
def test_conv_tc_tile_edges(kernel, shape):
    from styletts2_b200 import ops
    _, mode, Cout, tmajor = kernel
    B, Cin, K, dil, L, max_ctas = shape
    x, w = rnd(B, Cin, L, seed=1), rnd(Cout, Cin, K, seed=2, scale=1 / math.sqrt(Cin * K))
    a, b = 1 + 0.3 * rnd(B, Cin, seed=4), 0.2 * rnd(B, Cin, seed=5)
    pad = O.get_padding(K, dil)
    saved = ops.TC_TMAJOR_MAX_COUT
    ops.TC_TMAJOR_MAX_COUT = 128 if tmajor else 0
    try:
        y, stats = _run(ops, x, w, (a, b), mode, tmajor, K, dil, pad, max_ctas)
    finally:
        ops.TC_TMAJOR_MAX_COUT = saved
    what = f"{kernel[0]} {shape}"

    # outputs: per element against the recipe-exact reference
    z = R.prologue(x, a, b, "lrelu", 0.2)
    ref = R.conv1d(z, w, mode, padding=pad, dilation=dil)
    scale = R.sum_abs(F.conv1d, z, w, padding=pad, dilation=dil)
    e = float(((y - ref).abs() / (scale * 2.0 ** -20)).max())
    assert math.isfinite(e) and e <= R.KERNEL_BOUND_C[mode], (what, e)

    # statistics: exactly ceil(Lq / 64) partials per row, each the float64 (count, mean, M2) of its 64-frame slice
    Lq = y.shape[-1]
    nparts = (Lq + 63) // 64
    assert stats.shape[1] == nparts
    assert torch.isnan(stats[B * Cout]).all(), (what, "a partial was written past the last one of the last row")
    real = stats[: B * Cout].view(B, Cout, nparts, 3)
    assert torch.isfinite(real).all(), (what, "partials not written", torch.nonzero(~torch.isfinite(real[..., 0]))[:8].tolist())
    for p in range(nparts):
        sl = y[:, :, 64 * p: 64 * (p + 1)]
        n = sl.shape[-1]
        mean = sl.mean(-1)
        m2 = ((sl - mean[..., None]) ** 2).sum(-1)
        peak = sl.abs().amax(-1)
        assert (real[:, :, p, 0] == n).all(), (what, p, real[:, :, p, 0].unique().tolist(), n)
        assert ((real[:, :, p, 1] - mean).abs() <= 1e-5 * peak + 1e-30).all(), (what, p, "mean")
        assert ((real[:, :, p, 2] - m2).abs() <= 1e-4 * m2 + 1e-6 * n * peak ** 2).all(), (what, p, "M2")
