"""GPU tier: the epilogue modes of the tensor-core convs (csrc/conv_tc.cu) compose exactly with the plain conv.

Each conv runs twice on the same operands: once plain (bias only) and once with one epilogue mode -- residual, residual read
at half rate (res_shift = 1, the upsampling decoder block), out_div = sqrt(2), MRF accumulation (accum_mode 1 and 2) into a
pre-filled output, or tanh.  The epilogue applies its operations to the plain value in epi_combine's order, so the torch
fp32 epilogue applied to the plain output must reproduce the second run bit for bit (tanh: to a tolerance).  Both kernels run
at every time-major channel count and at two channel-major widths, at every Lq mod 128 that moves the edges of the output
slices.  The output is a view into a larger NaN-filled buffer: frames beyond Lq and the channel after the last one must stay
NaN."""
import ctypes as C
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

D = "cuda:0"

# (name, Cout, time-major)
KERNELS = [(f"tct nc{c}", c, True) for c in (16, 32, 64, 96, 128)] + [("tc c96", 96, False), ("tc c256", 256, False)]
LQS = [256, 257, 191, 193, 255]   # Lq mod 128 in {0, 1, 63, 65, 127}
MODES = ["res", "res_shift", "out_div", "accum1", "accum2", "tanh"]
GUARD = 5                          # NaN frames after Lq in every row of the output buffer


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _run(ops, x, w, bias, Cout, Lq, mode, y_init):
    """st2_conv1d_tc (K = 3, pad 1) into y = buf[:, :Cout, :Lq] of a [B, Cout + 1, Lq + GUARD] buffer (rows Lq + GUARD apart)"""
    from styletts2_b200 import lib as L
    from styletts2_b200.lib import ACT_TANH
    B = x.shape[0]
    buf = torch.full((B, Cout + 1, Lq + GUARD), float("nan"), device=D)
    if y_init is not None:
        buf[:, :Cout, :Lq] = y_init
    y = buf[:, :Cout]
    res, res_shift, out_div, accum_mode, accum_div, out_act = None, 0, 1.0, 0, 1.0, 0
    if mode in ("res", "res_shift"):
        res_shift = 1 if mode == "res_shift" else 0
        res = rnd(B, Cout, (Lq + res_shift) >> res_shift, seed=7).to(D)
    elif mode == "out_div":
        out_div = math.sqrt(2.0)
    elif mode in ("accum1", "accum2"):
        accum_mode, accum_div = (1, 1.0) if mode == "accum1" else (2, 3.0)
    elif mode == "tanh":
        out_act = ACT_TANH
    wtc = ops.conv_tc_weight_layout(w, L.TC_FAST)
    a = L.ConvArgs()
    ops._fill_conv_args(a, x, ops.conv_weight_layout(w), bias, y, K=3, stride=1, dil=1, pad=1, Lq=Lq, y_len=Lq + GUARD, pre=None,
                        pre_act=0, slope=0.0, alpha=None, res=res, res_shift=res_shift, out_div=out_div, accum_mode=accum_mode,
                        accum_div=accum_div, out_act=out_act, stats=None, nparts=0)
    L.call("st2_conv1d_tc", C.byref(a), L.ptr(wtc.buf), wtc.mode, 0, L.stream_ptr())
    torch.cuda.synchronize()
    ops.check_range()
    return buf.cpu(), (res.cpu() if res is not None else None), out_div, accum_div


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Lq", LQS)
@pytest.mark.parametrize("kernel", KERNELS, ids=[k[0] for k in KERNELS])
def test_epilogue_composes_with_plain_conv(kernel, Lq, mode):
    from styletts2_b200 import ops
    name, Cout, tmajor = kernel
    B, Cin = 2, 32
    x = rnd(B, Cin, Lq, seed=1).to(D)
    w = rnd(Cout, Cin, 3, seed=2, scale=1 / math.sqrt(Cin * 3)).to(D)
    bias = (0.1 * rnd(Cout, seed=3)).to(D)
    y_init = rnd(B, Cout, Lq, seed=5).to(D) if mode.startswith("accum") else None
    saved = ops.TC_TMAJOR_MAX_COUT
    ops.TC_TMAJOR_MAX_COUT = 128 if tmajor else 0
    try:
        plain_buf = _run(ops, x, w, bias, Cout, Lq, None, None)[0]
        buf, res, out_div, accum_div = _run(ops, x, w, bias, Cout, Lq, mode, y_init)
    finally:
        ops.TC_TMAJOR_MAX_COUT = saved
    what = f"{name} Lq {Lq} {mode}"
    for b_ in (plain_buf, buf):
        assert torch.isnan(b_[:, Cout]).all(), (what, "the channel after Cout was written")
        assert torch.isnan(b_[:, :Cout, Lq:]).all(), (what, "a frame beyond Lq was written")
    p = plain_buf[:, :Cout, :Lq]
    got = buf[:, :Cout, :Lq]
    assert torch.isfinite(p).all(), (what, "plain output not written everywhere")
    if mode == "res":
        want = p + res
    elif mode == "res_shift":
        want = p + res.repeat_interleave(2, dim=-1)[..., :Lq]
    elif mode == "out_div":
        want = p / torch.tensor(out_div, dtype=torch.float32)
    elif mode == "accum1":
        want = y_init.cpu() + p
    elif mode == "accum2":
        want = (y_init.cpu() + p) / torch.tensor(accum_div, dtype=torch.float32)
    else:
        want = torch.tanh(p)
        assert ((got - want).abs() <= 2e-6 * (1 + want.abs())).all(), (what, float((got - want).abs().max()))
        return
    assert torch.equal(got, want), (what, int((got != want).sum()), float((got - want).abs().max()))
