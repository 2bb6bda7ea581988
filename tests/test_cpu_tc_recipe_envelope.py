"""CPU tier: the precision envelope of the tensor-core conv recipes, from the recipe-exact reference (oracle/tc_recipes.py),
and the power of the GPU test that compares the kernel with that reference (tests/test_gpu_conv_tc_recipe.py).

Operands are scaled z' = 64 z, w' = 4096 w.  FAST's e4m3 correction operands saturate at 448: l(z') 2^8 from |z| = 64 on,
h(z') 2^-4 above |z| = 112.  Past that the correction is clipped and FAST falls towards single-fp16 accuracy; ACCURATE
(fp16 low planes) keeps ~1e-7 up to the fp16 range."""
import math

import pytest
import torch
import torch.nn.functional as F

import tc_recipes as R

FAST_TOL = 6e-5          # the fp64 tolerance of the FAST kernel tests (test_gpu_conv_tc.py TOL[0])


def _rel(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


def _shortcut_case(peak, whole=False, ci=514, co=256, T=512, seed=0):
    """the decoder's encode.conv1x1 shape (514 -> 256 here, K = 1); channel 512 (where F0_conv's output sits) peaks at
    `peak`, or the whole tensor is scaled to that peak"""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(1, ci, T, generator=g, dtype=torch.float64)
    if whole:
        z = z / z.abs().max() * peak
    else:
        z[0, 512] = peak * (0.5 + 0.5 * torch.rand(T, generator=g, dtype=torch.float64))
    w = (torch.rand(co, ci, 1, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(ci)
    return z.float(), w.float()


def _err(z, w, mode):
    return _rel(R.conv1d(z, w, mode), F.conv1d(z.double(), w.double()))


def test_e4m3_conversion_saturates_like_satfinite():
    """clamp-then-cast == __nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3) (values from the CUDA 12.9 host conversion)"""
    v = torch.tensor([447.0, 449.0, 464.0, 1000.0, -1000.0, 232.0, 2.0 ** -10, 3 * 2.0 ** -10])
    want = [448.0, 448.0, 448.0, 448.0, -448.0, 224.0, 0.0, 2.0 ** -8]        # round-to-nearest-even, subnormal ties too
    assert R.e4m3_satfinite(v).tolist() == want
    assert math.isnan(R.e4m3_satfinite(torch.tensor([float("nan")])).item())


def test_planes_reassemble_the_operands():
    """the planes of every recipe sum back to the scaled operand (to the precision the planes carry)"""
    g = torch.Generator().manual_seed(1)
    z = torch.randn(2, 32, 40, generator=g) * 3
    w = torch.randn(16, 32, 3, generator=g) * 0.05
    hz, lz = R.act_planes(z, R.ACCURATE)[:2]
    hw, _, lw = R.weight_planes(w, R.ACCURATE)
    assert float((hz + lz / 256 - z.double() * 64).abs().max()) <= float((z.double() * 64).abs().max()) * 2.0 ** -21
    assert float((hw + lw / 256 - w.double() * 4096).abs().max()) <= float((w.double() * 4096).abs().max()) * 2.0 ** -21
    fz = R.act_planes(z, R.FAST)
    assert torch.equal(fz[1], (fz[0] / 16).float().to(torch.float8_e4m3fn).double())   # |h(z')/16| < 448 here


@pytest.mark.parametrize("peak", [1, 16, 32, 64])
def test_fast_inside_envelope(peak):
    for whole in (False, True):
        e = _err(*_shortcut_case(peak, whole), R.FAST)
        assert e < FAST_TOL, (peak, whole, e)


@pytest.mark.parametrize("peak", [150, 225, 450, 900])
def test_fast_degrades_beyond_envelope(peak):
    """one channel past the e4m3 range: the correction of that channel is clipped, the error grows towards a single fp16
    pass (~5e-4) -- the decoder's shortcut convs must not run FAST on raw F0-scale input"""
    e = _err(*_shortcut_case(peak), R.FAST)
    assert 1.5e-4 < e < 1e-3, (peak, e)


@pytest.mark.parametrize("peak", [1, 64, 150, 300, 1000])
def test_accurate_and_f16x3_hold_to_the_fp16_range(peak):
    for whole in (False, True):
        for mode in (R.ACCURATE, R.F16X3):
            e = _err(*_shortcut_case(peak, whole), mode)
            assert e < 1e-6, (peak, whole, mode, e)


def test_fast_weight_magnitude_edge():
    """max |w| below ~1e-4 pushes FAST's e4m3 weight corrections subnormal (1.4e-4 at 1.3e-4); from ~1e-3 on it is exact"""
    z, w = _shortcut_case(1)
    errs = {s: _err(z, w / w.abs().max() * s, R.FAST) for s in (1.3e-4, 1e-3, 1.0, 8.0)}
    assert errs[1.3e-4] > FAST_TOL, errs
    assert all(errs[s] < FAST_TOL for s in (1e-3, 1.0, 8.0)), errs


def _fp32_accumulated(z, w, mode, pad, dil, zp=None, wp=None):
    """the recipe's plane products of one (16-channel block, tap) step at a time, summed in fp32 in the kernel's order:
    a stand-in for an honest kernel, whose only deviation from the float64 reference is its fp32 accumulation"""
    zp = R.act_planes(z, mode) if zp is None else zp
    wp = R.weight_planes(w, mode) if wp is None else wp
    B, Cin, L = z.shape
    K = w.shape[-1]
    Lo = L + 2 * pad - dil * (K - 1)
    y = torch.zeros(B, w.shape[0], Lo)
    for c0 in range(0, Cin, 16):
        for t in range(K):
            part = R.recipe_conv(F.conv1d, None, None, mode, zp=[p[:, c0:c0 + 16] for p in zp], wp=[p[:, c0:c0 + 16, t:t + 1] for p in wp])
            sh = t * dil - pad
            lo, hi = max(0, -sh), min(Lo, L - sh)
            step = torch.zeros_like(y)
            step[..., lo:hi] = part[..., lo + sh:hi + sh].float()
            y = y + step
    return y.double()


@pytest.mark.parametrize("Cin", [256, 512])
def test_gpu_bound_catches_a_lost_correction(Cin):
    """The GPU test's metric max |y - y_ref| / (2^-20 sum |w||z|) must reject a kernel that loses FAST's e4m3 correction on
    ONE tap of the last 16-channel block (a stager / weight-layout / descriptor bug of a tail block) by at least 10x its
    calibrated bound, while an fp32-accumulating kernel of the exact recipe passes it."""
    B, Cout, K, L = 2, 256, 3, 300
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / math.sqrt(Cin * K)
    a, b = 1 + 0.3 * torch.randn(B, Cin, generator=g), 0.2 * torch.randn(B, Cin, generator=g)
    z = R.prologue(x, a, b, "lrelu", 0.2)
    ref = R.conv1d(z, w, R.FAST, padding=1)
    scale = R.sum_abs(F.conv1d, z, w, padding=1) * 2.0 ** -20
    c = R.KERNEL_BOUND_C[R.FAST]
    honest = float(((_fp32_accumulated(z, w, R.FAST, 1, 1) - ref).abs() / scale).max())
    assert honest < c, (honest, c)
    wp = R.weight_planes(w, R.FAST)
    for tap in range(K):
        lost = [p.clone() for p in wp]
        for p in lost[1:]:
            p[:, Cin - 16:, tap] = 0
        y = R.recipe_conv(F.conv1d, z, w, R.FAST, wp=lost, padding=1)
        m = float(((y - ref).abs() / scale).max())
        assert m > 10 * c, (tap, m, c)
