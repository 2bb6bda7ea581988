"""Recipe-exact CPU reference of the tensor-core conv (styletts2_b200/csrc/conv_tc.cu).

Each precision recipe splits the two operands into planes with a fixed rounding -- power-of-two scales, fp16
round-to-nearest high planes, fp16 or e4m3 correction planes -- and multiplies plane pairs on the tensor core, which forms
every product exactly.  This module reproduces those planes bit for bit and convolves each plane pair in float64, so the
only thing it leaves out is the kernel's own fp32 accumulation.  A kernel that stages, lays out or folds a plane wrongly
differs from it by far more than that accumulation error (tests/test_cpu_tc_recipe_envelope.py, test_gpu_conv_tc_recipe.py).

    z   the fp32 activation operand after the prologue (AdaIN affine + activation; `prologue` computes it as the stagers do)
    w   the fp32 (folded) weight: [Cout, Cin, K] for conv1d, [Cin, Cout, K] for conv_transpose1d

Operands are scaled w' = w * 2^12, z' = z * 2^6 and the sum is scaled back by 2^-18 (conv_tc.cu W_SCALE / X_SCALE), with
h(.) = fp16(.) and l(.) = (.) - h(.) (exact in fp32):
    FAST      h(w') h(z')  +  e4m3(l(w') 2^4) e4m3(h(z') 2^-4)  +  e4m3(h(w') 2^-8) e4m3(l(z') 2^8)
    ACCURATE  h(w') h(z')  +  [h(w') fp16(l(z') 2^8)  +  fp16(l(w') 2^8) h(z')] 2^-8
    F16X3     h(w') h(z')  +   h(w') fp16(l(z'))      +  fp16(l(w')) h(z')
The e4m3 conversions saturate to +-448 (__NV_SATFINITE); torch's own e4m3 cast returns NaN from 464 on, so values are
clamped first.
"""
import torch
import torch.nn.functional as F

FAST, ACCURATE, F16X3 = 0, 1, 2          # include/styletts2_b200.h ST2_TC_*
RECIPES = {FAST: "FAST", ACCURATE: "ACCURATE", F16X3: "F16X3"}

W_SCALE, X_SCALE = 4096.0, 64.0
D_UNSCALE = 1.0 / (W_SCALE * X_SCALE)
ACC_LO_SCALE = 256.0
F8_WLO, F8_WHI, F8_XHI, F8_XLO = 16.0, 1.0 / 256.0, 1.0 / 16.0, 256.0
E4M3_MAX = 448.0
FP16_MAX = 65504.0

# Accumulation bound of the kernels: |y_kernel - y_ref| <= c * 2^-20 * sum|w||z| per output element, y_ref from this module.
# Measured on one H100 80GB HBM3 over tests/test_gpu_conv_tc_recipe.py: max 0.78 for FAST (both kernels) and ACCURATE, 2.08
# for F16X3 (its small plane products are added into the large running sum).  A FAST kernel that loses the e4m3 correction
# on one tap of one 16-channel block scores >= 16 (tests/test_cpu_tc_recipe_envelope.py).
KERNEL_BOUND_C = {FAST: 1.0, ACCURATE: 1.0, F16X3: 2.5}

# the functional convolutions as imported (tools that patch F.conv1d for an emulation still reach the real ones here)
_conv1d, _conv_transpose1d = F.conv1d, F.conv_transpose1d


def e4m3_satfinite(v: torch.Tensor) -> torch.Tensor:
    """fp32/fp16 -> e4m3 with round-to-nearest-even and saturation to +-448 (NaN stays NaN), returned as float64."""
    return v.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).double()


def _split(v: torch.Tensor, scale: float):
    """fp32 v * scale (exact) -> (fp16 high plane, fp32 remainder)"""
    vs = v.float() * scale
    h = vs.half()
    return h, vs - h.float()


def act_planes(z: torch.Tensor, mode: int):
    """activation operand planes of a recipe, as float64 tensors in the order weight_planes pairs them with"""
    h, l = _split(z, X_SCALE)
    hd = h.double()
    if mode == FAST:
        return [hd, e4m3_satfinite(h * F8_XHI), e4m3_satfinite(l * F8_XLO)]     # h(z')/16 is formed in fp16 (__hmul2)
    ls = ACC_LO_SCALE if mode == ACCURATE else 1.0
    return [hd, (l * ls).half().double(), hd]


def weight_planes(w: torch.Tensor, mode: int):
    h, l = _split(w, W_SCALE)
    hd = h.double()
    if mode == FAST:
        return [hd, e4m3_satfinite(l * F8_WLO), e4m3_satfinite(hd.float() * F8_WHI)]
    ls = ACC_LO_SCALE if mode == ACCURATE else 1.0
    return [hd, hd, (l * ls).half().double()]


def plane_scales(mode: int):
    """factor applied to each plane product before the sum (the 2^-18 unscale and ACCURATE's 2^-8 fold)"""
    lo = D_UNSCALE / ACC_LO_SCALE if mode == ACCURATE else D_UNSCALE
    return [D_UNSCALE, lo, lo]


def recipe_conv(fn, z, w, mode: int, zp=None, wp=None, **kw) -> torch.Tensor:
    """sum over the recipe's plane products of fn(z plane, w plane, None, **kw) in float64.
    zp / wp: precomputed (possibly edited) plane lists, e.g. to model a kernel that drops a correction term."""
    zp = act_planes(z, mode) if zp is None else zp
    wp = weight_planes(w, mode) if wp is None else wp
    return sum(s * fn(a, b, None, **kw) for a, b, s in zip(zp, wp, plane_scales(mode)))


def conv1d(z, w, mode: int, *, bias=None, padding=0, dilation=1, **kw) -> torch.Tensor:
    y = recipe_conv(_conv1d, z, w, mode, padding=padding, dilation=dilation, **kw)
    return y if bias is None else y + bias.double().view(1, -1, 1)


def conv_transpose1d(z, w, mode: int, *, stride, padding=0, output_padding=0, bias=None, **kw) -> torch.Tensor:
    y = recipe_conv(_conv_transpose1d, z, w, mode, stride=stride, padding=padding, output_padding=output_padding, **kw)
    return y if bias is None else y + bias.double().view(1, -1, 1)


def sum_abs(fn, z, w, **kw) -> torch.Tensor:
    """sum |w||z| of every output element (the scale of the accumulation error an fp32 dot product may make)"""
    return fn(z.double().abs(), w.double().abs(), None, **kw)


def prologue(x, a=None, b=None, act: str = "none", slope: float = 0.0) -> torch.Tensor:
    """fp32 z = act(a*x + b) as the stagers form it: one fused multiply-add (exact product, one rounding), then LeakyReLU
    in fp32 (the kernel works on 64 z; power-of-two scaling commutes with both roundings).  a, b: [B, C] or None."""
    x = x.float()
    if a is not None:
        z = (x.double() * a.double()[:, :, None] + b.double()[:, :, None]).float()
    else:
        z = x.clone()
    if act == "lrelu":
        z = torch.where(z > 0, z, z * torch.tensor(slope, dtype=torch.float32))
    elif act != "none":
        raise ValueError(act)
    return z
