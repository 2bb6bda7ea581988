"""Precision recipes of the tensor-core conv, EMULATED on the CPU oracle before any kernel was written (decision record):
every convolution / transposed convolution of the decoder that runs on the tensor-core kernel (stride 1, >= 16 channels) is
replaced by the arithmetic of a recipe; the waveform is compared with the exact fp32 oracle on the two decoder cases of
oracle/cases.py.  The shipped recipes (FAST, ACCURATE, F16X3) come from oracle/tc_recipes.py, the recipe-exact reference of
the kernel's operand rounding (float64 plane products); the rejected ones are plain fp32 emulations.
    python tools/emulate_precision.py        (CPU, a few minutes)"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import cases  # noqa: E402
import styletts2_oracle as O  # noqa: E402
import tc_recipes as R  # noqa: E402
from util import oracle_sds  # noqa: E402

oc, oct_ = F.conv1d, F.conv_transpose1d
SHIPPED = {"FAST": R.FAST, "ACCURATE": R.ACCURATE, "F16X3": R.F16X3}


def split16(t):
    hi = t.half().float()
    return hi, t - hi


def recipe_conv(fn, x, w, kw, mode):
    if mode == "tf32_like_fp16_both":           # one 16-bit pass
        return fn(x.half().float(), w.half().float(), None, **kw)
    if mode == "fp16_weights_x_two_planes":     # 2 MMAs: h(w) * (h(x) + l(x))
        xh, xl = split16(x)
        return fn(xh + xl.half().float(), w.half().float(), None, **kw)
    if mode == "bf16_hi_lo_x3":                 # round 1
        xb = x.bfloat16().float(); xl = (x - xb).bfloat16().float(); wb = w.bfloat16().float(); wl = (w - wb).bfloat16().float()
        return fn(xb, wb, None, **kw) + fn(xl, wb, None, **kw) + fn(xb, wl, None, **kw)
    if mode in SHIPPED:                         # the kernel's recipes, operand rounding reproduced exactly
        return R.recipe_conv(fn, x, w, SHIPPED[mode], **kw).to(x.dtype)
    raise ValueError(mode)


def patched(mode):
    def c1(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
        kw = dict(stride=stride, padding=padding, dilation=dilation, groups=groups)
        if not (groups == 1 and stride == 1 and w.shape[0] >= 16 and w.shape[1] >= 16):
            return oc(x, w, bias, **kw)
        y = recipe_conv(oc, x, w, kw, mode)
        return y if bias is None else y + bias.view(1, -1, 1)

    def ct(x, w, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
        kw = dict(stride=stride, padding=padding, output_padding=output_padding, groups=groups)
        if not (groups == 1 and w.shape[0] >= 16 and w.shape[1] >= 16):
            return oct_(x, w, bias, **kw)
        y = recipe_conv(oct_, x, w, kw, mode)
        return y if bias is None else y + bias.view(1, -1, 1)
    return c1, ct


def run(name, mode):
    case = cases.DECODER_CASES[name]
    mcfg = cases.MODEL_CFGS[case["model"]]
    sd = oracle_sds(case["model"])["decoder"]
    asr, f0, n, s = cases.decoder_inputs(case)
    rng = cases.ReplayRNG(case["seed"])
    L, B = case["T"] * 600, case["B"]
    ri, sn = rng.rand_ini((B, 9)), rng.sine_noise((B, L, 9))
    if mode != "exact":
        F.conv1d, F.conv_transpose1d = patched(mode)
    try:
        with torch.no_grad():
            return O.decoder(asr, f0, n, s, sd, mcfg["decoder"], rand_ini=ri, sine_noise=sn)
    finally:
        F.conv1d, F.conv_transpose1d = oc, oct_


if __name__ == "__main__":
    torch.set_num_threads(8)
    print("# waveform max-abs error of the whole decoder when every tensor-core conv uses the recipe (CPU emulation; fp32 accumulation"
          " for the rejected recipes, float64 for the shipped ones)")
    for name in ("lj_dec", "libri_dec"):
        ref = run(name, "exact")
        for mode in ("tf32_like_fp16_both", "fp16_weights_x_two_planes", "bf16_hi_lo_x3", *SHIPPED):
            o = run(name, mode)
            print(f"{name:10s} {mode:34s} max-abs {float((o - ref).abs().max()):.3e}   (waveform scale {float(ref.abs().max()):.2f})", flush=True)
