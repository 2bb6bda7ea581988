"""Tensor-level wrappers over the C ABI (one function per entry point family).

torch is used for device memory (allocation through the caching allocator) and streams only;
every arithmetic op on the path is a kernel of libstyletts2_b200.so.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Optional, Tuple

import torch

from . import lib as L
from .lib import ACT_GELU, ACT_LRELU, ACT_NONE, ACT_SNAKE, ACT_TANH, TC_ACCURATE, TC_FAST, TC_F16X3, TC_TMAJOR, ConvArgs, RowsArgs, ptr, stream_ptr

f32 = torch.float32


def _cl(x: torch.Tensor) -> torch.Tensor:
    """Require conv layout [B,C,L] with contiguous rows (batch stride free)."""
    assert x.dim() == 3 and x.dtype == f32
    if x.stride(2) != 1 or x.stride(1) != x.shape[2]:
        x = x.contiguous()
    return x


def empty(*shape, device, dtype=f32):
    return torch.empty(shape, device=device, dtype=dtype)


# ------------------------------------------------------------------ weight preparation
def fold_weight_norm(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    rows = v.shape[0]
    v2 = v.detach().contiguous().view(rows, -1)
    w = torch.empty_like(v2)
    L.call("st2_weight_norm_fold", ptr(v2), ptr(g.detach().contiguous()), ptr(w), rows, v2.shape[1], stream_ptr())
    return w.view_as(v)


def row_norm(v: torch.Tensor) -> torch.Tensor:
    """||v[r,:]||_2 per leading-dim row with the fold kernel's reduction -> [rows]"""
    rows = v.shape[0]
    v2 = v.detach().contiguous().view(rows, -1)
    out = torch.empty(rows, device=v.device, dtype=f32)
    L.call("st2_row_norm", ptr(v2), ptr(out), rows, v2.shape[1], stream_ptr())
    return out


def conv_weight_layout(w: torch.Tensor) -> torch.Tensor:
    """[Cout,Cin,K] -> [Cin,K,Cout]"""
    w = w.detach().contiguous()
    co, ci, k = w.shape
    wt = empty(ci, k, co, device=w.device)
    L.call("st2_conv_weight_layout", ptr(w), ptr(wt), co, ci, k, stream_ptr())
    return wt


def convT_weight_layout(w: torch.Tensor, stride: int, padding: int) -> torch.Tensor:
    """[Cin,Cout,K] -> [S,Cin,J,Cout]"""
    w = w.detach().contiguous()
    ci, co, k = w.shape
    j = (k + stride - 1) // stride
    wp = empty(stride, ci, j, co, device=w.device)
    L.call("st2_convT_weight_layout", ptr(w), ptr(wp), ci, co, k, stride, padding, stream_ptr())
    return wp


# ------------------------------------------------------------------ conv
def stats_parts(lq: int) -> int:
    return (lq + 255) // 256


def tc_stats_parts(lq: int) -> int:
    """InstanceNorm partials of the tensor-core conv kernels: one per 64-frame tile."""
    return (lq + 63) // 64


def _fill_conv_args(a: ConvArgs, x, wt, bias, y, *, K, stride, dil, pad, Lq, y_len, pre, pre_act, slope, alpha, res,
                    res_shift, out_div, accum_mode, accum_div, out_act, stats, nparts):
    B, Cin, Lin = x.shape
    a.x, a.x_bstride, a.Cin, a.Lin = ptr(x), x.stride(0), Cin, Lin
    a.w, a.bias = ptr(wt), ptr(bias)
    a.y, a.y_bstride, a.Cout, a.Lq, a.y_len = ptr(y), y.stride(0), y.shape[1], Lq, y_len
    a.y_tstride, a.y_toffset = 1, 0
    a.B, a.K, a.stride, a.dil, a.pad = B, K, stride, dil, pad
    if pre is not None:
        a.pre_a, a.pre_b = ptr(pre[0]), ptr(pre[1])
    else:
        a.pre_a, a.pre_b = None, None
    a.pre_act, a.pre_slope, a.pre_alpha = pre_act, slope, ptr(alpha)
    if res is not None:
        assert res.stride(2) == 1 and res.stride(1) == res.shape[2]
        a.res, a.res_bstride, a.res_len, a.res_shift = ptr(res), res.stride(0), res.shape[2], res_shift
    else:
        a.res, a.res_bstride, a.res_len, a.res_shift = None, 0, 0, 0
    a.out_div, a.accum_mode, a.accum_div, a.out_act = out_div, accum_mode, accum_div, out_act
    a.stats, a.stats_nparts, a.stats_part_offset = ptr(stats), nparts, 0
    a.dup_q0_to = -1


PROFILE = None  # bench.py sets this to a list: (name, algorithmic_flops, algorithmic_bytes, ev0, ev1, mma_per_product) per launch
NVTX = os.environ.get("ST2_NVTX", "0") != "0"   # NVTX range per kernel family / stage (nsys / ncu --nvtx)


class _prof:
    """CUDA events around one launch (or launch group) when bench.py profiling is on; NVTX range when ST2_NVTX=1."""
    __slots__ = ("name", "flops", "nbytes", "nmma", "e0")

    def __init__(self, name, flops=0.0, nbytes=0.0, nmma=0):
        self.name, self.flops, self.nbytes, self.nmma, self.e0 = name, flops, nbytes, nmma, None

    def __enter__(self):
        if NVTX:
            torch.cuda.nvtx.range_push(self.name.split(" ")[0])
        if PROFILE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.e0 is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            PROFILE.append((self.name, self.flops, self.nbytes, self.e0, e1, self.nmma))
        if NVTX:
            torch.cuda.nvtx.range_pop()
        return False


USE_TC = os.environ.get("ST2_TC", "1") != "0"   # tensor-core (wgmma) conv path where a wtc buffer is given
TC_MIN_WORK = 1 << 22                            # below this many MACs per utterance the SIMT kernel is used


def conv_tc_supported(Cin, Cout, K, stride, dil) -> bool:
    return bool(L.load().st2_conv_tc_supported(Cin, Cout, K, stride, dil))


class TCWeights:
    """Tensor-core weight blocks of one conv (opaque uint8 buffer) + the precision recipe they were laid out for."""
    __slots__ = ("buf", "mode")

    def __init__(self, buf, mode):
        self.buf, self.mode = buf, int(mode)


TC_MODE_OVERRIDE = os.environ.get("ST2_TC_MODE")   # A/B testing: force one recipe ("0" fast, "1" accurate, "2" f16x3)


# Layers with at most this many output channels run the TIME-MAJOR kernel (frames on the MMA's M axis, Cout on N): HiFi-GAN's
# C = 64 / 32 stages, conv_post, and -- faster there too -- the C = 128 resblock convs.  0 disables; 128 is the kernel's limit.
TC_TMAJOR_MAX_COUT = int(os.environ.get("ST2_TC_TMAJOR_MAX", "128"))


def _tc_mode(mode, cout=None):
    m = int(TC_MODE_OVERRIDE) if TC_MODE_OVERRIDE is not None else int(mode)
    if cout is not None and m == TC_FAST and cout <= min(TC_TMAJOR_MAX_COUT, 128):
        m |= TC_TMAJOR
    return m


def conv_tc_weight_layout(w: torch.Tensor, mode: int = TC_FAST) -> TCWeights:
    """folded fp32 [Cout,Cin,K] -> plane-split stage blocks for st2_conv1d_tc"""
    w = w.detach().contiguous()
    co, ci, k = w.shape
    mode = _tc_mode(mode, co)
    nbytes = int(L.load().st2_conv_tc_weight_bytes(co, ci, k))
    out = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    L.call("st2_conv_tc_weight_layout", ptr(w), ptr(out), co, ci, k, mode, stream_ptr())
    return TCWeights(out, mode)


def conv1d(x, wt, bias=None, *, K, stride=1, dil=1, pad=0, pre=None, pre_act=ACT_NONE, slope=0.0, alpha=None,
           res=None, res_shift=0, out_div=1.0, accum_mode=0, accum_div=1.0, out_act=ACT_NONE, out=None,
           want_stats=False, wtc=None, tc_max_ctas=0) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Fused Conv1d (see include/styletts2_b200.h).  wt is the [Cin,K,Cout] layout.
    wtc: optional tensor-core weight buffer (conv_tc_weight_layout) -> wgmma path when supported.
    Returns (y [B,Cout,Lout], stats [B,Cout,nparts,3] or None)."""
    x = _cl(x)
    B, Cin, Lin = x.shape
    assert wt.shape[0] == Cin and wt.shape[1] == K, (tuple(wt.shape), Cin, K)
    Cout = wt.shape[2]
    Lout = (Lin + 2 * pad - dil * (K - 1) - 1) // stride + 1
    if out is None:
        out = empty(B, Cout, Lout, device=x.device)
    assert out.shape == (B, Cout, Lout) and out.stride(2) == 1 and out.stride(1) == Lout
    use_tc = wtc is not None and USE_TC and stride == 1 and Cin * Cout * K * Lout >= TC_MIN_WORK
    nparts = tc_stats_parts(Lout) if use_tc else stats_parts(Lout)
    stats = empty(B, Cout, nparts, 3, device=x.device) if want_stats else None
    a = ConvArgs()
    _fill_conv_args(a, x, wt, bias, out, K=K, stride=stride, dil=dil, pad=pad, Lq=Lout, y_len=Lout, pre=pre,
                    pre_act=pre_act, slope=slope, alpha=alpha, res=res, res_shift=res_shift, out_div=out_div,
                    accum_mode=accum_mode, accum_div=accum_div, out_act=out_act, stats=stats, nparts=nparts)
    nbytes = 4.0 * B * (Lin * Cin + Lout * Cout * ((2 if res is not None else 1) + (1 if accum_mode else 0)))
    flops = 2.0 * B * Cin * Cout * K * Lout
    if use_tc:
        with _prof(f"conv1d_tc m{wtc.mode} ci{Cin} co{Cout} k{K} d{dil} L{Lout} B{B}", flops, nbytes, 2 if (wtc.mode & 15) == TC_FAST else 3):
            L.call("st2_conv1d_tc", C.byref(a), ptr(wtc.buf), wtc.mode, tc_max_ctas, stream_ptr())
    else:
        with _prof(f"conv1d_simt ci{Cin} co{Cout} k{K} s{stride} L{Lout} B{B}", flops, nbytes):
            L.call("st2_conv1d", C.byref(a), stream_ptr())
    return out, stats


def polyphase_gather(x, S: int, pad: int, Lp: int) -> torch.Tensor:
    """x [B,C,L] -> xp [B, C*S, Lp], xp[b, c*S + r, q] = x[b, c, q*S + r - pad] (zero outside)"""
    x = _cl(x)
    B, Cc, Ln = x.shape
    xp = empty(B, Cc * S, Lp, device=x.device)
    with _prof(f"polyphase_gather c{Cc} L{Ln} s{S} B{B}", 0.0, 4.0 * B * Cc * (Ln + S * Lp)):
        L.call("st2_polyphase_gather", ptr(x), x.stride(0), B, Cc, Ln, S, pad, Lp, ptr(xp), stream_ptr())
    return xp


def convT_tc_weight_layout(w: torch.Tensor, stride: int, padding: int, mode: int = TC_FAST) -> TCWeights:
    """folded fp32 ConvTranspose1d weight [Cin,Cout,K] -> per-phase tensor-core blocks"""
    w = w.detach().contiguous()
    ci, co, k = w.shape
    mode = _tc_mode(mode, co)
    nbytes = int(L.load().st2_convT_tc_weight_bytes(ci, co, k, stride))
    out = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    L.call("st2_convT_tc_weight_layout", ptr(w), ptr(out), ci, co, k, stride, padding, mode, stream_ptr())
    return TCWeights(out, mode)


def conv_transpose1d(x, wp, bias, *, K, stride, padding, pre_act=ACT_NONE, slope=0.0, alpha=None, res=None,
                     reflect_left1=False, want_stats=False, out=None, wtc=None):
    """Polyphase ConvTranspose1d; wp is the [S,Cin,J,Cout] layout; output length Lin*S (+1 if reflect)."""
    x = _cl(x)
    B, Cin, Lin = x.shape
    S = stride
    assert wp.shape[0] == S and wp.shape[1] == Cin
    Cout = wp.shape[3]
    Lout = Lin * S + (1 if reflect_left1 else 0)
    if out is None:
        out = empty(B, Cout, Lout, device=x.device)
    assert out.shape == (B, Cout, Lout) and out.stride(2) == 1 and out.stride(1) == Lout
    use_tc = wtc is not None and USE_TC
    nparts = 1 if use_tc else S * stats_parts(Lin)
    stats = empty(B, Cout, nparts, 3, device=x.device) if want_stats else None
    a = ConvArgs()
    _fill_conv_args(a, x, wp, bias, out, K=1, stride=1, dil=1, pad=0, Lq=Lin, y_len=Lout, pre=None, pre_act=pre_act,
                    slope=slope, alpha=alpha, res=res, res_shift=0, out_div=1.0, accum_mode=0, accum_div=1.0,
                    out_act=ACT_NONE, stats=stats, nparts=nparts)
    J = (K + S - 1) // S
    nbytes = 4.0 * B * (Lin * Cin + Lout * Cout * (2 if res is not None else 1))
    flops = 2.0 * B * Cin * Cout * J * S * Lin
    if use_tc:
        with _prof(f"convT_tc m{wtc.mode} ci{Cin} co{Cout} k{K} s{S} L{Lin} B{B}", flops, nbytes, 2 if (wtc.mode & 15) == TC_FAST else 3):
            tmp = empty(S * B * Cout * Lin, device=x.device)
            L.call("st2_conv_transpose1d_tc2", C.byref(a), ptr(wtc.buf), wtc.mode, K, S, padding, 1 if reflect_left1 else 0, ptr(tmp),
                   stream_ptr())
    else:
        with _prof(f"convT_simt ci{Cin} co{Cout} k{K} s{S} L{Lin} B{B}", flops, nbytes):
            L.call("st2_conv_transpose1d", C.byref(a), ptr(wp), K, S, padding, 1 if reflect_left1 else 0, stream_ptr())
    return out, stats


def instance_stats(x) -> torch.Tensor:
    x = _cl(x)
    B, Cc, Ln = x.shape
    st = empty(B, Cc, 1, 3, device=x.device)
    with _prof(f"instance_stats c{Cc} L{Ln} B{B}", 0.0, 4.0 * B * Cc * Ln):
        L.call("st2_instance_stats", ptr(x), x.stride(0), B, Cc, Ln, ptr(st), stream_ptr())
    return st


def adain_coef(stats, gb, eps=1e-5):
    """stats [B,C,nparts,3]; gb [B,2C] view (row stride free) -> (a,b) each [B,C]."""
    B, Cc, nparts, _ = stats.shape
    assert gb.shape == (B, 2 * Cc) and gb.stride(1) == 1
    a = empty(B, Cc, device=stats.device)
    b = empty(B, Cc, device=stats.device)
    L.call("st2_adain_coef", ptr(stats), nparts, ptr(gb), gb.stride(0), B, Cc, eps, ptr(a), ptr(b), stream_ptr())
    return a, b


def adain_lrelu_pool(x, a, b, pool_w, pool_b, slope=0.2):
    x = _cl(x)
    B, Cc, Ln = x.shape
    y = empty(B, Cc, 2 * Ln, device=x.device)
    with _prof(f"adain_lrelu_pool c{Cc} L{Ln} B{B}", 0.0, 4.0 * B * Cc * Ln * 3):
        L.call("st2_adain_lrelu_pool", ptr(x), x.stride(0), ptr(a), ptr(b), ptr(pool_w), ptr(pool_b), slope, B, Cc, Ln,
               ptr(y), y.stride(0), stream_ptr())
    return y


def channel_layernorm_lrelu(x, gamma, beta, lengths=None, eps=1e-5, slope=0.2):
    x = x.contiguous()
    B, Cc, Ln = x.shape
    y = torch.empty_like(x)
    L.call("st2_channel_layernorm_lrelu", ptr(x), ptr(y), ptr(gamma), ptr(beta), eps, slope, ptr(lengths), B, Cc, Ln,
           stream_ptr())
    return y


# ------------------------------------------------------------------ rows
def _rows_args(*, B, N, Cw, h_in=None, x=None, xs=1.0, emb=None, add=None, h_out=None, g1=None, b1=None, g2=None, b2=None,
               gb_bstride=0, ada=False, out1=None, out2=None, eps=1e-5, lengths=None):
    a = RowsArgs()
    a.h_in, a.h_in_ld = ptr(h_in), (h_in.stride(-2) if h_in is not None else 0)
    a.x, a.Cx, a.xs = ptr(x), (x.shape[-1] if x is not None else 0), xs
    a.emb, a.emb_ld = ptr(emb), (emb.stride(-2) if emb is not None else 0)
    a.add = ptr(add)
    a.h_out, a.h_out_ld = ptr(h_out), (h_out.stride(-2) if h_out is not None else 0)
    a.g1, a.b1, a.g2, a.b2, a.gb_bstride, a.ada = ptr(g1), ptr(b1), ptr(g2), ptr(b2), gb_bstride, 1 if ada else 0
    a.out1, a.out1_ld = ptr(out1), (out1.stride(-2) if out1 is not None else 0)
    a.out2, a.out2_ld = ptr(out2), (out2.stride(-2) if out2 is not None else 0)
    a.B, a.N, a.C, a.eps = B, N, Cw, eps
    a.lengths = ptr(lengths)
    return a


def rows_ln(*, B, N, Cw, **kw):
    L.call("st2_rows_ln", C.byref(_rows_args(B=B, N=N, Cw=Cw, **kw)), stream_ptr())


def rows_ln_packed(*, row_utt, M, B, Cw, **kw):
    """rows_ln over M packed token rows; row_utt (int32 [M]) gives each row's utterance, which selects x, add and the
    per-utterance g/b rows.  No row is masked: a packed buffer holds valid rows only."""
    with _prof(f"rows_ln_packed M{M} C{Cw} B{B}", 0.0, 4.0 * M * Cw * 3):
        L.call("st2_rows_ln_packed", C.byref(_rows_args(B=B, N=1, Cw=Cw, **kw)), ptr(row_utt), M, stream_ptr())


def bcast_cols(dst, col0, src, lengths=None):
    """dst [B,N,ld-view]; dst[:, :, col0:col0+W] = src[b] (masked rows -> 0)"""
    B, N = dst.shape[0], dst.shape[1]
    W = src.shape[1]
    L.call("st2_bcast_cols", ptr(dst), dst.stride(1), col0, ptr(src.contiguous()), B, N, W, ptr(lengths), stream_ptr())


def mean_rows(h, B, N):
    Cw = h.shape[-1]
    out = empty(B, Cw, device=h.device)
    L.call("st2_mean_rows", ptr(h), h.stride(-2), B, N, Cw, ptr(out), stream_ptr())
    return out


def mean_segments(h, offsets, B):
    """out[b] = mean of packed rows offsets[b] .. offsets[b+1]-1 of h (offsets int32 [B+1]), in mean_rows' summation order"""
    Cw = h.shape[-1]
    out = empty(B, Cw, device=h.device)
    with _prof(f"mean_segments M{h.shape[0]} C{Cw} B{B}", 0.0, 4.0 * (h.shape[0] + B) * Cw):
        L.call("st2_mean_segments", ptr(h), h.stride(-2), ptr(offsets), B, Cw, ptr(out), stream_ptr())
    return out


def _rows_view(t):
    """(tensor, rows, ld) for a [..., K] tensor whose rows are uniformly strided (else a contiguous copy)."""
    K = t.shape[-1]
    if t.stride(-1) != 1:
        t = t.contiguous()
    if t.dim() == 1:
        return t, 1, K
    if t.dim() == 2:
        return t, t.shape[0], t.stride(0)
    if t.dim() == 3 and (t.shape[0] == 1 or t.stride(0) == t.shape[1] * t.stride(1)):
        return t, t.shape[0] * t.shape[1], t.stride(1)
    t = t.contiguous()
    return t, t.numel() // K, K


LINEAR_TC_MIN_ROWS = 256
LINEAR_TC_PRESPLIT = os.environ.get("ST2_LINEAR_PRESPLIT", "1") != "0"


def linear_tc_weight_layout(W: torch.Tensor) -> torch.Tensor:
    """fp32 Linear weight [Nf,K] -> three-plane bf16 tensor-core blocks (opaque uint8 buffer)"""
    W = W.detach().contiguous()
    nf, k = W.shape
    out = torch.empty(int(L.load().st2_linear_tc_weight_bytes(nf, k)), dtype=torch.uint8, device=W.device)
    L.call("st2_linear_tc_weight_layout", ptr(W), ptr(out), nf, k, stream_ptr())
    return out


def linear(A, W, bias=None, *, act=ACT_NONE, R=None, out=None, wtc=None):
    """A [..., K] @ W[Nf,K]^T (+bias, act, +R) -> [..., Nf].  Rows may be strided (ld).
    wtc: optional tensor-core weight blocks (linear_tc_weight_layout) -> fp32-accurate wgmma path for big M."""
    K = A.shape[-1]
    A2, M, lda = _rows_view(A)
    Nf = W.shape[0]
    assert W.shape[1] == K and W.is_contiguous()
    if out is None:
        out = empty(*A.shape[:-1], Nf, device=A.device)
    o2, Mo, ldc = _rows_view(out)
    assert o2.data_ptr() == out.data_ptr() and Mo == M, "output rows must be uniformly strided"
    ldr = 0
    if R is not None:
        R2, Mr, ldr = _rows_view(R)
        assert R2.data_ptr() == R.data_ptr() and Mr == M
    if wtc is not None and USE_TC and M >= LINEAR_TC_MIN_ROWS:
        with _prof(f"linear_tc M{M} N{Nf} K{K}", 2.0 * M * Nf * K, 4.0 * (M * K + Nf * K + M * Nf * (2 if R is not None else 1)), 3):
            if Nf > 128 and LINEAR_TC_PRESPLIT:
                # split the activation rows into fp16 operand stages once (not once per 128-feature output block inside the GEMM)
                planes = torch.empty(int(L.load().st2_linear_tc_split_bytes(M, K)), dtype=torch.uint8, device=A.device)
                L.call("st2_linear_tc_split", ptr(A2), lda, M, K, ptr(planes), stream_ptr())
                L.call("st2_linear_tc_pre", ptr(A2), lda, ptr(planes), ptr(wtc), ptr(bias), ptr(R), ldr, ptr(out), ldc, M, Nf, K, act,
                       stream_ptr())
            else:
                L.call("st2_linear_tc", ptr(A2), lda, ptr(wtc), ptr(bias), ptr(R), ldr, ptr(out), ldc, M, Nf, K, act, stream_ptr())
    else:
        with _prof(f"linear_simt M{M} N{Nf} K{K}", 2.0 * M * Nf * K, 4.0 * (M * K + Nf * K + M * Nf)):
            L.call("st2_linear", ptr(A2), 0, lda, 1, M, ptr(W), ptr(bias), ptr(R), ldr, ptr(out), ldc, M, Nf, K, act, stream_ptr())
    return out


def check_range():
    """Raise if any fp16-plane operand of a tensor-core GEMM, attention or conv since the last check left fp16's range or
    was NaN (GEMM and attention: |x| >= 65504 for the activations, weights, q, k and v; conv, after its power-of-two operand
    scales: |z| >= 65504/64 after the prologue, |w| >= 65504/4096): the outputs of that pass hold inf/NaN.  Clears the
    flag.  Synchronises; not callable under CUDA-graph capture."""
    flag = C.c_int(0)
    L.call("st2_range_flag_fetch", C.byref(flag))
    if flag.value:
        raise FloatingPointError("styletts2_b200: an operand of a tensor-core GEMM, attention or conv exceeded the fp16 plane "
                                 "range (GEMM / attention |x| >= 65504; conv |activation| >= 1023.5 or |weight| >= 16) or was "
                                 "NaN; set ST2_TC=0 to run these layers on the fp32 SIMT kernels")


def linear_strided(x, B, Lr, K, bs, ls, ks, W, bias=None, *, act=ACT_NONE, out=None):
    """Rows (b,l) of x addressed with explicit strides (conv-layout inputs of LSTM projections)."""
    Nf = W.shape[0]
    M = B * Lr
    if out is None:
        out = empty(M, Nf, device=x.device)
    L.call("st2_linear", ptr(x), bs, ls, ks, Lr, ptr(W), ptr(bias), None, 0, ptr(out), out.stride(0), M, Nf, K, act,
           stream_ptr())
    return out


ATT_TC = os.environ.get("ST2_ATT_TC", "1") != "0"   # wgmma attention (fp32-accurate) where supported
ATT_TC_MIN_N = 32


def attention_ex(q, k, v, out, B, N, H, D, lengths=None):
    """softmax(q k^T / sqrt(D)) v per (utterance, head).  q / k / v / out: 2-D row views [B*N, >= H*D] (row strides free,
    head h in columns h*D..); lengths (int32 [B]) = key-padding mask.  wgmma kernel when the layout allows it."""
    scale = float(D) ** -0.5
    use_tc = (ATT_TC and USE_TC and N >= ATT_TC_MIN_N and k.stride(0) == v.stride(0)
              and bool(L.load().st2_attention_tc_supported(q.stride(0), k.stride(0), out.stride(0), D))
              and all(t.data_ptr() % 16 == 0 for t in (q, k, v, out)))
    with _prof(f"attention{'_tc' if use_tc else ''} B{B} N{N} H{H} D{D}", 4.0 * B * H * N * N * D, 4.0 * B * N * H * D * 4, 3 if use_tc else 0):
        L.call("st2_attention_tc" if use_tc else "st2_attention_ex", ptr(q), q.stride(0), ptr(k), ptr(v), k.stride(0), ptr(out),
               out.stride(0), ptr(lengths), B, N, H, D, scale, stream_ptr())
    return out


def attention_packed(q, kv, offsets, B, max_len, H=8, D=64, out=None):
    """q [M, H*D], kv [M, 2*H*D] (k | v) on packed token rows: utterance b owns rows offsets[b] .. offsets[b+1]-1
    (offsets int32 [B+1] on the device, max_len >= every row count) and attends over its own rows only -> [M, H*D].
    Runs the wgmma kernel; a layout it cannot take is an error."""
    M = q.shape[0]
    if out is None:
        out = empty(M, H * D, device=q.device)
    k, v = kv[:, :H * D], kv[:, H * D:]
    scale = float(D) ** -0.5
    ok = (k.stride(0) == v.stride(0) and bool(L.load().st2_attention_tc_supported(q.stride(0), k.stride(0), out.stride(0), D))
          and all(t.data_ptr() % 16 == 0 for t in (q, k, v, out)))
    if not ok:
        raise RuntimeError("attention_packed: head_features must be 64, row strides multiples of 4 floats, pointers 16-byte aligned")
    # the algorithmic work is sum_b n_b^2 per head; max_len * M bounds it without a host read of the offsets
    with _prof(f"attention_tc_packed M{M} B{B} maxN{max_len} H{H} D{D}", 4.0 * H * M * max_len * D, 4.0 * M * H * D * 4, 3):
        L.call("st2_attention_tc_packed", ptr(q), q.stride(0), ptr(k), ptr(v), k.stride(0), ptr(out), out.stride(0), ptr(offsets),
               B, max_len, H, D, scale, stream_ptr())
    return out


def attention(q, kv, B, N, H=8, D=64):
    """q [B*N, H*D], kv [B*N, 2*H*D] (k | v) -> [B*N, H*D]   (Modules/diffusion/modules.py:523-535)"""
    out = empty(B * N, H * D, device=q.device)
    return attention_ex(q, kv[:, :H * D], kv[:, H * D:], out, B, N, H, D)


def lstm_bidir(gx, whh, out, o_bs, o_ts, o_cs, B, Lr, H, lengths=None):
    work = empty(6 * B * H + 64, device=gx.device)
    with _prof(f"lstm_bidir B{B} L{Lr} H{H}", 16.0 * B * Lr * H * H, 0.0):
        L.call("st2_lstm_bidir", ptr(gx), ptr(whh), ptr(out), o_bs, o_ts, o_cs, ptr(lengths), B, Lr, H, ptr(work), stream_ptr())
    return out


# ------------------------------------------------------------------ sampler / glue
def kdiff_step(x_eval, x_pred, c_skip, c_out, sigma_eval, x_base, dt, eps=None, sigma_up=0.0, x_pred_masked=None,
               cfg_scale=1.0):
    out = torch.empty_like(x_base)
    L.call("st2_kdiff_step", ptr(x_eval), ptr(x_pred), ptr(x_pred_masked), cfg_scale, c_skip, c_out, sigma_eval,
           ptr(x_base), dt, ptr(eps), sigma_up, ptr(out), x_base.numel(), stream_ptr())
    return out


def scale(x, a):
    out = torch.empty_like(x)
    L.call("st2_scale", ptr(x.contiguous()), a, ptr(out), x.numel(), stream_ptr())
    return out


def axpby(x, a, y, b):
    x, y = x.contiguous(), y.contiguous()
    out = torch.empty_like(x)
    L.call("st2_axpby", ptr(x), a, ptr(y), b, ptr(out), x.numel(), stream_ptr())
    return out


def time_embedding(t, w):
    B, half = t.shape[0], w.shape[0]
    out = empty(B, 2 * half + 1, device=w.device)
    L.call("st2_time_embedding", ptr(t.contiguous()), ptr(w), half, B, ptr(out), out.stride(0), stream_ptr())
    return out


def embedding_cl(tokens, table, lengths=None):
    B, N = tokens.shape
    Cw = table.shape[1]
    out = empty(B, Cw, N, device=table.device)
    L.call("st2_embedding_cl", ptr(tokens.contiguous()), ptr(table), ptr(lengths), B, N, Cw, ptr(out), stream_ptr())
    return out


def durations(logits, last_plus=0, lengths=None):
    """lengths [B] int32 (optional): padded tokens get duration 0, `last_plus` lands on the last real token."""
    B, N, J = logits.shape
    pred = torch.empty(B, N, device=logits.device, dtype=torch.int32)
    durf = empty(B, N, device=logits.device)
    L.call("st2_durations", ptr(logits.contiguous()), B, N, J, last_plus, ptr(lengths), ptr(pred), ptr(durf), stream_ptr())
    return pred, durf


def frame_tokens(dur, T, shift_right=False):
    B, N = dur.shape
    tok = torch.empty(B, T, device=dur.device, dtype=torch.int32)
    total = torch.empty(B, device=dur.device, dtype=torch.int32)
    L.call("st2_frame_tokens", ptr(dur.contiguous()), B, N, T, 1 if shift_right else 0, ptr(tok), ptr(total), stream_ptr())
    return tok, total


def expand_rows(src, tok, out=None):
    """src [B,N,C] (row stride free) -> [B,T,C]"""
    B, N, Cw = src.shape
    T = tok.shape[1]
    if out is None:
        out = empty(B, T, Cw, device=src.device)
    assert src.stride(2) == 1 and src.stride(0) == N * src.stride(1)
    L.call("st2_expand_rows", ptr(src), src.stride(1), ptr(tok), B, N, T, Cw, ptr(out), out.stride(1), stream_ptr())
    return out


def expand_cl(src, tok, out=None):
    """src [B,C,N] contiguous -> out [B,C,T] (out may be a channel-prefix view of a wider buffer)"""
    src = src.contiguous()
    B, Cw, N = src.shape
    T = tok.shape[1]
    if out is None:
        out = empty(B, Cw, T, device=src.device)
    L.call("st2_expand_cl", ptr(src), ptr(tok), B, Cw, N, T, ptr(out), out.stride(0), stream_ptr())
    return out


# ------------------------------------------------------------------ source / stft
_RNG = {"seed": 0x5EED5EED, "offset": 0, "epoch": {}}


def manual_seed(seed: int):
    """Seed of the library's own Philox stream (throughput mode draws)."""
    _RNG["seed"], _RNG["offset"] = int(seed) & 0xFFFFFFFFFFFFFFFF, 0
    for e in _RNG["epoch"].values():
        e.zero_()


def _rng_epoch(device):
    """device-resident draw epoch (int64[1]); bumped by rng_advance() once per synthesize call."""
    dev = torch.device(device)
    key = dev.index if dev.index is not None else torch.cuda.current_device()
    e = _RNG["epoch"].get(key)
    if e is None:
        e = torch.zeros(1, dtype=torch.int64, device=dev)
        _RNG["epoch"][key] = e
    return e


def rng_advance(device):
    L.call("st2_rng_advance", ptr(_rng_epoch(device)), stream_ptr())


def _rng_take(n_counters: int):
    off = _RNG["offset"]
    _RNG["offset"] = off + int(n_counters)
    return _RNG["seed"], off


def randn_like(x):
    """N(0,1) draw with the library's Philox kernel (stands in for torch.randn_like on the path)."""
    out = torch.empty_like(x, memory_format=torch.contiguous_format)
    seed, off = _rng_take((x.numel() + 3) // 4)
    L.call("st2_randn", ptr(out), x.numel(), seed, off, ptr(_rng_epoch(x.device)), stream_ptr())
    return out


def sine_source(f0, scale_, noise, lin_w, lin_b):
    """f0 [B,F] -> [B, F*scale]; noise [B,F*scale,9] (injected) or None (drawn in the kernel)"""
    f0 = f0.contiguous()
    B, F = f0.shape
    out = empty(B, F * scale_, device=f0.device)
    work = empty(B * 9 * F, device=f0.device)
    seed, off = (0, 0) if noise is not None else _rng_take(B * F * scale_ * 3)
    with _prof(f"sine_source F{F} x{scale_} B{B}", 0.0, 4.0 * B * F * scale_ * (1 + (9 if noise is not None else 0))):
        L.call("st2_sine_source", ptr(f0), B, F, scale_, ptr(noise.contiguous() if noise is not None else None),
               ptr(lin_w.contiguous()), ptr(lin_b), ptr(out), ptr(work), seed, off,
               ptr(_rng_epoch(f0.device)) if noise is None else None, stream_ptr())
    return out


def stft20(x):
    x = x.contiguous()
    B, Ln = x.shape
    har = empty(B, 22, Ln // 5 + 1, device=x.device)
    with _prof(f"stft20 L{Ln} B{B}", 0.0, 4.0 * B * (Ln + 22 * (Ln // 5 + 1))):
        L.call("st2_stft20", ptr(x), B, Ln, ptr(har), stream_ptr())
    return har


def istft20_expsin(x):
    x = x.contiguous()
    B, _, Fr = x.shape
    wav = empty(B, 5 * (Fr - 1), device=x.device)
    with _prof(f"istft20 F{Fr} B{B}", 0.0, 4.0 * B * (22 * Fr + 5 * (Fr - 1))):
        L.call("st2_istft20_expsin", ptr(x), B, Fr, ptr(wav), stream_ptr())
    return wav


def pcm16(wav: torch.Tensor, gain: float = 1.0) -> torch.Tensor:
    """fp32 waveform (any shape) -> int16 PCM on the device: saturate(rint(x * 32767 * gain))"""
    wav = wav.contiguous()
    out = torch.empty(wav.shape, dtype=torch.int16, device=wav.device)
    with _prof(f"pcm16 n{wav.numel()}", 0.0, 6.0 * wav.numel()):
        L.call("st2_pcm16", ptr(wav), wav.numel(), float(gain), ptr(out), stream_ptr())
    return out


def kdiff_combine(out, out_masked, scale_):
    """classifier-free guidance: out_masked + (out - out_masked) * scale (modules.py:420-423)"""
    d = axpby(out, 1.0, out_masked, -1.0)
    return axpby(out_masked, 1.0, d, scale_)


# ------------------------------------------------------------------ reference-style path (SURVEY 8 f2)
def spectral_norm_fold(weight_orig, u, v):
    """eval-mode spectral_norm weight in the conv2d kernel layout [Cin/groups*KH*KW][Cout]; returns (wt, sigma[1])."""
    w = weight_orig.detach().contiguous()
    cout = w.shape[0]
    n = w.numel() // cout
    wt = empty(n, cout, device=w.device)
    sigma = empty(1, device=w.device)
    L.call("st2_spectral_norm_fold", ptr(w), ptr(u.contiguous()), ptr(v.contiguous()), cout, n, ptr(wt), ptr(sigma), stream_ptr())
    return wt, sigma


def conv2d(x, wt, bias, *, cout, kh, kw, pad, pre_act=False, slope=0.2, res=None, out_scale=1.0):
    from .lib import Conv2dArgs
    x = x.contiguous()
    B, Cin, H, W = x.shape
    Ho, Wo = H + 2 * pad - kh + 1, W + 2 * pad - kw + 1
    out = empty(B, cout, Ho, Wo, device=x.device)
    if res is not None:
        assert res.shape == out.shape and res.is_contiguous()
    a = Conv2dArgs()
    a.x, a.wt, a.bias, a.res, a.out = ptr(x), ptr(wt), ptr(bias), ptr(res), ptr(out)
    a.B, a.Cin, a.H, a.W, a.Cout, a.KH, a.KW, a.pad = B, Cin, H, W, cout, kh, kw, pad
    a.pre_act, a.slope, a.out_scale = int(bool(pre_act)), float(slope), float(out_scale)
    L.call("st2_conv2d", C.byref(a), stream_ptr())
    return out


def dwconv3x3_s2(x, wt, bias):
    x = x.contiguous()
    B, Cc, H, W = x.shape
    out = empty(B, Cc, (H - 1) // 2 + 1, (W - 1) // 2 + 1, device=x.device)
    L.call("st2_dwconv3x3_s2", ptr(x), ptr(wt), ptr(bias), ptr(out), B, Cc, H, W, stream_ptr())
    return out


def avgpool_half(x):
    x = x.contiguous()
    B, Cc, H, W = x.shape
    out = empty(B, Cc, H // 2, (W + 1) // 2, device=x.device)
    L.call("st2_avgpool_half", ptr(x), ptr(out), B * Cc, H, W, stream_ptr())
    return out


def mean_hw_lrelu(x, slope=0.2):
    x = x.contiguous()
    B, Cc, H, W = x.shape
    out = empty(B, Cc, device=x.device)
    L.call("st2_mean_hw_lrelu", ptr(x), ptr(out), B * Cc, H * W, float(slope), stream_ptr())
    return out


def mel_frames(wave, window, hop, n_fft):
    wave = wave.contiguous()
    B, Ln = wave.shape
    win = window.numel()
    F = 1 + Ln // hop
    frames = empty(B * F, win, device=wave.device)
    L.call("st2_mel_frames", ptr(wave), ptr(window), B, Ln, win, hop, n_fft, ptr(frames), stream_ptr())
    return frames, F


def mel_power(y, nf):
    rows = y.shape[0]
    p = empty(rows, nf, device=y.device)
    L.call("st2_mel_power", ptr(y), rows, nf, ptr(p), stream_ptr())
    return p


def logmel(mel, B, F, eps, mean, std):
    M = mel.shape[1]
    out = empty(B, M, F, device=mel.device)
    L.call("st2_logmel", ptr(mel), B, F, M, float(eps), float(mean), float(std), ptr(out), stream_ptr())
    return out
