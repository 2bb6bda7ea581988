"""nn.Module shells that keep the reference's class names, constructor arguments, forward
signatures and state-dict keys, and run every op through the C-ABI kernels.

Reference classes mirrored (SURVEY.md section 8b): models.py TextEncoder (:284-345), LayerNorm (:270-282),
AdaIN1d (:349-359), AdainResBlk1d (:372-416), AdaLayerNorm (:418-438), ProsodyPredictor (:440-515),
DurationEncoder (:517-569), LinearNorm (:166-176); Modules/istftnet.py + Modules/hifigan.py
AdaINResBlock1, SourceModuleHnNSF, Generator, Decoder.

Weight-norm parameters stay stored as weight_g / weight_v (checkpoint compatible); they are folded
and re-laid-out for the kernels once and cached until a parameter changes.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .lib import ACT_GELU, ACT_LRELU, ACT_NONE, ACT_SNAKE, ACT_TANH, TC_ACCURATE, TC_FAST


# =========================================================================== parameter holders
class _Cached(nn.Module):
    """Caches kernel-layout weights keyed on (data_ptr, version) of the parameters."""

    def _key(self):
        return tuple((p.data_ptr(), p._version, str(p.device)) for p in self.parameters(recurse=False))

    def prepared(self):
        k = self._key()
        c = self.__dict__.get("_prep")
        if c is None or c[0] != k:
            with torch.no_grad():
                c = (k, self._prepare())
            self.__dict__["_prep"] = c
        return c[1]


class WNConv1d(_Cached):
    """weight_norm(nn.Conv1d) holder: weight_g [Cout,1,1], weight_v [Cout,Cin,K], bias."""

    def __init__(self, cin, cout, k, stride=1, padding=0, dilation=1, bias=True):
        super().__init__()
        self.cin, self.cout, self.k, self.stride, self.padding, self.dilation = cin, cout, k, stride, padding, dilation
        self.weight_g = nn.Parameter(torch.ones(cout, 1, 1))
        self.weight_v = nn.Parameter(torch.empty(cout, cin, k).uniform_(-1, 1) / math.sqrt(cin * k))
        if bias:
            self.bias = nn.Parameter(torch.zeros(cout))
        else:
            self.register_parameter("bias", None)

    def _prepare(self):
        w = ops.fold_weight_norm(self.weight_v, self.weight_g)
        return ops.conv_weight_layout(w), w, _maybe_wtc(w, self.stride, self.dilation, getattr(self, "tc_mode", TC_FAST))

    def wt(self):
        return self.prepared()[0]

    def folded(self):
        return self.prepared()[1]

    def wtc(self):
        return self.prepared()[2]

    def forward(self, x, **kw):
        y, _ = ops.conv1d(x, self.wt(), self.bias, K=self.k, stride=self.stride, dil=self.dilation, pad=self.padding,
                          wtc=self.wtc(), **kw)
        return y


def _maybe_wtc(w, stride, dilation, mode=TC_FAST):
    """plane-split tensor-core weight blocks when the wgmma conv supports the shape and it is worth it.
    mode: precision recipe (TC_FAST for the decoder / vocoder, TC_ACCURATE for the F0/N predictor)."""
    co, ci, k = w.shape
    # Cout < 16 (conv_post of HiFi-GAN: one output channel) only through the time-major kernel, whose N is Cout rounded up to 16
    narrow_ok = co >= 16 or (mode == TC_FAST and ops.TC_TMAJOR_MAX_COUT >= 16 and ops.TC_MODE_OVERRIDE is None)
    if stride == 1 and narrow_ok and ci >= 16 and ops.conv_tc_supported(ci, co, k, stride, dilation):
        return ops.conv_tc_weight_layout(w, mode)
    return None


def set_tc_mode(root: nn.Module, mode: int):
    """Select the tensor-core precision recipe of every conv below `root` (before its weights are first prepared)."""
    for m in root.modules():
        if isinstance(m, (WNConv1d, Conv1d, WNConvTranspose1d)):
            m.tc_mode = mode
            m.__dict__.pop("_prep", None)


class Conv1d(_Cached):
    """plain nn.Conv1d holder (weight, bias)."""

    def __init__(self, cin, cout, k, stride=1, padding=0):
        super().__init__()
        self.cin, self.cout, self.k, self.stride, self.padding = cin, cout, k, stride, padding
        self.weight = nn.Parameter(torch.empty(cout, cin, k).uniform_(-1, 1) / math.sqrt(cin * k))
        self.bias = nn.Parameter(torch.zeros(cout))

    def _prepare(self):
        wt, wtc = ops.conv_weight_layout(self.weight), _maybe_wtc(self.weight.detach(), self.stride, 1, getattr(self, "tc_mode", TC_FAST))
        poly = None
        S, k = self.stride, self.k
        if S > 1 and k % S == 0 and self.cin * S >= 16 and self.cout >= 16 and ops.USE_TC and self.weight.is_cuda:
            # strided conv as a stride-1 conv over the polyphase input (ops.polyphase_gather): wp[co, c*S + r, j] = w[co, c, j*S + r]
            J = k // S
            wp = self.weight.detach().view(self.cout, self.cin, J, S).permute(0, 1, 3, 2).reshape(self.cout, self.cin * S, J).contiguous()
            if ops.conv_tc_supported(self.cin * S, self.cout, J, 1, 1):
                poly = (ops.conv_weight_layout(wp), ops.conv_tc_weight_layout(wp, getattr(self, "tc_mode", TC_FAST)), J)
        return wt, wtc, poly

    def wt(self):
        return self.prepared()[0]

    def wtc(self):
        return self.prepared()[1]

    def run(self, x, want_stats=False):
        """(y, stats) of the plain conv (no prologue); strided convs take the polyphase tensor-core route when prepared."""
        wt, wtc, poly = self.prepared()
        Lout = (x.shape[-1] + 2 * self.padding - self.k) // self.stride + 1
        if poly is not None and self.cin * self.cout * self.k * Lout >= ops.TC_MIN_WORK:
            wtp, wtcp, J = poly
            xp = ops.polyphase_gather(x, self.stride, self.padding, Lout + J - 1)
            return ops.conv1d(xp, wtp, self.bias, K=J, pad=0, want_stats=want_stats, wtc=wtcp)
        return ops.conv1d(x, wt, self.bias, K=self.k, stride=self.stride, pad=self.padding, want_stats=want_stats, wtc=wtc)

    def forward(self, x, **kw):
        y, _ = ops.conv1d(x, self.wt(), self.bias, K=self.k, stride=self.stride, pad=self.padding, wtc=self.wtc(), **kw)
        return y


class WNConvTranspose1d(_Cached):
    """weight_norm(nn.ConvTranspose1d): weight_g [Cin,1,1], weight_v [Cin,Cout/groups,K], bias [Cout]."""

    def __init__(self, cin, cout, k, stride, padding=0, output_padding=0, groups=1):
        super().__init__()
        self.cin, self.cout, self.k, self.stride, self.padding, self.groups = cin, cout, k, stride, padding, groups
        self.output_padding = output_padding
        self.weight_g = nn.Parameter(torch.ones(cin, 1, 1))
        self.weight_v = nn.Parameter(torch.empty(cin, cout // groups, k).uniform_(-1, 1) / math.sqrt(cin * k / groups))
        self.bias = nn.Parameter(torch.zeros(cout))

    def _prepare(self):
        w = ops.fold_weight_norm(self.weight_v, self.weight_g)
        if self.groups == 1:
            J = (self.k + self.stride - 1) // self.stride
            wtc = None
            if self.cin >= 16 and self.cout >= 16 and ops.conv_tc_supported(self.cin, self.cout, J, 1, 1):
                wtc = ops.convT_tc_weight_layout(w, self.stride, self.padding, getattr(self, "tc_mode", TC_FAST))
            return ops.convT_weight_layout(w, self.stride, self.padding), w, wtc
        return None, w.contiguous(), None

    def wp(self):
        return self.prepared()[0]

    def folded(self):
        return self.prepared()[1]

    def wtc(self):
        return self.prepared()[2]


class Linear(nn.Linear):
    """nn.Linear whose forward is the GEMM kernel (fp32 SIMT for small row counts, fp32-accurate wgmma otherwise)."""

    def _wtc(self):
        k = (self.weight.data_ptr(), self.weight._version, str(self.weight.device))
        c = self.__dict__.get("_wtc_cache")
        if c is None or c[0] != k:
            with torch.no_grad():
                c = (k, ops.linear_tc_weight_layout(self.weight))
            self.__dict__["_wtc_cache"] = c
        return c[1]

    def forward(self, x, act=ACT_NONE, R=None, out=None):
        rows = x.numel() // x.shape[-1]
        wtc = self._wtc() if (ops.USE_TC and rows >= ops.LINEAR_TC_MIN_ROWS and x.is_cuda) else None
        return ops.linear(x, self.weight, self.bias, act=act, R=R, out=out, wtc=wtc)


class LinearNorm(nn.Module):
    """models.py:166-176"""

    def __init__(self, in_dim, out_dim, bias=True, w_init_gain="linear"):
        super().__init__()
        self.linear_layer = Linear(in_dim, out_dim, bias=bias)

    def forward(self, x):
        return self.linear_layer(x)


class LayerNorm(nn.Module):
    """Channel LayerNorm holder of the TextEncoder (models.py:270-282): gamma, beta."""

    def __init__(self, channels, eps=1e-5):
        super().__init__()
        self.channels, self.eps = channels, eps
        self.gamma = nn.Parameter(torch.ones(channels))
        self.beta = nn.Parameter(torch.zeros(channels))


class LSTM(_Cached):
    """Single-layer bidirectional batch_first nn.LSTM look-alike (same parameter names)."""

    def __init__(self, input_size, hidden_size, num_layers=1, batch_first=True, bidirectional=True, dropout=0.0):
        super().__init__()
        assert num_layers == 1 and batch_first and bidirectional
        self.input_size, self.hidden_size = input_size, hidden_size
        k = 1.0 / math.sqrt(hidden_size)
        for sfx in ("", "_reverse"):
            self.register_parameter("weight_ih_l0" + sfx, nn.Parameter(torch.empty(4 * hidden_size, input_size).uniform_(-k, k)))
            self.register_parameter("weight_hh_l0" + sfx, nn.Parameter(torch.empty(4 * hidden_size, hidden_size).uniform_(-k, k)))
            self.register_parameter("bias_ih_l0" + sfx, nn.Parameter(torch.empty(4 * hidden_size).uniform_(-k, k)))
            self.register_parameter("bias_hh_l0" + sfx, nn.Parameter(torch.empty(4 * hidden_size).uniform_(-k, k)))

    def flatten_parameters(self):
        pass

    def _prepare(self):
        wih = torch.cat([self.weight_ih_l0, self.weight_ih_l0_reverse], 0).contiguous()
        bias = torch.cat([self.bias_ih_l0 + self.bias_hh_l0, self.bias_ih_l0_reverse + self.bias_hh_l0_reverse], 0).contiguous()
        whh = torch.stack([self.weight_hh_l0, self.weight_hh_l0_reverse], 0).contiguous()
        wtc = ops.linear_tc_weight_layout(wih) if (ops.USE_TC and wih.is_cuda) else None
        return wih, bias, whh, wtc

    def run(self, x, B, Lr, strides, out, out_strides, lengths=None):
        """x element (b,l,k) at strides (bs,ls,ks); out element (b,t,c) at out_strides."""
        wih, bias, whh, wtc = self.prepared()
        if wtc is not None and strides[2] == 1 and strides[0] == Lr * strides[1] and B * Lr >= ops.LINEAR_TC_MIN_ROWS:
            # row-layout input: input projection on the fp32-accurate tensor-core GEMM
            gx = ops.empty(B * Lr, wih.shape[0], device=x.device)
            ops.L.call("st2_linear_tc", ops.ptr(x), strides[1], ops.ptr(wtc), ops.ptr(bias), None, 0, ops.ptr(gx), gx.stride(0),
                       B * Lr, wih.shape[0], self.input_size, 0, ops.stream_ptr())
        else:
            gx = ops.linear_strided(x, B, Lr, self.input_size, strides[0], strides[1], strides[2], wih, bias)
        ops.lstm_bidir(gx, whh, out, out_strides[0], out_strides[1], out_strides[2], B, Lr, self.hidden_size, lengths)
        return out

    def forward(self, x, lengths=None):
        """x [B,L,In] (any strides) -> (out [B,L,2H], None)"""
        B, Lr, _ = x.shape
        H = self.hidden_size
        out = torch.zeros(B, Lr, 2 * H, device=x.device) if lengths is not None else ops.empty(B, Lr, 2 * H, device=x.device)
        self.run(x, B, Lr, x.stride(), out, out.stride(), lengths)
        return out, None


def _lengths_i32(input_lengths, device):
    if input_lengths is None:
        return None
    return input_lengths.to(device=device, dtype=torch.int32).contiguous()


# =========================================================================== style FC batching
class StyleFC:
    """All AdaIN1d / AdaLayerNorm `fc(s)` of a module tree in ONE GEMM (s is fixed per forward)."""

    def __init__(self, root: nn.Module, s: torch.Tensor):
        fcs = [m for m in root.modules() if isinstance(m, (AdaIN1d, AdaLayerNorm))]
        key = tuple((m.fc.weight.data_ptr(), m.fc.weight._version) for m in fcs)
        cache = root.__dict__.get("_stylefc")
        if cache is None or cache[0] != key:
            with torch.no_grad():
                W = torch.cat([m.fc.weight for m in fcs], 0).contiguous()
                b = torch.cat([m.fc.bias for m in fcs], 0).contiguous()
            offs, o = {}, 0
            for m in fcs:
                offs[id(m)] = (o, m.fc.weight.shape[0])
                o += m.fc.weight.shape[0]
            cache = (key, W, b, offs)
            root.__dict__["_stylefc"] = cache
        _, W, b, self.offs = cache
        self.h = ops.linear(s.contiguous(), W, b)  # [B, total]

    def gb(self, m) -> torch.Tensor:
        o, n = self.offs[id(m)]
        return self.h[:, o:o + n]


class AdaIN1d(nn.Module):
    """models.py:349-359 == istftnet.py:15-25.  forward(x, s) returns (1+gamma)*IN(x)+beta."""

    def __init__(self, style_dim, num_features):
        super().__init__()
        self.num_features = num_features
        self.fc = Linear(style_dim, num_features * 2)

    def coef(self, stats, fcs: Optional[StyleFC], s=None):
        gb = fcs.gb(self) if fcs is not None else self.fc(s)
        return ops.adain_coef(stats, gb)

    def forward(self, x, s):
        a, b = self.coef(ops.instance_stats(x), None, s)
        C = x.shape[1]
        eye = _identity_wt(C, x.device)
        y, _ = ops.conv1d(x, eye, None, K=1, pre=(a, b))
        return y


_EYE = {}


def _identity_wt(C, device):
    k = (C, str(device))
    if k not in _EYE:
        _EYE[k] = torch.eye(C, device=device).view(C, 1, C).contiguous()
    return _EYE[k]


class UpSample1d(nn.Module):
    def __init__(self, layer_type):
        super().__init__()
        self.layer_type = layer_type


class AdainResBlk1d(nn.Module):
    """models.py:372-416 (== istftnet.py:410-454 == hifigan.py:359-403)."""

    def __init__(self, dim_in, dim_out, style_dim=64, actv=None, upsample="none", dropout_p=0.0):
        super().__init__()
        self.upsample_type = upsample
        self.upsample = UpSample1d(upsample)
        self.learned_sc = dim_in != dim_out
        self.dim_in, self.dim_out = dim_in, dim_out
        self.conv1 = WNConv1d(dim_in, dim_out, 3, 1, 1)
        self.conv2 = WNConv1d(dim_out, dim_out, 3, 1, 1)
        self.norm1 = AdaIN1d(style_dim, dim_in)
        self.norm2 = AdaIN1d(style_dim, dim_out)
        if self.learned_sc:
            self.conv1x1 = WNConv1d(dim_in, dim_out, 1, 1, 0, bias=False)
        if upsample == "none":
            self.pool = nn.Identity()
        else:
            self.pool = WNConvTranspose1d(dim_in, dim_in, 3, 2, padding=1, output_padding=1, groups=dim_in)

    @property
    def has_upsample(self):
        return self.upsample_type != "none"

    def run(self, x, fcs: StyleFC, x_stats=None, out=None):
        """x [B,Cin,L] -> [B,Cout,L or 2L].  out: optional destination view."""
        if x_stats is None:
            x_stats = ops.instance_stats(x)
        a1, b1 = self.norm1.coef(x_stats, fcs)
        up = self.has_upsample
        if up:
            r = ops.adain_lrelu_pool(x, a1, b1, self.pool.folded().view(-1, 3), self.pool.bias, 0.2)
            h, hst = ops.conv1d(r, self.conv1.wt(), self.conv1.bias, K=3, pad=1, want_stats=True, wtc=self.conv1.wtc())
        else:
            h, hst = ops.conv1d(x, self.conv1.wt(), self.conv1.bias, K=3, pad=1, pre=(a1, b1), pre_act=ACT_LRELU, slope=0.2,
                                want_stats=True, wtc=self.conv1.wtc())
        a2, b2 = self.norm2.coef(hst, fcs)
        if self.learned_sc:
            sc, _ = ops.conv1d(x, self.conv1x1.wt(), None, K=1, wtc=self.conv1x1.wtc())
        else:
            sc = x
        y, _ = ops.conv1d(h, self.conv2.wt(), self.conv2.bias, K=3, pad=1, pre=(a2, b2), pre_act=ACT_LRELU, slope=0.2, res=sc,
                          res_shift=1 if up else 0, out_div=math.sqrt(2), out=out, wtc=self.conv2.wtc())
        return y

    def forward(self, x, s):
        return self.run(x, StyleFC(self, s))


class AdaLayerNorm(nn.Module):
    """models.py:418-438 / Modules/diffusion/modules.py:18-38 (holder; applied by rows_ln)."""

    def __init__(self, style_dim, channels, eps=1e-5):
        super().__init__()
        self.channels, self.eps = channels, eps
        self.fc = Linear(style_dim, channels * 2)

    def forward(self, x, s):
        """x [B,N,C] (as the reference is called after its transposes cancel) -> same shape."""
        B, N, Cw = x.shape
        gb = self.fc(s)
        out = ops.empty(B, N, Cw, device=x.device)
        x = x.contiguous()
        ops.rows_ln(B=B, N=N, Cw=Cw, h_in=x, g1=gb, b1=gb[:, Cw:], gb_bstride=gb.stride(0), ada=True, out1=out, eps=self.eps)
        return out


# =========================================================================== text side
class TextEncoder(nn.Module):
    """models.py:284-345.  forward(tokens [B,N] i64, input_lengths [B], mask [B,N] bool) -> [B,512,N]."""

    def __init__(self, channels, kernel_size, depth, n_symbols, actv=None):
        super().__init__()
        self.embedding = nn.Embedding(n_symbols, channels)
        padding = (kernel_size - 1) // 2
        self.cnn = nn.ModuleList()
        for _ in range(depth):
            self.cnn.append(nn.Sequential(WNConv1d(channels, channels, kernel_size, padding=padding), LayerNorm(channels),
                                          nn.LeakyReLU(0.2), nn.Dropout(0.2)))
        self.lstm = LSTM(channels, channels // 2, 1, batch_first=True, bidirectional=True)
        self.channels = channels

    def forward(self, x, input_lengths, m):
        B, N = x.shape
        dev = self.embedding.weight.device
        lens = _lengths_i32(input_lengths, dev)
        h = ops.embedding_cl(x.to(dev), self.embedding.weight, lens)
        for blk in self.cnn:
            conv, ln = blk[0], blk[1]
            y, _ = ops.conv1d(h, conv.wt(), conv.bias, K=conv.k, pad=conv.padding, wtc=conv.wtc())
            h = ops.channel_layernorm_lrelu(y, ln.gamma, ln.beta, lens, ln.eps, 0.2)
        C = self.channels
        out = torch.zeros(B, C, N, device=dev)
        # LSTM over tokens reading the conv layout directly; output written back in conv layout
        self.lstm.run(h, B, N, (C * N, 1, N), out, (C * N, 1, N), lens)
        return out


class DurationEncoder(nn.Module):
    """models.py:517-569.  forward(x [B,512,N], style [B,128], text_lengths, m) -> [B,N,640]."""

    def __init__(self, sty_dim, d_model, nlayers, dropout=0.1):
        super().__init__()
        self.lstms = nn.ModuleList()
        for _ in range(nlayers):
            self.lstms.append(LSTM(d_model + sty_dim, d_model // 2, num_layers=1, batch_first=True, bidirectional=True))
            self.lstms.append(AdaLayerNorm(sty_dim, d_model))
        self.dropout, self.d_model, self.sty_dim = dropout, d_model, sty_dim

    def forward(self, x, style, text_lengths, m):
        B, Cd, N = x.shape
        dev = x.device
        lens = _lengths_i32(text_lengths, dev)
        W = self.d_model + self.sty_dim
        style = style.contiguous()
        fcs = StyleFC(self, style)
        cur = ops.empty(B, N, W, device=dev)
        # x arrives as [B,512,N]; the reference works on its transpose.  Copy rows with the gather kernel
        # degenerate case (identity map) is overkill: a strided torch copy is pure data movement.
        cur[:, :, :Cd].copy_(x.transpose(1, 2))
        if lens is not None:
            mask = torch.arange(N, device=dev).unsqueeze(0) >= lens.unsqueeze(1)
            cur[:, :, :Cd].masked_fill_(mask.unsqueeze(-1), 0.0)
        ops.bcast_cols(cur, Cd, style, lens)
        H2 = self.d_model
        for i in range(0, len(self.lstms), 2):
            lstm, aln = self.lstms[i], self.lstms[i + 1]
            y = torch.zeros(B, N, H2, device=dev)
            lstm.run(cur, B, N, cur.stride(), y, y.stride(), lens)
            nxt = ops.empty(B, N, W, device=dev)
            gb = fcs.gb(aln)
            ops.rows_ln(B=B, N=N, Cw=H2, h_in=y, g1=gb, b1=gb[:, H2:], gb_bstride=gb.stride(0), ada=True,
                        out1=nxt, eps=aln.eps, lengths=lens)
            ops.bcast_cols(nxt, H2, style, lens)
            cur = nxt
        return cur


class ProsodyPredictor(nn.Module):
    """models.py:440-515."""

    def __init__(self, style_dim, d_hid, nlayers, max_dur=50, dropout=0.1):
        super().__init__()
        self.text_encoder = DurationEncoder(sty_dim=style_dim, d_model=d_hid, nlayers=nlayers, dropout=dropout)
        self.lstm = LSTM(d_hid + style_dim, d_hid // 2, 1, batch_first=True, bidirectional=True)
        self.duration_proj = LinearNorm(d_hid, max_dur)
        self.shared = LSTM(d_hid + style_dim, d_hid // 2, 1, batch_first=True, bidirectional=True)
        self.F0 = nn.ModuleList([AdainResBlk1d(d_hid, d_hid, style_dim, dropout_p=dropout),
                                 AdainResBlk1d(d_hid, d_hid // 2, style_dim, upsample=True, dropout_p=dropout),
                                 AdainResBlk1d(d_hid // 2, d_hid // 2, style_dim, dropout_p=dropout)])
        self.N = nn.ModuleList([AdainResBlk1d(d_hid, d_hid, style_dim, dropout_p=dropout),
                                AdainResBlk1d(d_hid, d_hid // 2, style_dim, upsample=True, dropout_p=dropout),
                                AdainResBlk1d(d_hid // 2, d_hid // 2, style_dim, dropout_p=dropout)])
        self.F0_proj = Conv1d(d_hid // 2, 1, 1, 1, 0)
        self.N_proj = Conv1d(d_hid // 2, 1, 1, 1, 0)
        self.d_hid = d_hid
        # F0 is integrated into a phase of 1e4..1e6 rad by the harmonic source downstream: this subtree runs the
        # fp32-accurate tensor-core recipe (two fp16 planes, separate correction accumulator)
        set_tc_mode(self, TC_ACCURATE)

    def forward(self, texts, style, text_lengths, alignment, m):
        d = self.text_encoder(texts, style, text_lengths, m)
        x, _ = self.lstm(d, _lengths_i32(text_lengths, d.device))
        duration = self.duration_proj(x)
        en = torch.matmul(d.transpose(-1, -2), alignment)  # training-time API kept for signature parity only
        return duration.squeeze(-1), en

    def F0Ntrain(self, x, s):
        """x = en [B,640,T] (any strides), s [B,128] -> (F0 [B,2T], N [B,2T])"""
        B, Ci, T = x.shape
        dev = x.device
        C = self.d_hid
        h = ops.empty(B, C, T, device=dev)
        xt = x.transpose(-1, -2)
        if xt.stride(2) != 1:
            # conv-layout input (the notebooks' `d.transpose(-1,-2) @ pred_aln_trg`): one transposing copy, so that the
            # LSTM input projection runs the same row-layout GEMM (same bits) whichever way the caller built `en`
            xt = xt.contiguous()
        self.shared.run(xt, B, T, xt.stride(), h, (C * T, 1, T))
        fcs = StyleFC(self, s.contiguous())
        hst = ops.instance_stats(h)
        outs = []
        for blocks, proj in ((self.F0, self.F0_proj), (self.N, self.N_proj)):
            y, st = h, hst
            for blk in blocks:
                y = blk.run(y, fcs, st)
                st = None
            o, _ = ops.conv1d(y, proj.wt(), proj.bias, K=1)
            outs.append(o.squeeze(1))
        return outs[0], outs[1]


# =========================================================================== vocoder blocks
def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


class AdaINResBlock1(nn.Module):
    """Modules/istftnet.py:27-75 == Modules/hifigan.py:26-74."""

    def __init__(self, channels, kernel_size=3, dilation=(1, 3, 5), style_dim=64):
        super().__init__()
        self.channels, self.kernel_size, self.dilation = channels, kernel_size, tuple(dilation)
        self.convs1 = nn.ModuleList([WNConv1d(channels, channels, kernel_size, 1, dilation=d, padding=get_padding(kernel_size, d))
                                     for d in dilation])
        self.convs2 = nn.ModuleList([WNConv1d(channels, channels, kernel_size, 1, dilation=1, padding=get_padding(kernel_size, 1))
                                     for _ in dilation])
        self.adain1 = nn.ModuleList([AdaIN1d(style_dim, channels) for _ in dilation])
        self.adain2 = nn.ModuleList([AdaIN1d(style_dim, channels) for _ in dilation])
        self.alpha1 = nn.ParameterList([nn.Parameter(torch.ones(1, channels, 1)) for _ in dilation])
        self.alpha2 = nn.ParameterList([nn.Parameter(torch.ones(1, channels, 1)) for _ in dilation])

    def run(self, x, fcs: StyleFC, x_stats=None, out=None, accum_mode=0, accum_div=1.0, final_stats=False):
        """3 x [AdaIN->Snake->dilated conv (stats) -> AdaIN->Snake->conv (+x, stats)].
        The last conv can accumulate into `out` (MRF mean)."""
        if x_stats is None:
            x_stats = ops.instance_stats(x)
        k = self.kernel_size
        n = len(self.convs1)
        st = x_stats
        for j in range(n):
            c1, c2 = self.convs1[j], self.convs2[j]
            a1, b1 = self.adain1[j].coef(st, fcs)
            h, hst = ops.conv1d(x, c1.wt(), c1.bias, K=k, dil=c1.dilation, pad=c1.padding, pre=(a1, b1), pre_act=ACT_SNAKE,
                                alpha=self.alpha1[j], want_stats=True, wtc=c1.wtc())
            a2, b2 = self.adain2[j].coef(hst, fcs)
            last = j == n - 1
            x, st = ops.conv1d(h, c2.wt(), c2.bias, K=k, dil=1, pad=c2.padding, pre=(a2, b2), pre_act=ACT_SNAKE,
                               alpha=self.alpha2[j], res=x, want_stats=(not last) or final_stats,
                               out=out if last else None, accum_mode=accum_mode if last else 0,
                               accum_div=accum_div if last else 1.0, wtc=c2.wtc())
        return x, st

    def forward(self, x, s):
        y, _ = self.run(x, StyleFC(self, s.contiguous()))
        return y


class SourceModuleHnNSF(nn.Module):
    """istftnet.py:250-297 (SineGen has no parameters; l_linear merges the 9 harmonics)."""

    def __init__(self, sampling_rate, upsample_scale, harmonic_num=0, sine_amp=0.1, add_noise_std=0.003, voiced_threshod=0):
        super().__init__()
        self.upsample_scale = int(upsample_scale)
        self.harmonic_num = harmonic_num
        self.l_linear = Linear(harmonic_num + 1, 1)

    def forward(self, f0_curve, noise=None):
        """f0_curve [B,2T] (NOT pre-upsampled: the nearest x300 upsample is fused) -> har_source [B, 600T].
        noise: the randn_like draw of istftnet.py:242 ([B,L,9]); generated on device if None."""
        return ops.sine_source(f0_curve, self.upsample_scale, noise, self.l_linear.weight.view(-1), self.l_linear.bias)


def _mrf(resblocks, x, x_stats, fcs, nk):
    """mean of nk AdaINResBlock1 outputs, accumulated in the last conv's epilogue (istftnet.py:369-375)."""
    acc = torch.empty_like(x)
    for j, rb in enumerate(resblocks):
        mode = 0 if j == 0 else (2 if j == nk - 1 else 1)
        rb.run(x, fcs, x_stats, out=acc, accum_mode=mode, accum_div=float(nk))
    return acc


class Generator(nn.Module):
    """iSTFTNet generator (Modules/istftnet.py:302-380)."""

    def __init__(self, style_dim, resblock_kernel_sizes, upsample_rates, upsample_initial_channel, resblock_dilation_sizes,
                 upsample_kernel_sizes, gen_istft_n_fft, gen_istft_hop_size):
        super().__init__()
        assert gen_istft_n_fft == 20 and gen_istft_hop_size == 5, "stft kernels are specialised for n_fft=20, hop=5"
        self.num_kernels = len(resblock_kernel_sizes)
        self.num_upsamples = len(upsample_rates)
        self.upsample_rates = list(upsample_rates)
        self.m_source = SourceModuleHnNSF(24000, int(np.prod(upsample_rates)) * gen_istft_hop_size, harmonic_num=8, voiced_threshod=10)
        self.noise_convs, self.noise_res, self.ups, self.resblocks = nn.ModuleList(), nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for i, (u, k) in enumerate(zip(upsample_rates, upsample_kernel_sizes)):
            self.ups.append(WNConvTranspose1d(upsample_initial_channel // (2 ** i), upsample_initial_channel // (2 ** (i + 1)), k, u,
                                              padding=(k - u) // 2))
        for i in range(len(self.ups)):
            ch = upsample_initial_channel // (2 ** (i + 1))
            for k, d in zip(resblock_kernel_sizes, resblock_dilation_sizes):
                self.resblocks.append(AdaINResBlock1(ch, k, d, style_dim))
            if i + 1 < len(upsample_rates):
                sf0 = int(np.prod(upsample_rates[i + 1:]))
                self.noise_convs.append(Conv1d(gen_istft_n_fft + 2, ch, sf0 * 2, stride=sf0, padding=(sf0 + 1) // 2))
                self.noise_res.append(AdaINResBlock1(ch, 7, [1, 3, 5], style_dim))
            else:
                self.noise_convs.append(Conv1d(gen_istft_n_fft + 2, ch, 1))
                self.noise_res.append(AdaINResBlock1(ch, 11, [1, 3, 5], style_dim))
        self.post_n_fft = gen_istft_n_fft
        self.conv_post = WNConv1d(ch, self.post_n_fft + 2, 7, 1, padding=3)

    def har_features(self, f0, sine_noise=None):
        return ops.stft20(self.m_source(f0, sine_noise))

    def forward(self, x, s, f0, sine_noise=None, har=None, fcs=None):
        """x [B,512,2T], s [B,128], f0 = F0_curve [B,2T] -> wav [B,1,600T].
        sine_noise / har: parity-mode injections (RNG draw; teacher-forced STFT features)."""
        fcs = fcs or StyleFC(self, s.contiguous())
        if har is None:
            har = self.har_features(f0, sine_noise)
        nk = self.num_kernels
        for i in range(self.num_upsamples):
            nc, up = self.noise_convs[i], self.ups[i]
            xs, xst = nc.run(har, want_stats=True)
            xs, _ = self.noise_res[i].run(xs, fcs, xst)
            x, st = ops.conv_transpose1d(x, up.wp(), up.bias, K=up.k, stride=up.stride, padding=up.padding, pre_act=ACT_LRELU,
                                         slope=0.1, res=xs, reflect_left1=(i == self.num_upsamples - 1), want_stats=True,
                                         wtc=up.wtc())
            x = _mrf(self.resblocks[i * nk:(i + 1) * nk], x, st, fcs, nk)
        y, _ = ops.conv1d(x, self.conv_post.wt(), self.conv_post.bias, K=7, pad=3, pre_act=ACT_LRELU, slope=0.01, wtc=self.conv_post.wtc())
        return ops.istft20_expsin(y).unsqueeze(1)


class HifiGenerator(nn.Module):
    """HiFi-GAN generator (Modules/hifigan.py:272-347)."""

    def __init__(self, style_dim, resblock_kernel_sizes, upsample_rates, upsample_initial_channel, resblock_dilation_sizes,
                 upsample_kernel_sizes):
        super().__init__()
        self.num_kernels = len(resblock_kernel_sizes)
        self.num_upsamples = len(upsample_rates)
        self.m_source = SourceModuleHnNSF(24000, int(np.prod(upsample_rates)), harmonic_num=8, voiced_threshod=10)
        self.noise_convs, self.ups, self.noise_res = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        for i, (u, k) in enumerate(zip(upsample_rates, upsample_kernel_sizes)):
            c_cur = upsample_initial_channel // (2 ** (i + 1))
            self.ups.append(WNConvTranspose1d(upsample_initial_channel // (2 ** i), c_cur, k, u, padding=(u // 2 + u % 2),
                                              output_padding=u % 2))
            if i + 1 < len(upsample_rates):
                sf0 = int(np.prod(upsample_rates[i + 1:]))
                self.noise_convs.append(Conv1d(1, c_cur, sf0 * 2, stride=sf0, padding=(sf0 + 1) // 2))
                self.noise_res.append(AdaINResBlock1(c_cur, 7, [1, 3, 5], style_dim))
            else:
                self.noise_convs.append(Conv1d(1, c_cur, 1))
                self.noise_res.append(AdaINResBlock1(c_cur, 11, [1, 3, 5], style_dim))
        self.resblocks = nn.ModuleList()
        self.alphas = nn.ParameterList([nn.Parameter(torch.ones(1, upsample_initial_channel, 1))])
        for i in range(len(self.ups)):
            ch = upsample_initial_channel // (2 ** (i + 1))
            self.alphas.append(nn.Parameter(torch.ones(1, ch, 1)))
            for k, d in zip(resblock_kernel_sizes, resblock_dilation_sizes):
                self.resblocks.append(AdaINResBlock1(ch, k, d, style_dim))
        self.conv_post = WNConv1d(ch, 1, 7, 1, padding=3)

    def forward(self, x, s, f0, sine_noise=None, har=None, fcs=None):
        fcs = fcs or StyleFC(self, s.contiguous())
        har = self.m_source(f0, sine_noise).unsqueeze(1)  # [B,1,L]
        nk = self.num_kernels
        for i in range(self.num_upsamples):
            nc, up = self.noise_convs[i], self.ups[i]
            xs, xst = nc.run(har, want_stats=True)
            xs, _ = self.noise_res[i].run(xs, fcs, xst)
            x, st = ops.conv_transpose1d(x, up.wp(), up.bias, K=up.k, stride=up.stride, padding=up.padding, pre_act=ACT_SNAKE,
                                         alpha=self.alphas[i], res=xs, want_stats=True, wtc=up.wtc())
            x = _mrf(self.resblocks[i * nk:(i + 1) * nk], x, st, fcs, nk)
        y, _ = ops.conv1d(x, self.conv_post.wt(), self.conv_post.bias, K=7, pad=3, pre_act=ACT_SNAKE,
                          alpha=self.alphas[self.num_upsamples], out_act=ACT_TANH, wtc=self.conv_post.wtc())
        return y


class Decoder(nn.Module):
    """Modules/istftnet.py:467-528 / Modules/hifigan.py:416-475.
    forward(asr [B,512,T], F0_curve [B,2T], N [B,2T], s [B,128]) -> wav [B,1,600T]."""

    def __init__(self, dim_in=512, F0_channel=512, style_dim=64, dim_out=80, resblock_kernel_sizes=[3, 7, 11],
                 upsample_rates=[10, 6], upsample_initial_channel=512, resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 3, 5]],
                 upsample_kernel_sizes=[20, 12], gen_istft_n_fft=None, gen_istft_hop_size=None):
        super().__init__()
        self.dim_in = dim_in
        self.encode = AdainResBlk1d(dim_in + 2, 1024, style_dim)
        self.decode = nn.ModuleList([AdainResBlk1d(1024 + 2 + 64, 1024, style_dim), AdainResBlk1d(1024 + 2 + 64, 1024, style_dim),
                                     AdainResBlk1d(1024 + 2 + 64, 1024, style_dim),
                                     AdainResBlk1d(1024 + 2 + 64, 512, style_dim, upsample=True)])
        self.F0_conv = WNConv1d(1, 1, 3, stride=2, padding=1)
        self.N_conv = WNConv1d(1, 1, 3, stride=2, padding=1)
        self.asr_res = nn.Sequential(WNConv1d(512, 64, 1))
        # The learned shortcut 1x1 convs read the cat buffers raw (no AdaIN in front), and one of their input channels is
        # F0_conv(F0 in Hz): a trained F0_conv puts 60..400 there, past the FAST recipe's envelope (its e4m3 corrections
        # saturate from |z| ~ 64 on and it falls to single-fp16 accuracy, ~4e-4).  ACCURATE keeps fp32-level accuracy up to
        # the fp16 range; these convs have K = 1 and run at the token-frame rate, so the third MMA costs little.
        for blk in [self.encode, *self.decode]:
            set_tc_mode(blk.conv1x1, TC_ACCURATE)
        if gen_istft_n_fft is not None:
            self.generator = Generator(style_dim, resblock_kernel_sizes, upsample_rates, upsample_initial_channel,
                                       resblock_dilation_sizes, upsample_kernel_sizes, gen_istft_n_fft, gen_istft_hop_size)
        else:
            self.generator = HifiGenerator(style_dim, resblock_kernel_sizes, upsample_rates, upsample_initial_channel,
                                           resblock_dilation_sizes, upsample_kernel_sizes)

    def forward(self, asr, F0_curve, N, s, sine_noise=None, har=None):
        B, Ca, T = asr.shape
        dev = asr.device
        s = s.contiguous()
        fcs = StyleFC(self, s)
        # channel concatenation is materialised once per buffer: producers write straight into their
        # channel slice (no torch.cat): cat0 = [asr | F0 | N], catA/B = [x | asr_res | F0 | N]
        cat0 = ops.empty(B, Ca + 2, T, device=dev)
        cat0[:, :Ca].copy_(asr)
        f0c, nc_ = self.F0_conv, self.N_conv
        ops.conv1d(F0_curve.unsqueeze(1), f0c.wt(), f0c.bias, K=3, stride=2, pad=1, out=cat0[:, Ca:Ca + 1])
        ops.conv1d(N.unsqueeze(1), nc_.wt(), nc_.bias, K=3, stride=2, pad=1, out=cat0[:, Ca + 1:Ca + 2])
        Cx = 1024
        Ccat = Cx + 64 + 2
        bufs = [ops.empty(B, Ccat, T, device=dev), ops.empty(B, Ccat, T, device=dev)]
        ar = self.asr_res[0]
        ops.conv1d(cat0[:, :Ca], ar.wt(), ar.bias, K=1, out=bufs[0][:, Cx:Cx + 64], wtc=ar.wtc())
        bufs[0][:, Cx + 64:].copy_(cat0[:, Ca:])
        bufs[1][:, Cx:].copy_(bufs[0][:, Cx:])
        self.encode.run(cat0, fcs, out=bufs[0][:, :Cx])
        cur = 0
        x = None
        for blk in self.decode:
            if blk.has_upsample:
                x = blk.run(bufs[cur], fcs)
            else:
                blk.run(bufs[cur], fcs, out=bufs[1 - cur][:, :Cx])
                cur = 1 - cur
        return self.generator(x, s, F0_curve, sine_noise=sine_noise, har=har, fcs=fcs)
