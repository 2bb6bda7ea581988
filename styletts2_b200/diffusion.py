"""Style-diffusion side: denoiser transformer and the EDM sampler, same names/signatures as
Modules/diffusion/{modules,sampler,diffusion}.py of the reference.

Mirrored: Transformer1d (modules.py:283-427), StyleTransformer1d (:40-185), TransformerBlock /
StyleTransformerBlock, Attention / StyleAttention / AttentionBase (:236-281,493-584), FeedForward
(:484-490), LearnedPositionalEmbedding / TimePositionalEmbedding / FixedEmbedding (:657-693),
KDiffusion (sampler.py:165-234), KarrasSchedule (:319-337), ADPM2Sampler (:481-519),
DiffusionSampler (:550-586), AudioDiffusionConditional (diffusion.py:66-94, container only).
"""
from __future__ import annotations

import math
from math import sqrt
from typing import Optional

import torch
import torch.nn as nn

from . import ops
from .lib import ACT_GELU, ACT_NONE
from .modules import AdaLayerNorm, Conv1d, Linear


class LearnedPositionalEmbedding(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        assert dim % 2 == 0
        self.weights = nn.Parameter(torch.randn(dim // 2))


class FixedEmbedding(nn.Module):
    def __init__(self, max_length: int, features: int):
        super().__init__()
        self.max_length = max_length
        self.embedding = nn.Embedding(max_length, features)

    def forward(self, x):
        B, N = x.shape[0], x.shape[1]
        assert N <= self.max_length, "Input sequence length must be <= max_length"
        return self.embedding.weight[:N].unsqueeze(0).expand(B, -1, -1)


class TokenPacking:
    """Packed token rows of a batch: only the valid rows of every utterance, concatenated (varlen layout).  Utterance b
    owns rows offsets[b] .. offsets[b+1]-1; row r belongs to utterance row_utt[r] at position pos[r].  The denoiser run on
    this layout confines attention and the token mean to each utterance's own rows, so every utterance gets the style it
    gets when it runs alone, whatever the other token counts of the batch."""

    def __init__(self, lengths, device):
        lengths = [int(n) for n in lengths]
        assert lengths and min(lengths) >= 1, lengths
        self.lengths = lengths
        self.B, self.M, self.max_len = len(lengths), sum(lengths), max(lengths)
        offs = [0]
        for n in lengths:
            offs.append(offs[-1] + n)
        utt = torch.repeat_interleave(torch.arange(self.B), torch.tensor(lengths))
        pos = torch.cat([torch.arange(n) for n in lengths])
        self.offsets = torch.tensor(offs, dtype=torch.int32).to(device)
        self.row_utt = utt.to(device=device, dtype=torch.int32)
        self._utt, self._pos = utt.to(device), pos.to(device)

    def pack(self, x):
        """[B, N, ...] (N >= every length) -> [M, ...] contiguous: the valid rows, utterance after utterance"""
        return x[self._utt, self._pos].contiguous()

    def pack_positions(self, table):
        """[L, ...] per-position table -> [M, ...]: row r takes table[r - offsets[b]] (the fixed embedding under guidance)"""
        assert self.max_len <= table.shape[0], "Input sequence length must be <= max_length"
        return table[self._pos].contiguous()


class AttentionBase(nn.Module):
    def __init__(self, features, *, head_features, num_heads, out_features=None):
        super().__init__()
        self.scale = head_features ** -0.5
        self.num_heads, self.head_features = num_heads, head_features
        self.to_out = Linear(head_features * num_heads, out_features or features)


class Attention(nn.Module):
    """pre-LN self attention (modules.py:538-584); style=True gives StyleAttention (:236-281)."""

    def __init__(self, features, *, head_features, num_heads, style_dim=None):
        super().__init__()
        mid = head_features * num_heads
        if style_dim is None:
            self.norm = nn.LayerNorm(features)
            self.norm_context = nn.LayerNorm(features)
        else:
            self.norm = AdaLayerNorm(style_dim, features)
            self.norm_context = AdaLayerNorm(style_dim, features)
        self.to_q = Linear(features, mid, bias=False)
        self.to_kv = Linear(features, mid * 2, bias=False)
        self.attention = AttentionBase(features, num_heads=num_heads, head_features=head_features)


class TransformerBlock(nn.Module):
    def __init__(self, features, num_heads, head_features, multiplier, style_dim=None):
        super().__init__()
        self.attention = Attention(features, num_heads=num_heads, head_features=head_features, style_dim=style_dim)
        mid = features * multiplier
        self.feed_forward = nn.Sequential(Linear(features, mid), nn.GELU(), Linear(mid, features))


class Transformer1d(nn.Module):
    """forward(x [B,1,256], time [B], embedding=[B,N,768], features=[B,256]|None, embedding_scale) -> [B,1,256]"""

    def __init__(self, num_layers, channels, num_heads, head_features, multiplier, use_context_time=True, use_rel_pos=False,
                 context_features_multiplier=1, rel_pos_num_buckets=None, rel_pos_max_distance=None, context_features=None,
                 context_embedding_features=None, embedding_max_length=512, _style=False):
        super().__init__()
        assert not use_rel_pos, "relative position bias is dead code in the reference configs (SURVEY section 2)"
        feats = channels + context_embedding_features
        self.channels, self.features = channels, feats
        self.num_heads, self.head_features = num_heads, head_features
        self.style = _style
        self.blocks = nn.ModuleList([TransformerBlock(feats, num_heads, head_features, multiplier,
                                                      style_dim=context_features if _style else None)
                                     for _ in range(num_layers)])
        self.to_out = nn.Sequential(nn.Identity(), Conv1d(feats, channels, 1))
        self.use_context_features = context_features is not None
        self.to_mapping = nn.Sequential(Linear(feats, feats), nn.GELU(), Linear(feats, feats), nn.GELU())
        self.to_time = nn.Sequential(nn.Sequential(LearnedPositionalEmbedding(channels), Linear(channels + 1, feats)), nn.GELU())
        if self.use_context_features:
            self.to_features = nn.Sequential(Linear(context_features, feats), nn.GELU())
        self.fixed_embedding = FixedEmbedding(max_length=embedding_max_length, features=context_embedding_features)

    def get_mapping(self, time, features=None):
        emb = ops.time_embedding(time, self.to_time[0][0].weights)
        m = self.to_time[0][1](emb, act=ACT_GELU)
        if self.use_context_features:
            assert features is not None, "context_features exists but no features provided"
            m = ops.axpby(m, 1.0, self.to_features[0](features.contiguous(), act=ACT_GELU), 1.0)
        m = self.to_mapping[0](m, act=ACT_GELU)
        return self.to_mapping[2](m, act=ACT_GELU)

    def run(self, x, time, embedding, features, packed=None):
        """embedding [B, N, E]; or, with packed = (offsets, row_utt, max_len), the packed token rows [M, E] of a
        TokenPacking (see run_packed)"""
        H, D = self.num_heads, self.head_features
        if packed is None:
            B, N, E = embedding.shape
            M = B * N
            emb = embedding if embedding.stride(-1) == 1 and embedding.stride(0) == N * embedding.stride(1) else embedding.contiguous()
            rows_ln = lambda **kw: ops.rows_ln(B=B, N=N, **kw)                   # noqa: E731
            attention = lambda q, kv: ops.attention(q, kv, B, N, H, D)           # noqa: E731
            mean = lambda h: ops.mean_rows(h, B, N)                              # noqa: E731
        else:
            offsets, row_utt, max_len = packed
            M, E = embedding.shape
            B = offsets.shape[0] - 1
            emb = embedding if embedding.stride(-1) == 1 else embedding.contiguous()
            rows_ln = lambda **kw: ops.rows_ln_packed(row_utt=row_utt, M=M, B=B, **kw)             # noqa: E731
            attention = lambda q, kv: ops.attention_packed(q, kv, offsets, B, max_len, H, D)     # noqa: E731
            mean = lambda h: ops.mean_segments(h, offsets, B)                                    # noqa: E731
        dev = embedding.device
        Cw = self.features
        mapping = self.get_mapping(time, features)
        x2 = x.reshape(B, self.channels).contiguous()
        h = ops.empty(M, Cw, device=dev)
        a = ops.empty(M, Cw, device=dev)
        c = ops.empty(M, Cw, device=dev)
        feats = features.contiguous() if features is not None else None
        for i, blk in enumerate(self.blocks):
            att = blk.attention
            if self.style:
                gb1, gb2 = att.norm.fc(feats), att.norm_context.fc(feats)
                kw = dict(g1=gb1, b1=gb1[:, Cw:], g2=gb2, b2=gb2[:, Cw:], gb_bstride=gb1.stride(0), ada=True)
            else:
                kw = dict(g1=att.norm.weight, b1=att.norm.bias, g2=att.norm_context.weight, b2=att.norm_context.bias)
            if i == 0:
                rows_ln(Cw=Cw, x=x2, xs=1.0, emb=emb, add=mapping, h_out=h, out1=a, out2=c, eps=1e-5, **kw)
            else:
                rows_ln(Cw=Cw, h_in=h, add=mapping, h_out=h, out1=a, out2=c, eps=1e-5, **kw)
            q = att.to_q(a)
            kv = att.to_kv(c)
            o = attention(q, kv)
            att.attention.to_out(o, R=h, out=h)
            f = blk.feed_forward[0](h, act=ACT_GELU)
            blk.feed_forward[2](f, R=h, out=h)
        hm = mean(h)
        conv = self.to_out[1]
        out = ops.linear(hm, conv.weight.view(conv.cout, conv.cin), conv.bias)
        return out.view(B, 1, self.channels)

    def run_packed(self, x, time, embedding, features, offsets, row_utt, max_len):
        """x [B,1,C], embedding [M,E] packed token rows (TokenPacking.pack), offsets int32 [B+1], row_utt int32 [M] ->
        [B,1,C]: each utterance attends over and averages its own rows only (the single-utterance result)"""
        return self.run(x, time, embedding, features, packed=(offsets, row_utt, max_len))

    def forward(self, x, time, embedding_mask_proba: float = 0.0, embedding=None, features=None, embedding_scale: float = 1.0):
        assert embedding_mask_proba == 0.0, "inference path only (no conditional dropout)"
        if embedding_scale != 1.0:
            fixed = self.fixed_embedding(embedding).contiguous()
            out = self.run(x, time, embedding, features)
            out_masked = self.run(x, time, fixed, features)
            # out_masked + (out - out_masked) * scale, fused into the sampler step when driven by
            # DiffusionSampler; standalone callers get it here
            return ops.kdiff_combine(out, out_masked, embedding_scale)
        return self.run(x, time, embedding, features)


class StyleTransformer1d(Transformer1d):
    def __init__(self, *a, **kw):
        super().__init__(*a, _style=True, **kw)


# ------------------------------------------------------------------------------------------ sampler side
class LogNormalDistribution:
    def __init__(self, mean: float, std: float):
        self.mean, self.std = mean, std


class KDiffusion(nn.Module):
    """sampler.py:165-234 (inference half: get_scale_weights, denoise_fn)."""
    alias = "k"

    def __init__(self, net, *, sigma_distribution=None, sigma_data: float, dynamic_threshold: float = 0.0):
        super().__init__()
        self.net = net
        self.sigma_data = sigma_data
        self.sigma_distribution = sigma_distribution
        self.dynamic_threshold = dynamic_threshold

    def scale_weights_host(self, sigma):
        """get_scale_weights evaluated with the reference's fp32 tensor arithmetic on the host
        (sampler.py:184-191); sigma: 0-dim fp32 CPU tensor or float."""
        sd = self.sigma_data
        sigmas = torch.full((1,), float(sigma), dtype=torch.float32)
        c_noise = torch.log(sigmas) * 0.25
        sg = sigmas.view(1, 1, 1)
        c_skip = (sd ** 2) / (sg ** 2 + sd ** 2)
        c_out = sg * sd * (sd ** 2 + sg ** 2) ** -0.5
        c_in = (sg ** 2 + sd ** 2) ** -0.5
        return float(c_skip), float(c_out), float(c_in), float(c_noise[0])

    def denoise_fn(self, x_noisy, sigmas=None, sigma=None, **kwargs):
        assert (sigma is None) != (sigmas is None), "Either sigma or sigmas must be provided"
        if sigma is None:
            s0 = float(sigmas.flatten()[0])
            assert bool((sigmas == s0).all()), "per-utterance sigmas are not used on the inference path"
            sigma = s0
        c_skip, c_out, c_in, c_noise = self.scale_weights_host(sigma)
        B = x_noisy.shape[0]
        xin = ops.scale(x_noisy, c_in)
        t = torch.full((B,), c_noise, device=x_noisy.device, dtype=torch.float32)
        x_pred = self.net(xin, t, **kwargs)
        return ops.axpby(x_noisy, c_skip, x_pred.reshape(x_noisy.shape), c_out)


class AudioDiffusionConditional(nn.Module):
    """Container whose .diffusion / .unet are overwritten by build_model (models.py:653-669)."""

    def __init__(self, **kw):
        super().__init__()
        self.unet = None
        self.diffusion = None


class Schedule(nn.Module):
    pass


class KarrasSchedule(Schedule):
    """sampler.py:319-337 (evaluated on the host: K+1 scalars)."""

    def __init__(self, sigma_min: float, sigma_max: float, rho: float = 7.0):
        super().__init__()
        self.sigma_min, self.sigma_max, self.rho = sigma_min, sigma_max, rho

    def forward(self, num_steps: int, device=None):
        rho_inv = 1.0 / self.rho
        steps = torch.arange(num_steps, dtype=torch.float32)
        sigmas = (self.sigma_max ** rho_inv + (steps / (num_steps - 1)) * (self.sigma_min ** rho_inv - self.sigma_max ** rho_inv)) ** self.rho
        return torch.nn.functional.pad(sigmas, pad=(0, 1), value=0.0)


class Sampler(nn.Module):
    diffusion_types = [KDiffusion]


class ADPM2Sampler(Sampler):
    """sampler.py:481-519."""

    def __init__(self, rho: float = 1.0):
        super().__init__()
        self.rho = rho

    def get_sigmas(self, sigma, sigma_next):
        r = self.rho
        sigma_up = sqrt(sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2)
        sigma_down = sqrt(sigma_next ** 2 - sigma_up ** 2)
        sigma_mid = ((sigma ** (1 / r) + sigma_down ** (1 / r)) / 2) ** r
        return sigma_up, sigma_down, sigma_mid

    def forward(self, noise, fn, sigmas, num_steps, step_noises=None):
        """fn: a _DenoiseEval (fused path).  sigmas: CPU fp32 tensor."""
        x = ops.scale(noise, float(sigmas[0]))
        for i in range(num_steps - 1):
            sigma, sigma_next = sigmas[i], sigmas[i + 1]
            sigma_up, sigma_down, sigma_mid = self.get_sigmas(sigma, sigma_next)
            dt_mid = float(sigma_mid - sigma)          # fp32 tensor arithmetic, as the reference
            dt_down = float(sigma_down - sigma)        # python float - fp32 tensor -> fp32 tensor
            eps = step_noises[i] if step_noises is not None else ops.randn_like(x)
            x_mid = fn.step(x, float(sigma), x, dt_mid)
            x = fn.step(x_mid, float(sigma_mid), x, dt_down, eps=eps, sigma_up=float(torch.tensor(sigma_up, dtype=torch.float32)))
        return x


class _DenoiseEval:
    """One denoiser evaluation + the elementwise half step, fused (sampler.py:193-208,499-510)."""

    def __init__(self, diffusion: KDiffusion, kwargs):
        self.kd, self.kw = diffusion, kwargs
        self.packing = kwargs.get("packing")        # TokenPacking: `embedding` holds its packed rows [M, 768]
        self.fixed_packed = None
        if self.packing is not None and kwargs.get("embedding_scale", 1.0) != 1.0:
            self.fixed_packed = self.packing.pack_positions(diffusion.net.fixed_embedding.embedding.weight)

    def step(self, x_eval, sigma_eval, x_base, dt, eps=None, sigma_up=0.0):
        kd = self.kd
        c_skip, c_out, c_in, c_noise = kd.scale_weights_host(sigma_eval)
        B = x_eval.shape[0]
        xin = ops.scale(x_eval, c_in)
        t = torch.full((B,), c_noise, device=x_eval.device, dtype=torch.float32)
        net = kd.net
        emb, feats = self.kw.get("embedding"), self.kw.get("features")
        scale = self.kw.get("embedding_scale", 1.0)
        pk = self.packing
        if pk is not None:
            packed = (pk.offsets, pk.row_utt, pk.max_len)
            pred = net.run_packed(xin, t, emb, feats, *packed)
            masked = None
            if scale != 1.0:
                masked = net.run_packed(xin, t, self.fixed_packed, feats, *packed)
        else:
            pred = net.run(xin, t, emb, feats)
            masked = None
            if scale != 1.0:
                masked = net.run(xin, t, net.fixed_embedding(emb).contiguous(), feats)
        return ops.kdiff_step(x_eval, pred.reshape(x_eval.shape), c_skip, c_out, float(torch.tensor(sigma_eval, dtype=torch.float32)),
                              x_base, dt, eps=eps, sigma_up=sigma_up,
                              x_pred_masked=None if masked is None else masked.reshape(x_eval.shape), cfg_scale=scale)


class DiffusionSampler(nn.Module):
    """sampler.py:550-586.  forward(noise [B,1,256], num_steps, embedding=..., embedding_scale=..., features=...)"""

    def __init__(self, diffusion, *, sampler, sigma_schedule, num_steps: Optional[int] = None, clamp: bool = True):
        super().__init__()
        self.diffusion = diffusion
        self.denoise_fn = diffusion.denoise_fn
        self.sampler = sampler
        self.sigma_schedule = sigma_schedule
        self.num_steps = num_steps
        self.clamp = clamp
        assert diffusion.alias in [t.alias for t in sampler.diffusion_types]

    def forward(self, noise, num_steps: Optional[int] = None, step_noises=None, **kwargs):
        num_steps = num_steps if num_steps is not None else self.num_steps
        assert num_steps is not None, "Parameter `num_steps` must be provided"
        sigmas = self.sigma_schedule(num_steps, "cpu")
        fn = _DenoiseEval(self.diffusion, kwargs)
        x = self.sampler(noise.contiguous(), fn=fn, sigmas=sigmas, num_steps=num_steps, step_noises=step_noises)
        return x.clamp(-1.0, 1.0) if self.clamp else x
