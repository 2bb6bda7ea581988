"""PL-BERT (phoneme-level ALBERT) on the library's kernels -- SURVEY.md section 8 f1, the first "next" row.

The reference wraps `transformers.AlbertModel` and returns `last_hidden_state` (Utils/PLBERT/util.py:6-12); its
config is Utils/PLBERT/config.yml:23-30 (vocab 178, hidden 768, 12 heads, intermediate 2048, 12 layers sharing ONE
set of weights, embedding size 128, gelu_new, LayerNorm eps 1e-12).  This module keeps AlbertModel's state-dict keys
(so `load_plbert`'s stripped checkpoint loads unchanged) and its call `bert(tokens, attention_mask=(~text_mask).int())`.
Its output feeds the duration path, so every GEMM runs at fp32 accuracy (SIMT fp32 or the 3-plane wgmma GEMM).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops
from .lib import ACT_GELU_TANH, ACT_NONE
from .modules import Linear


class _Cfg:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class _Embeddings(nn.Module):
    def __init__(self, vocab, emb, max_pos, eps):
        super().__init__()
        self.word_embeddings = nn.Embedding(vocab, emb)
        self.position_embeddings = nn.Embedding(max_pos, emb)
        self.token_type_embeddings = nn.Embedding(2, emb)
        self.LayerNorm = nn.LayerNorm(emb, eps=eps)


class _Attention(nn.Module):
    def __init__(self, hidden, eps):
        super().__init__()
        self.query, self.key, self.value = Linear(hidden, hidden), Linear(hidden, hidden), Linear(hidden, hidden)
        self.dense = Linear(hidden, hidden)
        self.LayerNorm = nn.LayerNorm(hidden, eps=eps)


class _Layer(nn.Module):
    def __init__(self, hidden, inter, eps):
        super().__init__()
        self.full_layer_layer_norm = nn.LayerNorm(hidden, eps=eps)
        self.attention = _Attention(hidden, eps)
        self.ffn = Linear(hidden, inter)
        self.ffn_output = Linear(inter, hidden)


class _Group(nn.Module):
    def __init__(self, hidden, inter, eps):
        super().__init__()
        self.albert_layers = nn.ModuleList([_Layer(hidden, inter, eps)])


class _Encoder(nn.Module):
    def __init__(self, emb, hidden, inter, eps):
        super().__init__()
        self.embedding_hidden_mapping_in = Linear(emb, hidden)
        self.albert_layer_groups = nn.ModuleList([_Group(hidden, inter, eps)])


class PLBert(nn.Module):
    """Drop-in for the reference's CustomAlbert: forward(input_ids, attention_mask=None) -> last_hidden_state [B,N,768]."""

    def __init__(self, vocab_size=178, hidden_size=768, num_attention_heads=12, intermediate_size=2048, max_position_embeddings=512,
                 num_hidden_layers=12, embedding_size=128, layer_norm_eps=1e-12, **unused):
        super().__init__()
        assert hidden_size // num_attention_heads == 64, "attention kernel is specialised for 64-wide heads"
        self.config = _Cfg(vocab_size=vocab_size, hidden_size=hidden_size, num_attention_heads=num_attention_heads,
                           intermediate_size=intermediate_size, max_position_embeddings=max_position_embeddings,
                           num_hidden_layers=num_hidden_layers, embedding_size=embedding_size, layer_norm_eps=layer_norm_eps)
        self.embeddings = _Embeddings(vocab_size, embedding_size, max_position_embeddings, layer_norm_eps)
        self.encoder = _Encoder(embedding_size, hidden_size, intermediate_size, layer_norm_eps)
        self.pooler = nn.Linear(hidden_size, hidden_size)   # present in the checkpoint; unused for last_hidden_state

    def _qkv(self):
        att = self.encoder.albert_layer_groups[0].albert_layers[0].attention
        key = tuple((p.data_ptr(), p._version) for p in (att.query.weight, att.key.weight, att.value.weight))
        c = self.__dict__.get("_qkv_cache")
        if c is None or c[0] != key:
            with torch.no_grad():
                W = torch.cat([att.query.weight, att.key.weight, att.value.weight], 0).contiguous()
                b = torch.cat([att.query.bias, att.key.bias, att.value.bias], 0).contiguous()
                wtc = ops.linear_tc_weight_layout(W) if (ops.USE_TC and W.is_cuda) else None
            c = (key, W, b, wtc)
            self.__dict__["_qkv_cache"] = c
        return c[1], c[2], c[3]

    @torch.no_grad()
    def forward(self, input_ids, attention_mask=None, **unused):
        cfg = self.config
        emb = self.embeddings
        dev = emb.word_embeddings.weight.device
        tokens = input_ids.to(dev).contiguous()
        B, N = tokens.shape
        assert N <= cfg.max_position_embeddings
        lengths = None
        if attention_mask is not None:
            # the reference passes a prefix mask (~length_to_mask).int(): keys beyond each length are excluded
            lengths = attention_mask.to(dev).to(torch.int32).sum(dim=1).to(torch.int32).contiguous()
        E, Hd = cfg.embedding_size, cfg.hidden_size
        e = ops.empty(B * N, E, device=dev)
        ops.L.call("st2_embedding_sum_rows", ops.ptr(tokens), ops.ptr(emb.word_embeddings.weight), ops.ptr(emb.position_embeddings.weight),
                   ops.ptr(emb.token_type_embeddings.weight), B, N, E, ops.ptr(e), ops.stream_ptr())
        en = ops.empty(B * N, E, device=dev)
        ops.rows_ln(B=B, N=N, Cw=E, h_in=e, g1=emb.LayerNorm.weight, b1=emb.LayerNorm.bias, out1=en, eps=cfg.layer_norm_eps)
        h = self.encoder.embedding_hidden_mapping_in(en)                      # [M,768]
        layer = self.encoder.albert_layer_groups[0].albert_layers[0]
        att = layer.attention
        Wqkv, bqkv, wtc = self._qkv()
        H, D = cfg.num_attention_heads, Hd // cfg.num_attention_heads
        M = B * N
        for _ in range(cfg.num_hidden_layers):
            use = wtc if M >= ops.LINEAR_TC_MIN_ROWS else None
            qkv = ops.linear(h, Wqkv, bqkv, wtc=use)                          # [M, 3*768] = q | k | v
            ctx = ops.empty(M, Hd, device=dev)
            ops.attention_ex(qkv[:, :Hd], qkv[:, Hd:2 * Hd], qkv[:, 2 * Hd:], ctx, B, N, H, D, lengths)
            y = att.dense(ctx, R=h)                                           # hidden + dense(attn)
            a_out = ops.empty(M, Hd, device=dev)
            ops.rows_ln(B=B, N=N, Cw=Hd, h_in=y, g1=att.LayerNorm.weight, b1=att.LayerNorm.bias, out1=a_out, eps=cfg.layer_norm_eps)
            f = layer.ffn(a_out, act=ACT_GELU_TANH)
            y2 = layer.ffn_output(f, R=a_out)
            h = ops.empty(M, Hd, device=dev)
            ops.rows_ln(B=B, N=N, Cw=Hd, h_in=y2, g1=layer.full_layer_layer_norm.weight, b1=layer.full_layer_layer_norm.bias, out1=h,
                        eps=cfg.layer_norm_eps)
        return h.view(B, N, Hd)


def load_plbert_state(bert: PLBert, checkpoint_net: dict):
    """Utils/PLBERT/util.py:30-40: strip `module.` and `encoder.` prefixes, drop position_ids, strict=False."""
    new = {}
    for k, v in checkpoint_net.items():
        name = k[7:] if k.startswith("module.") else k
        if name.startswith("encoder."):
            name = name[8:]
            if name != "embeddings.position_ids":
                new[name] = v
    bert.load_state_dict(new, strict=False)
    return bert
