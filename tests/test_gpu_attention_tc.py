"""GPU tier: the wgmma attention kernel (csrc/attention_tc.cu: QK^T and PV on the tensor cores, S / O in registers, fp16
two-plane split with separate correction accumulators) against a float64 reference, next to the fp32 SIMT kernel: the
durations are downstream of the denoiser, so the bar is fp32 accuracy (modules.py:523-535; PL-BERT key-padding mask)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from util import record

D = "cuda:0"


def _ref(q, k, v, B, N, H, Dh, lengths=None):
    qh = q.double().view(B, N, H, Dh).permute(0, 2, 1, 3)
    kh = k.double().view(B, N, H, Dh).permute(0, 2, 1, 3)
    vh = v.double().view(B, N, H, Dh).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * Dh ** -0.5
    if lengths is not None:
        mask = torch.arange(N)[None, :] >= lengths[:, None]
        s = s.masked_fill(mask[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vh).permute(0, 2, 1, 3).reshape(B * N, H * Dh)


@pytest.mark.parametrize("B,N,H,masked,scale", [(2, 128, 8, False, 1.0), (3, 40, 8, False, 1.0), (2, 200, 8, False, 3.0), (2, 512, 8, False, 1.0),
                                                (3, 145, 12, True, 2.0), (2, 500, 12, True, 1.0), (32, 128, 8, False, 1.0)])
def test_attention_tc_matches_float64(B, N, H, masked, scale):
    from styletts2_b200 import ops
    Dh = 64
    g = torch.Generator().manual_seed(N * 7 + H)
    qkv = torch.randn(B * N, 3 * H * Dh, generator=g) * scale          # one buffer, strided q | k | v views (PL-BERT layout)
    lengths = torch.tensor([N] + [max(5, N - 37 * (i + 1)) for i in range(B - 1)]) if masked else None
    q, k, v = qkv[:, :H * Dh], qkv[:, H * Dh:2 * H * Dh], qkv[:, 2 * H * Dh:]
    ref = _ref(q, k, v, B, N, H, Dh, lengths)
    d = qkv.to(D)
    ld = None if lengths is None else lengths.to(D, torch.int32)
    outs = {}
    for name, tc in (("tc", True), ("simt", False)):
        ops.ATT_TC = tc
        try:
            out = torch.full((B * N, H * Dh), float("nan"), device=D)
            ops.attention_ex(d[:, :H * Dh], d[:, H * Dh:2 * H * Dh], d[:, 2 * H * Dh:], out, B, N, H, Dh, ld)
            outs[name] = out.cpu().double()
        finally:
            ops.ATT_TC = True
    valid = torch.ones(B, N, dtype=torch.bool) if lengths is None else (torch.arange(N)[None] < lengths[:, None])
    valid = valid.reshape(-1)
    peak = float(ref[valid].abs().max())
    e_tc = float((outs["tc"] - ref)[valid].abs().max()) / peak
    e_simt = float((outs["simt"] - ref)[valid].abs().max()) / peak
    record("attention_tc", B=B, N=N, H=H, masked=masked, scale=scale, rel_err_tc=e_tc, rel_err_simt=e_simt)
    assert torch.isfinite(outs["tc"][valid]).all()
    assert e_tc < 2e-6, (e_tc, e_simt)


def test_denoiser_attention_entry_uses_the_tensor_core_kernel():
    from styletts2_b200 import lib, ops
    B, N, H, Dh = 4, 128, 8, 64
    g = torch.Generator().manual_seed(0)
    q, kv = torch.randn(B * N, H * Dh, generator=g), torch.randn(B * N, 2 * H * Dh, generator=g)
    ref = _ref(q, kv[:, :H * Dh], kv[:, H * Dh:], B, N, H, Dh)
    ops.PROFILE = []
    try:
        y = ops.attention(q.to(D), kv.to(D), B, N, H, Dh)
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert names and names[0].startswith("attention_tc"), names
    assert float((y.cpu().double() - ref).abs().max()) / float(ref.abs().max()) < 2e-6
