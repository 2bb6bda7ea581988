"""CPU tier: the recipe-exact references of the tensor-core GEMM and attention (oracle/tc_recipes.py) and the power of the
GPU test that compares the kernels with them (tests/test_gpu_linear_attention_tc.py).

The metric there is max |y - y_ref| / (2^-20 scale) per output element, bounded by LINEAR_BOUND_C / ATTENTION_BOUND_C.  Here
each defect a kernel could plausibly have -- a correction product lost on one K block or one 16-wide step, P's low plane
lost on the last key block, S's correction lost on one 16-wide d step, a mask off by one -- is modelled in the reference
and must score at least ten times the bound on the operand sets the GPU test uses."""
import pytest
import torch

import tc_recipes as R

# (M, K, Nf) of the GPU test's localised-contraction cases (the call sites and the tails)
from test_gpu_linear_attention_tc import ATT_CASES, GEMM_CASES, GEMM_TAILS  # noqa: E402

SCALE = 0.125    # 64 ** -0.5


def test_two_planes_hold_every_fp32_in_the_fp16_range():
    """h + l * 2^-11 == x to 2^-22 |x| for every |x| from 2^-14 to the fp16 limit.  The 2^11 pre-scaling is what keeps the
    low plane's rounding at that level: without it, l = fp16(x - h) falls below fp16's normal range from |x| < 2^-3 on."""
    g = torch.Generator().manual_seed(0)
    e = torch.rand(200000, generator=g) * 29.99 - 14                              # 2^-14 .. 2^15.99
    x = (2.0 ** e * (torch.randint(0, 2, e.shape, generator=g) * 2 - 1)).float()
    edges = torch.tensor([2.0 ** -14, 2.0 ** -14 * (1 + 2.0 ** -23), 65503.0, 65504.0 - 2.0 ** -8, 1.0 + 2.0 ** -12, 3.0 * 2.0 ** -13])
    x = torch.cat([x, edges.float(), -edges.float()])
    h, l = R.split2(x)
    assert torch.isfinite(h).all() and torch.isfinite(l).all()
    err = (h + l / R.LO_SCALE - x.double()).abs()
    assert float((err / x.double().abs()).max()) <= 2.0 ** -22
    # the planes are what the kernels' __floats2half2_rn forms: round-to-nearest-even of the exact fp32 values
    assert torch.equal(h, x.half().double()) and torch.equal(l, ((x - x.half().float()) * 2048).half().double())


def _gemm_subset(M, K, Nf, seed):
    """the GPU case's operands, restricted to rows that cover every K block three times, four dense rows and 64 features
    (a defect's score on a subset is a lower bound of its score on the whole case)"""
    a, w, _, _ = R.linear_operands(M, K, Nf, seed=seed)
    ncb = (K + R.GEMM_KB - 1) // R.GEMM_KB
    rows = torch.cat([torch.arange(min(M, 3 * ncb)), torch.arange(7, M, 61)[:4]])
    return a[rows], w[:64]


def _score(y, ref, scale):
    return float(((y - ref).abs() / (scale * 2.0 ** -20)).max())


@pytest.mark.parametrize("M,K,Nf", [c[:3] for c in GEMM_CASES + GEMM_TAILS])
def test_gemm_reference_is_fp64_accurate_and_its_defects_score_far_above_the_bound(M, K, Nf):
    a, w = _gemm_subset(M, K, Nf, seed=K)
    ref, scale = R.linear(a, w), R.sum_abs_linear(a, w)
    exact = _score(a.double() @ w.double().T, ref, scale)
    assert exact <= 0.5, exact                                     # within 2^-21 sum|a||w| of fp64
    ncb, nks = (K + R.GEMM_KB - 1) // R.GEMM_KB, (K + 15) // 16
    c = R.LINEAR_BOUND_C
    scores = {}
    for cb in sorted({0, ncb // 2, ncb - 1}):
        scores[f"hl block {cb}"] = _score(R.linear(a, w, drop_hl_block=cb), ref, scale)
    for st in sorted({0, nks // 2, nks - 1}):
        scores[f"lh step {st}"] = _score(R.linear(a, w, drop_lh_step=st), ref, scale)
    print(f"GEMM M{M} K{K} N{Nf}: c = {c}, weakest defect {min(scores.values()):.1f}", scores)
    assert all(s >= 10 * c for s in scores.values()), (c, scores)


@pytest.mark.parametrize("B,N,H,lengths", ATT_CASES)
def test_attention_defects_score_far_above_the_bound(B, N, H, lengths):
    """Per GPU case: B utterances with these key lengths (one head pair kept here); the defect-free recipe scores well
    below the bound (what is left for the kernel's fp32 accumulation), every defect at least ten times above it."""
    L = torch.tensor(lengths)
    q, k, v = R.attention_operands(B, N, H, L, seed=N)
    q, k, v = q[:, :, :2], k[:, :, :2], v[:, :, :2]
    o, E = R.attention_bound(q, k, v, L, SCALE)
    c = R.ATTENTION_BOUND_C
    score = lambda m: _score(R.attention_bound(q, k, v, L, SCALE, mutation=m)[0], o, E)   # noqa: E731
    honest = score("recipe")
    assert honest < c / 2, (honest, c)
    scores = {"p_low_last_block": score("p_low_last_block"), "mask_plus_one": score("mask_plus_one")}
    for i in range(4):
        scores[f"s_corr_step {i}"] = score(("s_corr_step", i))
    print(f"attention B{B} N{N} H{H}: c = {c}, recipe {honest:.2f}, weakest defect {min(scores.values()):.1f}", scores)
    if all(x >= N for x in lengths):
        scores.pop("mask_plus_one")                                # no key beyond the length to admit
    assert all(s >= 10 * c for s in scores.values()), (c, scores)
