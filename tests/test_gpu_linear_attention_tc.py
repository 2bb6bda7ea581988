"""GPU tier: the tensor-core GEMM (csrc/linear_tc.cu) and attention (csrc/attention_tc.cu) per output element, against the
recipe-exact references of oracle/tc_recipes.py, at the shapes and layouts of their call sites.

GEMM: |y - linear(a, w, bias)| <= LINEAR_BOUND_C * 2^-20 * (sum|a||w| + |bias| + |R|) on localised operands (every output is
dominated by one 32-wide K block), bit-identical results across the pre-split, on-the-fly and raw entry paths and across
strided / misaligned / in-place layouts, the epilogue activations against float64, and the fp16 range guard.
Attention: |o - o_ref| <= ATTENTION_BOUND_C * 2^-20 * E (tc_recipes.attention_bound) at the 64-query / 128-key block
edges, on peaked softmaxes and with every valid logit far below the masked keys' zero, bit-identical layouts, the SIMT
dispatch, and the range guard.  tests/test_cpu_gemm_attention_recipe.py shows each bound rejects the defects it targets."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import tc_recipes as R
from util import record

D = "cuda:0"
SCALE = 0.125    # 64 ** -0.5

# (M, K, Nf, call site) -- C2 shapes (M = 4096 rows unless noted); "inplace" cases write out = R = the residual stream
GEMM_CASES = [
    (4096, 1024, 512, "denoiser to_q"),
    (4096, 1024, 1024, "denoiser to_kv"),
    (4096, 512, 1024, "denoiser to_out inplace"),
    (4096, 1024, 2048, "denoiser ff0"),
    (4096, 2048, 1024, "denoiser ff2 inplace"),
    (4096, 768, 2304, "plbert qkv bias"),
    (4096, 768, 2048, "plbert ffn"),
    (4096, 2048, 768, "plbert ffn_output"),
    (4096, 128, 768, "plbert embedding mapping"),
    (4096, 640, 2048, "lstm input projection raw"),
    (1000, 1200, 2050, "mel dft"),
]
GEMM_TAILS = [(M, K, Nf, "tail") for K in (1, 16, 31, 33) for M, Nf in ((256, 1), (257, 127), (319, 129))]

# (B, N, H, key lengths): the 64-query / 128-key block edges; one length > N (clamped by the kernels)
_LENS = (1, 2, 63, 64, 65, 127, 128, 129)
ATT_CASES = [(len(ls), n, 8 if i % 2 == 0 else 12, ls) for i, (n, ls) in enumerate(
    (n, sorted({x for x in _LENS + (n - 1, n) if 1 <= x <= n}) + [n + 7]) for n in (32, 63, 64, 65, 127, 128, 129, 255, 256, 257, 512))]
ATT_CASES.append((32, 128, 8, [128 - 3 * i for i in range(32)]))                    # B = 32


def _bound_err(y, ref, scale):
    return float(((y - ref).abs() / (scale * 2.0 ** -20)).max())


def _gemm(ops, path, A, W, wtc, bias=None, R_=None, out=None, act=0):
    """one GEMM on the tensor cores: 'presplit' / 'fly' through ops.linear with LINEAR_TC_PRESPLIT on / off (Nf <= 128
    never pre-splits there, so 'presplit' calls st2_linear_tc_split + st2_linear_tc_pre itself), 'raw' = st2_linear_tc as
    the LSTM calls it"""
    M, K = A.shape
    Nf = W.shape[0]
    if out is None:
        out = torch.empty(M, Nf, device=D)
    ldr = R_.stride(0) if R_ is not None else 0
    if path == "raw" or (path == "presplit" and Nf <= 128):
        if path == "raw":
            ops.L.call("st2_linear_tc", ops.ptr(A), A.stride(0), ops.ptr(wtc), ops.ptr(bias), ops.ptr(R_), ldr, ops.ptr(out),
                       out.stride(0), M, Nf, K, act, ops.stream_ptr())
        else:
            planes = torch.empty(int(ops.L.load().st2_linear_tc_split_bytes(M, K)), dtype=torch.uint8, device=D)
            ops.L.call("st2_linear_tc_split", ops.ptr(A), A.stride(0), M, K, ops.ptr(planes), ops.stream_ptr())
            ops.L.call("st2_linear_tc_pre", ops.ptr(A), A.stride(0), ops.ptr(planes), ops.ptr(wtc), ops.ptr(bias), ops.ptr(R_), ldr,
                       ops.ptr(out), out.stride(0), M, Nf, K, act, ops.stream_ptr())
        return out
    old = ops.LINEAR_TC_PRESPLIT
    ops.LINEAR_TC_PRESPLIT = path == "presplit"
    try:
        return ops.linear(A, W, bias, act=act, R=R_, out=out, wtc=wtc)
    finally:
        ops.LINEAR_TC_PRESPLIT = old


@pytest.fixture(scope="module")
def ops():
    from styletts2_b200 import ops as o
    o.check_range()
    yield o
    o.check_range()


# ------------------------------------------------------------------ GEMM 1+2: localised contraction, every entry path
@pytest.mark.parametrize("M,K,Nf,site", GEMM_CASES + GEMM_TAILS)
def test_linear_tc_matches_recipe_reference_on_every_path(M, K, Nf, site, ops):
    a, w, b, r = R.linear_operands(M, K, Nf, seed=K, bias="bias" in site, residual="inplace" in site)
    A, W = a.to(D), w.to(D)
    bd = b.to(D) if b is not None else None
    wtc = ops.linear_tc_weight_layout(W)
    outs = {}
    for path in ("presplit", "fly", "raw"):
        if r is not None and path != "raw":
            out = r.to(D)                                          # in place: R and out are one buffer
            outs[path] = _gemm(ops, path, A, W, wtc, bd, out, out)
        else:
            outs[path] = _gemm(ops, path, A, W, wtc, bd, r.to(D) if r is not None else None)
    for path in ("fly", "raw"):
        assert torch.equal(outs["presplit"], outs[path]), (site, path)
    ref = R.linear(A, W, bd)
    scale = R.sum_abs_linear(A, W, bd)
    if r is not None:
        ref, scale = ref + r.to(D).double(), scale + r.to(D).double().abs()
    e = _bound_err(outs["presplit"].double(), ref, scale)
    record("linear_tc_recipe", M=M, K=K, Nf=Nf, site=site, bound_err=e)
    ops.check_range()
    assert math.isfinite(e) and e <= R.LINEAR_BOUND_C, (site, e)


# ------------------------------------------------------------------ GEMM 3: layouts
@pytest.mark.parametrize("M,K,Nf", [(300, 200, 200), (257, 1200, 2050), (260, 96, 100)])
@pytest.mark.parametrize("path", ["presplit", "fly"])
def test_linear_tc_layouts_are_bit_identical_to_contiguous(M, K, Nf, path, ops):
    a, w, b, r = R.linear_operands(M, K, Nf, seed=5, bias=True, residual=True)
    W, bd, Rd = w.to(D), b.to(D), r.to(D)
    wtc = ops.linear_tc_weight_layout(W)
    base = _gemm(ops, path, a.to(D), W, wtc, bd, Rd)
    # A as a column slice (lda > K, lda % 4 == 0, 16-byte aligned start)
    wide = torch.full((M, K + 8), float("nan"), device=D)
    wide[:, 4:4 + K] = a.to(D)
    assert torch.equal(_gemm(ops, path, wide[:, 4:4 + K], W, wtc, bd, Rd), base), "lda > K"
    # lda % 4 != 0
    odd = torch.full((M, K + 3), float("nan"), device=D)
    odd[:, :K] = a.to(D)
    assert torch.equal(_gemm(ops, path, odd[:, :K], W, wtc, bd, Rd), base), "lda % 4 != 0"
    # A one float off 16-byte alignment
    flat = torch.empty(M * K + 1, device=D)
    mis = flat[1:].view(M, K)
    mis.copy_(a.to(D))
    assert mis.data_ptr() % 16 == 4
    assert torch.equal(_gemm(ops, path, mis, W, wtc, bd, Rd), base), "misaligned A"
    # out as a column slice of a NaN-prefilled wider buffer (ldc > Nf); R with its own stride (ldr != ldc)
    ob = torch.full((M, Nf + 8), float("nan"), device=D)
    rb = torch.full((M, Nf + 5), float("nan"), device=D)
    rb[:, 1:1 + Nf] = Rd
    y = _gemm(ops, path, a.to(D), W, wtc, bd, rb[:, 1:1 + Nf], out=ob[:, 4:4 + Nf])
    assert torch.equal(y, base), "ldc > Nf, ldr != ldc"
    assert torch.isnan(ob[:, :4]).all() and torch.isnan(ob[:, 4 + Nf:]).all(), "write outside the output slice"
    # R and out are the same buffer
    io = Rd.clone()
    assert torch.equal(_gemm(ops, path, a.to(D), W, wtc, bd, io, out=io), base), "in-place residual"
    ops.check_range()


# ------------------------------------------------------------------ GEMM 4: epilogue activations
@pytest.mark.parametrize("act", ["gelu", "tanh", "gelu_tanh"])
def test_linear_tc_epilogue_activation_matches_float64(act, ops):
    """y_act = act(pre) + R against act64(pre) + R, with pre = the same GEMM with act = NONE (bit-identical accumulation):
    the epilogue's gelu_erf / tanhf / gelu_tanh within a few fp32 ulps of |pre| + |R| (measured max 1.58 ulps, tanh, on one
    H100 80GB HBM3 at 400 W)"""
    from styletts2_b200.lib import ACT_GELU, ACT_GELU_TANH, ACT_NONE, ACT_TANH
    code = {"gelu": ACT_GELU, "tanh": ACT_TANH, "gelu_tanh": ACT_GELU_TANH}[act]
    f64 = {"gelu": F.gelu, "tanh": torch.tanh, "gelu_tanh": lambda x: F.gelu(x, approximate="tanh")}[act]
    M, K, Nf = 1024, 256, 512
    g = torch.Generator().manual_seed(11)
    A = torch.randn(M, K, generator=g).to(D)
    W = (torch.randn(Nf, K, generator=g) * (3.0 / math.sqrt(K))).to(D)             # pre-activations over about +-10
    bd, Rd = (torch.randn(Nf, generator=g) * 0.5).to(D), torch.randn(M, Nf, generator=g).to(D)
    wtc = ops.linear_tc_weight_layout(W)
    worst = 0.0
    for path in ("presplit", "fly"):
        pre = _gemm(ops, path, A, W, wtc, bd, act=ACT_NONE).double()
        y = _gemm(ops, path, A, W, wtc, bd, Rd, act=code).double()
        ulps = float(((y - (f64(pre) + Rd.double())).abs() / ((pre.abs() + Rd.double().abs()) * 2.0 ** -23)).max())
        worst = max(worst, ulps)
    record("linear_tc_epilogue", act=act, ulps=worst)
    assert worst <= 2.4, (act, worst)


# ------------------------------------------------------------------ GEMM 5: range guard
def _guard_operands(ops):
    M, K, Nf = 300, 256, 256
    g = torch.Generator().manual_seed(2)
    A, W = torch.randn(M, K, generator=g).to(D), (torch.randn(Nf, K, generator=g) / 16).to(D)
    return A, W, ops.linear_tc_weight_layout(W)


@pytest.mark.parametrize("path", ["presplit", "fly"])
def test_linear_tc_range_guard_catches_a_nan_activation(path, ops):
    """the splitting threads of both paths (linear_tc_split_kernel, the GEMM's stagers) raise the flag on a NaN"""
    A, W, wtc = _guard_operands(ops)
    _gemm(ops, path, A, W, wtc)
    ops.check_range()                                              # clean operands: no flag
    A[7, 3] = float("nan")
    y = _gemm(ops, path, A, W, wtc)
    assert torch.isnan(y[7]).all() and torch.isfinite(y[8]).all()
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()                                              # the fetch cleared the flag


def test_linear_tc_range_guard_catches_a_nan_weight(ops):
    _, W, _ = _guard_operands(ops)
    W[5, 9] = float("nan")
    ops.linear_tc_weight_layout(W)
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()


# ------------------------------------------------------------------ attention
def _att(ops, q, k, v, lengths, B, N, H, out=None, expect_tc=True):
    """ops.attention_ex on [B*N, H*64] row views; returns the output and checks which kernel ran"""
    if out is None:
        out = torch.full((B * N, H * 64), float("nan"), device=D)
    ld = lengths.to(D, torch.int32) if lengths is not None else None
    ops.PROFILE = []
    try:
        ops.attention_ex(q, k, v, out, B, N, H, 64, ld)
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert len(names) == 1 and names[0].startswith("attention_tc" if expect_tc else "attention B"), names
    return out


def _rows(t):
    B, N, H, Dh = t.shape
    return t.reshape(B * N, H * Dh).to(D)


def _check_attention(ops, q, k, v, lengths, what, c=None, expect_tc=True, **kw):
    B, N, H, _ = q.shape
    y = _att(ops, _rows(q), _rows(k), _rows(v), lengths, B, N, H, expect_tc=expect_tc, **kw)
    o, E = R.attention_bound(q.to(D), k.to(D), v.to(D), lengths, SCALE)
    e = _bound_err(y.double().view(B, N, H, 64), o, E)
    record("attention_tc_recipe" if expect_tc else "attention_simt_recipe", case=what, bound_err=e)
    c = R.ATTENTION_BOUND_C if c is None else c
    assert math.isfinite(e) and e <= c, (what, e)
    return y


@pytest.mark.parametrize("B,N,H,lengths", ATT_CASES)
def test_attention_tc_matches_bound_at_block_edges(B, N, H, lengths, ops):
    L = torch.tensor(lengths)
    q, k, v = R.attention_operands(B, N, H, L, seed=N)
    _check_attention(ops, q, k, v, L, f"B{B} N{N} H{H}")
    ops.check_range()


@pytest.mark.parametrize("N", [64, 200, 300])
def test_attention_tc_peaked_tied_and_far_below_mask(N, ops):
    B, H = 3, 8
    g = torch.Generator().manual_seed(N)
    L = torch.tensor([N, N - 7, 40])
    k = torch.randn(B, N, H, 64, generator=g)
    k = k / k.norm(dim=-1, keepdim=True)
    v = torch.randn(B, N, H, 64, generator=g)
    # 1. logit gaps of 20 .. 80: q_i = t_i k_j(i) / scale with t in [20, 80], |k| = 1, other logits about t * N(0, 1/8)
    j = (torch.rand(B, N, H, generator=g) * L[:, None, None]).long()
    t = 20 + 60 * torch.rand(B, N, H, 1, generator=g)
    kj = torch.gather(k, 1, j[..., None].expand(B, N, H, 64))
    _check_attention(ops, (t * kj / SCALE).float(), k, v, L, f"peaked N{N}")
    # 2. ties: key 1 duplicates key 0; queries aligned with it see two equal maxima
    k2 = k.clone()
    k2[:, 1] = k2[:, 0]
    q2 = (40 * k2[:, :1] / SCALE).expand(B, N, H, 64).contiguous()
    y = _check_attention(ops, q2, k2, v, L, f"tie N{N}")
    assert torch.allclose(y.view(B, N, H, 64)[:, 5].cpu(), (v[:, 0] + v[:, 1]) / 2, atol=1e-6)
    # 3. every valid logit in [-130, -100] while a masked key (staged as zero) would score 0: the row maximum must ignore it
    u = torch.randn(B, 1, H, 64, generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    k3 = u + 0.02 * torch.randn(B, N, H, 64, generator=g)
    q3 = (-(100 + 30 * torch.rand(B, N, H, 1, generator=g)) * u / SCALE).float()
    logits = SCALE * torch.einsum("bnhd,bmhd->bhnm", q3.double(), k3.double())
    assert float(logits.max()) < -90
    _check_attention(ops, q3, k3.float(), v, L, f"below mask N{N}")
    ops.check_range()


@pytest.mark.parametrize("masked", [False, True])
def test_attention_tc_layouts_are_bit_identical(masked, ops):
    """PL-BERT layout (q | k | v views of one [M, 3 * 768] buffer) and the denoiser's (k | v of one [M, 1024] buffer), out
    into a slice of a NaN-prefilled buffer, against contiguous operands"""
    for B, N, H in ((4, 200, 12), (3, 129, 8)):
        L = torch.tensor([N, N - 60, 65, 1][:B]) if masked else None
        q, k, v = (_rows(t) for t in R.attention_operands(B, N, H, L, seed=3))
        base = _att(ops, q, k, v, L, B, N, H)
        HD = H * 64
        if H == 12:
            qkv = torch.cat([q, k, v], 1)
            qv, kv_, vv = qkv[:, :HD], qkv[:, HD:2 * HD], qkv[:, 2 * HD:]
        else:
            kvb = torch.cat([k, v], 1)
            qv, kv_, vv = q, kvb[:, :HD], kvb[:, HD:]
        wide = torch.full((B * N, HD + 8), float("nan"), device=D)
        y = _att(ops, qv, kv_, vv, L, B, N, H, out=wide[:, 4:4 + HD])
        assert torch.equal(y, base), (B, N, H)
        assert torch.isnan(wide[:, :4]).all() and torch.isnan(wide[:, 4 + HD:]).all()
    ops.check_range()


def test_attention_simt_dispatch_and_bound(ops):
    """N < 32 and a misaligned view take the SIMT kernel (rows.cu), which meets the same metric with its own constant"""
    for B, N, H in ((3, 31, 8), (2, 17, 12)):
        L = torch.tensor([N, 9, 1][:B])
        q, k, v = R.attention_operands(B, N, H, L, seed=N)
        _check_attention(ops, q, k, v, L, f"simt N{N}", c=R.ATTENTION_SIMT_BOUND_C, expect_tc=False)
    B, N, H = 2, 130, 8
    L = torch.tensor([130, 64])
    q, k, v = R.attention_operands(B, N, H, L, seed=7)
    flat = torch.empty(B * N * H * 64 + 1, device=D)
    qm = flat[1:].view(B * N, H * 64)
    qm.copy_(_rows(q))
    y = _att(ops, qm, _rows(k), _rows(v), L, B, N, H, expect_tc=False)
    o, E = R.attention_bound(q.to(D), k.to(D), v.to(D), L, SCALE)
    e = _bound_err(y.double().view(B, N, H, 64), o, E)
    record("attention_simt_recipe", case="misaligned q", bound_err=e)
    assert e <= R.ATTENTION_SIMT_BOUND_C, e


@pytest.mark.parametrize("which", ["q", "k", "v"])
@pytest.mark.parametrize("bad", [7.0e4, -1.0e5, float("nan")])
def test_attention_tc_range_guard(which, bad, ops):
    B, N, H = 2, 150, 8
    L = torch.tensor([150, 100])
    q, k, v = (_rows(t) for t in R.attention_operands(B, N, H, L, seed=1))
    _att(ops, q, k, v, L, B, N, H)
    ops.check_range()                                              # clean operands: no flag
    t = {"q": q, "k": k, "v": v}[which]
    keep = t[N + 130, 3 * 64 + 5].clone()                          # beyond utterance 1's length: masked for k and v
    t[N + 130, 3 * 64 + 5] = bad
    _att(ops, q, k, v, L, B, N, H)
    if which == "q":                                               # padded query rows are computed, so they are checked
        with pytest.raises(FloatingPointError):
            ops.check_range()
    else:
        ops.check_range()                                          # a masked key never reaches the planes
    t[N + 130, 3 * 64 + 5] = keep
    t[N + 40, 3 * 64 + 5] = bad                                    # a valid row / key of utterance 1, head 3
    y = _att(ops, q, k, v, L, B, N, H)
    assert not torch.isfinite(y.view(B, N, H, 64)[1, :, 3] if which != "q" else y.view(B, N, H, 64)[1, 40, 3]).all()
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()
