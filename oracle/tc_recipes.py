"""Recipe-exact references of the tensor-core conv (styletts2_b200/csrc/conv_tc.cu), GEMM (linear_tc.cu) and attention
(attention_tc.cu).  Plain torch: they run on the CPU, or in float64 on whatever device their inputs are on.

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


# ------------------------------------------------------------------ GEMM and attention (linear_tc.cu, attention_tc.cu)
# Both split every fp32 operand x into two fp16 planes, h = fp16(x) and l = fp16((x - h) * 2^11), and form a product as
# h*h + (h*l + l*h) * 2^-11 (l*l, 2^-22 relative, is left out), with h*h and the correction in separate fp32 accumulators.
LO_SCALE = 2048.0
GEMM_KB = 32            # K block of one GEMM pipeline stage (linear_tc.cu KB)
ATT_KB = 128            # key block of the attention kernel (attention_tc.cu KB)

# Accumulation bounds, metric |y - y_ref| <= c * 2^-20 * scale per output element:
#   GEMM       y_ref = linear(a, w, bias) (+ R), scale = sum_k |a_k||w_nk| + |bias_n| (+ |R|)       (sum_abs_linear)
#   attention  y_ref = the float64 attention of the fp32 operands, scale = E of attention_bound
# Measured on one H100 80GB HBM3 at a 400 W power limit over tests/test_gpu_linear_attention_tc.py: max 0.97 for the GEMM
# (K = 2048, dense rows), 2.45 for the tensor-core attention (a peaked softmax over two key blocks: the tensor core
# truncates each addition into the O accumulator, relative to the one dominant value), 0.80 for the SIMT attention.  The
# weakest modelled defect scores 84 (GEMM) and 48 (attention) in the same metric (tests/test_cpu_gemm_attention_recipe.py).
LINEAR_BOUND_C = 1.4
ATTENTION_BOUND_C = 3.5
ATTENTION_SIMT_BOUND_C = 1.2     # the fp32 SIMT attention kernel (rows.cu attention_kernel)     # the fp32 SIMT attention kernel (rows.cu), which st2_attention_ex runs


def split2(x: torch.Tensor):
    """fp32 x -> (h, l) as float64: h = fp16(x), l = fp16((x - h) * 2^11), as split2() of the GEMM and attention kernels.
    x - h is exact in fp32, and so is the scaling by 2^11; fp16 rounding is round-to-nearest-even on both sides."""
    x = x.float()
    h = x.half()
    return h.double(), ((x - h.float()) * LO_SCALE).half().double()


def linear(a, w, bias=None, *, drop_hl_block=None, drop_lh_step=None) -> torch.Tensor:
    """a [M,K] @ w[Nf,K]^T (+ bias) with the GEMM's operand planes, every plane product summed in float64.
    Defects of a kernel, for the power test of the bound (tests/test_cpu_gemm_attention_recipe.py):
      drop_hl_block = cb   the h(a)*l(w) product is lost on the 32-wide K block cb
      drop_lh_step = s     the l(a)*h(w) product is lost on the 16-wide K step s"""
    ah, al = split2(a)
    wh, wl = split2(w)
    hl, lh = ah @ wl.T, al @ wh.T
    if drop_hl_block is not None:
        k = slice(GEMM_KB * drop_hl_block, GEMM_KB * (drop_hl_block + 1))
        hl = hl - ah[:, k] @ wl[:, k].T
    if drop_lh_step is not None:
        k = slice(16 * drop_lh_step, 16 * (drop_lh_step + 1))
        lh = lh - al[:, k] @ wh[:, k].T
    y = ah @ wh.T + (hl + lh) / LO_SCALE
    return y if bias is None else y + bias.double()


def sum_abs_linear(a, w, bias=None) -> torch.Tensor:
    """sum_k |a_k||w_nk| (+ |bias_n|) of every output element: the scale of an fp32 dot product's rounding"""
    s = a.double().abs() @ w.double().abs().T
    return s if bias is None else s + bias.double().abs()


def _valid_keys(lengths, B, N, device, extra=0):
    klen = torch.full((B,), N, device=device) if lengths is None else lengths.to(device).long().clamp(max=N)
    return torch.arange(N, device=device)[None, :] < (klen + extra).clamp(max=N)[:, None]          # [B, N]


def attention_bound(q, k, v, lengths, scale, mutation=None, qchunk=64):
    """q, k, v [B, N, H, 64] fp32; lengths [B] (keys n >= lengths[b] masked; clamped to N, as the kernels do) or None.
    Returns (o, E), both [B, N, H, 64] float64:
      o     softmax(scale q k^T) v in float64 (padded query rows included)
      E     max_j(scale sum_e |q_ie||k_je|) * sum_j p_ij |v_jd - o_id|  +  sum_j p_ij |v_jd|   over valid keys j:
            how an error in the logits propagates through the softmax, plus the two-plane rounding of P and V.
    mutation: o is instead the kernel's two-plane recipe (operand planes of split2, P = exp(s - rowmax) split likewise,
    sums in float64) with one defect, for the power test of the bound:
      "recipe"             no defect (an accumulation-free kernel)
      "p_low_last_block"   P's low plane is lost on the last key block
      ("s_corr_step", i)   the correction products of S are lost on the 16-wide d step i
      "mask_plus_one"      the mask admits one key too many (klen + 1)"""
    B, N, H, Dh = q.shape
    dev = q.device
    qd, kd, vd = (t.double().permute(0, 2, 1, 3) for t in (q, k, v))               # [B, H, N, D]
    valid = _valid_keys(lengths, B, N, dev)[:, None, None, :]                        # [B, 1, 1, N]
    s = (qd @ kd.transpose(-1, -2)) * scale
    p = torch.softmax(s.masked_fill(~valid, float("-inf")), -1)
    o = p @ vd
    smax = ((qd.abs() @ kd.abs().transpose(-1, -2)) * scale).masked_fill(~valid, 0).amax(-1, keepdim=True)
    spread = torch.empty_like(o)
    for i0 in range(0, N, qchunk):                                                    # sum_j p_ij |v_jd - o_id|
        pi = p[:, :, i0:i0 + qchunk]
        spread[:, :, i0:i0 + qchunk] = (pi[..., None] * (vd[:, :, None] - o[:, :, i0:i0 + qchunk, None]).abs()).sum(-2)
    E = smax * spread + p @ vd.abs()
    if mutation is not None:
        o = _attention_recipe(q, k, v, lengths, scale, mutation)
    return o.permute(0, 2, 1, 3), E.permute(0, 2, 1, 3)


def _attention_recipe(q, k, v, lengths, scale, mutation):
    B, N, H, Dh = q.shape
    (qh, ql), (kh, kl), (vh, vl) = (tuple(x.permute(0, 2, 1, 3) for x in split2(t)) for t in (q, k, v))
    corr_q, corr_k = ql.clone(), kl.clone()
    if isinstance(mutation, tuple) and mutation[0] == "s_corr_step":
        d = slice(16 * mutation[1], 16 * (mutation[1] + 1))
        corr_q[..., d] = 0
        corr_k[..., d] = 0
    s = (qh @ kh.transpose(-1, -2) + (qh @ corr_k.transpose(-1, -2) + corr_q @ kh.transpose(-1, -2)) / LO_SCALE) * scale
    valid = _valid_keys(lengths, B, N, q.device, 1 if mutation == "mask_plus_one" else 0)[:, None, None, :]
    s = s.masked_fill(~valid, float("-inf"))
    P = torch.exp(s - s.amax(-1, keepdim=True))
    ph, pl = split2(P)
    if mutation == "p_low_last_block":
        nvalid = valid.sum(-1, keepdim=True)                                          # [B, 1, 1, 1]
        last0 = (nvalid - 1) // ATT_KB * ATT_KB
        pl = pl.masked_fill(torch.arange(N, device=q.device) >= last0, 0)
    o = (ph @ vh + (ph @ vl + pl @ vh) / LO_SCALE) / P.sum(-1, keepdim=True)
    return o


def linear_operands(M, K, Nf, seed=0, *, bias=False, residual=False):
    """Localised GEMM operands (a [M,K], w [Nf,K], bias [Nf] or None, R [M,Nf] or None; fp32): row m of a is non-zero only
    on the 32-wide K block m mod ncb, except every 61st row, which is dense; |a| log-uniform over 1e-3 .. 1e2, random signs.
    Every output element is then dominated by one K block (the tail block included), so a defect on one block or one
    16-wide step shows at full size instead of diluted over all K."""
    g = torch.Generator().manual_seed(seed)
    ncb = (K + GEMM_KB - 1) // GEMM_KB
    a = 10.0 ** (torch.rand(M, K, generator=g) * 5 - 3) * (torch.randint(0, 2, (M, K), generator=g) * 2 - 1)
    rows = torch.arange(M)[:, None]
    keep = (torch.arange(K)[None, :] // GEMM_KB == rows % ncb) | (rows % 61 == 7)
    a = (a * keep).float()
    w = torch.randn(Nf, K, generator=g) * 0.1
    b = torch.randn(Nf, generator=g) * 0.1 if bias else None
    r = torch.randn(M, Nf, generator=g) * 0.1 if residual else None
    return a, w, b, r


def attention_operands(B, N, H, lengths=None, seed=0, qscale=1.0):
    """q, k, v [B, N, H, 64] fp32.  Keys and values are N(0, 1); query i of every head is qscale * (k_a + k_b) + N(0, 0.1)
    for a random valid key a and a random key b of the utterance's LAST key block, so that (at scale 1/8) two keys carry
    most of each row's softmax and the last block a large share of it: a defect there shows at full size."""
    g = torch.Generator().manual_seed(seed)
    k = torch.randn(B, N, H, 64, generator=g)
    v = torch.randn(B, N, H, 64, generator=g)
    klen = torch.full((B,), N) if lengths is None else lengths.long().clamp(max=N)
    u1, u2 = torch.rand(B, N, H, generator=g), torch.rand(B, N, H, generator=g)
    last0 = (klen - 1) // ATT_KB * ATT_KB
    ia = (u1 * klen[:, None, None]).long()
    ib = last0[:, None, None] + (u2 * (klen - last0)[:, None, None]).long()
    take = lambda idx: torch.gather(k, 1, idx[..., None].expand(B, N, H, 64))     # noqa: E731
    q = qscale * (take(ia) + take(ib)) + 0.1 * torch.randn(B, N, H, 64, generator=g)
    return q.float(), k, v
