"""GPU tier: the style sampler on packed token rows (Synthesizer.synthesize(..., token_packing=True)).

Packed rows are only the valid rows of every utterance, concatenated (diffusion.TokenPacking).  The denoiser then attends
over and averages each utterance's own rows, so a batch of any token counts gives every utterance the style it gets alone.
Checked here: the packed attention kernel per output element and per row ownership, bit-identity with the padded entry
points at equal lengths, a ragged batch against the CPU oracle run on each utterance alone, that the padded default path
does NOT meet that bar (the test can tell the two apart), and the serving calls built on it."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

import cases
import styletts2_oracle as O
import tc_recipes as R
from util import gpu_model, maxdiff, oracle_sds, record

D = "cuda:0"
SCALE = 64 ** -0.5
S_TOL = 1e-4                                  # s_pred max-abs, as test_gpu_parity.py
WAV_TOL = 1e-3


@pytest.fixture(scope="module")
def ops():
    from styletts2_b200 import ops as o
    o.check_range()
    yield o
    o.check_range()


def _offsets(lengths):
    return torch.tensor([0] + np.cumsum(lengths).tolist(), dtype=torch.int32, device=D)


# ------------------------------------------------------------------ 1. packed attention per element and per row
LENS = [1, 31, 63, 64, 65, 127, 128, 129, 200]


def _packed_operands(H=8):
    qs, ks, vs = [], [], []
    for i, n in enumerate(LENS):
        q, k, v = R.attention_operands(1, n, H, None, seed=100 + i)
        qs.append(q[0]), ks.append(k[0]), vs.append(v[0])
    q, k, v = (torch.cat(t).reshape(-1, H * 64).to(D) for t in (qs, ks, vs))
    return q, torch.cat([k, v], 1).contiguous(), (qs, ks, vs)


def test_packed_attention_per_element_and_row_ownership(ops):
    H = 8
    q, kv, (qs, ks, vs) = _packed_operands(H)
    M, offs = q.shape[0], _offsets(LENS)
    out = torch.full((M, H * 64), float("nan"), device=D)
    ops.attention_packed(q, kv, offs, len(LENS), max(LENS), H, 64, out=out)
    ops.check_range()
    assert torch.isfinite(out).all(), "a packed row was never written"
    o0 = 0
    for b, n in enumerate(LENS):
        y = out[o0:o0 + n].double().view(1, n, H, 64)
        o, E = R.attention_bound(qs[b][None].to(D), ks[b][None].to(D), vs[b][None].to(D), None, SCALE)
        e = float(((y - o).abs() / (E * 2.0 ** -20)).max())
        record("attention_tc_packed", n=n, bound_err=e)
        assert math.isfinite(e) and e <= R.ATTENTION_BOUND_C, (n, e)
        # the rows hold this utterance's result, bit for bit as when it runs alone: written by its own CTAs and not
        # overwritten by a neighbour's
        solo = torch.full((n, H * 64), float("nan"), device=D)
        ops.attention_packed(q[o0:o0 + n], kv[o0:o0 + n], _offsets([n]), 1, n, H, 64, out=solo)
        assert torch.equal(solo, out[o0:o0 + n]), n
        o0 += n


def test_packed_attention_range_guard(ops):
    H = 8
    q, kv, _ = _packed_operands(H)
    offs = _offsets(LENS)
    ops.attention_packed(q, kv, offs, len(LENS), max(LENS), H, 64)
    ops.check_range()                                              # clean operands: no flag
    r = int(offs[6]) + 100                                         # a valid key row of the 128-token utterance, head 2
    kv[r, 2 * 64 + 7] = float("nan")
    y = ops.attention_packed(q, kv, offs, len(LENS), max(LENS), H, 64)
    with pytest.raises(FloatingPointError):
        ops.check_range()
    ops.check_range()
    blk = y[int(offs[6]):int(offs[7])].view(-1, H, 64)
    assert not torch.isfinite(blk[:, 2]).any() and torch.isfinite(y[:int(offs[6])]).all() and torch.isfinite(y[int(offs[7]):]).all()


# ------------------------------------------------------------------ 2. equal lengths: the padded entry points' bits
@pytest.mark.parametrize("B,N", [(4, 128), (3, 40)])
def test_equal_lengths_kernels_bit_identical(B, N, ops):
    H, Cx, E = 8, 256, 768
    C = Cx + E
    g = torch.Generator().manual_seed(B * 1000 + N)
    offs = _offsets([N] * B)
    row_utt = torch.arange(B, dtype=torch.int32).repeat_interleave(N).to(D)
    # attention
    q = torch.randn(B * N, H * 64, generator=g).to(D)
    kv = torch.randn(B * N, 2 * H * 64, generator=g).to(D)
    assert torch.equal(ops.attention_packed(q, kv, offs, B, N, H, 64), ops.attention(q, kv, B, N, H, 64))
    # rows_ln: the first block's form (x | emb + mapping, AdaLN rows per utterance) and a later block's (h_in)
    x = torch.randn(B, Cx, generator=g).to(D)
    emb = torch.randn(B * N, E, generator=g).to(D)
    add = torch.randn(B, C, generator=g).to(D)
    gb1, gb2 = torch.randn(B, 2 * C, generator=g).to(D), torch.randn(B, 2 * C, generator=g).to(D)
    ada = dict(g1=gb1, b1=gb1[:, C:], g2=gb2, b2=gb2[:, C:], gb_bstride=gb1.stride(0), ada=True)
    outs = {}
    for packed in (False, True):
        h, a, c = (torch.full((B * N, C), float("nan"), device=D) for _ in range(3))
        ln = (lambda **kw: ops.rows_ln_packed(row_utt=row_utt, M=B * N, B=B, **kw)) if packed else \
            (lambda **kw: ops.rows_ln(B=B, N=N, **kw))
        ln(Cw=C, x=x, xs=1.0, emb=emb, add=add, h_out=h, out1=a, out2=c, eps=1e-5, **ada)
        first = (h.clone(), a.clone(), c.clone())
        ln(Cw=C, h_in=h, add=add, h_out=h, out1=a, out2=c, eps=1e-5, **ada)
        outs[packed] = first + (h, a, c)
    for u, v in zip(outs[False], outs[True]):
        assert torch.equal(u, v)
    # token mean
    hh = torch.randn(B * N, C, generator=g).to(D)
    assert torch.equal(ops.mean_segments(hh, offs, B), ops.mean_rows(hh, B, N))


@pytest.mark.parametrize("B,N", [(4, 128), (3, 40)])
@pytest.mark.parametrize("model,scale", [("ljspeech", 1.5), ("libritts", 1.0)])
def test_equal_lengths_sampler_bit_identical(model, scale, B, N):
    from styletts2_b200.inference import Synthesizer
    m = gpu_model(model)
    syn = Synthesizer(m, cases.MODEL_CFGS[model], D)
    tokens, lengths, bert_dur, noise, ref_s = cases.e2e_inputs(dict(model=model, B=B, N=N, seed=B + N))
    rng = cases.ReplayRNG(B + N)
    steps = [rng.step_noise(i, (B, 1, 256)).to(D) for i in range(4)]
    sn = rng.sine_noise((B, 600 * 2 * N, 9)).to(D)
    outs = [syn.synthesize(tokens.to(D), lengths.to(D), bert_dur.to(D), noise.to(D), diffusion_steps=5, embedding_scale=scale,
                           ref_s=None if ref_s is None else ref_s.to(D), forced_durations=torch.full((B, N), 2.0),
                           rng=dict(step_noises=steps, sine_noise=sn), return_all=True, token_packing=tp) for tp in (False, True)]
    assert torch.equal(outs[0]["s_pred"], outs[1]["s_pred"])
    assert torch.equal(outs[0]["pred_dur"], outs[1]["pred_dur"])
    assert torch.equal(outs[0]["wav"], outs[1]["wav"])


# ------------------------------------------------------------------ 3 + 4. a ragged batch against each utterance alone
RAGGED = [9, 23, 64, 65, 128, 181]
RAGGED_CASES = {
    "lj_cfg": dict(model="ljspeech", embedding_scale=1.5, alpha=0.3, beta=0.7, seed=61),
    "libri_ref": dict(model="libritts", embedding_scale=1.0, alpha=0.2, beta=0.6, seed=62),
}
FPT = 2                        # frames per token of the teacher-forced durations under the F0 / waveform checks
PICKS = [1, 5]                 # utterances whose waveform is checked against the oracle


def _ragged_inputs(case):
    B, N = len(RAGGED), max(RAGGED)
    tokens, _, bert_dur, noise, ref_s = cases.e2e_inputs(dict(model=case["model"], B=B, N=N, seed=case["seed"]))
    lengths = torch.tensor(RAGGED)
    pad = torch.arange(N)[None] >= lengths[:, None]
    tokens = tokens.masked_fill(pad, 0)
    bert_dur = bert_dur.masked_fill(pad[..., None], 0.0)
    return tokens, lengths, bert_dur, noise, ref_s


@pytest.mark.parametrize("cname", list(RAGGED_CASES))
def test_ragged_batch_matches_each_utterance_alone(cname):
    from styletts2_b200.inference import Synthesizer
    case = RAGGED_CASES[cname]
    model = case["model"]
    mcfg = cases.MODEL_CFGS[model]
    m = gpu_model(model)
    sds = oracle_sds(model)
    syn = Synthesizer(m, mcfg, D)
    tokens, lengths, bert_dur, noise, ref_s = _ragged_inputs(case)
    B, N, K = len(RAGGED), max(RAGGED), 5
    rng = cases.ReplayRNG(case["seed"])
    steps = [rng.step_noise(i, (B, 1, 256)) for i in range(K - 1)]
    forced = (torch.arange(N)[None] < lengths[:, None]).float() * FPT
    L = 600 * FPT * N
    sine = rng.sine_noise((B, L, 9))
    common = dict(diffusion_steps=K, embedding_scale=case["embedding_scale"], alpha=case["alpha"], beta=case["beta"],
                  ref_s=None if ref_s is None else ref_s.to(D), forced_durations=forced, return_all=True)
    dev_in = (tokens.to(D), lengths.to(D), bert_dur.to(D), noise.to(D))
    inj = dict(step_noises=[s.to(D) for s in steps], sine_noise=sine.to(D))
    out = syn.synthesize(*dev_in, rng=inj, token_packing=True, **common)
    padded = syn.synthesize(*dev_in, rng=inj, **common)           # the default path on the same batch

    torch.set_num_threads(min(32, torch.get_num_threads() or 8))
    refs = {}
    for b, n in enumerate(RAGGED):
        sl = slice(b, b + 1)
        with torch.no_grad():
            refs[b] = O.synthesize(sds, mcfg, tokens[sl, :n], lengths[sl], bert_dur[sl, :n], noise[sl], diffusion_steps=K,
                                   embedding_scale=case["embedding_scale"], alpha=case["alpha"], beta=case["beta"],
                                   ref_s=None if ref_s is None else ref_s[sl],
                                   rng=dict(step_noises=[s[sl] for s in steps], sine_noise=sine[sl, :600 * FPT * n],
                                            rand_ini=torch.zeros(1, 9)),
                                   forced_durations=forced[sl, :n], skip_decoder=b not in PICKS)
    for b, n in enumerate(RAGGED):
        ref = refs[b]
        ds = maxdiff(out["s_pred"][b], ref["s_pred"][0])
        ds_padded = maxdiff(padded["s_pred"][b], ref["s_pred"][0])
        # integer durations: exact except where the oracle's own pre-rounding sum is within fp32 noise of x.5
        dur_f = torch.sigmoid(ref["logits"][0]).sum(-1).double()
        dur_err = float((out["dur_f"][b, :n].cpu().double() - dur_f).abs().max())
        guard = (dur_f - torch.floor(dur_f) - 0.5).abs()
        bad = out["pred_dur"][b, :n].cpu() != ref["pred_dur"][0].to(torch.int32)
        f0_rel = maxdiff(out["F0"][b, :2 * FPT * n], ref["F0"][0]) / max(1.0, float(ref["F0"].abs().max()))
        record("token_packing_ragged_" + cname, n=n, s_pred_maxabs=ds, s_pred_maxabs_padded_path=ds_padded,
               duration_mismatches=int(bad.sum()), duration_sum_maxabs_err=dur_err, F0_rel=f0_rel)
        assert ds <= S_TOL, (n, ds)
        assert dur_err < 1e-4, (n, dur_err)
        assert int(bad.sum()) <= 2 and bool((guard[bad] <= 4 * dur_err).all()), (n, guard[bad].tolist())
        assert bool((out["pred_dur"][b, n:] == 0).all())
        assert f0_rel <= 1e-4, (n, f0_rel)
    # 4. the padded default path misses the short utterances' single-utterance style by far more than the tolerance
    for b in (0, 1):
        assert maxdiff(padded["s_pred"][b], refs[b]["s_pred"][0]) >= 10 * S_TOL, b

    # waveforms of two utterances with the oracle's F0 / N (and har) teacher-forced
    F0i, Ni = out["F0"].clone(), out["N"].clone()
    for b in PICKS:
        T2 = 2 * FPT * RAGGED[b]
        F0i[b, :T2].copy_(refs[b]["F0"][0])
        Ni[b, :T2].copy_(refs[b]["N"][0])
    inj2 = dict(inj, F0=F0i, N=Ni)
    if mcfg["decoder"]["type"] == "istftnet":
        har = m.decoder.generator.har_features(F0i, inj["sine_noise"])
        sdg = O.sub(sds["decoder"], "generator")
        for b in PICKS:
            with torch.no_grad():
                hb = O.istftnet_har(refs[b]["F0"], sdg, mcfg["decoder"], torch.zeros(1, 9), sine[b:b + 1, :600 * FPT * RAGGED[b]])[0]
            har[b, :, :hb.shape[-1]].copy_(hb)
        inj2["har"] = har
    out2 = syn.synthesize(*dev_in, rng=inj2, token_packing=True, **common)
    for b in PICKS:
        Lb = 600 * FPT * RAGGED[b]
        assert int(out2["wav_lengths"][b]) == Lb
        d = maxdiff(out2["wav"][b, 0, :Lb], refs[b]["wav"].reshape(-1))
        record("token_packing_ragged_wav_" + cname, n=RAGGED[b], wav_maxabs_teacher_forced=d)
        assert d <= WAV_TOL, (RAGGED[b], d)


# ------------------------------------------------------------------ 5. serving calls
def test_synthesize_texts_matches_per_utterance_inference():
    from test_gpu_demo import _notebook
    nb, _, _ = _notebook("ljspeech")
    syn = nb.synthesizer
    g = torch.Generator().manual_seed(5)
    lens = [7, 30, 12, 65]
    token_lists = [[0] + torch.randint(1, 178, (n - 1,), generator=g).tolist() for n in lens]
    B, K = len(lens), 4
    noise = torch.randn(B, 1, 256, generator=g).to(D)
    steps = [torch.randn(B, 1, 256, generator=g).to(D) for _ in range(K - 1)]
    kw = dict(diffusion_steps=K, embedding_scale=1.3)
    N = max(lens)
    tk = torch.zeros(B, N, dtype=torch.long)
    for b, t in enumerate(token_lists):
        tk[b, :lens[b]] = torch.tensor(t)
    # PL-BERT's output for each utterance alone, padded into the batch.  (PL-BERT on the padded batch is masked correctly,
    # but its GEMMs run in other row-count regimes than alone, and the real checkpoint's magnitudes lift those last-bit
    # differences to ~3e-4 in s_pred: that is PL-BERT's batching, not the sampler's, and is kept out of this comparison.)
    with torch.no_grad():
        solo_bert = [syn.model.bert(torch.tensor([t], device=D), attention_mask=torch.ones(1, len(t), dtype=torch.int32, device=D))
                     for t in token_lists]
    bert_dur = torch.zeros(B, N, 768, device=D)
    for b in range(B):
        bert_dur[b, :lens[b]] = solo_bert[b][0]
    wavs = syn.synthesize_texts(token_lists, noise=noise, bert_dur=bert_dur, rng=dict(step_noises=steps), **kw)
    batch = syn.synthesize(tk.to(D), torch.tensor(lens, device=D), bert_dur, noise, token_packing=True, return_all=True,
                           rng=dict(step_noises=steps), **kw)
    assert len(wavs) == B
    for b, toks in enumerate(token_lists):
        # what Synthesizer.inference runs for this utterance alone, with its slice of the step noises injected
        one = syn._one(toks, solo_bert[b], noise[b:b + 1], rng=dict(step_noises=[s[b:b + 1] for s in steps]), return_all=True, **kw)
        solo_wav = one["wav"].squeeze().cpu().numpy()
        ds = maxdiff(batch["s_pred"][b], one["s_pred"][0])
        record("token_packing_synthesize_texts", n=lens[b], s_pred_maxabs=ds)
        assert ds <= S_TOL, (lens[b], ds)
        assert torch.equal(batch["pred_dur"][b, :lens[b]], one["pred_dur"][0])
        assert wavs[b].shape == solo_wav.shape, (wavs[b].shape, solo_wav.shape)


def test_inference_batch_is_synthesize_texts_over_the_notebook_tokens():
    from styletts2_b200 import ops
    from test_gpu_demo import _notebook, _texts
    nb, _, _ = _notebook("libritts")
    t0, t1 = _texts()
    texts = [t0, t1, t0[:-2] + " " + t1]
    ref_s = torch.randn(1, 256, generator=torch.Generator().manual_seed(3)).to(D) * 0.5
    ops.manual_seed(7)
    torch.manual_seed(7)
    got = nb.inference_batch(texts, ref_s, alpha=0.2, beta=0.6, diffusion_steps=3, embedding_scale=1.2)
    ops.manual_seed(7)
    torch.manual_seed(7)
    noise = torch.randn((len(texts), 256)).unsqueeze(1).to(D)
    toks = []
    for t in texts:
        ps = " ".join(nb.word_tokenize(nb.global_phonemizer.phonemize([t.strip()])[0]))
        toks.append([0] + nb.textclenaer(ps))
    want = nb.synthesizer.synthesize_texts(toks, noise=noise, ref_s=ref_s, alpha=0.2, beta=0.6, diffusion_steps=3,
                                           embedding_scale=1.2)
    assert len(got) == len(texts)
    for a, b in zip(got, want):
        assert a.shape == b.shape and np.array_equal(a, b)
