"""CPU oracle for the StyleTTS 2 text->waveform inference hot path.

TEST INFRASTRUCTURE -- NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / `--impl reference` legs may import this file.
The product path (styletts2_b200/) never routes through it and has no CPU
fallback.

What it is: a functional restatement (plain torch fp32 CPU ops on a flat
{key: tensor} state dict that uses the reference's own key names) of the
algorithm in yl4579/StyleTTS2 for the path SURVEY.md section 8(a) lists.  Every
function cites the reference file:line it follows.  It is written from the
reference's *behaviour*; it shares no class structure with it.

Pinning: oracle/make_golden.py (build container only, where the reference checkout ($STYLETTS2_REFERENCE) is
mounted) runs the UNMODIFIED reference modules and this restatement on the
same key-seeded weights and recorded RNG draws and asserts agreement
(bit-exact for the integer durations, <=1e-5 for every float boundary; the
measured figures are written to tests/golden/PINNING.json), then stores the
reference's outputs as fixtures in tests/golden/.  The reference itself has
no tests or golden vectors (SURVEY.md section 4), so those fixtures are the pin.

Conventions: B utterances, N tokens, T aligned frames, L = 600*T samples.
All tensors fp32 [B, C, time] unless noted.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]


# --------------------------------------------------------------------------- helpers
def sub(sd: SD, prefix: str) -> SD:
    """View of `sd` restricted to keys under `prefix.` (prefix stripped)."""
    p = prefix + "."
    return {k[len(p):]: v for k, v in sd.items() if k.startswith(p)}


def wn_weight(sd: SD, p: str) -> torch.Tensor:
    """Old-style torch.nn.utils.weight_norm (dim=0): w = v * g/||v|| over all dims
    but 0.  The reference never removes weight norm at inference, so it is
    re-evaluated per forward (Modules/istftnet.py:5,30-46; models.py:293,386-395)."""
    if p + ".weight" in sd:
        return sd[p + ".weight"]
    return torch._weight_norm(sd[p + ".weight_v"], sd[p + ".weight_g"], 0)


def conv1d(x, sd: SD, p: str, stride=1, padding=0, dilation=1, groups=1):
    return F.conv1d(x, wn_weight(sd, p), sd.get(p + ".bias"), stride, padding, dilation, groups)


def linear(x, sd: SD, p: str):
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def length_to_mask(lengths: torch.Tensor) -> torch.Tensor:
    """utils.py:42-45 / Demo/Inference_LJSpeech.ipynb#cell6: True where padded."""
    pos = torch.arange(int(lengths.max())).unsqueeze(0).expand(lengths.shape[0], -1).type_as(lengths)
    return torch.gt(pos + 1, lengths.unsqueeze(1))


def get_padding(k: int, d: int = 1) -> int:
    """Modules/utils.py:11-12."""
    return int((k * d - d) / 2)


def snake(x, alpha):
    """x + sin^2(alpha x)/alpha with learned per-channel alpha [1,C,1]
    (Modules/istftnet.py:69,72; Modules/hifigan.py:329,343)."""
    return x + (1 / alpha) * (torch.sin(alpha * x) ** 2)


# --------------------------------------------------------------------------- norms
def adain(x, s, sd: SD, p: str):
    """AdaIN1d (Modules/istftnet.py:15-25 == models.py:349-359): InstanceNorm1d
    (biased var, eps 1e-5, no affine) then (1+gamma)*xhat+beta, [gamma|beta]=fc(s)."""
    h = linear(s, sd, p + ".fc")
    h = h.view(h.size(0), h.size(1), 1)
    gamma, beta = torch.chunk(h, 2, dim=1)
    return (1 + gamma) * F.instance_norm(x, eps=1e-5) + beta


def ada_layer_norm(x, s, sd: SD, p: str, eps=1e-5):
    """AdaLayerNorm over the last axis of x [B,N,C] (models.py:418-438,
    Modules/diffusion/modules.py:18-38): LN without affine, then (1+gamma)*x+beta
    with per-utterance [gamma|beta]=fc(s)."""
    h = linear(s, sd, p + ".fc")
    gamma, beta = torch.chunk(h, 2, dim=-1)
    x = F.layer_norm(x, (x.shape[-1],), eps=eps)
    return (1 + gamma.unsqueeze(1)) * x + beta.unsqueeze(1)


# --------------------------------------------------------------------------- LSTM
def bilstm(x, sd: SD, p: str, lengths: Optional[torch.Tensor] = None):
    """Single-layer bidirectional LSTM, batch_first (models.py:300,450,453,523).
    With `lengths`, mirrors pack_padded_sequence/pad_packed_sequence as
    TextEncoder/DurationEncoder use it (models.py:314-322,545-560)."""
    names = ["weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0",
             "weight_ih_l0_reverse", "weight_hh_l0_reverse", "bias_ih_l0_reverse", "bias_hh_l0_reverse"]
    ws = [sd[p + "." + n] for n in names]
    hid = ws[1].shape[1]
    B = x.shape[0]
    h0 = x.new_zeros(2, B, hid)
    if lengths is None:
        out, _, _ = torch._VF.lstm(x, (h0, h0.clone()), ws, True, 1, 0.0, False, True, True)
        return out
    packed = torch.nn.utils.rnn.pack_padded_sequence(x, lengths.cpu(), batch_first=True, enforce_sorted=False)
    h0p = h0.index_select(1, packed.sorted_indices) if packed.sorted_indices is not None else h0
    out, _, _ = torch._VF.lstm(packed.data, packed.batch_sizes, (h0p, h0p.clone()), ws, True, 1, 0.0, False, True)
    packed_out = torch.nn.utils.rnn.PackedSequence(out, packed.batch_sizes, packed.sorted_indices, packed.unsorted_indices)
    out, _ = torch.nn.utils.rnn.pad_packed_sequence(packed_out, batch_first=True)
    return out


# --------------------------------------------------------------------------- a6 TextEncoder
def text_encoder(tokens, input_lengths, mask, sd: SD):
    """TextEncoder.forward (models.py:302-331): Embedding -> 3x[wn-Conv1d k5 p2 ->
    LayerNorm over channels -> LeakyReLU(.2)] (masked) -> packed biLSTM -> zero-pad,
    mask.  Returns t_en [B,512,N]."""
    x = F.embedding(tokens, sd["embedding.weight"]).transpose(1, 2)
    m = mask.unsqueeze(1)
    x = x.masked_fill(m, 0.0)
    depth = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("cnn."))
    for i in range(depth):
        x = conv1d(x, sd, f"cnn.{i}.0", padding=2)
        x = F.layer_norm(x.transpose(1, -1), (x.shape[1],), sd[f"cnn.{i}.1.gamma"], sd[f"cnn.{i}.1.beta"], 1e-5).transpose(1, -1)
        x = F.leaky_relu(x, 0.2)
        x = x.masked_fill(m, 0.0)
    x = bilstm(x.transpose(1, 2), sd, "lstm", input_lengths).transpose(-1, -2)
    out = torch.zeros(x.shape[0], x.shape[1], mask.shape[-1])
    out[:, :, : x.shape[-1]] = x
    return out.masked_fill(m, 0.0)


# --------------------------------------------------------------------------- a8/a9 predictor (duration side)
def duration_encoder(d_en, style, text_lengths, mask, sd: SD):
    """DurationEncoder.forward (models.py:536-569): x=[d_en^T | s]; 3x(biLSTM 640->512,
    AdaLayerNorm(512), concat style, mask).  d_en [B,512,N] -> d [B,N,640]."""
    B, _, N = d_en.shape
    s = style.unsqueeze(1).expand(B, N, -1)
    m = mask.unsqueeze(-1)
    x = torch.cat([d_en.transpose(1, 2), s], dim=-1).masked_fill(m, 0.0)
    nl = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("lstms."))
    for i in range(0, nl, 2):
        y = bilstm(x, sd, f"lstms.{i}", text_lengths)
        if y.shape[1] < N:
            y = torch.cat([y, y.new_zeros(B, N - y.shape[1], y.shape[2])], dim=1)
        y = ada_layer_norm(y, style, sd, f"lstms.{i + 1}")
        x = torch.cat([y, s], dim=-1).masked_fill(m, 0.0)
    return x


def duration_logits(d, sd_pred: SD):
    """predictor.lstm + duration_proj as the notebook glue calls them, un-packed
    (Demo/Inference_LJSpeech.ipynb#cell17; models.py:450-451,166-176)."""
    x = bilstm(d, sd_pred, "lstm")
    return linear(x, sd_pred, "duration_proj.linear_layer")


def predict_durations(logits, last_plus: int = 0):
    """round(sum_50 sigmoid(logit)) clamped to >=1; the LJSpeech demo adds 5 frames
    to the last token (Inference_LJSpeech.ipynb#cell17); LibriTTS does not
    (Inference_LibriTTS.ipynb#cell16).  Returns integral fp32 [B,N]."""
    dur = torch.sigmoid(logits).sum(dim=-1)
    pred = torch.round(dur).clamp(min=1)
    if last_plus:
        pred = pred.clone()
        pred[..., -1] += last_plus
    return pred


def alignment_from_durations(pred_dur_row: torch.Tensor) -> torch.Tensor:
    """One-hot monotonic alignment [N,T] built frame by frame (#cell17)."""
    n = pred_dur_row.shape[0]
    total = int(pred_dur_row.sum().item())
    aln = torch.zeros(n, total)
    c = 0
    for i in range(n):
        di = int(pred_dur_row[i].item())
        aln[i, c:c + di] = 1
        c += di
    return aln


def shift_right_one(x):
    """HiFi-GAN glue: frame 0 kept, the rest delayed by one (Inference_LibriTTS.ipynb#cell16)."""
    y = torch.zeros_like(x)
    y[:, :, 0] = x[:, :, 0]
    y[:, :, 1:] = x[:, :, :-1]
    return y


# --------------------------------------------------------------------------- a12 AdainResBlk1d
def adain_resblk1d(x, s, sd: SD, p: str):
    """AdainResBlk1d.forward (models.py:372-416 == istftnet.py:410-454 == hifigan.py:359-403).
    residual: AdaIN -> LeakyReLU(.2) -> [depthwise ConvT k3 s2 p1 op1] -> wn-Conv k3 ->
    AdaIN -> LeakyReLU -> wn-Conv k3; shortcut: [nearest x2] -> [wn-Conv1x1];
    (res+sc)/sqrt(2)."""
    upsample = (p + ".pool.weight_v") in sd
    learned_sc = (p + ".conv1x1.weight_v") in sd
    r = F.leaky_relu(adain(x, s, sd, p + ".norm1"), 0.2)
    if upsample:
        w = wn_weight(sd, p + ".pool")
        r = F.conv_transpose1d(r, w, sd[p + ".pool.bias"], stride=2, padding=1, output_padding=1, groups=w.shape[0])
    r = conv1d(r, sd, p + ".conv1", padding=1)
    r = F.leaky_relu(adain(r, s, sd, p + ".norm2"), 0.2)
    r = conv1d(r, sd, p + ".conv2", padding=1)
    sc = x
    if upsample:
        sc = F.interpolate(sc, scale_factor=2, mode="nearest")
    if learned_sc:
        sc = conv1d(sc, sd, p + ".conv1x1")
    return (r + sc) / math.sqrt(2)


# --------------------------------------------------------------------------- a11 F0Ntrain
def f0n_train(en, s, sd_pred: SD):
    """ProsodyPredictor.F0Ntrain (models.py:497-510): shared biLSTM over T, then two
    3-block AdainResBlk1d branches and a 1x1 projection each -> F0,N [B,2T]."""
    x = bilstm(en.transpose(-1, -2), sd_pred, "shared").transpose(-1, -2)
    outs = []
    for br in ("F0", "N"):
        y = x
        for i in range(3):
            y = adain_resblk1d(y, s, sd_pred, f"{br}.{i}")
        y = conv1d(y, sd_pred, f"{br}_proj")
        outs.append(y.squeeze(1))
    return outs[0], outs[1]


# --------------------------------------------------------------------------- a18 AdaINResBlock1
def adain_resblock1(x, s, sd: SD, p: str, k: int, dils=(1, 3, 5)):
    """AdaINResBlock1.forward (istftnet.py:66-75 == hifigan.py:65-74)."""
    for j, d in enumerate(dils):
        xt = snake(adain(x, s, sd, f"{p}.adain1.{j}"), sd[f"{p}.alpha1.{j}"])
        xt = conv1d(xt, sd, f"{p}.convs1.{j}", padding=get_padding(k, d), dilation=d)
        xt = snake(adain(xt, s, sd, f"{p}.adain2.{j}"), sd[f"{p}.alpha2.{j}"])
        xt = conv1d(xt, sd, f"{p}.convs2.{j}", padding=get_padding(k, 1))
        x = xt + x
    return x


# --------------------------------------------------------------------------- a14 SineGen / source
def sine_source(f0_curve, upsample_scale: int, sd_gen: SD, rand_ini=None, sine_noise=None,
                harmonic_num=8, sine_amp=0.1, noise_std=0.003, voiced_threshold=10.0, sr=24000):
    """f0_upsamp + SourceModuleHnNSF + SineGen (istftnet.py:146-247,283-297,352-355 ==
    hifigan.py:117-218,254-268,323-326).  f0_curve [B,2T] -> har_source [B, 2T*scale].

    Injected RNG (parity mode): rand_ini [B,9] (torch.rand, istftnet.py:155),
    sine_noise [B,L,9] (torch.randn_like, :242).  The third draw (:296) is unused.
    """
    B = f0_curve.shape[0]
    f0 = F.interpolate(f0_curve[:, None], scale_factor=float(upsample_scale), mode="nearest").transpose(1, 2)  # [B,L,1]
    harm = torch.arange(1, harmonic_num + 2, dtype=torch.float32).view(1, 1, -1)
    fn = f0 * harm
    rad = (fn / sr) % 1
    if rand_ini is None:
        rand_ini = torch.rand(B, harmonic_num + 1)
    rand_ini = rand_ini.clone()
    rand_ini[:, 0] = 0
    rad[:, 0, :] = rad[:, 0, :] + rand_ini
    rad = F.interpolate(rad.transpose(1, 2), scale_factor=1 / upsample_scale, mode="linear").transpose(1, 2)
    phase = torch.cumsum(rad, dim=1) * 2 * np.pi
    phase = F.interpolate(phase.transpose(1, 2) * upsample_scale, scale_factor=float(upsample_scale), mode="linear").transpose(1, 2)
    sines = torch.sin(phase) * sine_amp
    uv = (f0 > voiced_threshold).float()
    noise_amp = uv * noise_std + (1 - uv) * sine_amp / 3
    if sine_noise is None:
        sine_noise = torch.randn_like(sines)
    sines = sines * uv + noise_amp * sine_noise
    merged = torch.tanh(linear(sines, sd_gen, "m_source.l_linear"))  # [B,L,1]
    return merged.squeeze(-1)


# --------------------------------------------------------------------------- a15 STFT
def hann_periodic(n: int) -> torch.Tensor:
    """scipy.signal.get_window('hann', n, fftbins=True) as float32 (istftnet.py:89)."""
    k = np.arange(n, dtype=np.float64)
    return torch.from_numpy((0.5 - 0.5 * np.cos(2.0 * np.pi * k / n)).astype(np.float32))


def stft_mag_phase(x, n_fft=20, hop=5):
    """TorchSTFT.transform (istftnet.py:91-97): centered reflect-pad STFT -> |X|, angle X.

    NOTE (parity): angle X is ill-conditioned wherever |X| is at rounding-noise level and
    jumps by 2 pi when Im X changes sign with Re X < 0.  The first and last frames are
    exactly symmetric after reflect padding (hann[0]=0), so there Im X = 0 analytically
    and the reference's +-pi is FFT rounding noise.  Implementations that differ from the
    reference by 1 ulp anywhere upstream therefore differ by up to 2 pi in a handful of
    bins; waveform-parity tests teacher-force `har` (see generator_istftnet)."""
    X = torch.stft(x, n_fft, hop, n_fft, window=hann_periodic(n_fft), return_complex=True)
    return torch.abs(X), torch.angle(X)


def istft_from_mag_phase(mag, phase, n_fft=20, hop=5):
    """TorchSTFT.inverse (istftnet.py:99-104)."""
    y = torch.istft(mag * torch.exp(phase * 1j), n_fft, hop, n_fft, window=hann_periodic(n_fft))
    return y.unsqueeze(-2)


# --------------------------------------------------------------------------- a16 / a17 generators
def istftnet_har(f0_curve, sd: SD, cfg, rand_ini=None, sine_noise=None):
    """Harmonic-source features har=[|X| ; angle X] [B,22,120T+1] (istftnet.py:352-357)."""
    scale = int(np.prod(list(cfg["upsample_rates"])) * cfg["gen_istft_hop_size"])
    har_src = sine_source(f0_curve, scale, sd, rand_ini, sine_noise)
    mag, ph = stft_mag_phase(har_src, cfg["gen_istft_n_fft"], cfg["gen_istft_hop_size"])
    return torch.cat([mag, ph], dim=1)


def generator_istftnet(x, s, f0_curve, sd: SD, cfg, rand_ini=None, sine_noise=None, har=None):
    """Generator.forward, iSTFTNet (istftnet.py:350-380; ctor :303-347).
    `har`: teacher-forced STFT features (parity tests; see stft_mag_phase)."""
    rates, ks = list(cfg["upsample_rates"]), list(cfg["upsample_kernel_sizes"])
    rks, rds = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilation_sizes"]]
    n_fft, hop = cfg["gen_istft_n_fft"], cfg["gen_istft_hop_size"]
    if har is None:
        har = istftnet_har(f0_curve, sd, cfg, rand_ini, sine_noise)
    nk = len(rks)
    for i, (u, k) in enumerate(zip(rates, ks)):
        x = F.leaky_relu(x, 0.1)
        if i + 1 < len(rates):
            sf0 = int(np.prod(rates[i + 1:]))
            xs = F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"], stride=sf0, padding=(sf0 + 1) // 2)
            xs = adain_resblock1(xs, s, sd, f"noise_res.{i}", 7)
        else:
            xs = F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"])
            xs = adain_resblock1(xs, s, sd, f"noise_res.{i}", 11)
        x = F.conv_transpose1d(x, wn_weight(sd, f"ups.{i}"), sd[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        if i == len(rates) - 1:
            x = F.pad(x, (1, 0), mode="reflect")
        x = x + xs
        acc = None
        for j in range(nk):
            y = adain_resblock1(x, s, sd, f"resblocks.{i * nk + j}", rks[j], rds[j])
            acc = y if acc is None else acc + y
        x = acc / nk
    x = F.leaky_relu(x)
    x = conv1d(x, sd, "conv_post", padding=3)
    half = n_fft // 2 + 1
    return istft_from_mag_phase(torch.exp(x[:, :half]), torch.sin(x[:, half:]), n_fft, hop)


def generator_hifigan(x, s, f0_curve, sd: SD, cfg, rand_ini=None, sine_noise=None):
    """Generator.forward, HiFi-GAN (hifigan.py:321-347; ctor :273-319)."""
    rates, ks = list(cfg["upsample_rates"]), list(cfg["upsample_kernel_sizes"])
    rks, rds = list(cfg["resblock_kernel_sizes"]), [list(d) for d in cfg["resblock_dilation_sizes"]]
    scale = int(np.prod(rates))
    har = sine_source(f0_curve, scale, sd, rand_ini, sine_noise).unsqueeze(1)  # [B,1,L]
    nk = len(rks)
    for i, (u, k) in enumerate(zip(rates, ks)):
        x = snake(x, sd[f"alphas.{i}"])
        if i + 1 < len(rates):
            sf0 = int(np.prod(rates[i + 1:]))
            xs = F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"], stride=sf0, padding=(sf0 + 1) // 2)
            xs = adain_resblock1(xs, s, sd, f"noise_res.{i}", 7)
        else:
            xs = F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"])
            xs = adain_resblock1(xs, s, sd, f"noise_res.{i}", 11)
        x = F.conv_transpose1d(x, wn_weight(sd, f"ups.{i}"), sd[f"ups.{i}.bias"], stride=u,
                               padding=u // 2 + u % 2, output_padding=u % 2)
        x = x + xs
        acc = None
        for j in range(nk):
            y = adain_resblock1(x, s, sd, f"resblocks.{i * nk + j}", rks[j], rds[j])
            acc = y if acc is None else acc + y
        x = acc / nk
    x = snake(x, sd[f"alphas.{len(rates)}"])
    x = conv1d(x, sd, "conv_post", padding=3)
    return torch.tanh(x)


# --------------------------------------------------------------------------- a13 Decoder
def decoder(asr, f0_curve, n_curve, s, sd: SD, cfg, rand_ini=None, sine_noise=None, har=None):
    """Decoder.forward in eval mode (istftnet.py:499-528 == hifigan.py:446-475)."""
    f0 = conv1d(f0_curve.unsqueeze(1), sd, "F0_conv", stride=2, padding=1)
    n = conv1d(n_curve.unsqueeze(1), sd, "N_conv", stride=2, padding=1)
    x = torch.cat([asr, f0, n], dim=1)
    x = adain_resblk1d(x, s, sd, "encode")
    asr_res = conv1d(asr, sd, "asr_res.0")
    res = True
    nblk = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("decode."))
    for i in range(nblk):
        if res:
            x = torch.cat([x, asr_res, f0, n], dim=1)
        x = adain_resblk1d(x, s, sd, f"decode.{i}")
        if f"decode.{i}.pool.weight_v" in sd:
            res = False
    g = sub(sd, "generator")
    if cfg["type"] == "istftnet":
        return generator_istftnet(x, s, f0_curve, g, cfg, rand_ini, sine_noise, har)
    return generator_hifigan(x, s, f0_curve, g, cfg, rand_ini, sine_noise)


# --------------------------------------------------------------------------- a4/a5 denoiser
def _gelu(x):
    return F.gelu(x)  # exact erf form (nn.GELU default)


def denoiser_mapping(t, features, sd: SD):
    """get_mapping (modules.py:363-384 / :121-142): time embedding
    [t, sin(2 pi w t), cos(2 pi w t)] -> Linear(257->1024) -> GELU
    (+ GELU(Linear(256->1024)(features)) if multispeaker) -> 2x(Linear+GELU)."""
    w = sd["to_time.0.0.weights"]
    freqs = t.unsqueeze(1) * w.unsqueeze(0) * 2 * math.pi
    emb = torch.cat([t.unsqueeze(1), freqs.sin(), freqs.cos()], dim=-1)
    m = _gelu(linear(emb, sd, "to_time.0.1"))
    if "to_features.0.weight" in sd:
        m = torch.stack([m, _gelu(linear(features, sd, "to_features.0"))]).sum(0)
    m = _gelu(linear(m, sd, "to_mapping.0"))
    m = _gelu(linear(m, sd, "to_mapping.2"))
    return m


def _attention(x, ctx, sd: SD, p: str, heads=8):
    """Attention/StyleAttention core (modules.py:559-561,523-535): q from x, k|v from
    context, 8 heads x 64, softmax(q k^T / 8) v, Linear(512->1024)+bias.  No mask."""
    q = linear(x, sd, p + ".to_q")
    k, v = torch.chunk(linear(ctx, sd, p + ".to_kv"), 2, dim=-1)
    B, N, _ = q.shape
    sp = lambda z: z.view(B, N, heads, -1).permute(0, 2, 1, 3)
    q, k, v = sp(q), sp(k), sp(v)
    sim = torch.einsum("bhnd,bhmd->bhnm", q, k) * (q.shape[-1] ** -0.5)
    out = torch.einsum("bhnm,bhmd->bhnd", sim.softmax(dim=-1), v)
    out = out.permute(0, 2, 1, 3).reshape(B, N, -1)
    return linear(out, sd, p + ".attention.to_out")


def denoiser_run(x, t, embedding, features, sd: SD):
    """Transformer1d.run / StyleTransformer1d.run (modules.py:386-400 / :144-158)."""
    style = "blocks.0.attention.norm.fc.weight" in sd
    mapping = denoiser_mapping(t, features, sd).unsqueeze(1)
    N = embedding.size(1)
    h = torch.cat([x.expand(-1, N, -1), embedding], dim=-1)
    nb = 1 + max(int(k.split(".")[1]) for k in sd if k.startswith("blocks."))
    for i in range(nb):
        p = f"blocks.{i}"
        h = h + mapping
        if style:
            a = ada_layer_norm(h, features, sd, p + ".attention.norm")
            c = ada_layer_norm(h, features, sd, p + ".attention.norm_context")
        else:
            a = F.layer_norm(h, (h.shape[-1],), sd[p + ".attention.norm.weight"], sd[p + ".attention.norm.bias"])
            c = F.layer_norm(h, (h.shape[-1],), sd[p + ".attention.norm_context.weight"], sd[p + ".attention.norm_context.bias"])
        h = _attention(a, c, sd, p + ".attention") + h
        f = linear(_gelu(linear(h, sd, p + ".feed_forward.0")), sd, p + ".feed_forward.2")
        h = f + h
    h = h.mean(dim=1).unsqueeze(1)  # [B,1,1024]
    out = F.conv1d(h.transpose(1, 2), sd["to_out.1.weight"], sd["to_out.1.bias"])
    return out.transpose(-1, -2)


def denoiser_forward(x, t, embedding, features, sd: SD, embedding_scale=1.0):
    """Transformer1d.forward (modules.py:402-425): classifier-free guidance against the
    learned fixed embedding when embedding_scale != 1."""
    if embedding_scale != 1.0:
        N = embedding.shape[1]
        fixed = sd["fixed_embedding.embedding.weight"][:N].unsqueeze(0).expand(embedding.shape[0], -1, -1)
        out = denoiser_run(x, t, embedding, features, sd)
        out_masked = denoiser_run(x, t, fixed, features, sd)
        return out_masked + (out - out_masked) * embedding_scale
    return denoiser_run(x, t, embedding, features, sd)


# --------------------------------------------------------------------------- a1-a3, a19 sampler
def karras_sigmas(num_steps: int, sigma_min=1e-4, sigma_max=3.0, rho=9.0):
    """KarrasSchedule.forward (sampler.py:328-337); demo constants (#cell14)."""
    rho_inv = 1.0 / rho
    steps = torch.arange(num_steps, dtype=torch.float32)
    sig = (sigma_max ** rho_inv + (steps / (num_steps - 1)) * (sigma_min ** rho_inv - sigma_max ** rho_inv)) ** rho
    return F.pad(sig, (0, 1), value=0.0)


def kdiffusion_denoise(x_noisy, sigma, sd: SD, sigma_data, **kw):
    """KDiffusion.denoise_fn + get_scale_weights (sampler.py:184-208)."""
    B = x_noisy.shape[0]
    sigmas = torch.full((B,), float(sigma), dtype=torch.float32) if not torch.is_tensor(sigma) else sigma.expand(B).to(torch.float32)
    c_noise = torch.log(sigmas) * 0.25
    sg = sigmas.view(B, 1, 1)
    c_skip = (sigma_data ** 2) / (sg ** 2 + sigma_data ** 2)
    c_out = sg * sigma_data * (sigma_data ** 2 + sg ** 2) ** -0.5
    c_in = (sg ** 2 + sigma_data ** 2) ** -0.5
    x_pred = denoiser_forward(c_in * x_noisy, c_noise, sd=sd, **kw)
    return c_skip * x_noisy + c_out * x_pred


def adpm2_sample(noise, sd: SD, num_steps: int, embedding, features=None, embedding_scale=1.0,
                 sigma_data=0.2, step_noises: Optional[List[torch.Tensor]] = None):
    """DiffusionSampler.forward + ADPM2Sampler.forward/step/get_sigmas
    (sampler.py:573-586, 490-519), rho=1, clamp=False.  step_noises: injected
    randn_like draws, one per step (sampler.py:509)."""
    sigmas = karras_sigmas(num_steps)
    fn = lambda x, sigma: kdiffusion_denoise(x, sigma, sd, sigma_data, embedding=embedding,
                                             features=features, embedding_scale=embedding_scale)
    x = sigmas[0] * noise
    for i in range(num_steps - 1):
        sigma, sigma_next = sigmas[i], sigmas[i + 1]
        # get_sigmas: math.sqrt on 0-dim fp32 tensors -> python floats (fp64)
        sigma_up = math.sqrt(sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2)
        sigma_down = math.sqrt(sigma_next ** 2 - sigma_up ** 2)
        sigma_mid = ((sigma ** 1.0 + sigma_down ** 1.0) / 2) ** 1.0
        d = (x - fn(x, sigma)) / sigma
        x_mid = x + d * (sigma_mid - sigma)
        d_mid = (x_mid - fn(x_mid, sigma_mid)) / sigma_mid
        x = x + d_mid * (sigma_down - sigma)
        eps = step_noises[i] if step_noises is not None else torch.randn_like(x)
        x = x + eps * sigma_up
    return x


# --------------------------------------------------------------------------- end to end glue
def synthesize(sds: Dict[str, SD], model_cfg, tokens, input_lengths, bert_dur, noise, *,
               diffusion_steps=5, embedding_scale=1.0, ref_s=None, alpha=0.3, beta=0.7,
               rng=None, forced_durations=None, sigma_data=0.2, s_prev=None, t=0.7, skip_decoder=False, last_plus=None,
               front_only=False):
    """Batched (equal-length) version of the notebook `inference` glue
    (Demo/Inference_LJSpeech.ipynb#cell17 single-speaker; Demo/Inference_LibriTTS.ipynb#cell16
    multispeaker when ref_s is given).  `bert_dur` [B,N,768] is PL-BERT's output (an
    input producer, SURVEY section 8 f1).  rng: dict with optional 'step_noises' (list),
    'rand_ini', 'sine_noise', 'har' (teacher-forced STFT features).  s_prev / t: the long-form style carry-over of
    `LFinference` (Demo/Inference_LJSpeech.ipynb#cell29, Demo/Inference_LibriTTS.ipynb#cell42): s_pred = t*s_prev +
    (1-t)*s_pred before the split; 's_carry' is what the notebook returns as the next s_prev.
    last_plus: frames added to the last token's duration; None = the notebooks' `inference` convention (5 for the
    single-speaker cell 17, 0 for LibriTTS cell 16); the LJSpeech LFinference (cell 29) has NO increment -> pass 0.
    Returns a dict of every stage boundary."""
    rng = rng or {}
    dec_cfg = model_cfg["decoder"]
    multispeaker = ref_s is not None
    mask = length_to_mask(input_lengths)
    t_en = text_encoder(tokens, input_lengths, mask, sds["text_encoder"])
    d_en = F.linear(bert_dur, sds["bert_encoder"]["weight"], sds["bert_encoder"]["bias"]).transpose(-1, -2)
    s_pred = adpm2_sample(noise, sub(sds["diffusion"], "diffusion.net"), diffusion_steps, bert_dur,
                          features=ref_s, embedding_scale=embedding_scale, sigma_data=sigma_data,
                          step_noises=rng.get("step_noises")).squeeze(1)
    if s_prev is not None:
        s_pred = t * s_prev + (1 - t) * s_pred
    s = s_pred[:, 128:]
    ref = s_pred[:, :128]
    s_carry = s_pred
    if multispeaker:
        ref = alpha * ref + (1 - alpha) * ref_s[:, :128]
        s = beta * s + (1 - beta) * ref_s[:, 128:]
        s_carry = torch.cat([ref, s], dim=-1)
    pred = sds["predictor"]
    d = duration_encoder(d_en, s, input_lengths, mask, sub(pred, "text_encoder"))
    logits = duration_logits(d, pred)
    pred_dur = predict_durations(logits, (0 if multispeaker else 5) if last_plus is None else last_plus)
    if front_only:   # text side only (up to the integer boundary): any batch, totals need not agree
        return dict(t_en=t_en, d_en=d_en, s_pred=s_pred, s=s, ref=ref, d=d, logits=logits, pred_dur=pred_dur, s_carry=s_carry,
                    dur_f=torch.sigmoid(logits).sum(dim=-1))
    use_dur = pred_dur if forced_durations is None else forced_durations
    alns = [alignment_from_durations(use_dur[b]) for b in range(use_dur.shape[0])]
    T = alns[0].shape[1]
    assert all(a.shape[1] == T for a in alns), "batched oracle needs equal total durations"
    aln = torch.stack(alns)
    en = d.transpose(-1, -2) @ aln
    asr = t_en @ aln
    if dec_cfg["type"] == "hifigan":
        en, asr = shift_right_one(en), shift_right_one(asr)
    f0, n = f0n_train(en, s, pred)
    wav = None if skip_decoder else decoder(asr, f0, n, ref, sds["decoder"], dec_cfg, rng.get("rand_ini"), rng.get("sine_noise"),
                                            rng.get("har"))
    return dict(t_en=t_en, d_en=d_en, s_pred=s_pred, s=s, ref=ref, d=d, logits=logits, pred_dur=pred_dur,
                en=en, asr=asr, F0=f0, N=n, wav=wav, s_carry=s_carry)
