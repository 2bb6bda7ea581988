"""Text(tokens) -> waveform glue with the Demo notebooks' semantics, batched.

Follows Demo/Inference_LJSpeech.ipynb#cell17 (`inference(text, noise, diffusion_steps, embedding_scale)`)
and Demo/Inference_LibriTTS.ipynb#cell16 (`inference(text, ref_s, alpha, beta, ...)`): text encoder ->
bert_encoder -> style diffusion sampler -> duration encoder / duration head -> integer durations ->
alignment expansion (gather) -> F0Ntrain -> decoder.  The notebook-level entry points (raw text in, numpy out)
live in styletts2_b200/demo.py; this class is the batched engine under them.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional

import torch

from . import ops
from .diffusion import ADPM2Sampler, DiffusionSampler, KarrasSchedule, TokenPacking
from .models import Munch


def length_to_mask(lengths, n=None):
    """utils.py:42-45 (n given: no host sync on lengths.max(), needed under CUDA-graph capture)"""
    n = int(lengths.max()) if n is None else n
    mask = torch.arange(n, device=lengths.device).unsqueeze(0).expand(lengths.shape[0], -1).type_as(lengths)
    return torch.gt(mask + 1, lengths.unsqueeze(1))


def make_sampler(model):
    """notebook cell 14"""
    return DiffusionSampler(model.diffusion.diffusion, sampler=ADPM2Sampler(),
                            sigma_schedule=KarrasSchedule(sigma_min=0.0001, sigma_max=3.0, rho=9.0), clamp=False)


@contextlib.contextmanager
def _stage(name, marks):
    """NVTX range (ST2_NVTX=1) + optional CUDA event at the END of a stage of the path."""
    if ops.NVTX:
        torch.cuda.nvtx.range_push(name)
    try:
        yield
    finally:
        if ops.NVTX:
            torch.cuda.nvtx.range_pop()
        if marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append((name, ev))


class Synthesizer:
    """Batched text->waveform engine over a build_model() container (on one GPU).

    Utterances of a batch may have different token counts (`input_lengths` < N: tokens are padded) and different
    predicted lengths: after the integer durations are known the batch is grouped by total frame count and every group
    runs the prosody predictor and the decoder at its own T (every op on the path is per-utterance, so a group of one
    is exactly the reference's single-utterance call); the waveforms come back zero-padded with `wav_lengths`."""

    def __init__(self, model: Munch, model_cfg, device="cuda"):
        self.model, self.cfg, self.device = model, model_cfg, torch.device(device)
        self.multispeaker = bool(model_cfg["multispeaker"])
        self.hifigan = model_cfg["decoder"]["type"] == "hifigan"
        self.sampler = make_sampler(model)
        ops._rng_epoch(self.device)   # allocate the device-resident draw epoch outside any graph capture

    # ------------------------------------------------------------------ stages
    def _tail(self, d, t_en, s, ref, use, T, rng, marks, decoder_events):
        """durations [B,N] int32 (equal totals T) -> (wav [B,1,600T], F0, N, en, asr)"""
        m = self.model
        with _stage("f0n", marks):
            tok, _ = ops.frame_tokens(use, T, shift_right=self.hifigan)
            en_rows = ops.expand_rows(d, tok)                                         # [B,T,640]
            asr = ops.expand_cl(t_en, tok)                                            # [B,512,T]
            F0, Ncurve = m.predictor.F0Ntrain(en_rows.transpose(-1, -2), s)
        F0_used = rng["F0"] if "F0" in rng else F0
        N_used = rng["N"] if "N" in rng else Ncurve
        with _stage("decoder", marks):
            if decoder_events is not None:
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
            wav = m.decoder(asr, F0_used, N_used, ref, sine_noise=rng.get("sine_noise"), har=rng.get("har"))
            if decoder_events is not None:
                ev1.record()
                decoder_events.append((ev0, ev1))
        return wav, F0, Ncurve, en_rows, asr

    @torch.no_grad()
    def synthesize(self, tokens, input_lengths, bert_dur, noise, *, diffusion_steps=5, embedding_scale=1.0, ref_s=None,
                   alpha=0.3, beta=0.7, rng: Optional[Dict] = None, forced_durations=None, pin_frames_per_token=None,
                   return_all=False, decoder_events=None, stage_marks=None, s_prev=None, t=0.7, last_plus=None,
                   token_packing=False):
        """tokens [B,N] i64, input_lengths [B], bert_dur [B,N,768] (or None: model.bert runs), noise [B,1,256] (device tensors).
        rng (parity mode): 'step_noises' list of [B,1,256], 'sine_noise' [B,L,9], 'har' [B,22,F],
        'F0' / 'N' [B,2T] (teacher-forced prosody curves: the harmonic source integrates F0 into a phase
        of 1e4..1e6 rad, so waveform comparisons inject the reference's curves after checking ours); for a ragged
        batch these are padded to the longest utterance.
        forced_durations [B,N] int: teacher-forced durations (after the duration kernel has run).
        pin_frames_per_token: throughput mode of SURVEY section 8d (durations pinned so that T = N*k).
        last_plus: frames added to the last real token (None: 5 single-speaker / 0 multispeaker as the notebooks'
        `inference`; LFinference of the LJSpeech notebook passes 0).
        token_packing: run the style sampler on packed token rows (diffusion.TokenPacking): each utterance's denoiser
        attends over and averages its own tokens only, so its s_pred is the one it gets alone, whatever the token counts
        of the rest of the batch.  Off (the default), the sampler sees the padded batch as the reference's batched
        sampler does: padding an utterance changes its style.  The packed path reads input_lengths on the host (one sync)
        and cannot be captured into a CUDA graph.
        s_prev [B,256], t: long-form style carry-over of the notebooks' LFinference (LJSpeech cell 29, LibriTTS cell 42):
        s_pred = t*s_prev + (1-t)*s_pred before it is split; out['s_carry'] is the value to pass as the next s_prev."""
        m = self.model
        rng = rng or {}
        dev = self.device
        B, N = tokens.shape
        marks = stage_marks
        if marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            marks.append(("start", ev))
        if "step_noises" not in rng or "sine_noise" not in rng:
            ops.rng_advance(dev)   # throughput mode: new Philox epoch per call (also per CUDA-graph replay)
        with _stage("text_encoder", marks):
            mask = length_to_mask(input_lengths, N)
            lens32 = input_lengths.to(device=dev, dtype=torch.int32).contiguous()
            if bert_dur is None:   # PL-BERT on our kernels (styletts2_b200.plbert.PLBert passed to build_model)
                bert_dur = m.bert(tokens, attention_mask=(~mask).int())
            t_en = m.text_encoder(tokens, input_lengths, mask)                       # [B,512,N]
            d_en_rows = m.bert_encoder(bert_dur)                                      # [B,N,512]
        with _stage("sampler", marks):
            kw = dict(embedding=bert_dur, num_steps=diffusion_steps, embedding_scale=embedding_scale,
                      step_noises=rng.get("step_noises"))
            if token_packing:
                packing = TokenPacking(input_lengths.tolist(), dev)     # host lengths size the packed buffers
                assert packing.B == B and packing.max_len <= N, (input_lengths, N)
                kw.update(embedding=packing.pack(bert_dur), packing=packing)
            if self.multispeaker:
                kw["features"] = ref_s
            s_pred = self.sampler(noise, **kw).reshape(B, 256)
        with _stage("duration", marks):
            if s_prev is not None:
                s_pred = ops.axpby(s_prev.reshape(B, 256), t, s_pred, 1 - t)
            s = s_pred[:, 128:]
            ref = s_pred[:, :128]
            s_carry = s_pred
            if self.multispeaker:
                ref = ops.axpby(ref, alpha, ref_s[:, :128], 1 - alpha)
                s = ops.axpby(s, beta, ref_s[:, 128:], 1 - beta)
                s_carry = None   # assembled below from the blended halves (LibriTTS cell 42: torch.cat([ref, s]))
            s, ref = s.contiguous(), ref.contiguous()
            if s_carry is None:
                s_carry = torch.empty(B, 256, device=dev)
                s_carry[:, :128].copy_(ref)
                s_carry[:, 128:].copy_(s)
            d = m.predictor.text_encoder(d_en_rows.transpose(-1, -2), s, input_lengths, mask)   # [B,N,640]
            x, _ = m.predictor.lstm(d, lens32)
            logits = m.predictor.duration_proj(x)                                     # [B,N,50]
            lp = (0 if self.multispeaker else 5) if last_plus is None else int(last_plus)
            pred_dur, dur_f = ops.durations(logits, lp, lens32)
        if forced_durations is not None:
            use = forced_durations.to(device=dev, dtype=torch.int32).contiguous()
        elif pin_frames_per_token is not None:
            use = torch.full((B, N), int(pin_frames_per_token), device=dev, dtype=torch.int32)
        else:
            use = pred_dur
        groups = None
        if pin_frames_per_token is not None and forced_durations is None:
            T = N * int(pin_frames_per_token)   # known a priori: no host sync (the whole path is CUDA-graph capturable)
        else:
            totals = use.sum(dim=1).tolist()    # the one host sync of the path: buffer sizes depend on it
            T = max(totals)
            if any(tt != T for tt in totals):
                groups = {}
                for b, tt in enumerate(totals):
                    groups.setdefault(int(tt), []).append(b)
        if groups is None:
            wav, F0, Ncurve, en_rows, asr = self._tail(d, t_en, s, ref, use, T, rng, marks, decoder_events)
            out = dict(wav=wav, pred_dur=pred_dur, T=T, s_carry=s_carry,
                       wav_lengths=torch.full((B,), 600 * T, dtype=torch.int64))
        else:
            # ragged batch: one launch chain per distinct total length (per-utterance semantics == the reference's
            # single-utterance call); results are zero-padded to the longest utterance
            wav = torch.zeros(B, 1, 600 * T, device=dev)
            F0 = torch.zeros(B, 2 * T, device=dev)
            Ncurve = torch.zeros(B, 2 * T, device=dev)
            en_rows = asr = None
            wl = torch.zeros(B, dtype=torch.int64)
            for Tg, idx in sorted(groups.items()):
                ii = torch.tensor(idx, device=dev)
                sub = {}
                for k_, v_ in rng.items():
                    if k_ == "sine_noise":
                        sub[k_] = v_[ii, :600 * Tg].contiguous()
                    elif k_ in ("F0", "N"):
                        sub[k_] = v_[ii, :2 * Tg].contiguous()
                    elif k_ == "har":
                        sub[k_] = v_[ii, :, :120 * Tg + 1].contiguous()
                w_, f_, n_, _, _ = self._tail(d[ii].contiguous(), t_en[ii].contiguous(), s[ii].contiguous(), ref[ii].contiguous(),
                                              use[ii].contiguous(), Tg, sub, marks, decoder_events)
                wav[ii, :, :600 * Tg] = w_
                F0[ii, :2 * Tg] = f_
                Ncurve[ii, :2 * Tg] = n_
                wl[idx] = 600 * Tg
            out = dict(wav=wav, pred_dur=pred_dur, T=T, s_carry=s_carry, wav_lengths=wl)
        if not torch.cuda.is_current_stream_capturing() and (forced_durations is not None or pin_frames_per_token is None):
            ops.check_range()     # fp16-plane range guard of the tensor-core GEMMs (the path has synchronised already)
        if return_all:
            out.update(t_en=t_en, d_en=d_en_rows.transpose(-1, -2), s_pred=s_pred, s=s, ref=ref, d=d, logits=logits,
                       dur_f=dur_f, en=None if en_rows is None else en_rows.transpose(-1, -2), asr=asr, F0=F0, N=Ncurve)
        return out

    def _weights_token(self):
        """Changes whenever a parameter of the path is replaced or modified in place (load_state_dict after a capture)."""
        tok = []
        for k in ("bert", "bert_encoder", "predictor", "decoder", "text_encoder", "diffusion"):
            mod = self.model.get(k)
            if isinstance(mod, torch.nn.Module):
                tok.extend((p.data_ptr(), p._version) for p in mod.parameters())
        return hash(tuple(tok))

    @torch.no_grad()
    def synthesize_graphed(self, tokens, input_lengths, bert_dur, noise, *, diffusion_steps=5, embedding_scale=1.0, ref_s=None,
                           alpha=0.3, beta=0.7, pin_frames_per_token=4):
        """Throughput mode: the whole path (durations pinned, RNG drawn on the device) captured ONCE per shape into a
        CUDA graph and replayed -- removes the ~450 per-launch host overheads of a pass.  Inputs are copied into the
        graph's static buffers; returns the graph's static output waveform [B,1,L] (valid until the next replay).
        The cache key holds every host scalar baked into the captured launches (alpha, beta, guidance scale, steps) and a
        token of the weights (a load_state_dict after capture re-prepares the kernel layouts into new buffers)."""
        from . import lib
        key = (tuple(tokens.shape), int(diffusion_steps), float(embedding_scale), ref_s is not None, bert_dur is not None,
               int(pin_frames_per_token), float(alpha), float(beta), self._weights_token())
        cache = self.__dict__.setdefault("_graphs", {})
        ent = cache.get(key)
        if ent is None:
            st = dict(tokens=tokens.clone(), lengths=input_lengths.clone(), bert=None if bert_dur is None else bert_dur.clone(),
                      noise=noise.clone(), ref_s=None if ref_s is None else ref_s.clone())
            kw = dict(diffusion_steps=diffusion_steps, embedding_scale=embedding_scale, alpha=alpha, beta=beta,
                      pin_frames_per_token=pin_frames_per_token)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):   # warm-up: lazy weight preparation, cudaFuncSetAttribute, constant tables
                    self.synthesize(st["tokens"], st["lengths"], st["bert"], st["noise"], ref_s=st["ref_s"], **kw)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            n0 = lib.launch_count()
            with torch.cuda.graph(g):
                out = self.synthesize(st["tokens"], st["lengths"], st["bert"], st["noise"], ref_s=st["ref_s"], **kw)
            ent = dict(graph=g, st=st, wav=out["wav"], launches=lib.launch_count() - n0)
            cache[key] = ent
        st = ent["st"]
        st["tokens"].copy_(tokens, non_blocking=True)
        st["lengths"].copy_(input_lengths, non_blocking=True)
        if bert_dur is not None:
            st["bert"].copy_(bert_dur, non_blocking=True)
        st["noise"].copy_(noise, non_blocking=True)
        if ref_s is not None:
            st["ref_s"].copy_(ref_s, non_blocking=True)
        ent["graph"].replay()
        return ent["wav"], ent["launches"]

    @torch.no_grad()
    def synthesize_texts(self, token_lists: List[List[int]], noise=None, ref_s=None, bert_dur=None, **kw):
        """A batch of utterances with any token counts in one call, each with the notebooks' single-utterance `inference`
        result: the token lists (already cleaned, with the leading 0) are padded, the text side runs batched with the style
        sampler on packed token rows (token_packing=True), and one numpy waveform per utterance comes back (LJSpeech: last
        token +5 frames; LibriTTS: the last 50 samples cut).  After the durations the batch is grouped by total frame count
        and each group runs its own prosody / decoder launch chain.
        noise [B,1,256] (None: drawn on the device), ref_s [B,256] or [1,256] (multispeaker), bert_dur [B,N,768] padded PL-BERT output
        (None: model.bert runs on the padded batch with its attention mask); kw go to synthesize."""
        dev = self.device
        B = len(token_lists)
        lens = [len(t) for t in token_lists]
        N = max(lens)
        tk = torch.zeros(B, N, dtype=torch.long)
        for b, t in enumerate(token_lists):
            tk[b, :lens[b]] = torch.as_tensor(list(t), dtype=torch.long)
        if noise is None:
            noise = ops.randn_like(torch.empty(B, 1, 256, device=dev))
        if ref_s is not None:
            ref_s = ref_s.to(dev).reshape(-1, 256).expand(B, 256).contiguous()     # one row: the same voice for all
        out = self.synthesize(tk.to(dev), torch.tensor(lens, device=dev), None if bert_dur is None else bert_dur.to(dev),
                              noise.to(dev).reshape(B, 1, 256), ref_s=ref_s, token_packing=True, **kw)
        wav = out["wav"].reshape(B, -1).cpu().numpy()
        wl = out["wav_lengths"].tolist()
        wavs = [wav[b, :wl[b]] for b in range(B)]
        return [w[..., :-50] for w in wavs] if self.multispeaker else wavs

    # ------------------------------------------------------------------ single-utterance conveniences (token ids in)
    def _one(self, tokens: List[int], bert_dur, noise, **kw):
        dev = self.device
        tk = torch.tensor([list(tokens)], dtype=torch.long, device=dev)
        lens = torch.tensor([tk.shape[1]], dtype=torch.long, device=dev)
        if noise is None:
            noise = ops.randn_like(torch.empty(1, 1, 256, device=dev))
        for k_ in ("ref_s", "s_prev"):
            if kw.get(k_) is not None:
                kw[k_] = kw[k_].to(dev)
        return self.synthesize(tk, lens, None if bert_dur is None else bert_dur.to(dev), noise.to(dev), **kw)

    @torch.no_grad()
    def LFinference(self, tokens: List[int], bert_dur, s_prev, noise=None, ref_s=None, alpha=0.3, beta=0.7, t=0.7,
                    diffusion_steps=5, embedding_scale=1.0):
        """Long-form step with the notebooks' conventions.  LJSpeech cell 29 (`alpha` there is `t` here): NO `pred_dur[-1] += 5`,
        no trim.  LibriTTS cell 42: the last 100 samples are cut.  Returns (numpy waveform, s_pred to pass as the next
        sentence's s_prev)."""
        out = self._one(tokens, bert_dur, noise, diffusion_steps=diffusion_steps, embedding_scale=embedding_scale, ref_s=ref_s,
                        alpha=alpha, beta=beta, s_prev=s_prev, t=t, last_plus=0)
        wav = out["wav"].squeeze().cpu().numpy()
        return (wav[..., :-100] if self.multispeaker else wav), out["s_carry"]

    @torch.no_grad()
    def inference(self, tokens: List[int], bert_dur, noise=None, ref_s=None, alpha=0.3, beta=0.7, diffusion_steps=5,
                  embedding_scale=1.0):
        """Single-utterance call with the notebooks' conventions: `tokens` already cleaned (TextCleaner) with
        the leading 0; returns a numpy waveform (LJSpeech cell 17: last token +5 frames; LibriTTS cell 16: the last 50
        samples are cut)."""
        out = self._one(tokens, bert_dur, noise, diffusion_steps=diffusion_steps, embedding_scale=embedding_scale, ref_s=ref_s,
                        alpha=alpha, beta=beta)
        wav = out["wav"].squeeze().cpu().numpy()
        return wav[..., :-50] if self.multispeaker else wav
