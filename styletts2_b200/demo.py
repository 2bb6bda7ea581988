"""Notebook-level entry points with the reference's signatures (the drop-in boundary, SURVEY.md section 8b):

    inference(text, noise, diffusion_steps=5, embedding_scale=1)                      Demo/Inference_LJSpeech.ipynb#cell17
    LFinference(text, s_prev, noise, alpha=0.7, diffusion_steps=5, embedding_scale=1)  Demo/Inference_LJSpeech.ipynb#cell29
    inference(text, ref_s, alpha=0.3, beta=0.7, diffusion_steps=5, embedding_scale=1)  Demo/Inference_LibriTTS.ipynb#cell16
    LFinference(text, s_prev, ref_s, alpha, beta, t, diffusion_steps, embedding_scale) Demo/Inference_LibriTTS.ipynb#cell42
    STinference(text, ref_s, ref_text, alpha, beta, diffusion_steps, embedding_scale)  Demo/Inference_LibriTTS.ipynb#cell45
    compute_style(wave or path)                                                        Demo/Inference_LibriTTS.ipynb#cell5

and one batched call with the `inference` signature over a list of texts (no notebook counterpart):

    inference_batch(texts, noise [B,1,256], diffusion_steps=5, embedding_scale=1)                   single-speaker
    inference_batch(texts, ref_s [B,256], alpha=0.3, beta=0.7, diffusion_steps=5, embedding_scale=1)  multispeaker

which returns one waveform per text, each what `inference` gives for that text alone (the style sampler runs on packed
token rows, Synthesizer.synthesize_texts).

The notebooks define these as module-level functions over globals (`model`, `sampler`, `textclenaer`,
`global_phonemizer`, `device`); `bind(...)` builds the same set of callables over a `build_model()` container of this
package, so a notebook swaps its import and keeps its cells:

    from styletts2_b200.demo import bind
    nb = bind(model, model_params, device, phonemizer=global_phonemizer)   # or phonemizer=None for IPA input
    wav = nb.inference(text, noise, diffusion_steps=5, embedding_scale=1)

Every arithmetic op runs through the C-ABI kernels (Synthesizer); PL-BERT is `styletts2_b200.plbert.PLBert` when the
container's `bert` is one (no `transformers` on the path).  The phonemizer (espeak, GPL, not in this image) is the
caller's: `phonemizer.phonemize([text]) -> [ipa]`; with phonemizer=None the text must already be IPA phonemes.
"""
from __future__ import annotations

from typing import Callable, Optional

import numpy as np
import torch

from .inference import Synthesizer, length_to_mask, make_sampler
from .models import Munch
from .text import TextCleaner, word_tokenize as _word_tokenize


class _Identity:
    """phonemizer stand-in: the text is already a phoneme string (e.g. the rows of Data/val_list.txt)"""

    def phonemize(self, texts):
        return list(texts)


def bind(model: Munch, model_params, device="cuda", phonemizer=None, word_tokenize: Optional[Callable] = None):
    """Returns a namespace with the notebooks' functions for this model (single-speaker or multispeaker by config)."""
    cfg = model_params
    syn = Synthesizer(model, cfg, device)
    dev = syn.device
    textclenaer = TextCleaner()
    global_phonemizer = phonemizer if phonemizer is not None else _Identity()
    wt = word_tokenize or _word_tokenize
    multispeaker = bool(cfg["multispeaker"])

    def _tokens(text, strip_quotes, requote=False):
        text = text.strip()
        if strip_quotes:
            text = text.replace('"', '')
        ps = global_phonemizer.phonemize([text])
        ps = ' '.join(wt(ps[0]))
        if requote:                                   # LibriTTS cell 42
            ps = ps.replace('``', '"').replace("''", '"')
        tokens = textclenaer(ps)
        tokens.insert(0, 0)
        return tokens

    def _bert(tokens):
        """model.bert(tokens, attention_mask=(~text_mask).int()) of the notebooks, on whatever `bert` the container holds."""
        tk = torch.LongTensor(tokens).to(dev).unsqueeze(0)
        lens = torch.LongTensor([tk.shape[-1]]).to(dev)
        mask = length_to_mask(lens)
        with torch.no_grad():
            return model.bert(tk, attention_mask=(~mask).int())

    def _noise(B=1):
        return torch.randn((B, 256)).unsqueeze(1).to(dev)          # the multispeaker cells draw it themselves

    if not multispeaker:
        def inference(text, noise, diffusion_steps=5, embedding_scale=1):
            tokens = _tokens(text, strip_quotes=True)
            return syn.inference(tokens, _bert(tokens), noise=noise, diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

        def LFinference(text, s_prev, noise, alpha=0.7, diffusion_steps=5, embedding_scale=1):
            tokens = _tokens(text, strip_quotes=True)
            return syn.LFinference(tokens, _bert(tokens), s_prev, noise=noise, t=alpha, diffusion_steps=diffusion_steps,
                                   embedding_scale=embedding_scale)

        def inference_batch(texts, noise, diffusion_steps=5, embedding_scale=1):
            token_lists = [_tokens(t, strip_quotes=True) for t in texts]
            return syn.synthesize_texts(token_lists, noise=noise, diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

        STinference = None
    else:
        def inference_batch(texts, ref_s, alpha=0.3, beta=0.7, diffusion_steps=5, embedding_scale=1):
            token_lists = [_tokens(t, strip_quotes=False) for t in texts]
            return syn.synthesize_texts(token_lists, noise=_noise(len(texts)), ref_s=ref_s, alpha=alpha, beta=beta,
                                        diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

        def inference(text, ref_s, alpha=0.3, beta=0.7, diffusion_steps=5, embedding_scale=1):
            tokens = _tokens(text, strip_quotes=False)
            return syn.inference(tokens, _bert(tokens), noise=_noise(), ref_s=ref_s, alpha=alpha, beta=beta,
                                 diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

        def LFinference(text, s_prev, ref_s, alpha=0.3, beta=0.7, t=0.7, diffusion_steps=5, embedding_scale=1):
            tokens = _tokens(text, strip_quotes=False, requote=True)
            return syn.LFinference(tokens, _bert(tokens), s_prev, noise=_noise(), ref_s=ref_s, alpha=alpha, beta=beta, t=t,
                                   diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

        def STinference(text, ref_s, ref_text, alpha=0.3, beta=0.7, diffusion_steps=5, embedding_scale=1):
            """Cell 45 also runs PL-BERT on `ref_text`, but its result (`ref_bert_dur`) is never used by the shipped code:
            the output equals inference(text, ref_s, ...).  The reference text is still tokenised and encoded so that
            invalid input fails the same way."""
            tokens = _tokens(text, strip_quotes=False)
            ref_tokens = _tokens(ref_text, strip_quotes=False)
            _bert(ref_tokens)
            return syn.inference(tokens, _bert(tokens), noise=_noise(), ref_s=ref_s, alpha=alpha, beta=beta,
                                 diffusion_steps=diffusion_steps, embedding_scale=embedding_scale)

    def compute_style(wave_or_path, sr=24000):
        """Cell 5: waveform (numpy / tensor at 24 kHz, already trimmed) or a path readable by the caller's loader -> ref_s [1,256].
        librosa's load/trim are file I/O outside the accelerated path; arrays go straight to the GPU mel front-end."""
        from .style import compute_style as _cs
        if isinstance(wave_or_path, str):
            raise RuntimeError("pass the decoded 24 kHz waveform: librosa file loading/trimming is outside this package")
        wave = torch.as_tensor(np.asarray(wave_or_path), dtype=torch.float32)
        return _cs(model, wave.to(dev))

    return Munch(inference=inference, inference_batch=inference_batch, LFinference=LFinference, STinference=STinference, compute_style=compute_style,
                 textclenaer=textclenaer, length_to_mask=length_to_mask, sampler=make_sampler(model), synthesizer=syn,
                 device=dev, global_phonemizer=global_phonemizer, word_tokenize=wt)
