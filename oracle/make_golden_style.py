"""Pins oracle/style_oracle.py (SURVEY section 8 row f2) and writes tests/golden/style_libri.npz.

BUILD CONTAINER ONLY (needs the reference checkout ($STYLETTS2_REFERENCE) and torchaudio).  Checks, on key-seeded weights and a seeded
synthetic clip:
  1. oracle log-mel  == torchaudio.transforms.MelSpectrogram pipeline of the notebooks (cell 5 `preprocess`)
  2. oracle StyleEncoder == the UNMODIFIED reference StyleEncoder (models.py:139-164), both encoders
and stores the REFERENCE outputs as the fixture.  Run:  python -m oracle.make_golden_style
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cases, ref_import, style_oracle as SO  # noqa: E402
from styletts2_b200.synthetic import keyed_state_dict, synthetic_wave  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
CASE = dict(name="style_libri", B=2, samples=36000, seed=11)   # 1.5 s -> 121 frames (odd widths 121, 61, 31 on the way down)


def main():
    import torchaudio

    torch.manual_seed(0)
    torch.set_num_threads(8)
    nets, _ = ref_import.build_reference(cases.REF_CONFIG_FILE["libritts"])
    sds, shapes = {}, {}
    for k in ("style_encoder", "predictor_encoder"):
        shp = {n: tuple(v.shape) for n, v in nets[k].state_dict().items()}
        shapes[k] = {n: list(s) for n, s in shp.items()}
        sds[k] = keyed_state_dict(shp, k)
        nets[k].load_state_dict(sds[k])
        nets[k].eval()
    wave = synthetic_wave(CASE["B"], CASE["samples"], CASE["seed"])

    to_mel = torchaudio.transforms.MelSpectrogram(n_mels=80, n_fft=2048, win_length=1200, hop_length=300)
    with torch.no_grad():
        mel_ref = (torch.log(1e-5 + to_mel(wave)) - (-4)) / 4          # notebook preprocess(), batched
        mel_orc = SO.log_mel(wave)
        d_mel = float((mel_ref - mel_orc).abs().max())
        ref = torch.cat([nets["style_encoder"](mel_ref.unsqueeze(1)), nets["predictor_encoder"](mel_ref.unsqueeze(1))], dim=1)
        orc = SO.compute_style(sds, wave)
        orc_on_ref_mel = torch.cat([SO.style_encoder(mel_ref.unsqueeze(1), sds["style_encoder"]),
                                    SO.style_encoder(mel_ref.unsqueeze(1), sds["predictor_encoder"])], dim=1)
    d_s = float((ref - orc).abs().max())
    d_s_same_mel = float((ref - orc_on_ref_mel).abs().max())
    scale = float(ref.abs().max())
    print(f"log-mel: max|ref-oracle| = {d_mel:.3e}   (range {float(mel_ref.min()):.2f}..{float(mel_ref.max()):.2f})")
    print(f"ref_s  : max|ref-oracle| = {d_s:.3e} (same mel: {d_s_same_mel:.3e}), max|ref_s| = {scale:.3e}")
    assert d_mel <= 1e-4, d_mel
    assert d_s <= 1e-5 * max(1.0, scale) and d_s_same_mel <= 1e-5 * max(1.0, scale), (d_s, d_s_same_mel)
    np.savez_compressed(os.path.join(GOLD, CASE["name"] + ".npz"), wave=wave.numpy(), mel=mel_ref.numpy(), ref_s=ref.numpy())
    with open(os.path.join(GOLD, "state_shapes_style.json"), "w") as f:
        json.dump(shapes, f)
    pin_path = os.path.join(GOLD, "PINNING.json")
    pin = json.load(open(pin_path)) if os.path.exists(pin_path) else {}
    pin["style_libri"] = dict(case=CASE, log_mel_max_abs=d_mel, ref_s_max_abs=d_s, ref_s_same_mel_max_abs=d_s_same_mel,
                              ref_s_absmax=scale, torchaudio=torchaudio.__version__)
    json.dump(pin, open(pin_path, "w"), indent=1)
    print("wrote", CASE["name"] + ".npz")


if __name__ == "__main__":
    main()
