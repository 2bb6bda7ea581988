"""Extra pinning of the oracle against the UNMODIFIED reference on configurations other than the committed fixtures
(different seeds, batch sizes, token counts, sampler steps, guidance scales; both model families).  No fixtures are
written -- only the measured agreement, to tests/golden/PINNING_SWEEP.json.  BUILD CONTAINER ONLY (needs the reference checkout ($STYLETTS2_REFERENCE)).
Run:  python -m oracle.pin_sweep
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cases  # noqa: E402
import styletts2_oracle as O  # noqa: E402
from make_golden import GOLD, apply_patch, har_patch, load_models, reference_e2e  # noqa: E402

SWEEP = {
    "lj_b1_n5": dict(model="ljspeech", B=1, N=5, steps=3, embedding_scale=1.0, seed=101),
    "lj_b2_n19_cfg": dict(model="ljspeech", B=2, N=19, steps=5, embedding_scale=1.5, seed=102),
    "libri_b1_n7": dict(model="libritts", B=1, N=7, steps=4, embedding_scale=1.0, seed=103),
    "libri_b2_n13_cfg": dict(model="libritts", B=2, N=13, steps=6, embedding_scale=2.0, seed=104),
}


def style_sweep():
    """compute_style path (row f2): other clip lengths / batch sizes than the committed fixture."""
    import torchaudio

    import ref_import
    import style_oracle as SO
    from styletts2_b200.synthetic import keyed_state_dict, synthetic_wave
    nets, _ = ref_import.build_reference(cases.REF_CONFIG_FILE["libritts"])
    sds = {}
    for k in ("style_encoder", "predictor_encoder"):
        sds[k] = keyed_state_dict({n: tuple(v.shape) for n, v in nets[k].state_dict().items()}, k)
        nets[k].load_state_dict(sds[k])
        nets[k].eval()
    to_mel = torchaudio.transforms.MelSpectrogram(n_mels=80, n_fft=2048, win_length=1200, hop_length=300)
    res = {}
    for name, (B, samples, seed) in {"b1_101f": (1, 30000, 21), "b3_152f": (3, 45300, 22), "b1_80f": (1, 23999, 23)}.items():
        wave = synthetic_wave(B, samples, seed)
        with torch.no_grad():
            mel_ref = (torch.log(1e-5 + to_mel(wave)) + 4) / 4
            ref = torch.cat([nets["style_encoder"](mel_ref.unsqueeze(1)), nets["predictor_encoder"](mel_ref.unsqueeze(1))], dim=1)
            orc = SO.compute_style(sds, wave)
            d_mel = float((SO.log_mel(wave) - mel_ref).abs().max())
        d = float((orc - ref).abs().max())
        print("style", name, "frames", mel_ref.shape[-1], "log-mel", d_mel, "ref_s", d, "scale", float(ref.abs().max()))
        assert d_mel <= 1e-4 and d <= 1e-5
        res[name] = dict(B=B, samples=samples, frames=int(mel_ref.shape[-1]), log_mel_max_abs=d_mel, ref_s_max_abs=d,
                         ref_s_absmax=float(ref.abs().max()))
    return res


def main():
    torch.set_num_threads(8)
    models = load_models()   # also rewrites state_shapes_*.json with identical content
    out = {"torch": torch.__version__, "cases": {}}
    for cname, case in SWEEP.items():
        nets, sds = models[case["model"]]
        mcfg = cases.MODEL_CFGS[case["model"]]
        tokens, lengths, bert_dur, noise, ref_s = cases.e2e_inputs(case)
        ref, _ = reference_e2e(nets, mcfg, case, tokens, lengths, bert_dur, noise, ref_s)
        rng = cases.ReplayRNG(case["seed"])
        B, L = case["B"], ref["wav"].shape[-1]
        inj = dict(step_noises=[rng.step_noise(i, (B, 1, 256)) for i in range(case["steps"] - 1)],
                   rand_ini=rng.rand_ini((B, 9)), sine_noise=rng.sine_noise((B, L, 9)))
        if ref["har"] is not None:
            with torch.no_grad():
                har_o = O.istftnet_har(ref["F0"], O.sub(sds["decoder"], "generator"), mcfg["decoder"], inj["rand_ini"], inj["sine_noise"])
            pidx, pval, _ = har_patch(ref["har"], har_o)
            inj["har"] = apply_patch(har_o, pidx, pval)
        with torch.no_grad():
            orc = O.synthesize(sds, mcfg, tokens, lengths, bert_dur, noise, diffusion_steps=case["steps"],
                               embedding_scale=case["embedding_scale"], ref_s=ref_s, rng=inj, forced_durations=ref["forced_dur"])
        diffs = {k: float((orc[k] - ref[k]).abs().max()) for k in ["t_en", "s_pred", "d", "logits", "F0", "N"]}
        diffs["wav"] = float((orc["wav"].squeeze(1) - ref["wav"]).abs().max())
        diffs["pred_dur_mismatch"] = int((orc["pred_dur"] != ref["pred_dur"]).sum())
        scale = {k: float(ref[k].abs().max()) for k in ["s_pred", "F0", "wav"]}
        print(cname, diffs, scale)
        assert diffs["pred_dur_mismatch"] == 0
        for k, v in diffs.items():
            if k != "pred_dur_mismatch":
                assert v <= 1e-5 * max(1.0, float(ref[k].abs().max())), (cname, k, v)
        out["cases"][cname] = dict(case=case, diffs=diffs, scale=scale, T=int(ref["forced_dur"][0].sum()))
    out["style"] = style_sweep()
    with open(os.path.join(GOLD, "PINNING_SWEEP.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote PINNING_SWEEP.json")


if __name__ == "__main__":
    main()
