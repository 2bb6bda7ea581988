"""Pin the oracle against the UNMODIFIED reference and write tests/golden/ fixtures.

Runs ONLY in the build container (needs the reference checkout ($STYLETTS2_REFERENCE); see oracle/ref_import.py).
    python oracle/make_golden.py

For every case in oracle/cases.py it
  1. builds the reference modules (models.build_model) and loads the key-seeded
     weights (styletts2_b200/synthetic.py) through load_state_dict,
  2. drives them with the notebook glue (Demo/Inference_LJSpeech.ipynb#cell17,
     Demo/Inference_LibriTTS.ipynb#cell16), batched, with torch.randn_like/torch.rand
     patched to the deterministic ReplayRNG draws,
  3. runs oracle/styletts2_oracle.py on the same inputs and asserts agreement,
  4. stores the REFERENCE outputs as fixtures (+ PINNING.json with measured diffs,
     + state_shapes_*.json with the reference's state-dict schema).
"""
from __future__ import annotations

import json
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

import cases  # noqa: E402
import ref_import  # noqa: E402
import styletts2_oracle as O  # noqa: E402
from styletts2_b200.synthetic import keyed_state_dict  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
HOT = ["bert_encoder", "predictor", "decoder", "text_encoder", "diffusion"]


class PatchedRNG:
    """Context manager: torch.randn_like / torch.rand -> ReplayRNG in call order."""

    def __init__(self, rng: cases.ReplayRNG, n_steps: int):
        self.rng, self.n_steps, self.calls = rng, n_steps, []

    def __enter__(self):
        self._rl, self._r = torch.randn_like, torch.rand
        state = {"n": 0}

        def randn_like(x, *a, **k):
            shp = tuple(x.shape)
            i = state["n"]
            state["n"] += 1
            self.calls.append(("randn_like", shp))
            if shp[-1] == 256 and len(shp) == 3 and shp[1] == 1:
                return self.rng.step_noise(i, shp)
            if shp[-1] == 9:
                return self.rng.sine_noise(shp)
            return self.rng.unused(shp)

        def rand(*a, **k):
            shp = tuple(a[0]) if isinstance(a[0], (tuple, list, torch.Size)) else tuple(a)
            self.calls.append(("rand", shp))
            return self.rng.rand_ini(shp)

        torch.randn_like, torch.rand = randn_like, rand
        return self

    def __exit__(self, *e):
        torch.randn_like, torch.rand = self._rl, self._r


class HarRecorder:
    """Records the reference's har = [|X| ; angle X] (input of generator.noise_convs[0],
    iSTFTNet only).  angle X is ill-conditioned at near-zero |X| (oracle stft_mag_phase
    docstring), so fixtures carry a sparse patch = the bins where the reference's har
    differs from the oracle's by more than 1e-5; oracle har + patch == reference har."""

    def __init__(self, decoder):
        self.dec, self.har, self.h = decoder, None, None

    def __enter__(self):
        nc = self.dec.generator.noise_convs[0]
        if nc.in_channels > 1:
            def pre(m, inp):
                self.har = inp[0].clone()
            self.h = nc.register_forward_pre_hook(pre)
        return self

    def __exit__(self, *e):
        if self.h is not None:
            self.h.remove()


def har_patch(har_ref, har_orc, tol=1e-5):
    """(idx [n,3] int32, val [n] f32, stats) with har_orc[idx] := val giving har_ref to tol."""
    if har_ref is None:
        return np.zeros((0, 3), np.int32), np.zeros((0,), np.float32), {}
    d = (har_ref - har_orc).abs()
    idx = (d > tol).nonzero()
    val = har_ref[idx[:, 0], idx[:, 1], idx[:, 2]]
    half = har_ref.shape[1] // 2
    mags = har_ref[idx[:, 0], idx[:, 1] - half, idx[:, 2]] if len(idx) else torch.zeros(0)
    F = har_ref.shape[-1]
    stats = dict(n_bins=int(har_ref.numel()), n_patched=int(len(idx)),
                 n_edge=int(((idx[:, 2] == 0) | (idx[:, 2] == F - 1)).sum()) if len(idx) else 0,
                 max_mag_interior=float(mags[(idx[:, 2] != 0) & (idx[:, 2] != F - 1)].max()) if len(idx) and ((idx[:, 2] != 0) & (idx[:, 2] != F - 1)).any() else 0.0,
                 all_phase_channels=bool((idx[:, 1] >= half).all()) if len(idx) else True)
    return idx.numpy().astype(np.int32), val.numpy().astype(np.float32), stats


def apply_patch(har, idx, val):
    har = har.clone()
    if len(idx):
        i = torch.from_numpy(idx.astype(np.int64))
        har[i[:, 0], i[:, 1], i[:, 2]] = torch.from_numpy(val)
    return har


def load_models():
    out = {}
    for name, cfgfile in cases.REF_CONFIG_FILE.items():
        nets, args = ref_import.build_reference(cfgfile)
        sds, shapes = {}, {}
        for k in HOT:
            shp = {n: tuple(v.shape) for n, v in nets[k].state_dict().items()}
            shapes[k] = {n: list(s) for n, s in shp.items()}
            sds[k] = keyed_state_dict(shp, k)
            nets[k].load_state_dict(sds[k])
        with open(os.path.join(GOLD, f"state_shapes_{name}.json"), "w") as f:
            json.dump(shapes, f)
        out[name] = (nets, sds)
    return out


def reference_e2e(nets, model_cfg, case, tokens, lengths, bert_dur, noise, ref_s):
    """Notebook glue on the reference modules, batched over equal-length utterances."""
    from Modules.diffusion.sampler import ADPM2Sampler, DiffusionSampler, KarrasSchedule

    sampler = DiffusionSampler(nets["diffusion"].diffusion, sampler=ADPM2Sampler(),
                               sigma_schedule=KarrasSchedule(sigma_min=0.0001, sigma_max=3.0, rho=9.0), clamp=False)
    multispeaker = ref_s is not None
    hifigan = model_cfg["decoder"]["type"] == "hifigan"
    rng = cases.ReplayRNG(case["seed"])
    har_rec = HarRecorder(nets["decoder"])
    with torch.no_grad(), PatchedRNG(rng, case["steps"]) as pr, har_rec:
        mask = O.length_to_mask(lengths)
        t_en = nets["text_encoder"](tokens, lengths, mask)
        d_en = nets["bert_encoder"](bert_dur).transpose(-1, -2)
        kw = dict(embedding=bert_dur, num_steps=case["steps"], embedding_scale=case["embedding_scale"])
        if multispeaker:
            kw["features"] = ref_s
        s_pred = sampler(noise, **kw).squeeze(1)
        s, ref = s_pred[:, 128:], s_pred[:, :128]
        if multispeaker:
            ref = 0.3 * ref + (1 - 0.3) * ref_s[:, :128]
            s = 0.7 * s + (1 - 0.7) * ref_s[:, 128:]
        d = nets["predictor"].text_encoder(d_en, s, lengths, mask)
        x, _ = nets["predictor"].lstm(d)
        logits = nets["predictor"].duration_proj(x)
        duration = torch.sigmoid(logits).sum(axis=-1)
        pred_dur = torch.round(duration).clamp(min=1)
        if not multispeaker:
            pred_dur[:, -1] += 5
        # equalise total length across the batch so the batched decoder is legal
        # (InstanceNorm is per utterance; the reference demo itself is B=1)
        forced = pred_dur.clone()
        tot = forced.sum(1)
        forced[:, -1] += (tot.max() - tot)
        alns = torch.stack([O.alignment_from_durations(forced[b]) for b in range(forced.shape[0])])
        en = d.transpose(-1, -2) @ alns
        asr = t_en @ alns
        if hifigan:
            en, asr = O.shift_right_one(en), O.shift_right_one(asr)
        F0, N = nets["predictor"].F0Ntrain(en, s)
        wav = nets["decoder"](asr, F0, N, ref)
    return dict(t_en=t_en, d_en=d_en, s_pred=s_pred, d=d, logits=logits, pred_dur=pred_dur, forced_dur=forced,
                en=en, asr=asr, F0=F0, N=N, wav=wav.squeeze(1), har=har_rec.har), pr.calls


def main():
    os.makedirs(GOLD, exist_ok=True)
    torch.set_num_threads(8)
    models = load_models()
    pin = {"torch": torch.__version__, "threads": torch.get_num_threads(), "cases": {}}

    for cname, case in cases.E2E_CASES.items():
        nets, sds = models[case["model"]]
        mcfg = cases.MODEL_CFGS[case["model"]]
        tokens, lengths, bert_dur, noise, ref_s = cases.e2e_inputs(case)
        ref, calls = reference_e2e(nets, mcfg, case, tokens, lengths, bert_dur, noise, ref_s)
        rng = cases.ReplayRNG(case["seed"])
        B = case["B"]
        T = int(ref["forced_dur"][0].sum())
        L = ref["wav"].shape[-1]
        inj = dict(step_noises=[rng.step_noise(i, (B, 1, 256)) for i in range(case["steps"] - 1)],
                   rand_ini=rng.rand_ini((B, 9)), sine_noise=rng.sine_noise((B, L, 9)))
        pidx, pval, pstats = np.zeros((0, 3), np.int32), np.zeros((0,), np.float32), {}
        if ref["har"] is not None:
            with torch.no_grad():
                har_o = O.istftnet_har(ref["F0"], O.sub(sds["decoder"], "generator"), mcfg["decoder"],
                                       inj["rand_ini"], inj["sine_noise"])
            pidx, pval, pstats = har_patch(ref["har"], har_o)
            inj["har"] = apply_patch(har_o, pidx, pval)
        with torch.no_grad():
            orc = O.synthesize(sds, mcfg, tokens, lengths, bert_dur, noise, diffusion_steps=case["steps"],
                               embedding_scale=case["embedding_scale"], ref_s=ref_s, rng=inj,
                               forced_durations=ref["forced_dur"])
        diffs = {}
        for k in ["t_en", "d_en", "s_pred", "d", "logits", "en", "asr", "F0", "N"]:
            diffs[k] = float((orc[k] - ref[k]).abs().max())
        diffs["wav"] = float((orc["wav"].squeeze(1) - ref["wav"]).abs().max())
        diffs["pred_dur_mismatch"] = int((orc["pred_dur"] != ref["pred_dur"]).sum())
        scale = {k: float(ref[k].abs().max()) for k in ["s_pred", "F0", "N", "wav"]}
        print(cname, "T=", T, "L=", L, "diffs", diffs, "scale", scale, "rng calls", calls)
        assert diffs["pred_dur_mismatch"] == 0, "oracle durations differ from the reference"
        for k, v in diffs.items():
            if k != "pred_dur_mismatch":
                assert v <= 1e-5 * max(1.0, float(ref[k if k != 'wav' else 'wav'].abs().max())), (cname, k, v)
        pin["cases"][cname] = dict(diffs=diffs, scale=scale, T=T, L=L, har_patch=pstats,
                                   rng_calls=[[a, list(b)] for a, b in calls])
        np.savez_compressed(os.path.join(GOLD, cname + ".npz"),
                            pred_dur=ref["pred_dur"].numpy().astype(np.int32),
                            forced_dur=ref["forced_dur"].numpy().astype(np.int32),
                            s_pred=ref["s_pred"].numpy(), logits=ref["logits"].numpy(),
                            t_en=ref["t_en"].numpy(), d=ref["d"].numpy(),
                            F0=ref["F0"].numpy(), N=ref["N"].numpy(), wav=ref["wav"].numpy(),
                            har_patch_idx=pidx, har_patch_val=pval)

    for cname, case in cases.DECODER_CASES.items():
        nets, sds = models[case["model"]]
        mcfg = cases.MODEL_CFGS[case["model"]]
        asr, f0, n, s = cases.decoder_inputs(case)
        rng = cases.ReplayRNG(case["seed"])
        har_rec = HarRecorder(nets["decoder"])
        with torch.no_grad(), PatchedRNG(rng, 0) as pr, har_rec:
            wav_ref = nets["decoder"](asr, f0, n, s).squeeze(1)
        L = wav_ref.shape[-1]
        ri, sn = rng.rand_ini((case["B"], 9)), rng.sine_noise((case["B"], L, 9))
        har_inj, pidx, pval, pstats = None, np.zeros((0, 3), np.int32), np.zeros((0,), np.float32), {}
        if har_rec.har is not None:
            with torch.no_grad():
                har_o = O.istftnet_har(f0, O.sub(sds["decoder"], "generator"), mcfg["decoder"], ri, sn)
            pidx, pval, pstats = har_patch(har_rec.har, har_o)
            har_inj = apply_patch(har_o, pidx, pval)
        with torch.no_grad():
            wav_orc = O.decoder(asr, f0, n, s, sds["decoder"], mcfg["decoder"], ri, sn, har_inj).squeeze(1)
        diff = float((wav_orc - wav_ref).abs().max())
        print(cname, "L=", L, "wav diff", diff, "scale", float(wav_ref.abs().max()), pstats)
        assert diff <= 1e-5 * max(1.0, float(wav_ref.abs().max()))
        pin["cases"][cname] = dict(diffs=dict(wav=diff), scale=dict(wav=float(wav_ref.abs().max())), L=L, har_patch=pstats)
        np.savez_compressed(os.path.join(GOLD, cname + ".npz"), wav=wav_ref.numpy(),
                            har_patch_idx=pidx, har_patch_val=pval)

    pin_path = os.path.join(GOLD, "PINNING.json")
    if os.path.exists(pin_path):   # keep entries written by the other pinning scripts (make_golden_style.py)
        old = json.load(open(pin_path))
        for k, v in old.items():
            if k not in pin:
                pin[k] = v
    with open(pin_path, "w") as f:
        json.dump(pin, f, indent=1)
    print("golden fixtures written to", GOLD)


if __name__ == "__main__":
    main()
