"""Fixtures for the notebook-level boundary (TEST INFRASTRUCTURE; build container only: needs the reference checkout ($STYLETTS2_REFERENCE)).

Writes, from the UNMODIFIED reference tree:
  tests/golden/textcleaner_vocab.json   the 178-entry symbol table of text_utils.py and the ids of three val_list rows
  tests/golden/notebook_cells.json      the SOURCE of the inference cells of the two Demo notebooks, verbatim, so that
                                        tests/test_gpu_demo.py can exec() them over this package's modules
  tests/golden/plbert_real_fp16.npz     the bundled PL-BERT checkpoint (Utils/PLBERT/step_1000000.t7, loads under
                                        torch.load(weights_only=True)) rounded to fp16 (12 MB instead of 25), token rows
                                        from Data/val_list.txt, and transformers.AlbertModel's last_hidden_state on them
                                        WITH THE SAME fp16-rounded weights (so both sides of the parity test hold identical
                                        parameters with the real checkpoint's value distribution)
"""
import json
import os
import sys

import numpy as np
import torch
import yaml

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
REF = os.environ.get("STYLETTS2_REFERENCE", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "..", "StyleTTS2"))
GOLD = os.path.join(ROOT, "tests", "golden")


def main():
    sys.path.insert(0, REF)
    import text_utils as RT   # the reference's table (prints nothing at import)

    rows = [l.rstrip("\n").split("|") for l in open(os.path.join(REF, "Data", "val_list.txt"), encoding="utf-8").readlines()[:8]]
    dicts = RT.dicts
    sample = {}
    for r in rows[:3]:
        sample[r[1]] = [dicts[c] for c in r[1] if c in dicts]
    json.dump({"symbols": RT.symbols, "sample_ids": sample}, open(os.path.join(GOLD, "textcleaner_vocab.json"), "w"), ensure_ascii=False)

    cells = {}
    for key, nb, idx in (("lj_inference", "Inference_LJSpeech.ipynb", 17), ("lj_LFinference", "Inference_LJSpeech.ipynb", 29),
                         ("libri_inference", "Inference_LibriTTS.ipynb", 16), ("libri_LFinference", "Inference_LibriTTS.ipynb", 42),
                         ("libri_STinference", "Inference_LibriTTS.ipynb", 45)):
        d = json.load(open(os.path.join(REF, "Demo", nb)))
        cells[key] = {"notebook": nb, "cell": idx, "source": "".join(d["cells"][idx]["source"])}
    json.dump(cells, open(os.path.join(GOLD, "notebook_cells.json"), "w"), ensure_ascii=False, indent=1)

    # ---- PL-BERT with the real checkpoint (fp16-rounded on BOTH sides)
    from transformers import AlbertConfig, AlbertModel
    cfg = yaml.safe_load(open(os.path.join(REF, "Utils", "PLBERT", "config.yml")))["model_params"]
    ck = torch.load(os.path.join(REF, "Utils", "PLBERT", "step_1000000.t7"), map_location="cpu", weights_only=True)["net"]
    sd = {}
    for k, v in ck.items():
        name = k[7:] if k.startswith("module.") else k
        if name.startswith("encoder."):
            name = name[8:]
            if name != "embeddings.position_ids" and v.dtype == torch.float32:
                sd[name] = v.half()
    ref = AlbertModel(AlbertConfig(**cfg)).eval()
    missing, unexpected = ref.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not [m for m in missing if "position_ids" not in m], missing
    toks = [[0] + [dicts[c] for c in r[1] if c in dicts] for r in rows[:4]]
    N = max(len(t) for t in toks)
    lengths = torch.tensor([len(t) for t in toks])
    tokens = torch.zeros(len(toks), N, dtype=torch.long)
    for i, t in enumerate(toks):
        tokens[i, :len(t)] = torch.tensor(t)
    mask = (torch.arange(N)[None] < lengths[:, None]).int()
    torch.set_num_threads(8)
    with torch.no_grad():
        out = ref(tokens, attention_mask=mask).last_hidden_state
    stats = {k: float(v.float().abs().max()) for k, v in sd.items()}
    print("PL-BERT real weights: max |w| per tensor:", {k: round(v, 2) for k, v in sorted(stats.items(), key=lambda kv: -kv[1])[:6]})
    print("output abs max", float(out.abs().max()), "tokens", tuple(tokens.shape))
    np.savez_compressed(os.path.join(GOLD, "plbert_real_fp16.npz"), tokens=tokens.numpy(), lengths=lengths.numpy(),
                        last_hidden_state=out.numpy(), **{"w:" + k: v.numpy() for k, v in sd.items()})
    print("wrote", os.path.getsize(os.path.join(GOLD, "plbert_real_fp16.npz")) / 1e6, "MB")


if __name__ == "__main__":
    main()
