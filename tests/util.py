"""Shared helpers for the parity tests (test infrastructure)."""
import json
import os

import numpy as np
import torch

import cases
import styletts2_oracle as O
from styletts2_b200.synthetic import keyed_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def golden(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def ref_shapes(model_name):
    return json.load(open(os.path.join(GOLD, f"state_shapes_{model_name}.json")))


_SDS = {}


def oracle_sds(model_name, modules=("bert_encoder", "predictor", "decoder", "text_encoder", "diffusion")):
    """Key-seeded CPU state dicts with the reference's schema (no checkout of the reference needed)."""
    out = {}
    shapes = ref_shapes(model_name)
    for k in modules:
        key = (model_name, k)
        if key not in _SDS:
            _SDS[key] = keyed_state_dict({n: tuple(s) for n, s in shapes[k].items()}, k)
        out[k] = _SDS[key]
    return out


def apply_patch(har, idx, val):
    har = har.clone()
    if len(idx):
        i = torch.from_numpy(idx.astype(np.int64))
        har[i[:, 0], i[:, 1], i[:, 2]] = torch.from_numpy(val)
    return har


def maxdiff(a, b):
    return float((a.detach().cpu().float() - b.detach().cpu().float()).abs().max())


_MODELS = {}


def gpu_model(model_name):
    """build_model() on cuda:0 with the key-seeded weights."""
    from styletts2_b200.models import build_model, load_keyed_weights, recursive_munch
    if model_name not in _MODELS:
        m = build_model(recursive_munch(cases.MODEL_CFGS[model_name]))
        for k in m:
            m[k].to("cuda")
            m[k].eval()
        load_keyed_weights(m)
        _MODELS[model_name] = m
    return _MODELS[model_name]


def record(name, **vals):
    """Append measured parity figures to the JSON-lines file named by ST2_PARITY_REPORT (nothing is written without it)."""
    path = os.environ.get("ST2_PARITY_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(test=name, **{k: (float(v) if not isinstance(v, (int, str, bool)) else v) for k, v in vals.items()})) + "\n")
