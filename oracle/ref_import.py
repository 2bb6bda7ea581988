"""Import the UNMODIFIED reference (yl4579/StyleTTS2) read-only from the reference checkout ($STYLETTS2_REFERENCE).

TEST INFRASTRUCTURE ONLY.  Works only in the build container (the GPU box has no
the reference checkout ($STYLETTS2_REFERENCE)); used by oracle/make_golden.py to pin the oracle restatement
(oracle/styletts2_oracle.py) against the real reference forward and to emit the
fixtures under tests/golden/.  Nothing in the product path imports this.

The reference needs two third-party names that are not installed here
(SURVEY.md §8c): `munch.Munch` (models.py:24,672) and
`einops_exts.rearrange_many` (Modules/diffusion/modules.py:10,525).  They are
injected as in-memory stubs; no reference source is copied.
"""
import os
import sys
import types

REF_ROOT = os.environ.get("STYLETTS2_REFERENCE", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "..", "StyleTTS2"))


def available() -> bool:
    return os.path.isdir(os.path.join(REF_ROOT, "Modules"))


def _install_stubs():
    if "munch" not in sys.modules:
        m = types.ModuleType("munch")

        class Munch(dict):
            def __getattr__(self, k):
                try:
                    return self[k]
                except KeyError as e:
                    raise AttributeError(k) from e

            def __setattr__(self, k, v):
                self[k] = v

        m.Munch = Munch
        sys.modules["munch"] = m
    if "einops_exts" not in sys.modules:
        import einops

        m = types.ModuleType("einops_exts")

        def rearrange_many(tensors, pattern, **kw):
            return tuple(einops.rearrange(t, pattern, **kw) for t in tensors)

        m.rearrange_many = rearrange_many
        sys.modules["einops_exts"] = m


def import_reference():
    """Returns the reference's `models` module (and makes `Modules.*` importable)."""
    if not available():
        raise RuntimeError("reference tree not present at %s" % REF_ROOT)
    _install_stubs()
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    import models  # noqa: the reference's models.py

    return models


def recursive_munch(d):
    from munch import Munch

    if isinstance(d, dict):
        return Munch((k, recursive_munch(v)) for k, v in d.items())
    if isinstance(d, list):
        return [recursive_munch(v) for v in d]
    return d


class _BertCfg:
    hidden_size = 768
    max_position_embeddings = 512


class _FakeBert:
    """build_model only reads bert.config.{hidden_size,max_position_embeddings}
    (models.py:643-660); PL-BERT itself is an input producer (SURVEY §8 f1)."""
    config = _BertCfg()


def build_reference(config_name="config.yml"):
    import torch.nn as nn
    import yaml

    models = import_reference()
    cfg = yaml.safe_load(open(os.path.join(REF_ROOT, "Configs", config_name)))
    args = recursive_munch(cfg["model_params"])
    import torch
    bert = nn.Identity()
    bert.config = _BertCfg()
    nets = models.build_model(args, nn.Identity(), nn.Identity(), bert)
    for k in nets:
        nets[k].eval()
    return nets, args
