"""Loader of the UNMODIFIED reference for the baseline legs of bench.py (and nothing else).

The reference's pure-Python forward path is staged byte-identical under the git-ignored `oracle/_ref/reference/` by
`oracle/stage_reference.py` (called from `__graft_entry__.build()` where a reference checkout is present), so it is
available wherever the built tree is, including machines without the reference checkout.
This module puts that tree on sys.path and builds `spann3r.model.Spann3R` (`spann3r/model.py:214-226`) on the synthetic
checkpoint the product is benchmarked on.  Baseline infrastructure: nothing under `spann3r_b200/` imports it.
"""
from __future__ import annotations

import argparse
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
_REF_OUT = os.path.join(os.path.dirname(HERE), "oracle", "_ref")   # written by oracle/stage_reference.py
_CANDIDATES = (os.path.join(_REF_OUT, "reference"),)
CUROPE_DIR = os.path.join(_REF_OUT, "curope")
_REF_TOP = ("spann3r", "dust3r", "croco", "models", "curope")


def root():
    """Directory of the reference tree to import from, or None."""
    for c in _CANDIDATES:
        if os.path.isfile(os.path.join(c, "spann3r", "model.py")):
            return c
    return None


def curope_available() -> bool:
    return os.path.isfile(os.path.join(CUROPE_DIR, "curope.so"))


def _purge():
    for name in list(sys.modules):
        top = name.split(".")[0]
        if top in _REF_TOP:
            del sys.modules[name]
    for p in list(sys.path):
        if p in _CANDIDATES or p == CUROPE_DIR or p.rstrip("/").endswith("/croco"):
            sys.path.remove(p)


def load(with_curope: bool = False):
    """Import (or re-import) the reference's `spann3r.model`.  with_curope: put the local build of the reference's own
    CUDA RoPE extension (oracle/stage_reference.py --curope) on the path, so that `croco/models/pos_embed.py:106-111`
    binds RoPE2D to cuRoPE2D instead of the PyTorch fallback.  The choice is made at import time, hence the purge."""
    r = root()
    if r is None:
        raise ImportError("the reference is not staged: run `python -m oracle.stage_reference` where a reference checkout exists")
    _purge()
    if with_curope:
        if not curope_available():
            raise ImportError("oracle/_ref/curope/curope.so not built (python -m oracle.stage_reference --curope)")
        sys.path.insert(0, CUROPE_DIR)
    sys.path.insert(0, r)
    import spann3r.model as ref_model   # noqa: the reference
    rope_cls = sys.modules["models.pos_embed"].RoPE2D.__name__
    if with_curope and rope_cls != "cuRoPE2D":
        raise ImportError("the reference did not pick up the curope extension")
    return ref_model


def build_model(state_dict: dict, dust3r_args: str, with_curope: bool = False, mem_pos_enc: bool = False):
    """`Spann3R(dus3r_name=<checkpoint file>)` exactly as demo.py / eval.py construct it, then the full strict load."""
    import torch
    ref_model = load(with_curope)
    torch.serialization.add_safe_globals([argparse.Namespace])
    dsd = {k[len("dust3r."):]: v for k, v in state_dict.items() if k.startswith("dust3r.")}
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "synthetic_dust3r.pth")
        torch.save({"args": argparse.Namespace(model=dust3r_args), "model": dsd}, path)
        m = ref_model.Spann3R(dus3r_name=path, use_feat=False, mem_pos_enc=mem_pos_enc)
    m.load_state_dict(state_dict, strict=True)
    return m.eval()
