#!/usr/bin/env python
"""Build recipe of the reference peer: stage the UNMODIFIED reference's forward path under the git-ignored
`oracle/_ref/reference/` and build the reference's own CUDA RoPE extension under `oracle/_ref/curope/`, so that
`bench.py` can time the reference ITSELF -- `spann3r.model.Spann3R` (`spann3r/model.py:473-539` of the reference) -- as
the CPU arm (`--impl reference`) and as the PyTorch-eager peer on the same GPU, also where the reference checkout is
not present (only `oracle/_ref/` is needed there).

    python -m oracle.stage_reference              # copy the ~20 pure-Python files of the path (byte-identical)
    python -m oracle.stage_reference --curope     # also build the reference's own CUDA RoPE extension (sm_90)

The reference checkout is `$SPANN3R_REFERENCE`, else a `reference` directory next to this repository, else
`/root/reference` (where the golden vectors under tests/golden were made).  `__graft_entry__.build()` calls
`stage()` and `build_curope()` when one of them exists.  Nothing is written to tracked paths.

--curope: the reference's extension does not compile against this torch as shipped (`kernels.cu:101` uses the removed
`Tensor::type()` dispatch argument).  A COPY of its two source files is made under `oracle/_ref/curope/`, that one token
is replaced (`tokens.type()` -> `tokens.scalar_type()`), and the extension is built there for sm_90 (H100) with the
reference's own flags (`-O3 --use_fast_math`, setup.py:24-27).  The staged reference picks it up when
`oracle/_ref/curope` is on sys.path (`import curope`, curope2d.py:6-9); otherwise it falls back to its PyTorch RoPE2D.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import shutil
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(REPO, "oracle", "_ref", "reference")
DST_CUROPE = os.path.join(REPO, "oracle", "_ref", "curope")


def reference_dir():
    """The reference checkout to stage from, or None."""
    cands = [os.environ.get("SPANN3R_REFERENCE"), os.path.join(os.path.dirname(REPO), "reference"), "/root/reference"]
    for c in cands:
        if c and os.path.isfile(os.path.join(c, "spann3r", "model.py")):
            return c
    return None


# the import closure of spann3r.model (forward path) + what the training step of config 5 needs on top of it
FILES = [
    "spann3r/model.py",
    "spann3r/loss.py",
    "dust3r/__init__.py", "dust3r/model.py", "dust3r/patch_embed.py", "dust3r/losses.py", "dust3r/inference.py",
    "dust3r/heads/__init__.py", "dust3r/heads/dpt_head.py", "dust3r/heads/linear_head.py", "dust3r/heads/postprocess.py",
    "dust3r/utils/__init__.py", "dust3r/utils/misc.py", "dust3r/utils/path_to_croco.py", "dust3r/utils/geometry.py",
    "dust3r/utils/device.py",
    "croco/models/blocks.py", "croco/models/croco.py", "croco/models/pos_embed.py", "croco/models/dpt_block.py",
    "croco/models/masking.py",
    "croco/models/curope/__init__.py", "croco/models/curope/curope2d.py",
]
CUROPE_SRC = ["curope.cpp", "kernels.cu"]


def stage(verbose=True) -> dict:
    REF = reference_dir()
    if REF is None:
        raise SystemExit("no reference checkout found (set SPANN3R_REFERENCE)")
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(REF, rel), os.path.join(DST, rel)
        if not os.path.exists(src):
            if verbose:
                print("skip (absent in the reference):", rel)
            continue
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        manifest[rel] = hashlib.sha256(open(dst, "rb").read()).hexdigest()[:16]
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"source": REF, "files": manifest}, f, indent=1)
    if verbose:
        print(f"staged {len(manifest)} files under {DST}")
    return manifest


def build_curope(verbose=True) -> str:
    REF = reference_dir()
    if REF is None:
        raise SystemExit("no reference checkout found (set SPANN3R_REFERENCE)")
    os.makedirs(DST_CUROPE, exist_ok=True)
    for name in CUROPE_SRC:
        s = open(os.path.join(REF, "croco/models/curope", name)).read()
        if name == "kernels.cu":
            assert s.count("tokens.type()") == 1
            s = s.replace("tokens.type()", "tokens.scalar_type()")   # the ONE token (file docstring)
        open(os.path.join(DST_CUROPE, name), "w").write(s)
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0"    # the H100; the only change to the reference's build
    from torch.utils.cpp_extension import load
    load(name="curope", sources=[os.path.join(DST_CUROPE, n) for n in CUROPE_SRC], build_directory=DST_CUROPE,
         extra_cflags=["-O3"], extra_cuda_cflags=["-O3", "--use_fast_math"], verbose=verbose, is_python_module=False)
    so = os.path.join(DST_CUROPE, "curope.so")
    if verbose:
        print("built", so)
    return so


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--curope", action="store_true")
    a = ap.parse_args()
    stage()
    if a.curope:
        build_curope()
    sys.exit(0)
