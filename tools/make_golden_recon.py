#!/usr/bin/env python
"""Golden reconstruction metrics: runs the reference's OWN spann3r/tools/eval_recon.py (`accuracy`, `completion`,
`completion_ratio`, scipy cKDTree) on the seeded clouds of `spann3r_b200.synth.RECON_CASES` and writes
tests/golden/recon_eval.json: the metrics per case plus a seeded sample of (query, distance, index) triples of the
accuracy direction.  The reference checkout is found through SPANN3R_REFERENCE or as ../reference next to the repository.
Authoring tool: nothing under tests/ or bench.py imports it."""
import importlib.util
import json
import os
import sys

import numpy as np
import scipy

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from spann3r_b200 import synth  # noqa: E402

SAMPLES = 48


def _reference_eval_recon():
    for root in (os.environ.get("SPANN3R_REFERENCE"), os.path.join(os.path.dirname(REPO), "reference")):
        path = root and os.path.join(root, "spann3r", "tools", "eval_recon.py")
        if path and os.path.isfile(path):
            spec = importlib.util.spec_from_file_location("eval_recon", path)
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            return mod
    raise SystemExit("reference checkout not found (set SPANN3R_REFERENCE)")


def main():
    er = _reference_eval_recon()
    out = {"scipy": scipy.__version__, "numpy": np.__version__, "cases": []}
    for i, case in enumerate(synth.RECON_CASES):
        gt, pred, _ = synth.make_recon_case(*case)
        gt64, pred64 = gt.astype(np.float64), pred.astype(np.float64)
        scale = case[3]
        acc, acc_med = er.accuracy(gt64, pred64)
        comp, comp_med = er.completion(gt64, pred64)
        ratio = er.completion_ratio(gt64, pred64, dist_th=0.05 * scale)
        d, idx = er.KDTree(gt64).query(pred64)
        rng = np.random.default_rng(1000 + i)
        sel = np.sort(rng.choice(len(pred64), min(SAMPLES, len(pred64)), replace=False))
        out["cases"].append({"args": [case[0], case[1], case[2], case[3], case[4], case[5], case[6], list(case[7]),
                                      list(case[8]), case[9]],
                             "accuracy": [float(acc), float(acc_med)], "completion": [float(comp), float(comp_med)],
                             "completion_ratio": float(ratio), "dist_th": 0.05 * scale,
                             "sample": {"query": sel.tolist(), "dist": d[sel].tolist(), "index": idx[sel].tolist()}})
        print(case[0], len(gt), len(pred), acc, comp, ratio)
    path = os.path.join(REPO, "tests", "golden", "recon_eval.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
