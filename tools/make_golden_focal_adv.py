#!/usr/bin/env python
"""Golden values of the reference's focal estimate on adversarial pointmaps: the REAL
dust3r.post_process.estimate_focal_knowing_depth (CPU, fp32) in both modes on every frame of synth.FOCAL_ADV_CASES, plus
the fp64 weiszfeld value (the same reference function on pts.double()) and the fp32 reference's deviation from it
-> tests/golden/focal_adv.json.  NaN is written as JSON NaN.  The pointmaps are regenerated from their seeds by the tests."""
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")
from dust3r.post_process import estimate_focal_knowing_depth  # noqa: E402

from spann3r_b200 import synth  # noqa: E402


def _f(v):
    return float(v)


if __name__ == "__main__":
    torch.set_num_threads(1)        # the reference's CPU reductions in one fixed order
    cases = []
    for name in synth.FOCAL_ADV_CASES:
        pts = synth.make_focal_adv_case(name)
        B, H, W, _ = pts.shape
        pp = torch.tensor((W / 2, H / 2))
        f32 = estimate_focal_knowing_depth(pts, pp, focal_mode="weiszfeld")
        fm = estimate_focal_knowing_depth(pts, pp, focal_mode="median")
        f64 = estimate_focal_knowing_depth(pts.double(), pp.double(), focal_mode="weiszfeld")
        dev = [abs(float(a) - float(b)) if math.isfinite(float(a)) and math.isfinite(float(b)) else float("nan")
               for a, b in zip(f32.tolist(), f64.tolist())]
        cases.append(dict(name=name, B=B, H=H, W=W, underflow=name == "underflow",
                          focal=[_f(v) for v in f32], focal_f64=[_f(v) for v in f64], ref_err=dev,
                          focal_median=[_f(v) for v in fm]))
        print(name, cases[-1]["focal"], cases[-1]["focal_f64"], cases[-1]["focal_median"])
    with open(os.path.join(ROOT, "tests", "golden", "focal_adv.json"), "w") as fh:
        json.dump({"cases": cases}, fh, indent=1)
        fh.write("\n")
