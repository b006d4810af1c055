#!/usr/bin/env python
"""Golden criterion values: runs the reference's OWN spann3r/loss.py (with dust3r/losses.py) on CPU in strict fp32 on
the seeded synthetic views and predictions of `synth.make_loss_case` and writes tests/golden/loss_<case>.npz: loss,
factor_loss, details, the get_all_pts3d_t outputs and monitoring, and the autograd gradients with respect to every pred
map and conf map.  Maps are stored subsampled (every `sub`-th pixel row and column, sub = height // SUB_CELLS) to keep each file under 1 MB.
The reference checkout is found through SPANN3R_REFERENCE or as ../reference next to the repository.
Authoring tool: nothing under tests/ or bench.py imports it."""
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from spann3r_b200.synth import LOSS_CASES, make_loss_case  # noqa: E402

SUB_CELLS = 28    # stored maps: about SUB_CELLS x SUB_CELLS samples per image


def _reference():
    for root in (os.environ.get("SPANN3R_REFERENCE"), os.path.join(os.path.dirname(REPO), "reference")):
        if root and os.path.isfile(os.path.join(root, "spann3r", "loss.py")):
            sys.path.insert(0, root)
            import dust3r.losses  # noqa: F401
            import spann3r.loss as sl
            return sl
    raise SystemExit("reference checkout not found (set SPANN3R_REFERENCE)")


def main():
    sl = _reference()
    import dust3r.losses as dl
    ns = {**vars(dl), **vars(sl)}
    for name, case in LOSS_CASES.items():
        gts, preds = make_loss_case(**case["data"])
        sub = max(1, case["data"]["height"] // SUB_CELLS)
        leaves = []
        for pr in preds:
            for d in pr:
                for k in d:
                    d[k].requires_grad_(case["call"] == "loss")
                    leaves.append(d[k])
        crit = eval(case["criterion"], ns)
        out = {"criterion": case["criterion"], "case": json.dumps(case), "sub": sub}
        kw = case.get("kw", {})
        if case["call"] == "loss":
            loss, details, fl = crit.compute_frame_loss(gts, preds, **kw)
            total = loss + fl
            total.backward()
            out["loss"] = float(loss)
            out["factor_loss"] = float(fl)
            out["detail_keys"] = np.array(list(details.keys()))
            out["detail_vals"] = np.array([float(v) for v in details.values()])
            F = len(gts)
            for k in range(F - 1):
                for s, key in ((0, "pts3d" if k == 0 else "pts3d_in_other_view"), (1, "pts3d_in_other_view")):
                    out[f"grad_pts_{s}_{k}"] = preds[k][s][key].grad[:, ::sub, ::sub].detach().numpy()
                    g = preds[k][s]["conf"].grad
                    out[f"grad_conf_{s}_{k}"] = (g if g is not None else torch.zeros_like(preds[k][s]["conf"]))[:, ::sub, ::sub].detach().numpy()
        else:
            with torch.no_grad():
                gt_pts, (pl, pr), gf, pf, masks, mon = crit.get_all_pts3d_t(gts, preds, **kw)
            for i, g in enumerate(gt_pts):
                out[f"gt_{i}"] = g[:, ::sub, ::sub].detach().numpy()
                out[f"mask_{i}"] = masks[i][:, ::sub, ::sub].detach().numpy()
            for k in range(len(pl)):
                out[f"pr_l_{k}"] = pl[k][:, ::sub, ::sub].detach().numpy()
                out[f"pr_r_{k}"] = pr[k][:, ::sub, ::sub].detach().numpy()
            out["gt_factor"] = np.array([]) if gf is None else gf.flatten().numpy()
            out["pr_factor"] = np.array([]) if pf is None else pf.flatten().numpy()
            out["mon_keys"] = np.array(list(mon.keys()))
            out["mon_vals"] = np.array([float(v) for v in mon.values()])
        path = os.path.join(REPO, "tests", "golden", f"loss_{name}.npz")
        np.savez_compressed(path, **out)
        print(name, os.path.getsize(path), "bytes", out.get("loss"), out.get("factor_loss"))


if __name__ == "__main__":
    main()
