#!/usr/bin/env python
"""Adversarial golden criterion values: runs the reference's OWN spann3r/loss.py (with dust3r/losses.py) on CPU in strict
fp32 on the edited views and predictions of `synth.make_loss_adv_case` (empty and single-pixel batch elements, tied
medians, NaN at invalid pixels, a clipped norm factor, points at dist_clip, two frames, d == 0 pixels) and writes
tests/golden/loss_adv_<case>.npz: the get_all_pts3d_t outputs and monitoring at full resolution, and for the "loss"
cases loss, factor_loss, details and the autograd gradients with respect to every pred and conf map, at full resolution.
Where the reference raises, the file records the exception instead of the values.
The files are written byte-reproducibly (fixed zip timestamps, one CPU thread).
The reference checkout is found through SPANN3R_REFERENCE or as ../reference next to the repository.
Authoring tool: nothing under tests/ or bench.py imports it."""
import io
import json
import os
import sys
import zipfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from spann3r_b200.synth import LOSS_ADV_CASES, loss_slot, make_loss_adv_case  # noqa: E402


def _reference():
    for root in (os.environ.get("SPANN3R_REFERENCE"), os.path.join(os.path.dirname(REPO), "reference")):
        if root and os.path.isfile(os.path.join(root, "spann3r", "loss.py")):
            sys.path.insert(0, root)
            import dust3r.losses  # noqa: F401
            import spann3r.loss as sl
            return sl
    raise SystemExit("reference checkout not found (set SPANN3R_REFERENCE)")


def _savez(path, arrays):
    """np.savez_compressed with fixed member timestamps, so that a regeneration is byte-identical."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def _pts(crit, gts, preds, kw, out):
    pl_crit = getattr(crit, "pixel_loss", crit)
    with torch.no_grad():
        gt_pts, (pl, pr), gf, pf, masks, mon = pl_crit.get_all_pts3d_t(gts, preds, **kw)
    for i, g in enumerate(gt_pts):
        out[f"gt_{i}"] = g.numpy()
        out[f"mask_{i}"] = masks[i].numpy()
    for k in range(len(pl)):
        out[f"pr_l_{k}"] = pl[k].numpy()
        out[f"pr_r_{k}"] = pr[k].numpy()
    out["gt_factor"] = np.array([], np.float32) if gf is None else gf.flatten().numpy()
    out["pr_factor"] = np.array([], np.float32) if pf is None else pf.flatten().numpy()
    out["mon_keys"] = np.array(list(mon.keys()), dtype="U32")
    out["mon_vals"] = np.array([float(v) for v in mon.values()], np.float64)


def main():
    torch.set_num_threads(1)
    sl = _reference()
    import dust3r.losses as dl
    ns = {**vars(dl), **vars(sl)}
    for name, case in LOSS_ADV_CASES.items():
        kw = case.get("kw", {})
        crit = eval(case["criterion"], ns)
        out = {"criterion": np.array(case["criterion"]), "case": np.array(json.dumps(case, sort_keys=True)),
               "raises": np.array("")}
        gts, preds = make_loss_adv_case(name)
        _pts(crit, gts, preds, kw, out)
        if case["call"] == "loss":
            gts, preds = make_loss_adv_case(name)
            F = len(gts)
            for k in range(F - 1):
                for side in (0, 1):
                    loss_slot(preds, k, side).requires_grad_(True)
                    preds[k][side]["conf"].requires_grad_(True)
            try:
                loss, details, fl = crit.compute_frame_loss(gts, preds, **kw)
                (loss + fl).backward()
            except Exception as ex:      # recorded: the native path must refuse the same case
                out["raises"] = np.array(type(ex).__name__)
            else:
                out["loss"] = np.float64(float(loss))
                out["factor_loss"] = np.float64(float(fl))
                out["detail_keys"] = np.array(list(details.keys()), dtype="U64")
                out["detail_vals"] = np.array([float(v) for v in details.values()], np.float64)
                for k in range(F - 1):
                    for side in (0, 1):
                        gp = loss_slot(preds, k, side).grad
                        gc = preds[k][side]["conf"].grad
                        out[f"grad_pts_{side}_{k}"] = gp.numpy()
                        out[f"grad_conf_{side}_{k}"] = (gc if gc is not None else torch.zeros_like(gp[..., 0])).numpy()
        path = os.path.join(REPO, "tests", "golden", f"loss_adv_{name}.npz")
        _savez(path, out)
        print(name, os.path.getsize(path), "bytes", str(out["raises"]) or (out.get("loss"), out.get("factor_loss")))


if __name__ == "__main__":
    main()
