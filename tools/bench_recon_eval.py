#!/usr/bin/env python
"""Reconstruction metrics of one eval.py scene on the GPU (spann3r_b200.recon_eval) vs scipy on the host.

A seeded 50-frame 224x224 scene (synth.make_eval_scene: 2.5 M predicted + 2.5 M ground-truth points before masking).
CUDA-event times of the index build, ICP (with its pass count), normals of both clouds, accuracy + completion, and the
whole of evaluate_reconstruction; scipy cKDTree accuracy + completion (tree builds + both 1-NN queries, default single
worker, as eval_recon.py calls it) on the same clouds in the same run.  Open3D's ICP and normals are not measured (not
installed).  Prints one JSON line:  python tools/bench_recon_eval.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import recon_eval as R  # noqa: E402
from spann3r_b200 import synth  # noqa: E402


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best, out = float("inf"), None
    for _ in range(reps):
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return best, out


def main():
    pts, pts_gt, masks = synth.make_eval_scene()
    keep = masks > 0
    pred_np, gt_np = pts[keep].astype(np.float64), pts_gt[keep].astype(np.float64)
    pred, gt = torch.from_numpy(pts[keep]).cuda(), torch.from_numpy(pts_gt[keep]).cuda()
    res = {"what": "eval.py reconstruction metrics, 50 x 224 x 224 scene, 1 % far outliers",
           "n_pred": int(len(pred)), "n_gt": int(len(gt))}
    res["index_build_ms"], gt_index = timed(lambda: R.PointIndex(gt))
    res["icp_ms"], out = timed(lambda: R._icp(pred, gt_index, 0.1, None, 30, 1e-6, 1e-6))
    res["icp_passes"] = int(out[18].item())
    pred_index = R.PointIndex(pred)
    res["normals_both_ms"], _ = timed(lambda: (gt_index.normals(30), pred_index.normals(30)))
    res["accuracy_completion_ms"], _ = timed(lambda: (R.accuracy(gt, pred), R.completion(gt, pred)))
    res["evaluate_reconstruction_ms"], m = timed(
        lambda: R.evaluate_reconstruction(torch.from_numpy(pts).cuda(), torch.from_numpy(pts_gt).cuda(),
                                          torch.from_numpy(masks).cuda(), 0.1))
    res["metrics"] = m._asdict()
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    d1, _ = cKDTree(gt_np).query(pred_np)
    d2, _ = cKDTree(pred_np).query(gt_np)
    res["scipy_accuracy_completion_ms"] = (time.perf_counter() - t0) * 1e3
    res["scipy_mean_distances"] = [float(np.mean(d1)), float(np.mean(d2))]
    res["host_cores"] = os.cpu_count()
    res["open3d_icp_and_normals"] = "not measured"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res["gpu"] = q.stdout.strip() or torch.cuda.get_device_name()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
