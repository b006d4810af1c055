#!/usr/bin/env python
"""Time Spann3R's criteria: the native kernels (spann3r_b200.loss) against the reference's own criterion from the copy
that `__graft_entry__.build()` stages under oracle/_ref (absent: the native arm alone), on synthetic views
(synth.make_loss_case), with CUDA events, mean over --iters calls after --warmup.  Prints the card and its power limit,
then one JSON line per workload:
  train  ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4) forward + backward, B=4, F=10, 224^2
  eval   Regr3D_t_ScaleShiftInv(L21, norm_mode=False, gt_scale=True).get_all_pts3d_t, B=1, F=50, 224^2
  eval   the same at F=10, 512x384
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [
    ("train", "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)", 4, 10, 224, 224),
    ("eval", "Regr3D_t_ScaleShiftInv(L21, norm_mode=False, gt_scale=True)", 1, 50, 224, 224),
    ("eval", "Regr3D_t_ScaleShiftInv(L21, norm_mode=False, gt_scale=True)", 1, 10, 384, 512),
]


def namespaces():
    ns_native = {}
    exec("from spann3r_b200.loss import *", ns_native)
    ns_ref = None
    try:
        from baseline import ref_loader
        if ref_loader.root() is not None:
            sys.path.insert(0, ref_loader.root())
            import dust3r.losses as dl
            import spann3r.loss as sl
            ns_ref = {**vars(dl), **vars(sl)}
    except ImportError as ex:
        print("reference criterion not available:", ex)
    return ns_native, ns_ref


def time_one(kind, crit, gts, preds, iters, warmup):
    leaves = [t for p in preds for d in p for t in d.values()]

    def once():
        if kind == "train":
            for t in leaves:
                t.grad = None
            loss, details, fl = crit.compute_frame_loss(gts, preds)
            (loss + fl).backward()
        else:
            with torch.no_grad():
                # the reference modifies norm_mode=False predictions in place: give it fresh copies each call
                p = [tuple({k: v.clone() for k, v in d.items()} for d in pr) for pr in preds] if fresh else preds
                crit.get_all_pts3d_t(gts, p)

    fresh = kind == "eval"
    for _ in range(warmup):
        once()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        once()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loss needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q or torch.cuda.get_device_name(0), flush=True)
    from spann3r_b200 import synth
    ns_native, ns_ref = namespaces()
    for kind, crit_str, B, F, H, W in WORKLOADS:
        gts, preds = synth.make_loss_case(B, F, H, W, invalid=0.3, seed=0, device="cuda:0")
        if kind == "train":
            for p in preds:
                for d in p:
                    for t in d.values():
                        t.requires_grad_(True)
        row = {"workload": kind, "criterion": crit_str, "batch": B, "frames": F, "height": H, "width": W,
               "iters": a.iters, "card": q}
        row["native_ms"] = time_one(kind, eval(crit_str, ns_native), gts, preds, a.iters, a.warmup)
        if ns_ref is not None:
            row["reference_ms"] = time_one(kind, eval(crit_str, ns_ref).to("cuda:0"), gts, preds, a.iters, a.warmup)
            row["speedup"] = row["reference_ms"] / row["native_ms"]
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
