#!/usr/bin/env python
"""Milliseconds per training view with ColorJitter, over a synthetic Co3d-layout tree (640x480 JPEG + 16-bit PNG depth
+ mask, spann3r_b200.synth.write_co3d_tree; resolution 224 by default):

  cpu_ref          a CPU restatement of the reference's per-item work (not the reference's code, which this tool does not
                   import): spann3r_b200.synth.Co3dLike's decoding and sampling, Pillow crop + Lanczos (geometry from
                   plan_view), torchvision ColorJitter + ImgNorm, cv2 nearest depth, numpy unprojection; 1 thread
  worker           the worker half of TrainViews on the same items (decoding, planning, host depth crop, jitter draws),
                   1 thread
  build            TrainViews.build of B items x F views (one build_planned call: host packing, one copy, four
                   launches, one synchronise), CUDA events, with every geometry's tables already cached
  build_cold       the same with the geometry cache emptied first (host wall clock around build + synchronise)
  jitter_kernel    views_color_jitter_kernel alone, from torch.profiler's CUDA activity, per launch of B x F views

The card's name and power limit are read in the same run and written beside the numbers.

    python tools/bench_train_views.py [--batch 4] [--frames 10] [--res 224] [--reps 5] [--out results/bench_train_views.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spann3r_b200 import synth  # noqa: E402
from spann3r_b200.train_views import TrainViews  # noqa: E402
from spann3r_b200.views import plan_view  # noqa: E402


def cpu_getitem(ds, idx):
    """BaseStereoViewDataset.__getitem__ on the CPU for a Co3dLike (unpatched): the reference's per-view work (Pillow
    crop + Lanczos, cv2 nearest depth, the transform, the numpy unprojection), geometry from plan_view."""
    import cv2
    import PIL.Image

    def crop(image, depthmap, intrinsics, resolution, rng=None, info=None):
        rgb = np.asarray(image)
        p = plan_view(rgb.shape[0], rgb.shape[1], intrinsics, resolution, ds.aug_crop, rng)
        l, t, r, b = p["crop1"]
        l2, t2, r2, b2 = p["crop2"]
        img = PIL.Image.fromarray(rgb).crop((l, t, r, b)).resize(p["scaled"], resample=PIL.Image.Resampling.LANCZOS)
        d = cv2.resize(depthmap[t:b, l:r], p["scaled"], interpolation=cv2.INTER_NEAREST)[t2:b2, l2:r2]
        return img.crop((l2, t2, r2, b2)), d, p["K"]

    ds._crop_resize_if_necessary = crop
    try:
        ds._rng = np.random.default_rng(seed=ds.seed + idx)
        views = ds._get_views(idx, ds._resolutions[0], ds._rng)
        for v in views:
            v["img"] = ds.transform(v["img"])
            d, K, pose = v["depthmap"], v["camera_intrinsics"], v["camera_pose"]
            u, w = np.meshgrid(np.arange(d.shape[1]), np.arange(d.shape[0]))
            X = np.stack(((u - K[0, 2]) * d / K[0, 0], (w - K[1, 2]) * d / K[1, 1], d), axis=-1).astype(np.float32)
            v["pts3d"] = np.einsum("ik, vuk -> vui", pose[:3, :3], X) + pose[:3, 3][None, None, :]
            v["valid_mask"] = (d > 0) & np.isfinite(v["pts3d"]).all(axis=-1)
        for v in views:
            v["rng"] = int.from_bytes(ds._rng.bytes(4), "big")
        return views
    finally:
        del ds._crop_resize_if_necessary


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power = (s.strip() for s in out[0].split(","))
        return {"name": name, "power_limit": power}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"not read ({e!r})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--frames", type=int, default=10)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_views needs a CUDA device")
    torch.set_num_threads(1)
    import cv2
    cv2.setNumThreads(1)
    B, F = args.batch, args.frames
    res = {"card": card(), "batch": B, "frames": F, "resolution": args.res}
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_co3d_tree(tmp, frames=60, width=640, height=480, seed=0, zero_frames=())
        kw = dict(resolution=args.res, num_frames=F, mask_bg="rand", seed=5, min_thresh=2, max_thresh=5, num_seq=50)
        ref = synth.Co3dLike(tmp, **kw)
        idxs = list(range(B))
        t = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            for i in idxs:
                cpu_getitem(ref, i)
            t.append((time.perf_counter() - t0) * 1e3 / (B * F))
        res["cpu_ref_ms_per_view"] = statistics.median(t)

        ds = synth.Co3dLike(tmp, **kw)
        tv = TrainViews(ds)
        t = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            items = [ds[i] for i in idxs]
            t.append((time.perf_counter() - t0) * 1e3 / (B * F))
        res["worker_ms_per_view"] = statistics.median(t)

        tv.build(items)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        t = []
        for _ in range(max(args.reps, 10)):
            ev[0].record()
            tv.build(items)
            ev[1].record()
            torch.cuda.synchronize()
            t.append(ev[0].elapsed_time(ev[1]))
        res["build_ms_per_batch"] = statistics.median(t)
        res["build_ms_per_view"] = res["build_ms_per_batch"] / (B * F)
        t = []
        for _ in range(max(args.reps, 10)):      # cold: every geometry's tables built and copied again
            tv._builders.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            tv.build(items)
            torch.cuda.synchronize()
            t.append((time.perf_counter() - t0) * 1e3)
        res["build_cold_ms_per_batch"] = statistics.median(t)
        res["geometries_per_batch"] = len(next(iter(tv._builders.values()))._tables)

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(10):
                tv.build(items)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                for name in ("views_color_jitter_kernel", "views_resample_v_u8_kernel", "views_resample_h_kernel",
                             "views_depth_kernel"):
                    if name in e.name:
                        kern.setdefault(name, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
        res["kernel_us_per_launch"] = {k: statistics.median(v) for k, v in kern.items()}
        if "views_color_jitter_kernel" in kern:
            res["jitter_kernel_us_per_view"] = res["kernel_us_per_launch"]["views_color_jitter_kernel"] / (B * F)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
