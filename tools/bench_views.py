#!/usr/bin/env python
"""Milliseconds per dataset view over one 50-view 7Scenes-layout sequence (640x480 PNG colour + 16-bit PNG depth +
pose text, resolution 224 by default):

  cpu              the CPU path the device replaces, as the reference runs it per view: Pillow Lanczos, cv2 nearest,
                   ImgNorm and the numpy unprojection (geometry from plan_view), 1 thread, decoded arrays in memory
  cpu_e2e          the same with the files decoded per view (what eval.py's loader does per view)
  device_e2e       DeviceViews over the same scene, decoding included, until the views are on the device
  device_build     ViewBuilder.build_planned alone (host packing, one copy, three launches, one synchronise), CUDA events
  device_kernels   the three view kernels alone, from torch.profiler's CUDA activity

    python tools/bench_views.py [--views 50] [--res 224] [--reps 5] [--out results/bench_views.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import cv2
import numpy as np
import PIL.Image
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spann3r_b200.synth import SevenScenesLike, write_7scenes_sequence  # noqa: E402
from spann3r_b200.views import plan_view  # noqa: E402


def cpu_view(rgb, depth, K, pose, resolution, rng):
    """One view on the CPU the way the reference computes it (crops, PIL LANCZOS, cv2 INTER_NEAREST, ImgNorm,
    fp64 unprojection, fp32 einsum, valid mask)."""
    p = plan_view(rgb.shape[0], rgb.shape[1], K, resolution, 0, rng)
    l, t, r, b = p["crop1"]
    l2, t2, r2, b2 = p["crop2"]
    img = PIL.Image.fromarray(rgb).crop((l, t, r, b)).resize(p["scaled"], resample=PIL.Image.Resampling.LANCZOS)
    img = np.asarray(img.crop((l2, t2, r2, b2))).astype(np.float32) / np.float32(255.0)
    img = ((img - np.float32(0.5)) / np.float32(0.5)).transpose(2, 0, 1)
    d = cv2.resize(depth[t:b, l:r], p["scaled"], interpolation=cv2.INTER_NEAREST)[t2:b2, l2:r2]
    Kf = p["K"]
    u, v = np.meshgrid(np.arange(d.shape[1]), np.arange(d.shape[0]))
    X = np.stack(((u - Kf[0, 2]) * d / Kf[0, 0], (v - Kf[1, 2]) * d / Kf[1, 1], d), axis=-1).astype(np.float32)
    pts = np.einsum("ik, vuk -> vui", pose[:3, :3], X) + pose[:3, 3][None, None, :]
    return img, d, pts, (d > 0) & np.isfinite(pts).all(axis=-1)


def decode_item(ds):
    """The dataset's own decoding of item 0 -> [(rgb, depth, K, pose)], stopping where the crop would start."""
    calls = []
    ds._crop_resize_if_necessary = lambda im, d, K, r, rng=None, info=None: (calls.append((im, d, K)), (None, None, K))[1]
    metas = ds._get_views(0, ds._resolutions[0], np.random.default_rng(ds.seed))
    del ds._crop_resize_if_necessary
    return [(rgb, d, K, m["camera_pose"]) for (rgb, d, K), m in zip(calls, metas)]


def cpu_item(ds, inputs=None):
    """cpu_view over every frame of item 0, decoding the files first unless `inputs` are given."""
    rng = np.random.default_rng(ds.seed)
    return [cpu_view(rgb, d, K, pose, ds._resolutions[0], rng) for rgb, d, K, pose in inputs or decode_item(ds)]


def timed(fn, reps):
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        out.append(time.perf_counter() - t0)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from spann3r_b200.views import DeviceViews, ViewBuilder

    torch.set_num_threads(1)
    cv2.setNumThreads(1)
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "chess", "seq-01")
        write_7scenes_sequence(root, frames=a.views)
        ds = SevenScenesLike(root, resolution=a.res, kf_every=1)
        inputs = decode_item(ds)                   # decoded arrays, for the arithmetic-only legs
        n = len(inputs)
        res["cpu_ms_per_view"] = 1e3 * timed(lambda: cpu_item(ds, inputs), max(1, a.reps // 2)) / n
        res["cpu_e2e_ms_per_view"] = 1e3 * timed(lambda: cpu_item(ds), max(1, a.reps // 2)) / n

        dv = DeviceViews(SevenScenesLike(root, resolution=a.res, kf_every=1))
        dv[0]
        torch.cuda.synchronize()
        res["device_e2e_ms_per_view"] = 1e3 * timed(lambda: (dv[0], torch.cuda.synchronize()), a.reps) / n

        vb = ViewBuilder(a.res)
        rng = np.random.default_rng(1)
        planned = [(rgb, d, pose, vb.plan(rgb.shape[0], rgb.shape[1], K, rng)) for rgb, d, K, pose in inputs]
        vb.build_planned(planned)
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            vb.build_planned(planned)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        res["device_build_ms_per_view"] = statistics.median(ms) / n

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                vb.build_planned(planned)
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "views_" in ev.key:
                kern[ev.key.split("(")[0]] = ev.device_time_total / 1e3 / a.reps     # ms per sequence
        res["device_kernels_ms_per_view"] = sum(kern.values()) / n
        res["kernels_ms_per_sequence"] = kern
    res.update(views=n, resolution=a.res, torch_threads=1, device=torch.cuda.get_device_name(0))
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:      # the numbers stand without it; say so
        res["power_limit"] = f"unavailable: {ex!r}"
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
