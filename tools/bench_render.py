#!/usr/bin/env python
"""Headless rendering (spann3r_b200.vis.render_frames) on the GPU vs the numpy rasteriser on the host.

Workloads, all drawn at 1920x1080 from a seeded scene of points in front of the camera (80 % kept by the mask):
  * demo:      50 frames of 224x224 points, static (the accumulated cloud), as demo.py --vis draws a sequence;
  * 512x384:   100 frames of 512x384 points, static and dynamic.
Device time: CUDA events around whole render_frames calls after a warm-up (best of 3).  Host encoding of the same frames
(PNG per frame + the 10 fps mp4v video, OpenCV, into a temporary directory) is timed separately.  The CPU peer is the
same rasteriser in vectorised numpy on the same host (oracle/render_oracle.py's algorithm, restated here because tools/
do not import the oracle), incremental like the kernels (one z-buffer kept across frames in static mode); its last frame
is compared with the GPU's byte for byte.  Open3D's window renderer is not measured (not installed).  Prints one JSON
line:  python tools/bench_render.py"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import vis  # noqa: E402

W_OUT, H_OUT = 1920, 1080


def scene(T, H, W, seed):
    rng = np.random.default_rng(seed)
    pts = np.empty((T, H, W, 3), np.float32)
    pts[..., :2] = rng.uniform(-1, 1, (T, H, W, 2))
    pts[..., 2] = rng.uniform(1.0, 3.0, (T, H, W))
    cols = rng.uniform(0, 1, (T, H, W, 3)).astype(np.float32)
    return pts, cols, rng.random((T, H, W)) < 0.8


def device_ms(fn, reps=3):
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


EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def host_peer(pts, cols, mask, cam, dynamic):
    """-> (ms, last frame [H_OUT, W_OUT, 3] uint8): s3r_render_* semantics in numpy, fp64 in the kernel's order."""
    T, H, W, _ = pts.shape
    per = H * W
    R = np.asarray(cam.extrinsic, np.float64)
    K = np.asarray(cam.intrinsic.intrinsic_matrix, np.float64)
    colors = cols.reshape(-1, 3).astype(np.float64)
    t0 = time.perf_counter()
    zbuf = np.full(H_OUT * W_OUT, EMPTY, np.uint64)
    for i in range(T):
        if dynamic:
            zbuf[:] = EMPTY
        p = pts[i].reshape(per, 3).astype(np.float64)
        q = [((R[r, 0] * p[:, 0] + R[r, 1] * p[:, 1]) + R[r, 2] * p[:, 2]) + R[r, 3] for r in range(3)]
        with np.errstate(all="ignore"):
            col = np.floor((K[0, 0] * (q[0] / q[2]) + K[0, 2]) + 0.5)
            row = np.floor((K[1, 1] * (q[1] / q[2]) + K[1, 2]) + 0.5)
        keep = mask[i].reshape(per) & np.isfinite(q[0]) & np.isfinite(q[1]) & np.isfinite(q[2]) & (q[2] > 0)
        keep &= (col >= 0) & (col < W_OUT) & (row >= 0) & (row < H_OUT)
        depth = q[2][keep].astype(np.float32).view(np.uint32).astype(np.uint64)
        ids = np.nonzero(keep)[0].astype(np.uint64) + np.uint64(i * per)
        pix = row[keep].astype(np.int64) * W_OUT + col[keep].astype(np.int64)
        np.minimum.at(zbuf, pix, (depth << np.uint64(32)) | ids)
        frame = np.zeros((H_OUT * W_OUT, 3), np.uint8)
        hit = zbuf != EMPTY
        c = colors[(zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
        frame[hit] = np.floor(np.fmin(1.0, np.fmax(0.0, c)) * 255.0 + 0.5).astype(np.uint8)
    return (time.perf_counter() - t0) * 1e3, frame.reshape(H_OUT, W_OUT, 3)


def workload(name, T, H, W, dynamic, seed, write_files):
    pts, cols, mask = scene(T, H, W, seed)
    cam = vis.camera_from_pose(np.eye(4), 700.0, W_OUT, H_OUT)
    p, c, m = torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), torch.from_numpy(mask).cuda()
    ms, frames = device_ms(lambda: vis.render_frames(p, c, cam, mask=m, dynamic=dynamic))
    r = {"workload": name, "frames": T, "points_per_frame": H * W, "mode": "dynamic" if dynamic else "static",
         "device_ms": round(ms, 3), "device_ms_per_frame": round(ms / T, 4),
         "lit_pixels_last_frame": int(frames[-1].any(-1).sum())}
    if write_files:
        with tempfile.TemporaryDirectory() as d:
            t0 = time.perf_counter()
            vis.write_frames(frames, d, cam, save_video=True)
            r["png_mp4_write_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    host_ms, last = host_peer(pts, cols, mask, cam, dynamic)
    r["numpy_host_ms"] = round(host_ms, 1)
    r["last_frame_equal_to_numpy"] = bool(np.array_equal(frames[-1].cpu().numpy(), last))
    return r


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res = {"gpu": q.stdout.strip() or torch.cuda.get_device_name(), "host_cores": os.cpu_count(),
           "render_size": [W_OUT, H_OUT], "open3d": "not measured",
           "runs": [workload("demo 224x224", 50, 224, 224, False, 0, True),
                    workload("512x384", 100, 384, 512, False, 1, True),
                    workload("512x384", 100, 384, 512, True, 2, False)]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
