#!/usr/bin/env python
"""Times the mesh path on the GPU (run on the H100):

  * app.py's post-processing of a reconstruction: its host numpy face build (`host_faces`, app.py's per-frame
    pts3d_to_trimesh + cat_meshes restated) plus a GLB write, against `mesh.pts3d_to_mesh` + `write_glb`, at
    50 frames of 224 x 224 and 10 frames of 512 x 384;
  * `render_depth_maps`' draws on a seeded DTU-sized mesh (a bumpy sphere of a few million triangles) from 49 views at
    1600 x 1200, device time per view with CUDA events.

    python tools/bench_mesh.py [--out results/bench_mesh.json]

Prints the card's name and power limit beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spann3r_b200 import mesh  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:   # the numbers still stand with the torch name
        q = f"{torch.cuda.get_device_name()} (power limit unknown: {ex!r})"
    return q


def events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def host_faces(img_all, pts_all, valid_all):
    """app.py's host face build: per frame, the four blocks of two triangles per pixel quad (each in both windings),
    the faces with an invalid corner removed, then the frames joined with their vertex offsets."""
    faces, colors = [], []
    for t, (img, valid) in enumerate(zip(img_all, valid_all)):
        H, W, _ = img.shape
        idx = np.arange(H * W).reshape(H, W)
        i1, i2, i3, i4 = idx[:-1, :-1].ravel(), idx[:-1, 1:].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()
        f = np.concatenate([np.c_[i1, i2, i3], np.c_[i3, i2, i1], np.c_[i2, i3, i4], np.c_[i4, i3, i2]])
        tl, br = img[:-1, :-1].reshape(-1, 3), img[1:, 1:].reshape(-1, 3)
        c = np.concatenate([tl, tl, br, br])
        keep = valid.ravel()[f].all(-1)
        faces.append(f[keep] + t * H * W)
        colors.append(c[keep])
    return np.concatenate(faces), np.concatenate(colors)


def app_post(T, H, W, tmp):
    rng = np.random.default_rng(T * H)
    pts = rng.normal(0, 1, (T, H, W, 3)).astype(np.float32)
    img = rng.uniform(0, 1, (T, H, W, 3)).astype(np.float32)
    valid = rng.random((T, H, W)) < 0.8
    path = os.path.join(tmp, "scene.glb")
    M = mesh.app_scene_matrix()
    t0 = time.perf_counter()
    faces, _ = host_faces(img, pts, valid)
    t1 = time.perf_counter()
    mesh.write_glb(path, pts.reshape(-1, 3), faces, img.reshape(-1, 3), M)
    t2 = time.perf_counter()
    P, I, V = (torch.from_numpy(x).cuda() for x in (pts, img, valid))
    dev_ms = events_ms(lambda: mesh.pts3d_to_mesh(P, I, V), 5)
    t3 = time.perf_counter()
    v, f, _ = mesh.pts3d_to_mesh(P, I, V)
    mesh.write_glb(path, v, f, I.reshape(-1, 3), M)
    t4 = time.perf_counter()
    assert np.array_equal(f.cpu().numpy(), faces.astype(np.int32))
    return {"T": T, "H": H, "W": W, "faces": int(len(faces)), "candidates": 4 * T * (H - 1) * (W - 1),
            "host_faces_ms": 1e3 * (t1 - t0), "host_glb_ms": 1e3 * (t2 - t1), "device_faces_ms": dev_ms,
            "device_faces_plus_glb_ms": 1e3 * (t4 - t3), "glb_bytes": os.path.getsize(path)}


def sphere(n_lat, n_lon, radius, bump, seed):
    rng = np.random.default_rng(seed)
    th, ph = np.meshgrid(np.linspace(0.01, np.pi - 0.01, n_lat), np.linspace(0, 2 * np.pi, n_lon, endpoint=False),
                         indexing="ij")
    r = radius * (1 + bump * np.sin(7 * th) * np.cos(5 * ph) + 0.002 * rng.standard_normal(th.shape))
    v = np.stack([r * np.sin(th) * np.cos(ph), r * np.sin(th) * np.sin(ph), r * np.cos(th)], -1).reshape(-1, 3)
    i = np.arange(n_lat * n_lon).reshape(n_lat, n_lon)
    a, b = i[:-1], np.roll(i, -1, 1)[:-1]
    c, d = i[1:], np.roll(i, -1, 1)[1:]
    f = np.concatenate([np.stack([a, c, b], -1).reshape(-1, 3), np.stack([b, c, d], -1).reshape(-1, 3)])   # outward
    return v.astype(np.float32), f


def dtu_render():
    v, f = sphere(1000, 1500, 300.0, 0.05, 0)             # ~3.0 M triangles, DTU's millimetre scale
    K = np.array([[2892.0, 0, 824.0], [0, 2883.0, 605.0], [0, 0, 1]])   # a DTU camera at 1600 x 1200
    poses = []
    for k in range(49):
        ang = 2 * np.pi * k / 49
        eye = np.array([700 * np.cos(ang), 700 * np.sin(ang), 200.0 * np.sin(3 * ang)])
        fwd = -eye / np.linalg.norm(eye)
        right = np.cross(fwd, [0, 0, 1.0])
        right /= np.linalg.norm(right)
        down = np.cross(fwd, right)
        P = np.eye(4)
        P[:3, 0], P[:3, 1], P[:3, 2], P[:3, 3] = right, -down, -fwd, eye
        poses.append(P)
    cams = [mesh.pyrender_camera(p, K) for p in poses]
    V, F = mesh._to_device_mesh((v, f), "cuda")
    run = lambda: mesh._depth_maps(V, F, cams, 1200, 1600, 0.01, 5000.0)
    ms = events_ms(run, 3)
    d = run().cpu().numpy()
    return {"triangles": int(len(f)), "views": 49, "size": "1600x1200", "all_views_ms": ms, "per_view_ms": ms / 49,
            "covered_fraction": float((d > 0).mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--render-only", action="store_true", help="only the DTU-sized draws (A/B of library builds)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_mesh needs a GPU")
    res = {"card": card(), "library": mesh._lib.LIB_PATH}
    if args.render_only:
        res["dtu_render"] = dtu_render()
        print(json.dumps(res))
        return
    with tempfile.TemporaryDirectory() as tmp:
        res["app_post"] = [app_post(50, 224, 224, tmp), app_post(10, 384, 512, tmp)]
    res["dtu_render"] = dtu_render()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
