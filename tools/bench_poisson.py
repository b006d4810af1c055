"""Screened Poisson reconstruction (spann3r_b200.mesh.create_from_point_cloud_poisson + get_mesh_from_ply's trim) on
synthetic scan-like clouds: a bumpy closed surface of 1M and 4M samples at depth 8 and 9.

Per case, CUDA-event times of each stage of the C ABI (one warm-up run first, then the median of --reps runs):
  setup    bounding box, sort by cell, splat of v, screening blocks, right-hand side b, density grid
  solve    multigrid-preconditioned conjugate gradients to a relative residual of 1e-8 (iterations reported), iso value
  extract  marching tetrahedra: counts, scans, one size read, vertex / face / per-vertex density writes
  trim     np.quantile(densities, 0.1) by exact selection, then remove_vertices_by_mask
plus the peak allocated memory, the card and its power limit.  Prints one JSON line per case.

    python tools/bench_poisson.py [--reps 3] [--out bench_poisson.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import mesh  # noqa: E402


def scan_like(n, seed=0):
    """A closed, bumpy surface r(d) = 1 + 0.15 sin(5 x) sin(4 y) sin(3 z) on unit directions d, with exact normals, in
    millimetre-like units (DTU's clouds are a few hundred mm across)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x, y, z = d.T
    f = 0.15 * np.sin(5 * x) * np.sin(4 * y) * np.sin(3 * z)
    g = 0.15 * np.stack([5 * np.cos(5 * x) * np.sin(4 * y) * np.sin(3 * z), 4 * np.sin(5 * x) * np.cos(4 * y) * np.sin(3 * z),
                         3 * np.sin(5 * x) * np.sin(4 * y) * np.cos(3 * z)], 1)
    r = 1.0 + f
    # normal of the level set |p| - r(p / |p|) = 0: d - grad_tangential(r) / r
    gt = g - (g * d).sum(1, keepdims=True) * d
    nrm = d - gt / r[:, None]
    return (200.0 * r[:, None] * d).astype(np.float32), (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:   # nvidia-smi missing: the name from torch, the power limit unknown
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def run_once(P, N, depth):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    info = _stages(P, N, depth, ev)
    torch.cuda.synchronize()
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(("setup", "solve", "extract", "trim"))}, info


def _stages(P, N, depth, ev):
    import ctypes as C
    from spann3r_b200 import _lib
    L = _lib.lib()
    n = len(P)
    ws_bytes = int(L.s3r_poisson_workspace_bytes(n, depth))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    info, out, sizes = np.zeros(8), np.zeros(3), np.zeros(2, np.int64)
    stream = _lib.stream_ptr()
    ev[0].record()
    _lib.check(L.s3r_poisson_setup(_lib.ptr(P), _lib.ptr(N), 0, n, depth, 1.1, _lib.ptr(ws), ws_bytes,
                                   C.c_void_p(info.ctypes.data), stream), "setup")
    ev[1].record()
    _lib.check(L.s3r_poisson_solve(n, depth, mesh.POISSON_TOL, mesh.POISSON_MAX_ITER, _lib.ptr(ws), ws_bytes,
                                   C.c_void_p(out.ctypes.data), stream), "solve")
    ev[2].record()
    _lib.check(L.s3r_poisson_extract_count(n, depth, _lib.ptr(ws), ws_bytes, C.c_void_p(sizes.ctypes.data), stream),
               "extract_count")
    v = torch.empty((int(sizes[0]), 3), dtype=torch.float32, device="cuda")
    f = torch.empty((int(sizes[1]), 3), dtype=torch.int64, device="cuda")
    d = torch.empty(int(sizes[0]), dtype=torch.float64, device="cuda")
    _lib.check(L.s3r_poisson_extract(n, depth, _lib.ptr(ws), ws_bytes, _lib.ptr(v), _lib.ptr(f), _lib.ptr(d), stream),
               "extract")
    ev[3].record()
    vt, ft = mesh.remove_vertices_by_mask(v, f, d < mesh.quantile(d, 0.1))
    ev[4].record()
    return dict(iterations=int(out[0]), residual=float(out[1]), vertices=len(v), faces=len(f), kept_vertices=len(vt),
                kept_faces=len(ft), workspace_gb=ws_bytes / 1e9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sizes", default="1000000,4000000")
    ap.add_argument("--depths", default="8,9")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    rows = []
    for n in [int(s) for s in a.sizes.split(",")]:
        p, nrm = scan_like(n)
        P, N = torch.from_numpy(p).cuda(), torch.from_numpy(nrm).cuda()
        for depth in [int(s) for s in a.depths.split(",")]:
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            run_once(P, N, depth)                              # warm-up: module loads, allocator
            times = []
            for _ in range(a.reps):
                t, info = run_once(P, N, depth)
                times.append(t)
            med = {k: float(np.median([t[k] for t in times])) for k in times[0]}
            row = dict(samples=n, depth=depth, ms=med, total_ms=sum(med.values()), **info,
                       peak_allocated_gb=torch.cuda.max_memory_allocated() / 1e9, card=name, power_limit=power)
            print(json.dumps(row), flush=True)
            rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
