#!/usr/bin/env python
"""How close the GEMM engine's main loop comes to the tensor cores' rate, on the flagship workload's shapes.

    python tools/ring_ab.py [--label NAME]                                   # the in-tree library
    S3R_LIB=ab/libspann3r_b200_parent.so python tools/ring_ab.py --label parent

1. The CTA-0 timeline of tools/trace_gemm.py on enc.fc2 (7680 x 4096 -> 1024, BN = 128, 4096 channels of K): from
   CTA 0's first operands landing to its first accumulator being ready, per 64 channels of K.  64 channels of a
   128 x 128 tile are 2 warpgroups x 4 k16 steps x 3 m64n128k16 MMAs = 6.3 MFLOP, 1536 clocks at 4096 dense bf16 FLOP
   per clock per SM; the ideal is printed at the SM clock nvidia-smi reports during the measurement.  Time above it is
   the tensor cores waiting, mostly for operands.
2. Every shape of tools/gemm_sweep.py at the planner's tile width with its bias + residual epilogue: CUDA-event time
   of 30 back-to-back launches after 3 warm-ups, TFLOP/s of algorithmic 2MNK work.

Prints the card, its power limit and SM clock beside the numbers, then one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gemm_sweep import SHAPES  # noqa: E402
from spann3r_b200 import _lib as L  # noqa: E402

CLOCKS_PER_64CH = 1536


def _smi(fields):
    r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={fields}",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    return [f.strip() for f in r.stdout.strip().splitlines()[0].split(",")]


def _desc(xp, wp, b, r, out, G, rows, K, N, trace=None):
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, 1, rows, K, 1, N
    d.bias = b.data_ptr()
    d.res1, d.ldr1 = r.data_ptr(), N
    d.out_f32, d.ldo = out.data_ptr(), N
    if trace is not None:
        d.trace = trace.data_ptr()
    return d


def _operands(G, rows, K, N):
    x = torch.randn(G * rows, K, device="cuda")
    w = torch.randn(G * N, K, device="cuda") * K ** -0.5
    return (L.split(x), L.split(w), torch.randn(G * N, device="cuda"), torch.randn(G * rows, N, device="cuda"),
            torch.empty(G * rows, N, device="cuda"))


def fc2_timeline(n_launch=1500):
    """Median main-loop ns per 64 channels of CTA 0's first tile over n_launch launches, and the SM clock (MHz, median
    of nvidia-smi samples taken while the launches run)."""
    G, rows, K, N = 1, 7680, 4096, 1024
    xp, wp, b, r, out = _operands(G, rows, K, N)
    trace = torch.zeros(n_launch, 16, dtype=torch.int64, device="cuda")
    descs = [_desc(xp, wp, b, r, out, G, rows, K, N, trace[i]) for i in range(n_launch)]
    for d in descs[:3]:
        L.gemm(d)
    torch.cuda.synchronize()
    smi = subprocess.Popen(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=clocks.sm",
                            "--format=csv,noheader,nounits", "-lms", "50"], stdout=subprocess.PIPE, text=True)
    try:
        for d in descs:
            L.gemm(d)
        torch.cuda.synchronize()
    finally:
        smi.terminate()
        rows_out, _ = smi.communicate(timeout=30)
    clocks = [float(v) for v in rows_out.split() if v.replace(".", "").isdigit()]
    t = trace.cpu().double()
    per64 = [(t[i, 4] - t[i, 3]).item() / (K / 64) for i in range(3, n_launch)]
    return statistics.median(per64), (statistics.median(clocks) if clocks else float("nan")), len(clocks)


def sweep(iters=30):
    res = {}
    for name, G, rows, K, N in SHAPES:
        xp, wp, b, r, out = _operands(G, rows, K, N)
        d = _desc(xp, wp, b, r, out, G, rows, K, N)
        for _ in range(3):
            L.gemm(d)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            L.gemm(d)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / iters * 1e3
        res[name] = (us, 2.0 * G * rows * N * K / us / 1e6)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--label", default="tree")
    args = ap.parse_args()
    L.require_device()
    torch.manual_seed(0)
    name, plimit, max_sm = _smi("name,power.limit,clocks.max.sm")
    ns64, sm_mhz, n_samples = fc2_timeline()
    ideal_ns = CLOCKS_PER_64CH / sm_mhz * 1e3
    shapes = sweep()
    print(f"[{args.label}] {L.LIB_PATH}")
    print(f"[{args.label}] {name}, power limit {plimit} W, max SM clock {max_sm} MHz, SM clock during the enc.fc2 launches "
          f"{sm_mhz:.0f} MHz (median of {n_samples} samples)")
    print(f"[{args.label}] enc.fc2 CTA-0 main loop: {ns64 / 1e3:.3f} us per 64 channels of K, ideal {ideal_ns / 1e3:.3f} us "
          f"({CLOCKS_PER_64CH} clocks) -> {ideal_ns / ns64:.2f} of the tensor-core rate")
    for k, (us, tf) in shapes.items():
        print(f"[{args.label}]   {k:9s} {us:8.1f} us {tf:6.1f} TFLOP/s")
    total = sum(us for us, _ in shapes.values())
    print(f"[{args.label}]   sum of the shapes {total:.1f} us")
    print(json.dumps({"label": args.label, "gpu": name, "power_limit_w": plimit, "sm_clock_mhz": sm_mhz,
                      "fc2_us_per_64ch": ns64 / 1e3, "ideal_us_per_64ch": ideal_ns / 1e3, "sum_us": total,
                      "shapes": {k: {"us": us, "tflops": tf} for k, (us, tf) in shapes.items()}}), flush=True)


if __name__ == "__main__":
    main()
