#!/usr/bin/env python
"""fp32-grade vs bf16 precision on BASELINE config 2 (one 10-frame 384 x 512 sequence, sharpened checkpoint) and on the
GEMM shapes of tools/gemm_sweep.py, in one process on one GPU.

    python tools/bench_precision.py [--reps 5] [--out DIR]

1. Frames/s of Spann3R.forward at precision "fp32" and "bf16", timed alternately after warm-up (host clock around work
   that ends in a device synchronise), median and spread over --reps.
2. Per stage: the tensor-core launch time of one frame step (CUDA events per launch, s3r_engine_profile_list), and the
   TFLOP/s of the one-product (kind 2) launches.
3. The 14 gemm_sweep shapes with the planner's tile, split (3 products) against bf16 (1 product), CUDA events over 30
   back-to-back launches.
The card's name and power limit are printed beside the numbers; --out also writes them as JSON.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import Spann3R, synth  # noqa: E402
from spann3r_b200 import _lib as L  # noqa: E402
from tools.gemm_sweep import SHAPES  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers are still the numbers; say that the card could not be read
        q = f"unknown ({e})"
    return q


def fps(m, frames, precision):
    m.set_precision(precision)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        m(frames)
    torch.cuda.synchronize()
    return len(frames) / (time.perf_counter() - t0)


def stage_profile(m, frames, precision):
    """Tensor-core time [ms] per stage of the first frame step, and (ms, flops) of its kind-2 launches."""
    m.set_precision(precision)
    eng = m._engine_for(1, 384, 512, n_frames=len(frames))
    img = torch.cat([f["img"] for f in frames[:2]]).contiguous()
    out, k2 = {}, [0.0, 0.0]

    def prof(name, fn):
        eng.profile(True)
        r = fn()
        lst = eng.profile_list()
        eng.profile_read()
        eng.profile(False)
        out[name] = sum(ms for ms, _, _ in lst)
        for ms, fl, kd in lst:
            if kd == 2:
                k2[0] += ms
                k2[1] += fl
        return r

    with torch.no_grad():
        feats = prof("encode (2 images)", lambda: eng.encode(img))
        f1, f2 = feats[:1].contiguous(), feats[1:].contiguous()
        prof("decode", lambda: eng.decode(f1, f2))
        k1, _ = prof("keyheads", lambda: eng.keyheads(f1, f2))
        pts, _ = prof("heads", lambda: eng.heads())
        prof("value", lambda: eng.value(pts[0].contiguous(), k1))
    return out, (k2[1] / (k2[0] * 1e9) if k2[0] else 0.0)


def sweep(iters=30):
    rows = []
    for name, G, M, K, N in SHAPES:
        x = torch.randn(G * M, K, device="cuda")
        w = torch.randn(G * N, K, device="cuda") * K ** -0.5
        b = torch.randn(G * N, device="cuda")
        xp, wp = L.split(x), L.split(w)
        out = torch.empty(G * M, N, device="cuda")
        t = {}
        for prec in (L.PRECISION_SPLIT, L.PRECISION_BF16):
            d = L.GemmDesc()
            d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
            d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, 1, M, K, 1, N
            d.bias = b.data_ptr()
            d.out_f32, d.ldo = out.data_ptr(), N
            d.precision = prec
            for _ in range(3):
                L.gemm(d)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                L.gemm(d)
            e1.record()
            torch.cuda.synchronize()
            t[prec] = e0.elapsed_time(e1) / iters * 1e3
        fl = 2.0 * G * M * N * K
        rows.append(dict(shape=name, G=G, M=M, K=K, N=N, split_us=t[0], bf16_us=t[1], split_tflops=fl / t[0] / 1e6,
                         bf16_tflops=fl / t[1] / 1e6, speedup=t[0] / t[1]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    L.require_device()
    gpu = card()
    print("card (name, power limit, max SM clock):", gpu, flush=True)
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(synth.make_state_dict(seed=0, sharpen=True), strict=True)   # the golden vectors' checkpoint
    m = m.cuda().eval()
    frames = [{"img": f["img"].cuda()} for f in synth.make_frames(10, 384, 512)]
    for p in ("fp32", "bf16", "fp32", "bf16"):     # warm-up: engines, plans, modules
        fps(m, frames, p)
    res = {"fp32": [], "bf16": []}
    for _ in range(a.reps):
        for p in ("fp32", "bf16"):
            res[p].append(fps(m, frames, p))
    summary = {p: dict(median=statistics.median(v), min=min(v), max=max(v)) for p, v in res.items()}
    for p, s in summary.items():
        print(f"config 2 {p}: {s['median']:.1f} frames/s (min {s['min']:.1f}, max {s['max']:.1f}, {a.reps} alternated runs)")
    print(f"config 2 speed-up bf16 / fp32: {summary['bf16']['median'] / summary['fp32']['median']:.2f}x", flush=True)
    stages = {}
    for p in ("fp32", "bf16"):
        st, k2 = stage_profile(m, frames, p)
        stages[p] = dict(stages_ms=st, kind2_tflops=k2)
        print(f"{p} tensor-core ms per stage (one frame step): " + ", ".join(f"{k} {v:.2f}" for k, v in st.items()) +
              (f"; kind-2 launches {k2:.0f} TFLOP/s" if k2 else ""), flush=True)
    rows = sweep()
    for r in rows:
        print(f"{r['shape']:9s} G{r['G']} M{r['M']} K{r['K']} N{r['N']}: split {r['split_us']:7.1f} us "
              f"({r['split_tflops']:5.0f} TF)  bf16 {r['bf16_us']:7.1f} us ({r['bf16_tflops']:5.0f} TF)  x{r['speedup']:.2f}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_precision.json"), "w") as f:
            json.dump(dict(card=gpu, fps=res, summary=summary, stages=stages, sweep=rows), f, indent=1)


if __name__ == "__main__":
    main()
