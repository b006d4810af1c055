#!/usr/bin/env python
"""Forward + backward of the training recompute's attentions: the native kernels of `_native_attn` against eager `_sdpa`
in strict fp32 and in TF32, and against `F.scaled_dot_product_attention` (whichever backend PyTorch picks, named).

    python tools/bench_attn_train.py [--iters 20] [--warmup 5] [--only NAME,...]

Shapes: every attention of a 224 x 224 training step at B = 4, F = 10 (the encoder stage recomputes all 40 images at once)
plus the 512 x 384 encoder.  Per shape one JSON line: mean ms of forward + backward (dQ, dK, dV) over `--iters` calls timed
with CUDA events after `--warmup` untimed ones, and the peak allocated memory of one call above its inputs.  Every path
returns [B, nq, heads * dh], as `_recompute._attn` does.  The first line names the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (name, images, heads, nq, nk, dh)
SHAPES = [
    ("encoder_224", 40, 16, 196, 196, 64),
    ("decoder_self_224", 4, 12, 196, 196, 64),
    ("decoder_cross_224", 4, 12, 196, 196, 64),
    ("value_encoder_224", 4, 16, 196, 196, 64),
    ("value_encoder_use_feat_224", 4, 16, 196, 196, 48),
    ("encoder_512x384", 40, 16, 768, 768, 64),
]


def time_it(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def sdpa_backend(q, k, v):
    try:
        from torch.nn.attention import SDPBackend
        return SDPBackend(torch._fused_sdp_choice(q, k, v)).name
    except Exception as e:   # the private chooser moved: say so rather than guess
        return "unknown (%s)" % type(e).__name__


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_attn_train: no CUDA device (timings need the GPU)")
    from spann3r_b200 import _native_attn as NA, _recompute as R
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(), "nvidia_smi": smi, "iters": a.iters, "warmup": a.warmup}),
          flush=True)
    only = set(filter(None, a.only.split(",")))
    g = torch.Generator().manual_seed(0)
    for name, B, H, nq, nk, dh in SHAPES:
        if only and name not in only:
            continue
        q = torch.randn(B, H, nq, dh, generator=g).cuda().requires_grad_(True)
        k = torch.randn(B, H, nk, dh, generator=g).cuda().requires_grad_(True)
        v = torch.randn(B, H, nk, dh, generator=g).cuda().requires_grad_(True)
        go = torch.randn(B, nq, H * dh, generator=g).cuda()
        scale = dh ** -0.5

        def eager():
            return R._sdpa(q, k, v).transpose(1, 2).reshape(B, nq, H * dh)

        def fused():
            return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, nq, H * dh)

        paths = {"native": (lambda: NA.attention(q, k, v, scale), False), "sdpa_eager_fp32": (eager, False),
                 "sdpa_eager_tf32": (eager, True), "F_sdpa": (fused, False)}
        row = {"shape": name, "images": B, "heads": H, "nq": nq, "nk": nk, "dh": dh,
               "F_sdpa_backend": sdpa_backend(q, k, v),
               "eager_probabilities_mb": B * H * nq * nk * 4 / 2 ** 20}
        for pname, (fwd, tf32) in paths.items():
            torch.backends.cuda.matmul.allow_tf32 = tf32

            def step():
                torch.autograd.grad(fwd(), (q, k, v), go)
            row[pname + "_ms"] = round(time_it(step, a.iters, a.warmup), 4)
            row[pname + "_peak_mb"] = round(peak_mb(step), 1)
        torch.backends.cuda.matmul.allow_tf32 = False
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
