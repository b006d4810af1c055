#!/usr/bin/env python
"""Forward, dgrad and wgrad of the DPT-head / patch-embedding convolutions: the native path of `_native_conv` against cuDNN
in strict fp32 and in TF32.

    python tools/bench_conv_bwd.py [--res 224x224] [--batch 4] [--iters 20] [--warmup 5] [--only NAME,...]

Per conv shape (one DPT head, `_recompute._dpt`, plus the patch embeddings) and pass, one JSON line: mean time over `--iters`
launches timed with CUDA events after `--warmup` untimed ones, and the achieved TFLOP/s of 2 * MACs (from the shapes,
below).  Native forward = the `s3r_gemm` launch(es) of the recompute, dgrad = the input-gradient GEMM (+ col2im / fold),
wgrad = `s3r_conv_wgrad`; each includes the NCHW <-> NHWC copies and plane splits the Function does.  cuDNN passes are
`F.conv2d`, `torch.nn.grad.conv2d_input` / `conv2d_weight` (ConvTranspose: the adjoint calls).  The first line names the
card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def convs(H, W):
    gh, gw = H // 16, W // 16
    h3, w3 = (gh + 1) // 2, (gw + 1) // 2
    return [("act_postprocess.0.0", "1x1", 1024, 96, gh, gw), ("act_postprocess.1.0", "1x1", 768, 192, gh, gw),
            ("act_postprocess.2.0", "1x1", 768, 384, gh, gw), ("act_postprocess.3.0", "1x1", 768, 768, gh, gw),
            ("act_postprocess.0.1", "convT4", 96, 96, gh, gw), ("act_postprocess.1.1", "convT2", 192, 192, gh, gw),
            ("act_postprocess.3.1", "3x3s2", 768, 768, gh, gw),
            ("layer_rn.0", "3x3nb", 96, 256, 4 * gh, 4 * gw), ("layer_rn.1", "3x3nb", 192, 256, 2 * gh, 2 * gw),
            ("layer_rn.2", "3x3nb", 384, 256, gh, gw), ("layer_rn.3", "3x3nb", 768, 256, h3, w3),
            ("refinenet4.rcu", "3x3", 256, 256, h3, w3), ("refinenet3.rcu", "3x3", 256, 256, gh, gw),
            ("refinenet2.rcu", "3x3", 256, 256, 2 * gh, 2 * gw), ("refinenet1.rcu", "3x3", 256, 256, 4 * gh, 4 * gw),
            ("refinenet4.out_conv", "1x1", 256, 256, gh, gw), ("refinenet3.out_conv", "1x1", 256, 256, 2 * gh, 2 * gw),
            ("refinenet2.out_conv", "1x1", 256, 256, 4 * gh, 4 * gw), ("refinenet1.out_conv", "1x1", 256, 256, 8 * gh, 8 * gw),
            ("head.0", "3x3", 256, 128, H // 2, W // 2), ("head.2", "3x3", 128, 128, H, W),
            ("pos_patch_embed", "patch", 3, 1024, H, W)]


def macs(kind, cin, cout, h, w, nb):
    """Multiply-adds of one pass (forward, dgrad and wgrad all have the same count); (h, w) = the input map."""
    if kind.startswith("convT"):
        return nb * h * w * cin * cout * int(kind[-1]) ** 2
    if kind == "3x3s2":
        return nb * ((h + 1) // 2) * ((w + 1) // 2) * cout * cin * 9
    if kind == "patch":
        return nb * (h // 16) * (w // 16) * cout * cin * 256
    return nb * h * w * cout * cin * (9 if kind.startswith("3x3") else 1)


def make(kind, cin, cout, h, w, nb, g):
    if kind.startswith("convT"):
        s = int(kind[-1])
        wt = torch.randn(cin, cout, s, s, generator=g) * cin ** -0.5
    else:
        k = {"1x1": 1, "patch": 16}.get(kind, 3)
        wt = torch.randn(cout, cin, k, k, generator=g) * (cin * k * k) ** -0.5
    x = torch.randn(nb, cin, h, w, generator=g)
    b = None if kind == "3x3nb" else torch.randn(cout, generator=g)
    return x.cuda(), wt.cuda(), (b.cuda() if b is not None else None)


def torch_fwd(kind, x, w, b):
    if kind == "1x1":
        return F.conv2d(x, w, b)
    if kind in ("3x3", "3x3nb"):
        return F.conv2d(x, w, b, padding=1)
    if kind == "3x3s2":
        return F.conv2d(x, w, b, stride=2, padding=1)
    if kind == "patch":
        return F.conv2d(x, w, b, stride=16)
    return F.conv_transpose2d(x, w, b, stride=int(kind[-1]))


def torch_passes(kind, x, w, b, gy):
    st, pad = {"3x3s2": (2, 1), "patch": (16, 0), "3x3": (1, 1), "3x3nb": (1, 1)}.get(kind, (1, 0))
    if kind.startswith("convT"):
        s = int(kind[-1])
        # ConvTranspose2d(x; W) is the input gradient of Conv2d(W, stride s): its dgrad / wgrad are that conv's forward / wgrad
        return {"forward": lambda: F.conv_transpose2d(x, w, b, stride=s),
                "dgrad": lambda: F.conv2d(gy, w, None, stride=s),
                "wgrad": lambda: torch.nn.grad.conv2d_weight(gy, w.shape, x, stride=s)}
    return {"forward": lambda: torch_fwd(kind, x, w, b),
            "dgrad": lambda: torch.nn.grad.conv2d_input(x.shape, w, gy, stride=st, padding=pad),
            "wgrad": lambda: torch.nn.grad.conv2d_weight(x, w.shape, gy, stride=st, padding=pad)}


def native_passes(kind, x, w, b, gy):
    from spann3r_b200 import _native_conv as NC
    cls = {"1x1": NC._Conv1x1, "3x3": NC._Conv3x3, "3x3nb": NC._Conv3x3, "3x3s2": NC._Conv3x3s2, "patch": NC._PatchConv}
    def call(xi, wi):
        return NC._ConvT.apply(xi, wi, b, int(kind[-1])) if kind.startswith("convT") else cls[kind].apply(xi, wi, b)

    def fwd():
        with torch.no_grad():
            return call(x, w)

    def bwd(want):
        # a graph in which only the wanted input requires a gradient: its backward runs that pass alone (the bias is a
        # constant here)
        xi, wi = x.detach().requires_grad_(want == 0), w.detach().requires_grad_(want == 1)
        with torch.enable_grad():
            y = call(xi, wi)
        return lambda: torch.autograd.grad(y, xi if want == 0 else wi, gy, retain_graph=True)
    return {"forward": fwd, "dgrad": bwd(0), "wgrad": bwd(1)}


def time_it(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="224x224", help="H x W of the frame")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="", help="comma-separated conv names")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv_bwd: no CUDA device (timings need the GPU)")
    H, W = (int(v) for v in a.res.lower().split("x"))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(), "nvidia_smi": q, "res": [H, W], "batch": a.batch,
                      "iters": a.iters, "warmup": a.warmup}), flush=True)
    g = torch.Generator().manual_seed(0)
    only = set(filter(None, a.only.split(",")))
    for name, kind, cin, cout, h, w in convs(H, W):
        if only and name not in only:
            continue
        x, wt, b = make(kind, cin, cout, h, w, a.batch, g)
        with torch.no_grad():
            y = torch_fwd(kind, x, wt, b)
        gy = torch.randn(y.shape, generator=g).cuda()
        flop = 2.0 * macs(kind, cin, cout, h, w, a.batch)
        row = {"conv": name, "kind": kind, "cin": cin, "cout": cout, "map": [h, w], "batch": a.batch, "gflop_per_pass": flop / 1e9}
        for impl in ("native", "cudnn_fp32", "cudnn_tf32"):
            torch.backends.cudnn.allow_tf32 = impl == "cudnn_tf32"
            passes = native_passes(kind, x, wt, b, gy) if impl == "native" else torch_passes(kind, x, wt, b, gy)
            for pname, fn in passes.items():
                ms = time_it(fn, a.iters, a.warmup)
                row[f"{impl}_{pname}_ms"] = round(ms, 4)
                row[f"{impl}_{pname}_tflops"] = round(flop / ms / 1e9, 1)
        torch.backends.cudnn.allow_tf32 = False
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
