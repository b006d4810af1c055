#!/usr/bin/env python
"""Time the wgmma GEMM engine over the path's shapes and tile widths (CUDA events, back-to-back launches)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import _lib as L  # noqa: E402

SHAPES = [  # (name, groups, rows, K, N)
    ("dec.qkv", 2, 768, 768, 2304), ("dec.proj", 2, 768, 768, 768), ("dec.kv", 2, 768, 768, 1536),
    ("dec.fc1", 2, 768, 768, 3072), ("dec.fc2", 2, 768, 3072, 768), ("key.fc1", 2, 768, 1792, 1792),
    ("val.qkv", 1, 768, 1024, 3072), ("val.proj", 1, 768, 1024, 1024), ("val.fc1", 1, 768, 1024, 4096),
    ("val.fc2", 1, 768, 4096, 1024),
    ("enc.qkv", 1, 7680, 1024, 3072), ("enc.proj", 1, 7680, 1024, 1024), ("enc.fc1", 1, 7680, 1024, 4096),
    ("enc.fc2", 1, 7680, 4096, 1024),
]


def main():
    iters = 30
    for name, G, rows, K, N in SHAPES:
        x = torch.randn(G * rows, K, device="cuda")
        w = torch.randn(G * N, K, device="cuda") * K ** -0.5
        b = torch.randn(G * N, device="cuda")
        r = torch.randn(G * rows, N, device="cuda")
        xp, wp = L.split(x), L.split(w)
        res = []
        for bn in (64, 128, 256, 2128, 2256):
            if (bn % 1000) // 2 >= N:
                continue
            for _ in range(3):
                L.linear(xp, wp, bias=b, res=r, groups=G, force_bn=bn)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            out = torch.empty(G * rows, N, device="cuda")
            d = L.GemmDesc()
            d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
            d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, 1, rows, K, 1, N
            d.force_bn = bn
            d.bias = b.data_ptr()
            d.res1, d.ldr1 = r.data_ptr(), N
            d.out_f32, d.ldo = out.data_ptr(), N
            e0.record()
            for _ in range(iters):
                L.gemm(d)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / iters * 1e3
            tf = 2.0 * G * rows * N * K / us / 1e6
            res.append(f"bn{bn}: {us:7.1f}us {tf:6.1f}TF")
        print(f"{name:9s} G{G} M{rows} K{K} N{N}  " + " | ".join(res), flush=True)


if __name__ == "__main__":
    main()
