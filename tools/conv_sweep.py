#!/usr/bin/env python
"""Time the DPT-head conv / GEMM shapes at B=1 (2 heads as groups) through the op-level ABI.  With S3R_LIB pointing at
an older build this is a same-box A/B of the GEMM engine (the descriptor's leading fields are layout-compatible)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import _lib as L  # noqa: E402

if os.environ.get("S3R_LIB"):
    L._PROTOS.pop("s3r_abi_sizeof", None)

SHAPES = [  # (name, H, W, Cin, Cout, taps, mode)   mode: "relu" = act ReLU -> planes; "res" = +res1 -> fp32 + relu planes
    ("act1_conv", 24, 32, 1024, 96, 1, "planes"), ("layer_rn1", 96, 128, 96, 256, 9, "res"),
    ("rn4.rcu", 12, 16, 256, 256, 9, "relu"), ("rn3.rcu", 24, 32, 256, 256, 9, "relu"), ("rn2.rcu", 48, 64, 256, 256, 9, "relu"),
    ("rn1.rcu.c1", 96, 128, 256, 256, 9, "relu"), ("rn1.rcu.c2", 96, 128, 256, 256, 9, "res"),
    ("rn1.out_conv", 96, 128, 256, 256, 1, "f32"), ("head0", 192, 256, 256, 128, 9, "f32"), ("head2-like", 384, 512, 128, 128, 9, "relu"),
    ("enc.fc1-like", 1, 7680, 1024, 4096, 1, "relu"), ("enc.proj-like", 1, 7680, 1024, 1024, 1, "res"),
    ("dec.proj", 1, 768, 768, 768, 1, "res"), ("dec.fc1", 1, 768, 768, 3072, 1, "relu"),
]
G = 2
for name, H, W, Cin, Cout, taps, mode in SHAPES:
    x = torch.randn(G, H, W, Cin, device="cuda")
    w = torch.randn(G * Cout, taps * Cin, device="cuda") * (taps * Cin) ** -0.5
    b = torch.randn(G * Cout, device="cuda")
    res = torch.randn(G, H, W, Cout, device="cuda")
    xp, wp = L.split(x), L.split(w)
    out = torch.empty(G, H, W, Cout, device="cuda")
    oh = torch.empty(out.shape, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, H, W, Cin, taps, Cout
    d.epi = L.EPI_PLAIN
    d.bias = b.data_ptr()
    if mode == "relu":
        d.act = L.ACT_RELU
        d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), Cout
    elif mode == "planes":
        d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), Cout
    elif mode == "res":
        d.res1, d.ldr1 = res.data_ptr(), Cout
        d.out_f32, d.ldo = out.data_ptr(), Cout
        d.out_hi, d.out_lo, d.ldp, d.plane_relu = oh.data_ptr(), ol.data_ptr(), Cout, 1
    else:
        d.out_f32, d.ldo = out.data_ptr(), Cout
    res_txt = []
    sweep = [0] + ([b for b in (64, 96, 128) if b <= Cout] if "--sweep" in sys.argv else [])
    for fb in sweep:
        d.force_bn = fb
        try:
            for _ in range(3):
                L.gemm(d)
        except Exception:
            continue
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 20
        e0.record()
        for _ in range(iters):
            L.gemm(d)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / iters * 1e3
        bn = L.lib().s3r_gemm_tile_n(d)
        res_txt.append(f"{'auto' if fb == 0 else fb}(bn{bn}) {us:7.1f}us")
    tf = 2.0 * G * H * W * Cout * Cin * taps / 1e6
    print(f"{name:14s} {H:3d}x{W:<4d} {Cin:4d}->{Cout:<4d} taps{taps} {mode:6s} " + " | ".join(res_txt) + f"   [{tf:.0f} MFLOP]", flush=True)
