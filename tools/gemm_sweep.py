#!/usr/bin/env python
"""Time the wgmma GEMM engine over the path's shapes and tile widths (CUDA events, back-to-back launches).

Every shape runs at each forced tile width (64 / 96 / 128) and at the planner's choice ("plan"), split and, with --bf16,
one-product.  The bias + residual shapes are followed by the decoder's N = 768 launches with their real epilogues: `q`
(folded LayerNorm + EPI_QKV with RoPE), and proj / fc2 (in-place residual + stats_out of the next folded LayerNorm)."""
import argparse
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import _lib as L  # noqa: E402

SHAPES = [  # (name, groups, rows, K, N)
    ("dec.qkv", 2, 768, 768, 2304), ("dec.proj", 2, 768, 768, 768), ("dec.kv", 2, 768, 768, 1536),
    ("dec.fc1", 2, 768, 768, 3072), ("dec.fc2", 2, 768, 3072, 768), ("key.fc1", 2, 768, 1792, 1792),
    ("key.fc2", 2, 768, 1792, 1024),
    ("val.qkv", 1, 768, 1024, 3072), ("val.proj", 1, 768, 1024, 1024), ("val.fc1", 1, 768, 1024, 4096),
    ("val.fc2", 1, 768, 4096, 1024),
    ("enc.qkv", 1, 7680, 1024, 3072), ("enc.proj", 1, 7680, 1024, 1024), ("enc.fc1", 1, 7680, 1024, 4096),
    ("enc.fc2", 1, 7680, 4096, 1024),
]
# the decoder's N = 768 launches as the engine issues them: (name, K, epilogue)
DEC_EPI = [("dec.q+ln+qkv", 768, "qkv"), ("dec.proj+res+stats", 768, "stats"), ("dec.fc2+res+stats", 3072, "stats")]
WIDTHS = (64, 96, 128, 0)


def _time(d, iters):
    for _ in range(3):
        L.gemm(d)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        L.gemm(d)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def _desc(xp, wp, G, rows, K, N, precision):
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, 1, rows, K, 1, N
    d.precision = precision
    return d


def _row(name, G, rows, K, N, make, iters, precision):
    res = []
    for bn in WIDTHS:
        d, keep = make()
        d.force_bn = bn
        chosen = L.lib().s3r_gemm_tile_n(d)
        us = _time(d, iters)
        del keep
        tf = 2.0 * G * rows * N * K / us / 1e6
        res.append(f"{'plan' if bn == 0 else 'bn%d' % bn}{'(%d)' % chosen if bn == 0 else ''}: {us:7.1f}us {tf:6.1f}TF")
    print(f"{name:20s} {'bf16' if precision else 'split'} G{G} M{rows} K{K} N{N}  " + " | ".join(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--bf16", action="store_true", help="also time the one-product precision")
    ap.add_argument("--only", default="", help="comma-separated name prefixes")
    args = ap.parse_args()
    L.require_device()
    try:
        info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        info = torch.cuda.get_device_name()
    print(f"# {info}", flush=True)
    only = [p for p in args.only.split(",") if p]
    want = lambda name: not only or any(name.startswith(p) for p in only)  # noqa: E731
    g = torch.Generator(device="cpu").manual_seed(0)
    for precision in ((0, 1) if args.bf16 else (0,)):
        for name, G, rows, K, N in SHAPES:
            if not want(name):
                continue
            x = torch.randn(G * rows, K, generator=g).cuda()
            w = (torch.randn(G * N, K, generator=g) * K ** -0.5).cuda()
            b = torch.randn(G * N, generator=g).cuda()
            r = torch.randn(G * rows, N, generator=g).cuda()
            out = torch.empty(G * rows, N, device="cuda")
            xp, wp = L.split(x), L.split(w)

            def make():
                d = _desc(xp, wp, G, rows, K, N, precision)
                d.bias = b.data_ptr()
                d.res1, d.ldr1 = r.data_ptr(), N
                d.out_f32, d.ldo = out.data_ptr(), N
                return d, None
            _row(name, G, rows, K, N, make, args.iters, precision)

        G, rows, N = 2, 768, 768
        for name, K, kind in DEC_EPI:
            if not want(name):
                continue
            x = torch.randn(G * rows, K, generator=g).cuda()
            w = (torch.randn(G * N, K, generator=g) * K ** -0.5).cuda()
            b = torch.randn(G * N, generator=g).cuda()
            xp, wp = L.split(x), L.split(w)
            if kind == "qkv":
                ntok, heads = rows, N // 64
                st = torch.stack((x.view(G * rows, K // 32, 32).sum(-1), x.view(G * rows, K // 32, 32).pow(2).sum(-1)), -1)
                cs = w.view(G, N, K).sum(-1).reshape(-1).contiguous()
                pos = torch.randint(0, 32, (G * rows, 2), generator=g).to(torch.int32).cuda()
                ang = torch.rand(32, 16, generator=g) * 2 * math.pi
                qcs = torch.stack((ang.cos(), ang.sin()), -1).contiguous().cuda()
                qo = torch.empty(G * heads * ntok * 64, device="cuda")

                def make():
                    d = _desc(xp, wp, G, rows, K, N, precision)
                    d.epi, d.bias = L.EPI_QKV, b.data_ptr()
                    d.q_c, d.q_role_base, d.q_ntok, d.q_ntok_pad, d.q_rope, d.q_nb = N, 0, ntok, ntok, 1, 1
                    d.q_pos, d.q_cs, d.q_scale, d.q_out = pos.data_ptr(), qcs.data_ptr(), 0.125, qo.data_ptr()
                    d.ln_stats, d.ln_np, d.ln_eps, d.ln_cs = st.data_ptr(), K // 32, 1e-6, cs.data_ptr()
                    return d, None
            else:
                out = torch.randn(G * rows, N, generator=g).cuda()
                oh = torch.empty(G * rows, N, dtype=torch.bfloat16, device="cuda")
                ol = torch.empty_like(oh)
                sto = torch.empty(G * rows, N // 32, 2, device="cuda")

                def make():
                    d = _desc(xp, wp, G, rows, K, N, precision)
                    d.bias = b.data_ptr()
                    d.res1, d.ldr1 = out.data_ptr(), N           # in place, as the engine's proj / fc2
                    d.out_f32, d.ldo = out.data_ptr(), N
                    d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), N
                    d.stats_out = sto.data_ptr()
                    return d, None
            _row(name, G, rows, K, N, make, args.iters, precision)


if __name__ == "__main__":
    main()
