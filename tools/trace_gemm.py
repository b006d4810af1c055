#!/usr/bin/env python
"""Where do the ~7 us of fixed cost of a small GEMM launch go?  CTA 0 of each launch stamps %globaltimer at: entry,
prologue done, dependency (PDL) wait done, first operands landed, accumulator ready, epilogue done, exit.  A chain of
dependent launches (each reads the previous one's planes) in steady state."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from spann3r_b200 import _lib as L  # noqa: E402

G, rows, N = 2, 768, 768
for K in (64, 768):
    n_launch = 24
    w = torch.randn(G * N, K, device="cuda") * K ** -0.5
    wp = L.split(w)
    bufs = [L.split(torch.randn(G * rows, max(K, N), device="cuda")[:, :K].contiguous()) for _ in range(2)]
    outs = [(torch.empty(G * rows, N, dtype=torch.bfloat16, device="cuda"), torch.empty(G * rows, N, dtype=torch.bfloat16, device="cuda"))
            for _ in range(2)]
    trace = torch.zeros(n_launch, 16, dtype=torch.int64, device="cuda")
    b = torch.randn(G * N, device="cuda")
    descs = []
    for i in range(n_launch):
        d = L.GemmDesc()
        # launch i reads the planes launch i-1 wrote when K == N (true dependency chain); otherwise fixed inputs
        src = outs[(i + 1) % 2] if K == N else bufs[i % 2]
        d.a_hi, d.a_lo, d.b_hi, d.b_lo = src[0].data_ptr(), src[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
        d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, 1, rows, K, 1, N
        d.force_bn = 64
        d.bias = b.data_ptr()
        d.out_hi, d.out_lo, d.ldp = outs[i % 2][0].data_ptr(), outs[i % 2][1].data_ptr(), N
        d.trace = trace[i].data_ptr()
        descs.append(d)
    for rep in range(3):
        for d in descs:
            L.gemm(d)
    torch.cuda.synchronize()
    t = trace.cpu().double()
    names = ["entry", "prologue", "pdl_wait", "operands", "accum", "epilogue", "exit"]   # the stamps gemm.cu writes
    print(f"K={K}: per-launch timeline of CTA 0, ns relative to the previous launch's exit stamp (launches 8..15)")
    for i in range(8, 16):
        base = t[i - 1, 6]
        print("   " + "  ".join(f"{n}={t[i, j] - base:7.0f}" for j, n in enumerate(names)))
    per = (t[8:20, 6] - t[7:19, 6]).mean()
    print(f"   mean exit-to-exit period {per:.0f} ns")
