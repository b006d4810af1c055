"""`nn.Linear` forward AND backward on the wgmma GEMM engine -- the first native piece of the training backward
(SURVEY.md §8f rank 1).

`_recompute.py` (the PyTorch recompute that `train.py` differentiates) routes every Linear through `linear()` below.  With the
switch off (default) that is `F.linear` and PyTorch autograd.  With it on, the three GEMMs of a Linear -- y = x W^T + b in the
recompute, dx = dy W (dgrad) and dW = dy^T x (wgrad) in the backward -- run as split-bf16 (`bf16x3`, ~fp32-accurate) launches of
`s3r_gemm` through the C ABI: the same `gemm_bf16x3_kernel` the forward path uses, operands re-laid-out by
plain data movement (transpose, zero-pad of the contraction to a multiple of 8, split into planes).  Linears carry ~85 % of the
backward's FLOPs; attention, LayerNorm, GELU, the DPT convolutions and the elementwise glue remain PyTorch autograd.

Enable with `spann3r_b200.train.set_native_linear(True)` or `S3R_TRAIN_NATIVE_LINEAR=1`.  CUDA tensors only; on the CPU (tests of
the recompute against the oracle) the call is `F.linear`.
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F

from . import _lib

ENABLED = os.environ.get("S3R_TRAIN_NATIVE_LINEAR", "0") == "1"


def _pad8(t: torch.Tensor) -> torch.Tensor:
    """Zero-pad the last (contraction) dimension to a multiple of 8 elements: the TMA row pitch must be 16 bytes."""
    k = t.shape[-1]
    return t if k % 8 == 0 else F.pad(t, (0, 8 - k % 8))


def gemm_nt(a: torch.Tensor, b: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """a [rows, K] @ b[N, K]^T (+ bias) -> fp32 [rows, N] on the split-bf16 wgmma engine (N % 32 == 0)."""
    assert a.dim() == 2 and b.dim() == 2 and a.shape[1] == b.shape[1] and b.shape[0] % 32 == 0, (tuple(a.shape), tuple(b.shape))
    a, b = _pad8(a.float()).contiguous(), _pad8(b.float()).contiguous()
    out, _, _ = _lib.linear(_lib.split(a), _lib.split(b), bias=None if bias is None else bias.float().contiguous())
    return out


class _NativeLinear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        x2 = x.reshape(-1, x.shape[-1])
        ctx.save_for_backward(x2, w)
        ctx.x_shape, ctx.has_bias = x.shape, b is not None
        return gemm_nt(x2, w, b).view(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        x2, w = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gx = gemm_nt(g2, w.t()).view(ctx.x_shape) if ctx.needs_input_grad[0] else None          # dgrad: dy [rows, N] @ W [N, K]
        gw = gemm_nt(g2.t(), x2.t()) if ctx.needs_input_grad[1] else None                        # wgrad: dy^T [N, rows] @ x [rows, K]
        gb = g2.sum(dim=0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb


def linear(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None) -> torch.Tensor:
    if ENABLED and x.is_cuda and w.shape[0] % 32 == 0 and w.shape[1] % 32 == 0:
        return _NativeLinear.apply(x, w, b)
    return F.linear(x, w, b)
