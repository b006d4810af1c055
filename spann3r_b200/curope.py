"""Drop-in for the reference's ONLY native boundary: the pybind module `curope` and its `cuRoPE2D` wrapper
(croco/models/curope/curope.cpp:49-69, kernels.cu:83-108, curope2d.py:12-40) -- SURVEY.md §8b.

    from spann3r_b200 import curope            # instead of `import curope` / `from . import curope`
    curope.rope_2d(tokens, positions, base, fwd)        # in place; tokens [B, N, H, D], positions [B, N, 2] int64
    rope = curope.cuRoPE2D(freq=100.0)                  # rope(tokens [B, H, N, D], positions) -> tokens (rotated in place)

Same argument meaning, in-place semantics, checks and messages as the pybind function (raised as RuntimeError, which is
what a failed TORCH_CHECK surfaces as in Python), same autograd rule (`backward` = the rotation with `-F0`,
curope2d.py:24-29).  Differences, both deliberate: fp32 only (the reference also dispatches fp16 / fp64), and the kernel
runs on PyTorch's CURRENT stream instead of the legacy default stream the reference launches on (kernels.cu:102).  On the
fused fast path RoPE never runs as a separate op (it lives in the QKV-projection epilogue, csrc/gemm_epilogue.cuh); this
module exists so that reference code which calls curope directly keeps working.  No CPU path: CPU tensors raise.
"""
from __future__ import annotations

import torch

from . import _lib


def _launch(tokens: torch.Tensor, positions: torch.Tensor, base: float, fwd: float) -> None:
    B, N, H, D = tokens.shape
    st = tokens.stride()
    if B == 1 or st[0] == N * st[1]:            # one uniform token stride across the batch: a single launch
        _lib.call("s3r_rope2d_inplace", tokens, _lib.ptr(tokens), _lib.ptr(positions), B * N, H, D, st[1], st[2],
                  float(base), float(fwd))
        return
    for b in range(B):
        _lib.call("s3r_rope2d_inplace", tokens, _lib.ptr(tokens[b]), _lib.ptr(positions[b]), N, H, D, st[1], st[2],
                  float(base), float(fwd))


def rope_2d(tokens: torch.Tensor, positions: torch.Tensor, base: float, fwd: float) -> None:
    """curope.rope_2d (curope.cpp:49-65 + the checks of rope_2d_cuda, kernels.cu:83-94).  Mutates `tokens`."""
    def check(cond, msg):
        if not cond:
            raise RuntimeError(msg)
    check(tokens.dim() == 4, "tokens must have 4 dimensions")
    check(positions.dim() == 3, "positions must have 3 dimensions")
    check(tokens.size(0) == positions.size(0), "batch size differs between tokens & positions")
    check(tokens.size(1) == positions.size(1), "seq_length differs between tokens & positions")
    check(positions.size(2) == 2, "positions.shape[2] must be equal to 2")
    check(tokens.is_cuda == positions.is_cuda, "tokens and positions are not on the same device")
    check(tokens.is_cuda, "spann3r_b200.curope has no CPU path (the reference falls back to rope_2d_cpu)")
    D = tokens.size(3)
    check(tokens.stride(3) == 1 and tokens.stride(2) == D, "tokens are not contiguous")
    check(positions.is_contiguous(), "positions are not contiguous")
    check(D % 4 == 0, "token dim must be multiple of 4")
    check(tokens.dtype == torch.float32, "spann3r_b200.curope supports float32 tokens only")
    check(positions.dtype == torch.int64, "positions must be int64")
    _lib.require_device()
    _launch(tokens, positions, base, fwd)


class cuRoPE2D_func(torch.autograd.Function):
    """In-place rotation with the inverse rotation as its gradient (curope2d.py:12-29)."""

    @staticmethod
    def forward(ctx, tokens, positions, base, F0=1):
        ctx.save_for_backward(positions)
        ctx.rope_args = (base, F0)
        rope_2d(tokens, positions, base, F0)
        ctx.mark_dirty(tokens)
        return tokens

    @staticmethod
    def backward(ctx, grad_res):
        (positions,), (base, F0) = ctx.saved_tensors, ctx.rope_args
        if not (grad_res.stride(3) == 1 and grad_res.stride(2) == grad_res.size(3)):
            grad_res = grad_res.contiguous()     # the reference would raise "tokens are not contiguous" here
        rope_2d(grad_res, positions, base, -F0)
        ctx.mark_dirty(grad_res)
        return grad_res, None, None, None


class cuRoPE2D(torch.nn.Module):
    """croco/models/curope/curope2d.py:32-40: tokens [B, H, N, D] (a view whose transpose(1, 2) has head stride D, as
    the q / k views of croco/models/blocks.py:94-112 do), positions [B, N, 2] int64 (y, x)."""

    def __init__(self, freq=100.0, F0=1.0):
        super().__init__()
        self.base = freq
        self.F0 = F0

    def forward(self, tokens, positions):
        cuRoPE2D_func.apply(tokens.transpose(1, 2), positions, self.base, self.F0)
        return tokens
