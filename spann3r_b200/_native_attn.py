"""Attention of the training backward on the library's own kernels -- the third switch of the native recompute backward,
next to `_native_linear` and `_native_conv`.

`_recompute.py` routes every self- and cross-attention (24 encoder blocks, 2 x 12 decoder blocks, 6 value-encoder blocks)
through `_attn`, which calls `attention()` below when the switch is on and the tensors are on the GPU.  `attention` is an
autograd Function over `s3r_attn_train_forward` / `s3r_attn_train_backward` (csrc/attention_train.cu):

* forward: a flash forward that returns O already in the [B, nq, heads * dh] layout the attention's `proj` reads, and
  keeps O and one log-sum-exp per row for the backward -- not the [B * heads, nq, nk] probabilities autograd would keep;
* backward: D = rowsum(dO o O), then dK / dV (one pass over the queries per key tile) and dQ (one pass over the keys per
  query tile), probabilities rebuilt from the log-sum-exp.

Every product is split-bf16 (`bf16x3`, ~fp32-accurate) whatever `torch.backends.cuda.matmul.allow_tf32` says, and the
result is bitwise reproducible (no float atomics).  dh = 48 (the use_feat value encoder) is zero-padded to 64 inside the
kernels.  RoPE stays PyTorch.  CPU tensors keep the PyTorch ops.

Enable with `spann3r_b200.train.set_native_attention(True)` or `S3R_TRAIN_NATIVE_ATTN=1`; independent of the other two.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib

ENABLED = os.environ.get("S3R_TRAIN_NATIVE_ATTN", "0") == "1"


def use(q: torch.Tensor) -> bool:
    return ENABLED and q.is_cuda and q.shape[-1] in (48, 64)


def _operand(t: torch.Tensor) -> torch.Tensor:
    """fp32 with dh contiguous, strides multiples of 4 elements and a 16-byte aligned start (the qkv views already are)."""
    t = t.float()
    if t.stride(-1) != 1 or any(s % 4 for s in t.stride()[:3]) or t.data_ptr() % 16:
        t = t.contiguous()
    return t


def _desc(q, k, v, scale: float) -> _lib.AttnTrainDesc:
    B, H, nq, dh = q.shape
    d = _lib.AttnTrainDesc()
    d.batch, d.heads, d.nq, d.nk, d.dh, d.scale = B, H, nq, k.shape[2], dh, float(scale)
    d.q, d.k, d.v = q.data_ptr(), k.data_ptr(), v.data_ptr()
    for name, t in (("q_stride", q), ("k_stride", k), ("v_stride", v)):
        getattr(d, name)[:] = list(t.stride()[:3])
    return d


def _forward(q, k, v, scale: float):
    q, k, v = _operand(q), _operand(k), _operand(v)
    B, H, nq, dh = q.shape
    d = _desc(q, k, v, scale)
    o = torch.empty((B, nq, H * dh), dtype=torch.float32, device=q.device)
    lse = torch.empty((B * H, nq), dtype=torch.float32, device=q.device)
    _lib.call("s3r_attn_train_forward", q, C.byref(d), _lib.ptr(o), _lib.ptr(lse))
    return q, k, v, o, lse


class _Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale):
        q, k, v, o, lse = _forward(q, k, v, scale)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.scale = scale
        return o

    @staticmethod
    def backward(ctx, go):
        q, k, v, o, lse = ctx.saved_tensors
        go = go.float().contiguous()
        d = _desc(q, k, v, ctx.scale)
        ws_bytes = _lib.lib().s3r_attn_train_workspace_bytes(C.byref(d))
        ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=q.device)
        dq = torch.empty(q.shape, dtype=torch.float32, device=q.device)
        dk = torch.empty(k.shape, dtype=torch.float32, device=q.device)
        dv = torch.empty(v.shape, dtype=torch.float32, device=q.device)
        _lib.call("s3r_attn_train_backward", q, C.byref(d), _lib.ptr(o), _lib.ptr(lse), _lib.ptr(go), _lib.ptr(ws),
                  ws_bytes, _lib.ptr(dq), _lib.ptr(dk), _lib.ptr(dv))
        return dq, dk, dv, None


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float) -> torch.Tensor:
    """softmax(scale q k^T) v of q [B, heads, nq, dh], k / v [B, heads, nk, dh] (dh 48 or 64, CUDA) -> [B, nq, heads * dh]."""
    return _Attention.apply(q, k, v, scale)


def attention_with_lse(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float):
    """The forward alone, without autograd: (O [B, nq, heads * dh], LSE [B * heads, nq])."""
    return _forward(q, k, v, scale)[3:]
