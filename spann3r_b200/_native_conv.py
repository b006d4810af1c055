"""The convolutions of the training backward on the wgmma GEMM engine, with the conv weight gradient on its own kernel.

`_recompute.py` routes every `F.conv2d` / `F.conv_transpose2d` through `conv2d()` / `conv_transpose2d()` below.  With the
switch off (default) those are the PyTorch calls and PyTorch autograd.  With it on, each convolution the DPT heads and the
two patch embeddings issue is an autograd Function whose three passes run split-bf16 (`bf16x3`, ~fp32-accurate) kernels
of libspann3r_b200.so:

* forward (the recompute): `s3r_gemm` as the eval path uses it -- 9 shifted taps for a 3x3 stride-1 conv, im2col for the
  3x3 stride-2 conv and the k = s = 16 patch conv, the `EPI_PIXSHUF` epilogue for ConvTranspose2d with kernel == stride;
* dgrad: `s3r_gemm` -- flipped, transposed weights [Cin, 9, Cout] for 3x3 stride 1; dY . W then `s3r_col2im_3x3s2` for
  stride 2; the un-shuffled dY against W as [Cin, s*s*Cout] for ConvTranspose; dY . W folded back to pixels for the patch
  conv.  Skipped when the input needs no gradient;
* wgrad: `s3r_conv_wgrad`, the pixel contraction read straight from the NHWC planes (conv_wgrad.cu);
* bias gradient: a sum over the pixels.

Layout changes between NCHW and the engine's NHWC planes, the weight flip / transposes and the ConvTranspose un-shuffle are
plain PyTorch data movement.  Anything else -- CPU tensors, and channel counts the engine does not take (`head.4`, 128 -> 4)
-- is the PyTorch call.

Enable with `spann3r_b200.train.set_native_conv(True)` or `S3R_TRAIN_NATIVE_CONV=1`; independent of `set_native_linear`.
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F

from . import _lib

ENABLED = os.environ.get("S3R_TRAIN_NATIVE_CONV", "0") == "1"


def _nhwc(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 2, 3, 1).float().contiguous()


def _planes(t: torch.Tensor):
    return _lib.split(t.float().contiguous())


def _gemm(a, nb, h, w, b, n, taps, bias=None, ps_s=0):
    """s3r_gemm on planes a [nb, h, w, kc] (taps 9: 3x3 stride 1 pad 1) and b [n, taps * kc] -> fp32 NHWC [nb, h, w, n]
    (ps_s > 0: ConvTranspose pixel shuffle, [nb, h * s, w * s, n / s^2])."""
    ah, al = a
    bh, bl = b
    dev = ah.device
    d = _lib.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = ah.data_ptr(), al.data_ptr(), bh.data_ptr(), bl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = 1, nb, h, w, ah.shape[-1], taps, n
    if ps_s:
        cout = n // (ps_s * ps_s)
        out = torch.empty((nb, h * ps_s, w * ps_s, cout), dtype=torch.float32, device=dev)
        d.epi, d.ps_s, d.ps_cout, d.ldo = _lib.EPI_PIXSHUF, ps_s, cout, cout
    else:
        out = torch.empty((nb, h, w, n), dtype=torch.float32, device=dev)
        d.epi, d.ldo = _lib.EPI_PLAIN, n
    if bias is not None:
        bias = bias.float().contiguous()
        d.bias = bias.data_ptr()
    d.out_f32 = out.data_ptr()
    _lib.gemm(d, dev)
    return out


def _nchw(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 3, 1, 2)


class _Conv1x1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        nb, _, h, wd = x.shape
        xp = _planes(_nhwc(x))
        ctx.xp, ctx.has_bias = xp, b is not None
        ctx.save_for_backward(w)
        return _nchw(_gemm(xp, nb, h, wd, _planes(w.flatten(1)), w.shape[0], 1, b))

    @staticmethod
    def backward(ctx, gy):
        (w,) = ctx.saved_tensors
        nb, _, h, wd = gy.shape
        gp = _planes(_nhwc(gy))
        gx = _nchw(_gemm(gp, nb, h, wd, _planes(w.flatten(1).t()), w.shape[1], 1)) if ctx.needs_input_grad[0] else None
        gw = _lib.conv_wgrad(gp, ctx.xp, 1).view(w.shape) if ctx.needs_input_grad[1] else None
        gb = gy.sum(dim=(0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb


class _Conv3x3(torch.autograd.Function):
    """3x3, stride 1, padding 1."""

    @staticmethod
    def forward(ctx, x, w, b):
        nb, c, h, wd = x.shape
        xp = _planes(_nhwc(x))
        ctx.xp, ctx.has_bias = xp, b is not None
        ctx.save_for_backward(w)
        return _nchw(_gemm(xp, nb, h, wd, _planes(w.permute(0, 2, 3, 1).reshape(w.shape[0], 9 * c)), w.shape[0], 9, b))

    @staticmethod
    def backward(ctx, gy):
        (w,) = ctx.saved_tensors
        n, c = w.shape[:2]
        nb, _, h, wd = gy.shape
        gp = _planes(_nhwc(gy))
        gx = None
        if ctx.needs_input_grad[0]:   # dx[p, c] = sum_{tap, n} dY[p + shift(tap), n] W[n, c, 2 - ky, 2 - kx]
            wf = w.flip(2, 3).permute(1, 2, 3, 0).reshape(c, 9 * n)
            gx = _nchw(_gemm(gp, nb, h, wd, _planes(wf), c, 9))
        gw = _lib.conv_wgrad(gp, ctx.xp, 9).view(n, 3, 3, c).permute(0, 3, 1, 2) if ctx.needs_input_grad[1] else None
        gb = gy.sum(dim=(0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb


class _Conv3x3s2(torch.autograd.Function):
    """3x3, stride 2, padding 1 (im2col + GEMM; the input gradient by col2im)."""

    @staticmethod
    def forward(ctx, x, w, b):
        nb, c, h, wd = x.shape
        ho, wo = (h + 1) // 2, (wd + 1) // 2
        xh, xl = _planes(_nhwc(x))
        ch = torch.empty((nb, ho, wo, 9 * c), dtype=torch.bfloat16, device=x.device)
        cl = torch.empty_like(ch)
        _lib.call("s3r_im2col_3x3s2", x, _lib.ptr(xh), _lib.ptr(xl), nb, h, wd, c, ho, wo, _lib.ptr(ch), _lib.ptr(cl))
        ctx.cols, ctx.in_shape, ctx.has_bias = (ch, cl), (nb, h, wd, c), b is not None
        ctx.save_for_backward(w)
        return _nchw(_gemm((ch, cl), nb, ho, wo, _planes(w.permute(0, 2, 3, 1).reshape(w.shape[0], 9 * c)), w.shape[0], 1, b))

    @staticmethod
    def backward(ctx, gy):
        (w,) = ctx.saved_tensors
        n = w.shape[0]
        nb, h, wd, c = ctx.in_shape
        _, _, ho, wo = gy.shape
        gp = _planes(_nhwc(gy))
        gx = None
        if ctx.needs_input_grad[0]:
            gcols = _gemm(gp, nb, ho, wo, _planes(w.permute(0, 2, 3, 1).reshape(n, 9 * c).t()), 9 * c, 1)
            gx = _nchw(_lib.col2im_3x3s2(gcols, nb, h, wd, c))
        gw = _lib.conv_wgrad(gp, ctx.cols, 1).view(n, 3, 3, c).permute(0, 3, 1, 2) if ctx.needs_input_grad[1] else None
        gb = gy.sum(dim=(0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb


class _PatchConv(torch.autograd.Function):
    """Conv2d(3, E, kernel 16, stride 16): im2col (k = c * 256 + i * 16 + j) + GEMM."""

    @staticmethod
    def forward(ctx, x, w, b):
        nb, _, h, wd = x.shape
        gh, gw_ = h // 16, wd // 16
        xf = x.float()
        ch = torch.empty((nb, gh, gw_, 768), dtype=torch.bfloat16, device=x.device)
        cl = torch.empty_like(ch)
        sb, sc, sy, sx = xf.stride()
        _lib.call("s3r_im2col_patch16", x, _lib.ptr(xf), sb, sc, sy, sx, nb, gh, gw_, _lib.ptr(ch), _lib.ptr(cl))
        ctx.cols, ctx.in_shape, ctx.has_bias = (ch, cl), x.shape, b is not None
        ctx.save_for_backward(w)
        return _nchw(_gemm((ch, cl), nb, gh, gw_, _planes(w.reshape(w.shape[0], 768)), w.shape[0], 1, b))

    @staticmethod
    def backward(ctx, gy):
        (w,) = ctx.saved_tensors
        nb, _, h, wd = ctx.in_shape
        _, _, gh, gw_ = gy.shape
        gp = _planes(_nhwc(gy))
        gx = None
        if ctx.needs_input_grad[0]:
            gcols = _gemm(gp, nb, gh, gw_, _planes(w.reshape(w.shape[0], 768).t()), 768, 1)
            gx = gcols.view(nb, gh, gw_, 3, 16, 16).permute(0, 3, 1, 4, 2, 5).reshape(nb, 3, h, wd)
        gw = _lib.conv_wgrad(gp, ctx.cols, 1).view(w.shape) if ctx.needs_input_grad[1] else None
        gb = gy.sum(dim=(0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb


class _ConvT(torch.autograd.Function):
    """ConvTranspose2d(Cin, Cout, kernel s, stride s): weight [Cin, Cout, s, s]; GEMM columns (i, j, co)."""

    @staticmethod
    def forward(ctx, x, w, b, s):
        nb, cin, h, wd = x.shape
        cout = w.shape[1]
        xp = _planes(_nhwc(x))
        ctx.xp, ctx.s, ctx.has_bias = xp, s, b is not None
        ctx.save_for_backward(w)
        return _nchw(_gemm(xp, nb, h, wd, _planes(w.permute(2, 3, 1, 0).reshape(s * s * cout, cin)), s * s * cout, 1, b, ps_s=s))

    @staticmethod
    def backward(ctx, gy):
        (w,) = ctx.saved_tensors
        s = ctx.s
        cin, cout = w.shape[:2]
        nb, _, hs, ws = gy.shape
        h, wd = hs // s, ws // s
        # un-shuffle: dY [nb, h s, w s, co] -> [nb, h, w, (i, j, co)]
        gu = _nhwc(gy).view(nb, h, s, wd, s, cout).permute(0, 1, 3, 2, 4, 5).reshape(nb, h, wd, s * s * cout)
        gp = _planes(gu)
        gx = None
        if ctx.needs_input_grad[0]:
            gx = _nchw(_gemm(gp, nb, h, wd, _planes(w.permute(0, 2, 3, 1).reshape(cin, s * s * cout)), cin, 1))
        gw = None
        if ctx.needs_input_grad[1]:
            gw = _lib.conv_wgrad(gp, ctx.xp, 1).view(s, s, cout, cin).permute(3, 2, 0, 1)
        gb = gy.sum(dim=(0, 2, 3)) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return gx, gw, gb, None


def _engine_channels(*cs) -> bool:
    return all(c % 32 == 0 for c in cs)


def conv2d(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, stride: int = 1, padding: int = 0) -> torch.Tensor:
    if ENABLED and x.is_cuda and x.dim() == 4 and w.shape[-1] == w.shape[-2]:
        n, c, k = w.shape[0], w.shape[1], w.shape[-1]
        h, wd = x.shape[-2:]
        if k == 1 and stride == 1 and padding == 0 and _engine_channels(n, c):
            return _Conv1x1.apply(x, w, b)
        if k == 3 and stride == 1 and padding == 1 and _engine_channels(n, c):
            return _Conv3x3.apply(x, w, b)
        if k == 3 and stride == 2 and padding == 1 and _engine_channels(n, c):
            return _Conv3x3s2.apply(x, w, b)
        if k == 16 and stride == 16 and padding == 0 and c == 3 and n % 32 == 0 and h % 16 == 0 and wd % 16 == 0:
            return _PatchConv.apply(x, w, b)
    return F.conv2d(x, w, b, stride=stride, padding=padding)


def conv_transpose2d(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, stride: int) -> torch.Tensor:
    if (ENABLED and x.is_cuda and x.dim() == 4 and w.shape[-1] == w.shape[-2] == stride and
            _engine_channels(w.shape[0], w.shape[1])):
        return _ConvT.apply(x, w, b, stride)
    return F.conv_transpose2d(x, w, b, stride=stride)
