"""Input adapter on the GPU (SURVEY.md section 8f rank 3): decoded RGB frames -> network inputs.

Replaces, for the demo / eval callers, the CPU preprocessing the reference runs per frame with PIL, batch 1,
`num_workers=0` (spann3r/datasets/demo.py:57-86 -> dust3r/datasets/base/base_stereo_view_dataset.py:143-194
`_crop_resize_if_necessary` -> dust3r/datasets/utils/cropping.py:55-124 -> dust3r/utils/image.py:23 `ImgNorm`):
centre crop on the principal point, Lanczos down-scale so that the image contains the target resolution, centred
crop, ToTensor + Normalize(0.5, 0.5).  The arithmetic runs in libspann3r_b200.so (csrc/preprocess.cu) and is
bit-identical to the reference's output: the down-scale is Pillow's 8-bit separable resampler (integer arithmetic),
the rest is index bookkeeping and one fp32 affine map.

Host side = the small, shape-only parts: the crop / scale geometry of `_crop_resize_if_necessary` and Pillow's
coefficient tables (`precompute_coeffs` + `normalize_coeffs_8bpc` of src/libImaging/Resample.c), computed once per
(image size, resolution) and cached on the device.  No CPU fallback: without the library / an H100 this raises.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import _lib

PRECISION_BITS = 32 - 8 - 2      # Pillow, Resample.c


def plan_frame(h: int, w: int, resolution=(512, 384), square_flip: bool = False) -> dict:
    """Integer geometry of `_crop_resize_if_necessary` (base_stereo_view_dataset.py:143-194) for an [h, w] image with the
    demo's pseudo intrinsics (cx = w // 2, cy = h // 2, demo.py:73-74): crop1 (l, t, r, b) on the source, scaled (W2, H2)
    = PIL resize target, crop2 (l, t, r, b) on the scaled image, out (W, H).  `square_flip` is the reference's
    `rng.integers(2)` draw for (nearly) square images (:176-178)."""
    cx, cy = w // 2, h // 2
    mx, my = min(cx, w - cx), min(cy, h - cy)
    if not (mx > w / 5 and my > h / 5):
        raise ValueError("bad principal point")            # the reference asserts the same (:160-161)
    l, t, r, b = cx - mx, cy - my, cx + mx, cy + my
    W, H = r - l, b - t
    res = tuple(int(v) for v in resolution)
    if res[0] < res[1]:
        raise ValueError("resolution must be (W, H) with W >= H")
    if H > 1.1 * W:
        res = res[::-1]
    elif 0.9 < H / W < 1.1 and res[0] != res[1] and square_flip:
        res = res[::-1]
    scale_final = max(res[0] / W, res[1] / H) + 1e-8          # cropping.py:69
    W2, H2 = int(np.floor(W * scale_final)), int(np.floor(H * scale_final))
    # principal point through crop 1, the rescale and the centred crop (cropping.py:87-124): float32 intrinsics,
    # colmap <-> opencv +-0.5, offset = 0.5 * margins, bbox = round(cx_in - cx_out)
    f32 = np.float32
    cx1, cy1 = f32(cx - l), f32(cy - t)
    cx2 = f32((cx1 + f32(0.5)) * f32(scale_final) - f32(0.5))
    cy2 = f32((cy1 + f32(0.5)) * f32(scale_final) - f32(0.5))
    margins = np.asarray((W2, H2)) * 1.0 - np.asarray(res)
    if not np.all(margins >= 0.0):
        raise ValueError("rescaled image does not contain the target resolution")
    off = 0.5 * margins
    cx3 = f32(f32(cx2 + f32(0.5)) - off[0]) - f32(0.5)
    cy3 = f32(f32(cy2 + f32(0.5)) - off[1]) - f32(0.5)
    l2 = int(np.int32(np.round(cx2 - cx3)))
    t2 = int(np.int32(np.round(cy2 - cy3)))
    return dict(crop1=(l, t, r, b), scaled=(W2, H2), crop2=(l2, t2, l2 + res[0], t2 + res[1]), out=res)


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def lanczos_coeffs(in_size: int, out_size: int):
    """Pillow's coefficient table for resizing `in_size` -> `out_size` pixels with LANCZOS (Resample.c:
    precompute_coeffs, lanczos_filter, normalize_coeffs_8bpc), in C-double arithmetic via Python floats / libm:
    (bounds [out, 2] int32 = (first source index, tap count), kk [out, ksize] int32 fixed point, ksize)."""
    scale = filterscale = in_size / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 3.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    ss = 1.0 / filterscale
    one = float(1 << PRECISION_BITS)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        n = xmax - xmin
        ws = []
        ww = 0.0
        for x in range(n):
            a = (x + xmin - center + 0.5) * ss
            wv = _sinc(a) * _sinc(a / 3.0) if -3.0 <= a < 3.0 else 0.0
            ws.append(wv)
            ww += wv
        for x in range(n):
            k = ws[x] / ww if ww != 0.0 else ws[x]
            kk[xx, x] = int(-0.5 + k * one) if k < 0 else int(0.5 + k * one)
        bounds[xx] = (xmin, n)
    return bounds, kk, ksize


class FrameAdapter:
    """uint8 RGB frame [H, W, 3] (numpy or torch, host or device) -> float32 [1, 3, H_out, W_out] on the device,
    bit-identical to `ImgNorm(_crop_resize_if_necessary(...))` of the reference.  Tables are cached per geometry."""

    def __init__(self, resolution=(512, 384), device="cuda"):
        _lib.require_device()
        self.resolution = tuple(resolution)
        self.device = torch.device(device)
        self._plans = {}

    def _plan(self, h, w, square_flip):
        key = (h, w, bool(square_flip))
        p = self._plans.get(key)
        if p is None:
            g = plan_frame(h, w, self.resolution, square_flip)
            l, t, r, b = g["crop1"]
            W1, H1 = r - l, b - t
            W2, H2 = g["scaled"]
            l2, t2, r2, b2 = g["crop2"]
            bh, kh, ksh = lanczos_coeffs(W1, W2)
            bv, kv, ksv = lanczos_coeffs(H1, H2)
            bh, kh = bh[l2:r2].copy(), kh[l2:r2].copy()              # only the columns / rows the final crop keeps
            bv, kv = bv[t2:b2].copy(), kv[t2:b2].copy()
            row0 = int(bv[0, 0])                                      # source rows the vertical pass reads
            row1 = int(bv[-1, 0] + bv[-1, 1])
            bv[:, 0] -= row0
            n = bh.shape[0]
            span = 0
            for x0 in range(0, n, 128):
                xl = min(x0 + 127, n - 1)
                span = max(span, int(bh[xl, 0] + bh[xl, 1] - bh[x0, 0]))
            dev = self.device
            p = dict(geom=g, src_row0=t + row0, rows=row1 - row0, src_col0=l, out_w=r2 - l2, out_h=b2 - t2, span=span,
                     bh=torch.from_numpy(bh).to(dev), kh=torch.from_numpy(kh).to(dev), ksh=ksh,
                     bv=torch.from_numpy(bv).to(dev), kv=torch.from_numpy(kv).to(dev), ksv=ksv,
                     tmp=torch.empty((row1 - row0, r2 - l2, 3), dtype=torch.uint8, device=dev))
            self._plans[key] = p
        return p

    @torch.no_grad()
    def __call__(self, rgb, square_flip: bool = False) -> torch.Tensor:
        if isinstance(rgb, np.ndarray):
            rgb = torch.from_numpy(np.ascontiguousarray(rgb))
        if rgb.dtype != torch.uint8 or rgb.dim() != 3 or rgb.shape[2] != 3:
            raise ValueError("expected a uint8 RGB image [H, W, 3]")
        h, w = int(rgb.shape[0]), int(rgb.shape[1])
        p = self._plan(h, w, square_flip)
        src = rgb.to(self.device, non_blocking=True).contiguous()
        out = torch.empty((1, 3, p["out_h"], p["out_w"]), dtype=torch.float32, device=self.device)
        L = _lib.lib()
        src_ptr = src.data_ptr() + (p["src_row0"] * w + p["src_col0"]) * 3
        with _lib.on_device(out):
            sp = _lib.stream_ptr(out.device)
            _lib.check(L.s3r_resample_h_u8(src_ptr, w * 3, p["rows"], p["out_w"], _lib.ptr(p["bh"]), _lib.ptr(p["kh"]), p["ksh"],
                                           p["span"], _lib.ptr(p["tmp"]), sp), "s3r_resample_h_u8")
            _lib.check(L.s3r_resample_v_u8_norm(_lib.ptr(p["tmp"]), p["out_w"], p["out_h"], _lib.ptr(p["bv"]), _lib.ptr(p["kv"]),
                                                p["ksv"], _lib.ptr(out), sp), "s3r_resample_v_u8_norm")
        return out


def load_frames(images, resolution=(512, 384), device="cuda", adapter: FrameAdapter = None):
    """List of decoded uint8 RGB frames -> the list of view dicts `Spann3R.forward` takes ({'img': [1, 3, H, W] fp32 on the
    device, 'true_shape': [[H, W]]}), i.e. what `Demo(...)[0]` + the DataLoader collate produce for the model (the
    geometry entries demo.py derives for visualisation are not needed by the forward path)."""
    adapter = adapter or FrameAdapter(resolution, device)
    views = []
    for im in images:
        x = adapter(im)
        views.append({"img": x, "true_shape": torch.tensor([[x.shape[2], x.shape[3]]], dtype=torch.int32)})
    return views
