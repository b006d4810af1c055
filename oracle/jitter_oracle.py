"""ORACLE (test infrastructure, not product code): numpy restatement of torchvision's ColorJitter on a PIL RGB image
(Pillow's ImageEnhance / Image.blend / HSV conversions), and of one training item of the reference's datasets built on
the CPU -- the path spann3r_b200/train_views.py runs on the device.

Rules (each pinned against Pillow / torchvision by tests/test_train_views.py):
  L            (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16
  blend        t = in1 + a * (in2 - in1) in fp32; 0 <= a <= 1: trunc(t), otherwise clamp t to [0, 255] and truncate
  brightness   blend(0, x, f); saturation blend(L, x, f); contrast blend(int(mean(L) + 0.5), x, f)
  hue          RGB -> HSV (fp32 ratios, fp64 sextant arithmetic), h += int32(hue * 255) mod 256, HSV -> RGB
"""
from __future__ import annotations

import numpy as np

from . import views_oracle as VO

f32, f64 = np.float32, np.float64


def luma(rgb) -> np.ndarray:
    c = rgb.astype(np.int64)
    return ((c[..., 0] * 19595 + c[..., 1] * 38470 + c[..., 2] * 7471 + 0x8000) >> 16).astype(np.uint8)


def blend(in1, in2, alpha) -> np.ndarray:
    a = f32(alpha)
    d = (np.asarray(in2, np.int64) - np.asarray(in1, np.int64)).astype(f32)
    t = np.asarray(in1, np.int64).astype(f32) + a * d
    if 0 <= a <= 1:
        return np.trunc(t).astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.trunc(np.clip(t, 0, 255)))).astype(np.uint8)


def contrast_mean(img) -> int:
    L = luma(img)
    return int(float(L.astype(np.int64).sum()) / float(L.size) + 0.5)


def rgb_to_hsv(rgb) -> np.ndarray:
    c = rgb.astype(np.int64)
    r, g, b = c[..., 0], c[..., 1], c[..., 2]
    mx, mn = c.max(-1), c.min(-1)
    grey = mx == mn
    cr = np.where(grey, 1, mx - mn).astype(f32)
    s = cr / np.where(grey, 1, mx).astype(f32)
    rc, gc, bc = ((mx - r).astype(f32) / cr, (mx - g).astype(f32) / cr, (mx - b).astype(f32) / cr)
    h = np.where(r == mx, (bc - gc).astype(f64),
                 np.where(g == mx, (2.0 + rc.astype(f64)) - bc.astype(f64), (4.0 + gc.astype(f64)) - rc.astype(f64)))
    h = h.astype(f32).astype(f64)
    h = np.fmod(h / 6.0 + 1.0, 1.0).astype(f32)
    uh = np.clip(np.trunc(h.astype(f64) * 255.0), 0, 255).astype(np.int64)
    us = np.clip(np.trunc(s.astype(f64) * 255.0), 0, 255).astype(np.int64)
    return np.stack([np.where(grey, 0, uh), np.where(grey, 0, us), mx], -1).astype(np.uint8)


def _round_half_away(x):
    fl = np.floor(x)
    return np.where(x - fl >= 0.5, fl + 1, fl)


def hsv_to_rgb(hsv) -> np.ndarray:
    c = hsv.astype(np.int64)
    h, s, v = c[..., 0], c[..., 1], c[..., 2]
    h6 = h.astype(f64) * 6.0 / 255.0
    i = np.floor(h6).astype(np.int64)
    f = (h6 - i.astype(f64)).astype(f32)
    fs = (s.astype(f64) / 255.0).astype(f32)
    vd = v.astype(f64)
    p = np.clip(_round_half_away(vd * (1.0 - fs.astype(f64))), 0, 255).astype(np.int64)
    q = np.clip(_round_half_away(vd * (1.0 - (fs * f).astype(f64))), 0, 255).astype(np.int64)
    t = np.clip(_round_half_away(vd * (1.0 - fs.astype(f64) * (1.0 - f.astype(f64)))), 0, 255).astype(np.int64)
    sel = i % 6
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    out = np.zeros(c.shape, np.int64)
    for k, chans in enumerate(table):
        m = sel == k
        for ch in range(3):
            out[..., ch] = np.where(m, chans[ch], out[..., ch])
    grey = s == 0
    out = np.where(grey[..., None], v[..., None], out)
    return out.astype(np.uint8)


def shift_hue(rgb, hue) -> np.ndarray:
    hsv = rgb_to_hsv(rgb)
    hsv[..., 0] = (hsv[..., 0].astype(np.int64) + int(np.int32(hue * 255))) & 255
    return hsv_to_rgb(hsv)


def color_jitter(rgb, params) -> np.ndarray:
    """uint8 [H, W, 3] + one view's draw (dict(order, brightness, contrast, saturation, hue); None = no jitter)."""
    img = np.asarray(rgb, np.uint8)
    if params is None:
        return img
    for op in params["order"]:
        if op == 0 and params["brightness"] is not None:
            img = blend(np.zeros_like(img), img, params["brightness"])
        elif op == 1 and params["contrast"] is not None:
            img = blend(np.full_like(img, contrast_mean(img)), img, params["contrast"])
        elif op == 2 and params["saturation"] is not None:
            img = blend(np.repeat(luma(img)[..., None], 3, -1), img, params["saturation"])
        elif op == 3 and params["hue"] is not None:
            img = shift_hue(img, params["hue"])
    return img


def build_view(rgb, depth, K, pose, plan_args, params) -> dict:
    """views_oracle.build_view with ColorJitter between the crop / rescale and ImgNorm."""
    image, depth, Kf, _ = VO.crop_resize(rgb, depth, K, *plan_args)
    _, pts3d, valid = VO.unproject(depth, Kf, pose)
    W, H = image.size
    view = dict(img=VO.img_norm(color_jitter(np.asarray(image), params)), depthmap=depth, camera_intrinsics=Kf,
                camera_pose=pose, pts3d=pts3d, valid_mask=valid, true_shape=np.int32((H, W)))
    if W < H:
        view["img"] = view["img"].swapaxes(1, 2)
        view["valid_mask"] = view["valid_mask"].swapaxes(0, 1)
        view["depthmap"] = view["depthmap"].swapaxes(0, 1)
        view["pts3d"] = view["pts3d"].swapaxes(0, 1)
        view["camera_intrinsics"] = view["camera_intrinsics"][[1, 0, 2]]
    return {k: np.ascontiguousarray(v) for k, v in view.items()}


class _Crop:
    def __init__(self, rgb, depth, K):
        self.rgb, self.depth, self.K = rgb, depth, K


def getitem(ds, idx) -> list:
    """One item of a training dataset of spann3r_b200.synth (unpatched), built on the CPU as the reference's
    BaseStereoViewDataset.__getitem__ builds it: `_get_views` with a real crop (views_oracle) so its checks read the
    reference's cropped depth, one ColorJitter draw per view in view order, then the base tail."""
    from spann3r_b200.train_views import draw_jitter, split_transform
    import torch  # noqa: F401  (the draws use torch's global RNG)
    pending = {}

    def crop(image, depthmap, intrinsics, resolution, rng=None, info=None):
        rgb = np.asarray(image)
        state = rng.bit_generator.state
        _, d, Kf, _ = VO.crop_resize(rgb, depthmap, intrinsics, resolution, ds.aug_crop, rng)
        key = id(d)
        pending[key] = (rgb, depthmap, intrinsics, resolution, state)
        return _Crop(rgb, d, Kf), d, Kf

    ds._crop_resize_if_necessary = crop
    try:
        if isinstance(idx, tuple):
            idx, ar_idx = idx
        else:
            ar_idx = 0
        if ds.seed:
            ds._rng = np.random.default_rng(seed=ds.seed + idx)
        resolution = ds._resolutions[ar_idx]
        views = ds._get_views(idx, resolution, ds._rng)
        cj = split_transform(ds.transform)
        out = []
        for v, view in enumerate(views):
            rgb, depth0, K0, res, state = pending[id(view["depthmap"])]
            rng = np.random.default_rng()
            rng.bit_generator.state = state                     # replay the crop's own draws
            params = draw_jitter(cj) if cj is not None else None
            built = build_view(rgb, depth0, K0, view["camera_pose"], (res, ds.aug_crop, rng), params)
            extra = {k: val for k, val in view.items() if k not in ("img", "depthmap", "camera_pose", "camera_intrinsics")}
            built.update(extra, idx=(idx, ar_idx, v))
            out.append(built)
        for view in out:
            view["rng"] = int.from_bytes(ds._rng.bytes(4), "big")
        return out
    finally:
        del ds._crop_resize_if_necessary
