"""ORACLE (test infrastructure, not product code): CPU restatement of how the reference turns a decoded view into the
view dict its datasets yield, with numpy, Pillow and cv2 -- the path spann3r_b200/views.py runs on the device.

What the reference does per view (dust3r/datasets/base/base_stereo_view_dataset.py:63-194, cropping.py, geometry.py):

  1. crop centred on the rounded principal point (np.round, half to even); the margins must exceed a fifth of the size
  2. portrait crop -> transposed resolution; nearly square crop and non-square resolution -> rng.integers(2) decides
  3. aug_crop > 1 -> target = resolution + rng.integers(0, aug_crop)
  4. scale = max(target / size) + 1e-8; PIL LANCZOS resize of the image and cv2 INTER_NEAREST resize of the depth to
     floor(size * scale); intrinsics through camera_matrix_of_crop (colmap +-0.5, scaled, minus half the floor margin)
  5. centred crop to the resolution (bbox from the intrinsics before / after a centred camera_matrix_of_crop)
  6. ImgNorm; pts3d = R (K^-1 [u, v, 1] z) + t in numpy's promotion (fp64 unprojection rounded to fp32, fp32 einsum);
     valid_mask = (depth > 0) & isfinite(pts3d).all(-1); true_shape = (H, W)
  7. transpose_to_landscape for W < H; after all views, rng.bytes(4) per view
"""
from __future__ import annotations

import cv2
import numpy as np
import PIL.Image

LANCZOS = PIL.Image.Resampling.LANCZOS


def _camera_matrix_of_crop(K, in_res, out_res, scaling=1, offset_factor=0.5):
    margins = np.asarray(in_res) * scaling - out_res
    assert np.all(margins >= 0.0)
    offset = offset_factor * margins
    Kc = K.copy()
    Kc[0, 2] += 0.5
    Kc[1, 2] += 0.5
    Kc[:2, :] *= scaling
    Kc[:2, 2] -= offset
    Kc[0, 2] -= 0.5
    Kc[1, 2] -= 0.5
    return Kc


def _crop(image, depth, K, bbox):
    l, t, r, b = bbox
    K = K.copy()
    K[0, 2] -= l
    K[1, 2] -= t
    return image.crop((l, t, r, b)), depth[t:b, l:r], K


def crop_resize(rgb, depth, K, resolution, aug_crop=0, rng=None):
    """Steps 1-5 -> (PIL image, depth, K, geometry dict as spann3r_b200.views.plan_view returns it)."""
    image = PIL.Image.fromarray(rgb)
    W, H = image.size
    cx, cy = K[:2, 2].round().astype(int)
    mx, my = min(cx, W - cx), min(cy, H - cy)
    if not (mx > W / 5 and my > H / 5):
        raise ValueError("bad principal point")
    crop1 = (cx - mx, cy - my, cx + mx, cy + my)
    image, depth, K = _crop(image, depth, K, crop1)
    W, H = image.size
    res = tuple(resolution)
    if H > 1.1 * W:
        res = res[::-1]
    elif 0.9 < H / W < 1.1 and res[0] != res[1]:
        if rng.integers(2):
            res = res[::-1]
    target = np.array(res)
    if aug_crop > 1:
        target += rng.integers(0, aug_crop)
    in_res = np.array(image.size)
    scale = max(target / image.size) + 1e-8
    out_res = np.floor(in_res * scale).astype(int)
    image = image.resize(tuple(out_res), resample=LANCZOS)
    depth = cv2.resize(depth, out_res, fx=scale, fy=scale, interpolation=cv2.INTER_NEAREST)
    K = _camera_matrix_of_crop(K, in_res, out_res, scaling=scale)
    K2 = _camera_matrix_of_crop(K, image.size, res, offset_factor=0.5)
    l, t = np.int32(np.round(K[:2, 2] - K2[:2, 2]))
    crop2 = (l, t, l + res[0], t + res[1])
    image, depth, K = _crop(image, depth, K, crop2)
    geom = dict(crop1=tuple(int(v) for v in crop1), scaled=(int(out_res[0]), int(out_res[1])),
                crop2=tuple(int(v) for v in crop2), out=res, K=K, portrait=res[0] < res[1])
    return image, depth, K, geom


def unproject(depth, K, pose):
    """depthmap_to_absolute_camera_coordinates + the validity rule -> (camera points, world points, valid_mask)."""
    K = np.float32(K)
    H, W = depth.shape
    fu, fv, cu, cv = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    x = (u - cu) * depth / fu
    y = (v - cv) * depth / fv
    X_cam = np.stack((x, y, depth), axis=-1).astype(np.float32)
    X_world = np.einsum("ik, vuk -> vui", pose[:3, :3], X_cam) + pose[:3, 3][None, None, :]
    valid = (depth > 0.0) & np.isfinite(X_world).all(axis=-1)
    return X_cam, X_world, valid


def img_norm(image) -> np.ndarray:
    """ImgNorm (ToTensor + Normalize(0.5, 0.5)) -> float32 [3, H, W]."""
    x = np.asarray(image).astype(np.float32) / np.float32(255.0)
    x = (x - np.float32(0.5)) / np.float32(0.5)
    return np.ascontiguousarray(x.transpose(2, 0, 1))


def build_view(rgb, depth, K, pose, resolution, aug_crop=0, rng=None) -> dict:
    """Steps 1-7 for one view (without the trailing rng bytes): numpy arrays, transposed to landscape."""
    image, depth, Kf, _ = crop_resize(rgb, depth, K, resolution, aug_crop, rng)
    if pose is None:
        pose = np.full((4, 4), np.nan, dtype=np.float32)
    _, pts3d, valid = unproject(depth, Kf, pose)
    W, H = image.size
    view = dict(img=img_norm(image), depthmap=depth, camera_intrinsics=Kf, camera_pose=pose, pts3d=pts3d,
                valid_mask=valid, true_shape=np.int32((H, W)))
    if W < H:
        view["img"] = view["img"].swapaxes(1, 2)
        view["valid_mask"] = view["valid_mask"].swapaxes(0, 1)
        view["depthmap"] = view["depthmap"].swapaxes(0, 1)
        view["pts3d"] = view["pts3d"].swapaxes(0, 1)
        view["camera_intrinsics"] = view["camera_intrinsics"][[1, 0, 2]]
    return {k: np.ascontiguousarray(v) for k, v in view.items()}


def build_item(inputs, resolution, aug_crop, seed) -> list:
    """One dataset item: the views of `inputs` [(rgb, depth, K, pose)] with the item's rng (seeded as the reference's
    __getitem__ seeds it for idx 0), then rng.bytes(4) per view."""
    rng = np.random.default_rng(seed)
    views = [build_view(rgb, depth, K, pose, resolution, aug_crop, rng) for rgb, depth, K, pose in inputs]
    for v in views:
        v["rng"] = int.from_bytes(rng.bytes(4), "big")
    return views
