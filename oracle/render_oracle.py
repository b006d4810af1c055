"""ORACLE -- TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ only; nothing under spann3r_b200/ touches it).

numpy restatement of the headless point rasteriser (spann3r_b200/vis.py, csrc/render.cu): the semantics stated in
include/spann3r_b200.h for s3r_render_*, vectorised.  The projection is formed element by element in fp64 in the
kernel's operation order (no `@` / `einsum`, whose summation order is unspecified), so every (col, row, key) is
bit-identical to the device's; the z-buffer is `np.minimum.at` on the uint64 keys.  Static mode re-renders the
cumulative cloud of frames 0..i from scratch for every frame, so it also checks the kernel's incremental shortcut.
"""
from __future__ import annotations

import numpy as np

EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def camera_array(extrinsic, intrinsic_matrix) -> np.ndarray:
    """World->camera 4x4 (or 3x4) and the 3x3 K -> the 16 doubles of s3r_render_splat: [R | t] row-major, fx, fy, cx, cy."""
    E = np.asarray(extrinsic, np.float64)
    K = np.asarray(intrinsic_matrix, np.float64)
    return np.concatenate([E[:3, :4].reshape(-1), [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]])


def project(pts, cam, z_near: float, w: int, h: int, id0: int = 0):
    """fp32 points [N, 3] with global indices id0 + i -> (pix int64 [N]: row * w + col, -1 where dropped; col, row
    int64 (-1 where dropped); key uint64 [N]: bits(fp32(qz)) << 32 | index, EMPTY where dropped)."""
    p = np.asarray(pts, np.float32).reshape(-1, 3).astype(np.float64)
    cam = np.asarray(cam, np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    fx, fy, cx, cy = cam[12:16]
    with np.errstate(all="ignore"):
        q = [((cam[4 * r] * x + cam[4 * r + 1] * y) + cam[4 * r + 2] * z) + cam[4 * r + 3] for r in range(3)]
        keep = np.isfinite(q[0]) & np.isfinite(q[1]) & np.isfinite(q[2]) & (q[2] > z_near)
        u = fx * (q[0] / q[2]) + cx
        v = fy * (q[1] / q[2]) + cy
        col = np.floor(u + 0.5)
        row = np.floor(v + 0.5)
        keep &= (col >= 0) & (col < w) & (row >= 0) & (row < h)
        col = np.where(keep, col, -1.0).astype(np.int64)
        row = np.where(keep, row, -1.0).astype(np.int64)
        depth = q[2].astype(np.float32).view(np.uint32).astype(np.uint64)
    ids = np.arange(len(p), dtype=np.uint64) + np.uint64(id0)
    key = np.where(keep, (depth << np.uint64(32)) | ids, EMPTY)
    pix = np.where(keep, row * w + col, -1)
    return pix, col, row, key


def color_u8(c) -> np.ndarray:
    """floor(min(1, max(0, c)) * 255 + 0.5) in fp64, NaN -> 0: the rounding of s3r_render_resolve."""
    s = np.fmin(1.0, np.fmax(0.0, np.asarray(c, np.float32).astype(np.float64)))
    return np.floor(s * 255.0 + 0.5).astype(np.uint8)


def splat(zbuf: np.ndarray, pts, cam, z_near, w, h, id0=0, mask=None):
    """zbuf [h * w] uint64 <- min(zbuf, keys of the points) in place."""
    pix, _, _, key = project(pts, cam, z_near, w, h, id0)
    keep = pix >= 0
    if mask is not None:
        keep &= np.asarray(mask, bool).reshape(-1)
    np.minimum.at(zbuf, pix[keep], key[keep])


def resolve(zbuf: np.ndarray, colors, w: int, h: int) -> np.ndarray:
    """zbuf [h * w] and colours [N, 3] fp32 by global index -> RGB [h, w, 3] uint8, black where empty."""
    colors = np.asarray(colors, np.float32).reshape(-1, 3)
    out = np.zeros((h * w, 3), np.uint8)
    hit = zbuf != EMPTY
    out[hit] = color_u8(colors[(zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)])
    return out.reshape(h, w, 3)


def render_frames(pts_all, image_all, cam, w: int, h: int, mask=None, dynamic: bool = False, z_near: float = 0.0):
    """pts_all, image_all [T, H, W, 3] fp32, mask [T, H, W] bool or None -> frames [T, h, w, 3] uint8.  Frame i draws
    frame i's points (dynamic) or the points of frames 0..i (static), each frame from an empty z-buffer."""
    pts_all = np.asarray(pts_all, np.float32)
    T = pts_all.shape[0]
    per = int(np.prod(pts_all.shape[1:3]))
    pts = pts_all.reshape(T, per, 3)
    colors = np.asarray(image_all, np.float32).reshape(-1, 3)
    m = None if mask is None else np.asarray(mask, bool).reshape(T, per)
    out = np.zeros((T, h, w, 3), np.uint8)
    for i in range(T):
        zbuf = np.full(h * w, EMPTY, np.uint64)
        for j in ([i] if dynamic else range(i + 1)):
            splat(zbuf, pts[j], cam, z_near, w, h, id0=j * per, mask=None if m is None else m[j])
        out[i] = resolve(zbuf, colors, w, h)
    return out
