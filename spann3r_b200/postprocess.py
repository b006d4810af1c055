"""Post-path geometry on the GPU (SURVEY.md section 8f rank 4): the reference's focal estimate and per-frame camera pose.

`demo.py:148-150` copies `preds[0]['pts3d']` to the CPU and runs `estimate_focal_knowing_depth(pts3d, pp,
focal_mode='weiszfeld')` (dust3r/post_process.py:12-60); `demo.py:166-180` then calls `cv2.solvePnPRansac` on a CPU copy of
every frame's pointmap (~0.3 s per 512x384 frame).  Same functions (names, argument meaning, outputs) here, computed on
the device by libspann3r_b200.so (csrc/geometry.cu, csrc/pnp.cu), batched over frames; no CPU fallback."""
from __future__ import annotations

import math

import torch

from . import _lib


def estimate_focal_knowing_depth(pts3d: torch.Tensor, pp, focal_mode: str = "median", min_focal: float = 0.0,
                                 max_focal: float = float("inf")) -> torch.Tensor:
    """pts3d [B, H, W, 3] fp32 on the device, pp = (cx, cy) (tensor or pair) -> focal [B] on the device."""
    if focal_mode not in ("weiszfeld", "median"):
        raise ValueError(f"bad {focal_mode=}")
    _lib.require_device()
    if not (pts3d.is_cuda and pts3d.dtype == torch.float32 and pts3d.dim() == 4 and pts3d.shape[-1] == 3):
        raise ValueError("expected pts3d [B, H, W, 3] float32 on the GPU")
    pts3d = pts3d.contiguous()
    B, H, W, _ = pts3d.shape
    ppx, ppy = (float(v) for v in (pp.flatten().tolist() if torch.is_tensor(pp) else pp))
    base = max(H, W) / (2 * math.tan(math.radians(60) / 2))
    lo = min_focal * base
    hi = max_focal * base           # max_focal = inf -> no upper clip; a NaN focal stays NaN in both modes
    focal = torch.empty(B, dtype=torch.float32, device=pts3d.device)
    if focal_mode == "median":      # nanmedian of the per-pixel votes: an exact selection, bit-identical to the reference
        scratch = torch.empty(B * 260, dtype=torch.int32, device=pts3d.device)
        _lib.call("s3r_focal_median", pts3d, _lib.ptr(pts3d), B, H, W, ppx, ppy, lo, hi, _lib.ptr(scratch), _lib.ptr(focal))
        return focal
    scratch = torch.empty(B * 148 * 2, dtype=torch.float32, device=pts3d.device)
    _lib.call("s3r_focal_weiszfeld", pts3d, _lib.ptr(pts3d), B, H, W, ppx, ppy, 10, lo, hi, _lib.ptr(scratch), _lib.ptr(focal))
    return focal


def solve_pnp_ransac(pts3d: torch.Tensor, camera_matrix, image_points: torch.Tensor | None = None, dist_coeffs=None,
                     iterations_count: int = 100, reprojection_error: float = 8.0, refine_iters: int = 15, seed: int = 0):
    """`cv2.solvePnPRansac(objectPoints, imagePoints, cameraMatrix, distCoeffs)` as demo.py:166-180 uses it, for a batch of
    frames at once and without leaving the device.

    pts3d [B, H, W, 3] fp32 (device): the world-frame pointmaps; their image points are the pixel grid (u = column,
    v = row) exactly as demo.py builds `points_2d` -- or pass pts3d [B, n, 3] with image_points [B, n, 2].
    camera_matrix: 3x3 (array / tensor / nested list) shared by the batch; dist_coeffs must be None or zeros (demo.py).
    iterations_count / reprojection_error: cv2's parameters of the same name (defaults 100 / 8.0).
    Returns (success [B] bool, rvec [B, 3] fp64, tvec [B, 3] fp64, inliers [B, H, W] or [B, n] bool), all on the device,
    nothing synchronised: x_cam = Rodrigues(rvec) x_world + tvec, like cv2; `inliers` is cv2's index list as a mask.
    The pose is the least-squares optimum of the reprojection error on the RANSAC model's inliers (what cv2's final
    SOLVEPNP_ITERATIVE refinement computes); deterministic for a given seed."""
    _lib.require_device()
    if dist_coeffs is not None and any(float(v) != 0.0 for v in torch.as_tensor(dist_coeffs).flatten().tolist()):
        raise NotImplementedError("lens distortion is not modelled (demo.py passes zeros)")
    if not (pts3d.is_cuda and pts3d.dtype == torch.float32 and pts3d.shape[-1] == 3 and pts3d.dim() in (3, 4)):
        raise ValueError("expected pts3d [B, H, W, 3] or [B, n, 3] float32 on the GPU")
    K = torch.as_tensor(camera_matrix, dtype=torch.float64).cpu().reshape(3, 3)
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    pts3d = pts3d.contiguous()
    B = pts3d.shape[0]
    if pts3d.dim() == 4:
        if image_points is not None:
            raise ValueError("image_points only with pts3d [B, n, 3]")
        n, width, out_shape = pts3d.shape[1] * pts3d.shape[2], pts3d.shape[2], tuple(pts3d.shape[:3])
    else:
        if image_points is None or tuple(image_points.shape) != (B, pts3d.shape[1], 2):
            raise ValueError("pts3d [B, n, 3] needs image_points [B, n, 2]")
        if not (image_points.is_cuda and image_points.dtype == torch.float32):
            raise ValueError("image_points must be float32 on the GPU")
        image_points = image_points.contiguous()
        n, width, out_shape = pts3d.shape[1], 0, tuple(pts3d.shape[:2])
    ws = torch.empty(int(_lib.lib().s3r_pnp_workspace_bytes(B, int(iterations_count))), dtype=torch.uint8, device=pts3d.device)
    out = torch.empty(B, 18, dtype=torch.float64, device=pts3d.device)
    mask = torch.empty(B, n, dtype=torch.uint8, device=pts3d.device)
    _lib.call("s3r_pnp_ransac", pts3d, _lib.ptr(pts3d), _lib.ptr(image_points), B, n, width, fx, fy, cx, cy,
              float(reprojection_error), int(iterations_count), int(refine_iters), int(seed), _lib.ptr(ws), _lib.ptr(out),
              _lib.ptr(mask))
    return out[:, 17] > 0.5, out[:, 12:15], out[:, 9:12], mask.view(out_shape).bool()
