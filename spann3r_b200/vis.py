"""Headless rendering and PLY export: the reference's spann3r/tools/vis.py `render_frames` and Open3D's
`o3d.io.write_point_cloud` / `read_pinhole_camera_parameters` / `write_pinhole_camera_parameters` without Open3D or a
display.

`render_frames` draws the reconstruction with a deterministic z-buffered point rasteriser on the device
(csrc/render.cu, through libspann3r_b200.so; there is no CPU fallback): one pixel per point (Open3D's point_size 1) on a
black background, the nearest point of a pixel winning at fp32 depth resolution and equal depths going to the smaller
point index.  Static mode keeps the z-buffer across frames and splats only each new frame's points, which gives exactly
what re-rendering the accumulated cloud from scratch gives.  Differences from the Open3D window: INTEGRATION.md,
"Headless rendering and PLY export".
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np
import torch

from . import _lib


class PinholeCameraIntrinsic:
    """Open3D's PinholeCameraIntrinsic: image `width`, `height` and the 3x3 `intrinsic_matrix` (fx 0 cx; 0 fy cy; 0 0 1)."""

    def __init__(self, width: int, height: int, intrinsic_matrix):
        self.width = int(width)
        self.height = int(height)
        self.intrinsic_matrix = np.array(intrinsic_matrix, dtype=np.float64).reshape(3, 3)


class PinholeCameraParameters:
    """Open3D's PinholeCameraParameters: `.intrinsic` (PinholeCameraIntrinsic) and `.extrinsic` (4x4, world -> camera)."""

    def __init__(self, intrinsic: PinholeCameraIntrinsic, extrinsic):
        self.intrinsic = intrinsic
        self.extrinsic = np.array(extrinsic, dtype=np.float64).reshape(4, 4)


def read_pinhole_camera_parameters(path: str) -> PinholeCameraParameters:
    """Open3D's camera.json (what `o3d.io.write_pinhole_camera_parameters` writes; matrices column-major)."""
    with open(path) as f:
        d = json.load(f)
    if d.get("class_name") != "PinholeCameraParameters" or d.get("version_major") != 1:
        raise ValueError(f"{path}: not an Open3D PinholeCameraParameters file (version 1.x)")
    intr = d["intrinsic"]
    if len(d["extrinsic"]) != 16 or len(intr["intrinsic_matrix"]) != 9:
        raise ValueError(f"{path}: expected 16 extrinsic and 9 intrinsic_matrix values")
    K = np.array(intr["intrinsic_matrix"], dtype=np.float64).reshape(3, 3).T
    E = np.array(d["extrinsic"], dtype=np.float64).reshape(4, 4).T
    return PinholeCameraParameters(PinholeCameraIntrinsic(intr["width"], intr["height"], K), E)


def write_pinhole_camera_parameters(path: str, camera) -> None:
    """Write `camera` (.intrinsic, .extrinsic: this module's types or Open3D's) as Open3D's camera.json."""
    K = np.asarray(camera.intrinsic.intrinsic_matrix, dtype=np.float64)
    E = np.asarray(camera.extrinsic, dtype=np.float64)
    d = {
        "class_name": "PinholeCameraParameters",
        "extrinsic": [float(v) for v in E.reshape(-1, order="F")],
        "intrinsic": {"height": int(camera.intrinsic.height),
                      "intrinsic_matrix": [float(v) for v in K.reshape(-1, order="F")],
                      "width": int(camera.intrinsic.width)},
        "version_major": 1,
        "version_minor": 0,
    }
    with open(path, "w") as f:
        json.dump(d, f, indent=4)
        f.write("\n")


def camera_from_pose(cam_to_world, focal: float, width: int = 1920, height: int = 1080) -> PinholeCameraParameters:
    """A camera at a camera-to-world pose (e.g. demo.py's `poses_all[0]`) with focal length `focal` in pixels of the
    width x height image and the principal point at (width / 2 - 0.5, height / 2 - 0.5), as Open3D's view control
    requires.  For a headless run, which has no window to pick a view in."""
    P = np.asarray(cam_to_world.cpu() if isinstance(cam_to_world, torch.Tensor) else cam_to_world, dtype=np.float64)
    if P.shape != (4, 4) or not np.isfinite(P).all():
        raise ValueError(f"cam_to_world: expected a finite 4x4 pose, got shape {P.shape}")
    R, t = P[:3, :3], P[:3, 3]
    E = np.eye(4)
    E[:3, :3] = R.T
    E[:3, 3] = -(R.T @ t)
    K = np.array([[focal, 0.0, width / 2 - 0.5], [0.0, focal, height / 2 - 0.5], [0.0, 0.0, 1.0]])
    return PinholeCameraParameters(PinholeCameraIntrinsic(width, height, K), E)


def _camera_array(camera):
    """-> (the 16 doubles of s3r_render_splat, width, height); ValueError for a camera the rasteriser cannot draw."""
    try:
        K = np.asarray(camera.intrinsic.intrinsic_matrix, dtype=np.float64)
        E = np.asarray(camera.extrinsic, dtype=np.float64)
        w, h = int(camera.intrinsic.width), int(camera.intrinsic.height)
    except AttributeError as ex:
        raise ValueError(f"camera_parameters: expected .intrinsic (width, height, intrinsic_matrix) and .extrinsic: {ex}")
    if K.shape != (3, 3) or E.shape != (4, 4):
        raise ValueError(f"camera_parameters: expected a 3x3 intrinsic and a 4x4 extrinsic, got {K.shape}, {E.shape}")
    if not (np.isfinite(K).all() and np.isfinite(E).all()):
        raise ValueError("camera_parameters: non-finite values")
    if K[0, 1] != 0 or K[1, 0] != 0 or K[2].tolist() != [0.0, 0.0, 1.0]:
        raise ValueError(f"camera_parameters: the intrinsic must be [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] (no skew), got "
                         f"{K.tolist()}")
    if E[3].tolist() != [0.0, 0.0, 0.0, 1.0]:
        raise ValueError(f"camera_parameters: the extrinsic's last row must be [0, 0, 0, 1], got {E[3].tolist()}")
    if not (w >= 1 and h >= 1 and w * h < 2 ** 31):
        raise ValueError(f"camera_parameters: image size {w}x{h} out of range")
    cam = np.ascontiguousarray(np.concatenate([E[:3, :4].reshape(-1), [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]]))
    return cam, w, h


def _frames_input(pts_all, image_all, mask):
    for name, x in (("pts_all", pts_all), ("image_all", image_all)):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise ValueError(f"{name}: expected a CUDA tensor [T, H, W, 3], got "
                             f"{x.device if isinstance(x, torch.Tensor) else type(x).__name__}")
        if x.dtype != torch.float32 or x.dim() != 4 or x.shape[-1] != 3 or x.numel() == 0:
            raise ValueError(f"{name}: expected float32 [T, H, W, 3], got {tuple(x.shape)} {x.dtype}")
    if image_all.shape != pts_all.shape or image_all.device != pts_all.device:
        raise ValueError(f"image_all {tuple(image_all.shape)} on {image_all.device} must match pts_all "
                         f"{tuple(pts_all.shape)} on {pts_all.device}")
    if pts_all.shape[0] * pts_all.shape[1] * pts_all.shape[2] >= 2 ** 32:
        raise ValueError(f"pts_all: T * H * W must be below 2^32, got {tuple(pts_all.shape[:3])}")
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or tuple(mask.shape) != tuple(pts_all.shape[:3]) \
                or mask.device != pts_all.device:
            raise ValueError(f"mask: expected a bool tensor {tuple(pts_all.shape[:3])} on {pts_all.device}, got "
                             f"{tuple(mask.shape) if isinstance(mask, torch.Tensor) else type(mask).__name__}")
        mask = mask.contiguous().view(torch.uint8)
    return pts_all.contiguous(), image_all.contiguous(), mask


def render_frames(pts_all, image_all, camera_parameters, output_dir=None, mask=None, save_video=True, save_camera=True,
                  dynamic=False, z_near=0.0):
    """spann3r/tools/vis.py `render_frames` on the device, with its arguments.

    pts_all, image_all: [T, H, W, 3] fp32 CUDA tensors (colours in [0, 1], as demo.py builds `images_all`); mask:
    [T, H, W] bool or None (demo.py passes `conf_sig_all > conf_thresh`); camera_parameters: `.intrinsic` (width,
    height, intrinsic_matrix without skew) and `.extrinsic` (4x4 world -> camera), e.g. from
    `read_pinhole_camera_parameters` or `camera_from_pose`.  Frame i draws frame i's points (dynamic=True) or those of
    frames 0..i; points with camera depth <= z_near (>= 0) are not drawn, and there is no far plane.

    Returns the frames as a uint8 CUDA tensor [T, h, w, 3] (RGB) at the camera's image size: 6.2 MB per frame at
    1920x1080.  With `output_dir`, also writes the reference's layout: render_frames/frame_{i:03d}.png,
    render_frames/camera.json (save_camera) and render_frame.mp4 at 10 fps (save_video; OpenCV, 'mp4v')."""
    pts_all, image_all, mask = _frames_input(pts_all, image_all, mask)
    cam, w, h = _camera_array(camera_parameters)
    if not (math.isfinite(z_near) and z_near >= 0):
        raise ValueError(f"z_near must be finite and >= 0, got {z_near}")
    _lib.require_device()
    T, H, W, _ = pts_all.shape
    per = H * W
    dev = pts_all.device
    keys = torch.empty(int(_lib.lib().s3r_render_workspace_bytes(w, h)) // 8, dtype=torch.int64, device=dev)
    frames = torch.empty((T, h, w, 3), dtype=torch.uint8, device=dev)
    cam_p = C.c_void_p(cam.ctypes.data)
    for i in range(T):
        if dynamic or i == 0:
            _lib.call("s3r_render_clear", dev, _lib.ptr(keys), w, h)
        _lib.call("s3r_render_splat", dev, _lib.ptr(pts_all[i]), _lib.ptr(None if mask is None else mask[i]), per, i * per,
                  cam_p, float(z_near), w, h, _lib.ptr(keys))
        _lib.call("s3r_render_resolve", dev, _lib.ptr(keys), _lib.ptr(image_all), w, h, _lib.ptr(frames[i]))
    if output_dir is not None:
        write_frames(frames, output_dir, camera_parameters if save_camera else None, save_video)
    return frames


def render_mesh_frames(pts_all, image_all, camera_parameters, output_dir=None, mask=None, save_video=True,
                       save_camera=True, dynamic=False, z_near=0.0):
    """`render_frames`' contract, drawing app.py's reconstruction mesh (`mesh.pts3d_to_mesh`) instead of points.

    Frame i draws the triangles of frame i (dynamic=True) or of frames 0..i with the triangle rasteriser of
    `mesh.rasterize` (back faces culled: app.py's mesh carries both windings, so none of it is hidden); each pixel takes
    the colour of its face, rounded as render_frames rounds.  Static mode keeps the key buffer across frames and draws
    only each new frame's triangles.  mask: [T, H, W] bool (the valid pixels) or None; points and colours of valid
    pixels must be finite.  Returns uint8 [T, h, w, 3] CUDA frames and writes render_frames' files with `write_frames`."""
    from . import mesh
    pts_all, image_all, mask = _frames_input(pts_all, image_all, mask)
    cam, w, h = _camera_array(camera_parameters)
    if not (math.isfinite(z_near) and z_near >= 0):
        raise ValueError(f"z_near must be finite and >= 0, got {z_near}")
    T, H, W, _ = pts_all.shape
    verts, faces, colors = mesh.pts3d_to_mesh(pts_all, image_all, None if mask is None else mask.view(torch.bool))
    # faces come frame by frame: the frame of a face is its first vertex // (H W)
    bounds = torch.searchsorted(torch.div(faces[:, 0], H * W, rounding_mode="floor").contiguous(),
                                torch.arange(T + 1, dtype=torch.int32, device=faces.device)).cpu().tolist()
    if len(colors) == 0:
        colors = torch.zeros((1, 3), dtype=torch.float32, device=pts_all.device)   # never read: no face is drawn
    dev = pts_all.device
    keys = torch.empty(int(_lib.lib().s3r_render_workspace_bytes(w, h)) // 8, dtype=torch.int64, device=dev)
    frames = torch.empty((T, h, w, 3), dtype=torch.uint8, device=dev)
    cam_p = C.c_void_p(cam.ctypes.data)
    for i in range(T):
        if dynamic or i == 0:
            _lib.call("s3r_render_clear", dev, _lib.ptr(keys), w, h)
        f = faces[bounds[i]:bounds[i + 1]]
        if len(f):
            _lib.call("s3r_raster_triangles", dev, _lib.ptr(verts), len(verts), _lib.ptr(f), len(f), bounds[i], cam_p,
                      float(z_near), math.inf, w, h, _lib.ptr(keys))
        # the keys hold face ids: the render resolve gathers the face colours
        _lib.call("s3r_render_resolve", dev, _lib.ptr(keys), _lib.ptr(colors), w, h, _lib.ptr(frames[i]))
    if output_dir is not None:
        write_frames(frames, output_dir, camera_parameters if save_camera else None, save_video)
    return frames


def write_frames(frames: torch.Tensor, output_dir: str, camera_parameters=None, save_video: bool = True) -> None:
    """The files of render_frames: output_dir/render_frames/frame_{i:03d}.png, .../camera.json (when a camera is given)
    and output_dir/render_frame.mp4 (10 fps, 'mp4v'), from RGB uint8 frames [T, h, w, 3] on any device.  Host I/O by
    OpenCV; raises if a file cannot be written."""
    import cv2
    T, h, w, _ = frames.shape
    frame_dir = os.path.join(output_dir, "render_frames")
    os.makedirs(frame_dir, exist_ok=True)
    if camera_parameters is not None:
        write_pinhole_camera_parameters(os.path.join(frame_dir, "camera.json"), camera_parameters)
    writer = None
    if save_video:
        video = os.path.join(output_dir, "render_frame.mp4")
        writer = cv2.VideoWriter(video, cv2.VideoWriter_fourcc(*"mp4v"), 10, (w, h))
        if not writer.isOpened():
            raise RuntimeError(f"cv2.VideoWriter could not open {video} ('mp4v', {w}x{h})")
    try:
        for i in range(T):
            bgr = np.ascontiguousarray(frames[i].cpu().numpy()[..., ::-1])
            path = os.path.join(frame_dir, f"frame_{i:03d}.png")
            if not cv2.imwrite(path, bgr):
                raise RuntimeError(f"cv2.imwrite could not write {path}")
            if writer is not None:
                writer.write(bgr)
    finally:
        if writer is not None:
            writer.release()


def _host_array(x, name: str) -> np.ndarray:
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    if x.ndim < 1 or x.shape[-1] != 3 or not (np.issubdtype(x.dtype, np.floating) or np.issubdtype(x.dtype, np.integer)):
        raise ValueError(f"{name}: expected a real array [..., 3], got {x.shape} {x.dtype}")
    return x.reshape(-1, 3).astype(np.float64)


def _color_u8(c: np.ndarray) -> np.ndarray:
    """Open3D's ColorToUint8: round(min(1, max(0, c)) * 255), half away from zero (not numpy's half to even); NaN -> 0.
    Exact for any double c: x - floor(x) is exact for 0 <= x <= 255."""
    x = np.fmin(1.0, np.fmax(0.0, c)) * 255.0
    f = np.floor(x)
    return (f + (x - f >= 0.5)).astype(np.uint8)


def write_point_cloud(path: str, points, colors=None) -> None:
    """`o3d.io.write_point_cloud(path, pcd)` for a coloured cloud: binary little-endian PLY with `double x y z` and, with
    colours, `uchar red green blue` (Open3D's default layout and rounding).  points [..., 3] and colors [..., 3] (in
    [0, 1]) are tensors on any device or arrays; demo.py's cloud is `pts_all[conf_sig_all > thresh]` with
    `images_all[conf_sig_all > thresh]`.  The write is host I/O."""
    p = _host_array(points, "points")
    fields = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    c = None
    if colors is not None:
        c = _host_array(colors, "colors")
        if len(c) != len(p):
            raise ValueError(f"colors: {len(c)} colours for {len(p)} points")
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    rec = np.empty(len(p), dtype=np.dtype(fields))
    rec["x"], rec["y"], rec["z"] = p[:, 0], p[:, 1], p[:, 2]
    if c is not None:
        u8 = _color_u8(c)
        rec["red"], rec["green"], rec["blue"] = u8[:, 0], u8[:, 1], u8[:, 2]
    props = "".join(f"property double {a}\n" for a in "xyz")
    if c is not None:
        props += "".join(f"property uchar {a}\n" for a in ("red", "green", "blue"))
    header = f"ply\nformat binary_little_endian 1.0\nelement vertex {len(p)}\n{props}end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())
