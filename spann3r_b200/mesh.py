"""Triangle meshes on the GPU: the reference app.py's reconstruction mesh (`pts3d_to_trimesh` + `cat_meshes`) with a GLB
writer, and spann3r/tools/render_dtu.py's depth maps, without trimesh, pyrender, Open3D or an OpenGL context.

* `pts3d_to_mesh` builds app.py's face list and face colours on the device (csrc/mesh.cu, through libspann3r_b200.so;
  there is no CPU fallback) in app.py's order, with one device -> host read for the face count.
* `rasterize` draws triangles with a deterministic z-buffered rasteriser on the device: fp64 projection and edge
  functions with a top-left rule, perspective-correct fp32 depth, the nearest depth winning and equal depths going to
  the smaller face id.  Back faces and degenerate triangles are culled, triangles with a vertex at depth <= z_near are
  skipped (no near-plane clipping), depths > z_far are dropped.
* `render_depth_maps`, `load_cam_mvsnet` and `render_dtu_scenes` take render_dtu.py's arguments and write its files.
* `write_glb` writes app.py's scene as glTF 2.0 binary; `read_ply_mesh` reads a triangle mesh PLY.

Differences from app.py's trimesh scene and render_dtu.py's pyrender: INTEGRATION.md, "Meshes: app.py and render_dtu".
"""
from __future__ import annotations

import ctypes as C
import json
import math
import os
import struct

import numpy as np
import torch

from . import _lib

# app.py's OPENGL axis flip
OPENGL = np.array([[1, 0, 0, 0], [0, -1, 0, 0], [0, 0, -1, 0], [0, 0, 0, 1]])


def _cuda(x, name: str, dtypes, last=None, dim=None) -> torch.Tensor:
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise ValueError(f"{name}: expected a CUDA tensor, got "
                         f"{x.device if isinstance(x, torch.Tensor) else type(x).__name__}")
    if x.dtype not in dtypes or (dim is not None and x.dim() != dim) or (last is not None and x.shape[-1] != last):
        raise ValueError(f"{name}: expected {'/'.join(str(d) for d in dtypes)} with {dim} dims and last dim {last}, got "
                         f"{tuple(x.shape)} {x.dtype}")
    return x.contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# app.py's mesh
# ----------------------------------------------------------------------------------------------------------------------
def pts3d_to_mesh(pts_all, images_all, mask=None):
    """app.py's `cat_meshes([pts3d_to_trimesh(images_all[i], pts_all[i], mask[i]) for i in range(T)])` on the device.

    pts_all, images_all: [T, H, W, 3] fp32 CUDA tensors; mask: [T, H, W] bool (app.py: `conf_sig_all > conf_thresh`)
    or None (every pixel valid).  Returns CUDA tensors (vertices [T H W, 3] fp32: every pixel, as app.py keeps them;
    faces [F, 3] int32; face colours [F, 3] fp32), the faces and colours in app.py's order.  Points and colours of
    valid pixels must be finite."""
    pts_all = _cuda(pts_all, "pts_all", (torch.float32,), 3, 4)
    images_all = _cuda(images_all, "images_all", (torch.float32,), 3, 4)
    if images_all.shape != pts_all.shape or images_all.device != pts_all.device or pts_all.numel() == 0:
        raise ValueError(f"images_all {tuple(images_all.shape)} must match the non-empty pts_all {tuple(pts_all.shape)} "
                         f"on {pts_all.device}")
    T, H, W, _ = pts_all.shape
    if T * H * W >= 2 ** 31:
        raise ValueError(f"pts_all: T * H * W must be below 2^31 (int32 faces), got {(T, H, W)}")
    if mask is None:
        mask = torch.ones((T, H, W), dtype=torch.bool, device=pts_all.device)
    if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or tuple(mask.shape) != (T, H, W) \
            or mask.device != pts_all.device:
        raise ValueError(f"mask: expected a bool tensor {(T, H, W)} on {pts_all.device}, got "
                         f"{tuple(mask.shape) if isinstance(mask, torch.Tensor) else type(mask).__name__}")
    mask = mask.contiguous()
    finite = torch.isfinite(pts_all).all(-1) & torch.isfinite(images_all).all(-1)
    if not bool((finite | ~mask).all()):
        raise ValueError("pts_all / images_all: non-finite values at valid pixels")
    _lib.require_device()
    dev = pts_all.device
    valid = mask.view(torch.uint8)
    ws_bytes = int(_lib.lib().s3r_mesh_grid_workspace_bytes(T, H, W))
    ws = torch.empty(ws_bytes // 8, dtype=torch.int64, device=dev)
    n = C.c_int64(0)
    _lib.call("s3r_mesh_grid_count", dev, _lib.ptr(valid), T, H, W, _lib.ptr(ws), ws_bytes, C.byref(n))
    faces = torch.empty((n.value, 3), dtype=torch.int32, device=dev)
    colors = torch.empty((n.value, 3), dtype=torch.float32, device=dev)
    if n.value:
        _lib.call("s3r_mesh_grid_faces", dev, _lib.ptr(valid), _lib.ptr(images_all), T, H, W, _lib.ptr(ws), ws_bytes,
                  _lib.ptr(faces), _lib.ptr(colors))
    return pts_all.reshape(-1, 3), faces, colors


def app_scene_matrix() -> np.ndarray:
    """app.py's `np.linalg.inv(OPENGL @ rot)` with rot a 180 degree turn about y, computed as app.py computes it."""
    from scipy.spatial.transform import Rotation
    rot = np.eye(4)
    rot[:3, :3] = Rotation.from_euler('y', np.deg2rad(180)).as_matrix()
    return np.linalg.inv(OPENGL @ rot)


def _host(x, name):
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    return np.asarray(x)


def _rgba_u8(c: np.ndarray) -> np.ndarray:
    """float colours in [0, 1] -> uint8 by floor(min(1, max(0, c)) * 255 + 0.5) (the renderers' rounding); uint8 kept;
    alpha 255 when there are three channels."""
    if c.dtype != np.uint8:
        c = np.floor(np.fmin(1.0, np.fmax(0.0, c.astype(np.float64))) * 255.0 + 0.5).astype(np.uint8)
    if c.shape[1] == 3:
        c = np.concatenate([c, np.full((len(c), 1), 255, np.uint8)], 1)
    return np.ascontiguousarray(c)


def write_glb(path: str, vertices, faces=None, colors=None, matrix=None) -> None:
    """A glTF 2.0 binary file with one mesh on one node, as app.py's `scene.export(...glb)` writes the reconstruction.

    vertices [N, 3] (N >= 1, finite) become float32 POSITION with min / max; colors [N, 3] or [N, 4] (floats in [0, 1],
    or uint8) become normalized uint8 RGBA COLOR_0, one colour per vertex (for app.py's mesh: the vertex's own pixel,
    `images_all.reshape(-1, 3)`; trimesh's face -> vertex colour averaging is not reproduced); faces [F, 3] become
    UNSIGNED_INT indices of a TRIANGLES primitive, and faces=None writes a POINTS primitive (app.py's
    `as_pointcloud=True`).  matrix: the node's 4x4 transform (app.py: `app_scene_matrix()`), or None.  Tensors on any
    device or arrays; the write is host I/O."""
    v = _host(vertices, "vertices").reshape(-1, 3).astype(np.float32)
    if len(v) == 0 or not np.isfinite(v).all():
        raise ValueError(f"vertices: expected a non-empty finite [N, 3] array, got {v.shape}")
    chunks, views, accessors = [], [], []

    def add(arr: np.ndarray, target: int, acc: dict) -> int:
        offset = sum(len(c) for c in chunks)
        data = arr.tobytes()
        chunks.append(data + b"\0" * (-len(data) % 4))
        views.append({"buffer": 0, "byteOffset": offset, "byteLength": len(data), "target": target})
        accessors.append({"bufferView": len(views) - 1, **acc})
        return len(accessors) - 1

    attributes = {"POSITION": add(v, 34962, {"componentType": 5126, "count": len(v), "type": "VEC3",
                                             "min": [float(x) for x in v.min(0)], "max": [float(x) for x in v.max(0)]})}
    if colors is not None:
        c = _host(colors, "colors")
        if c.ndim != 2 or c.shape[0] != len(v) or c.shape[1] not in (3, 4) or \
                not (c.dtype == np.uint8 or np.issubdtype(c.dtype, np.floating)) or not np.isfinite(c).all():
            raise ValueError(f"colors: expected finite [{len(v)}, 3 or 4] floats or uint8, got {c.shape} {c.dtype}")
        attributes["COLOR_0"] = add(_rgba_u8(c), 34962, {"componentType": 5121, "normalized": True, "count": len(v),
                                                         "type": "VEC4"})
    primitive = {"attributes": attributes, "mode": 0}
    if faces is not None:
        f = _host(faces, "faces")
        if f.ndim != 2 or f.shape[1] != 3 or not np.issubdtype(f.dtype, np.integer) or \
                (f.size and (f.min() < 0 or f.max() >= len(v))):
            raise ValueError(f"faces: expected integer [F, 3] indices into {len(v)} vertices, got {f.shape} {f.dtype}")
        primitive["mode"] = 4
        if len(f):
            primitive["indices"] = add(f.astype(np.uint32).reshape(-1), 34963, {"componentType": 5125,
                                                                                 "count": f.size, "type": "SCALAR"})
    node = {"mesh": 0}
    if matrix is not None:
        m = np.asarray(matrix, np.float64)
        if m.shape != (4, 4) or not np.isfinite(m).all():
            raise ValueError(f"matrix: expected a finite 4x4 transform, got {m.shape}")
        node["matrix"] = [float(x) for x in m.T.reshape(-1)]      # glTF matrices are column-major
    binary = b"".join(chunks)
    doc = {"asset": {"version": "2.0", "generator": "spann3r_b200"}, "scene": 0, "scenes": [{"nodes": [0]}],
           "nodes": [node], "meshes": [{"primitives": [primitive]}], "accessors": accessors, "bufferViews": views,
           "buffers": [{"byteLength": len(binary)}]}
    js = json.dumps(doc, separators=(",", ":")).encode("utf-8")
    js += b" " * (-len(js) % 4)
    total = 12 + 8 + len(js) + 8 + len(binary)
    with open(path, "wb") as fh:
        fh.write(struct.pack("<4sII", b"glTF", 2, total))
        fh.write(struct.pack("<I4s", len(js), b"JSON") + js)
        fh.write(struct.pack("<I4s", len(binary), b"BIN\0") + binary)


# ----------------------------------------------------------------------------------------------------------------------
# Rasteriser
# ----------------------------------------------------------------------------------------------------------------------
def _camera16(camera) -> np.ndarray:
    """camera: 16 doubles ([R | t] 3x4 row-major world -> camera, fx, fy, cx, cy) or (extrinsic 4x4 / 3x4, K 3x3)."""
    if isinstance(camera, (tuple, list)) and len(camera) == 2:
        E = np.asarray(camera[0], np.float64)
        K = np.asarray(camera[1], np.float64)
        if E.shape not in ((4, 4), (3, 4)) or K.shape != (3, 3):
            raise ValueError(f"camera: expected (extrinsic 4x4 or 3x4, K 3x3), got {E.shape}, {K.shape}")
        if K[0, 1] != 0 or K[1, 0] != 0 or K[2].tolist() != [0.0, 0.0, 1.0]:
            raise ValueError(f"camera: K must be [[fx, 0, cx], [0, fy, cy], [0, 0, 1]], got {K.tolist()}")
        cam = np.concatenate([E[:3, :4].reshape(-1), [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]])
    else:
        cam = np.asarray(camera, np.float64).reshape(-1)
    if cam.shape != (16,) or not np.isfinite(cam).all():
        raise ValueError(f"camera: expected 16 finite values, got shape {cam.shape}")
    return np.ascontiguousarray(cam)


def _mesh_input(vertices, faces):
    v = _cuda(vertices, "vertices", (torch.float32,), 3, 2)
    f = _cuda(faces, "faces", (torch.int32, torch.int64), 3, 2)
    if f.device != v.device:
        raise ValueError(f"faces on {f.device} must be on the vertices' device {v.device}")
    if len(v) >= 2 ** 31 or len(f) >= 2 ** 31:
        raise ValueError(f"at most 2^31 - 1 vertices and faces, got {len(v)}, {len(f)}")
    if not bool(torch.isfinite(v).all()):
        raise ValueError("vertices: non-finite values")
    if len(f) and (int(f.min()) < 0 or int(f.max()) >= len(v)):
        raise ValueError(f"faces: indices must lie in [0, {len(v)})")
    return v, f.to(torch.int32).contiguous()


def _size(w, h):
    w, h = int(w), int(h)
    if not (w >= 1 and h >= 1 and w * h < 2 ** 31):
        raise ValueError(f"image size {w}x{h} out of range")
    return w, h


def _planes(z_near, z_far):
    z_near, z_far = float(z_near), float(z_far)
    if not (math.isfinite(z_near) and z_near >= 0 and z_far > z_near):
        raise ValueError(f"need a finite z_near >= 0 and z_far > z_near (inf allowed), got {z_near}, {z_far}")
    return z_near, z_far


def _draw(keys, v, f, cam, z_near, z_far, w, h, id0=0):
    if len(f) == 0:
        return
    _lib.call("s3r_raster_triangles", keys, _lib.ptr(v), len(v), _lib.ptr(f), len(f), id0, C.c_void_p(cam.ctypes.data),
              z_near, z_far, w, h, _lib.ptr(keys))


def _resolve(keys, w, h, depth, face):
    _lib.call("s3r_raster_resolve", keys, _lib.ptr(keys), w, h, _lib.ptr(depth), _lib.ptr(face))


def rasterize(vertices, faces, camera, w, h, z_near=0.0, z_far=math.inf):
    """Draws the triangles faces [F, 3] (int32 / int64 indices) of vertices [N, 3] fp32 (CUDA tensors) into a w x h
    image -> (depth [h, w] fp32, 0 where empty; face [h, w] int32, the face index drawn, -1 where empty).

    camera: 16 doubles ([R | t] 3x4 row-major world -> camera, fx, fy, cx, cy) or (extrinsic, K); pixel centres at
    integer (u, v) = (col, row).  Front faces are counter-clockwise on the image; back faces and degenerate triangles
    are culled, triangles with a vertex at camera depth <= z_near are skipped, depths > z_far are dropped."""
    v, f = _mesh_input(vertices, faces)
    cam = _camera16(camera)
    w, h = _size(w, h)
    z_near, z_far = _planes(z_near, z_far)
    _lib.require_device()
    dev = v.device
    keys = torch.empty(int(_lib.lib().s3r_render_workspace_bytes(w, h)) // 8, dtype=torch.int64, device=dev)
    depth = torch.empty((h, w), dtype=torch.float32, device=dev)
    face = torch.empty((h, w), dtype=torch.int32, device=dev)
    _lib.call("s3r_render_clear", keys, _lib.ptr(keys), w, h)
    _draw(keys, v, f, cam, z_near, z_far, w, h)
    _resolve(keys, w, h, depth, face)
    return depth, face


# ----------------------------------------------------------------------------------------------------------------------
# render_dtu.py
# ----------------------------------------------------------------------------------------------------------------------
def pyrender_camera(pose, K) -> np.ndarray:
    """A c2w pose in the OpenGL convention (render_dtu.py's, the columns 1 and 2 of an OpenCV c2w negated) and
    pyrender's IntrinsicsCamera intrinsics -> the 16 camera values of `rasterize`.  The axis flip is undone, and the
    principal point moves by -0.5: pyrender samples pixel (r, c) at (u, v) = (c + 0.5, r + 0.5) (derived in
    oracle/mesh_oracle.py's docstring; not checked against pyrender, which is not a dependency)."""
    P = np.array(pose, dtype=np.float64)
    K = np.asarray(K, dtype=np.float64)
    if P.shape != (4, 4) or not np.isfinite(P).all() or K.shape[0] < 3 or K.shape[1] < 3:
        raise ValueError(f"pose: expected a finite 4x4 c2w and K at least 3x3, got {P.shape}, {K.shape}")
    P[:, 1:3] *= -1.0
    E = np.linalg.inv(P)
    return _camera16(np.concatenate([E[:3, :4].reshape(-1), [K[0, 0], K[1, 1], K[0, 2] - 0.5, K[1, 2] - 0.5]]))


def _mesh_arrays(mesh):
    if isinstance(mesh, (tuple, list)) and len(mesh) == 2:
        verts, faces = mesh
    else:
        try:
            verts, faces = mesh.vertices, mesh.faces
        except AttributeError:
            raise ValueError("mesh: expected (vertices, faces) or an object with .vertices and .faces")
    return verts, faces


def _to_device_mesh(mesh, device):
    verts, faces = _mesh_arrays(mesh)
    v = torch.as_tensor(np.asarray(verts.cpu() if isinstance(verts, torch.Tensor) else verts, np.float32)).to(device)
    f = faces.to(device) if isinstance(faces, torch.Tensor) else torch.as_tensor(np.asarray(faces, np.int64)).to(device)
    return _mesh_input(v, f)


def _depth_maps(v, f, cams, H, W, near, far):
    """[len(cams), H, W] fp32 CUDA: one draw per camera against the same device mesh."""
    dev = v.device
    keys = torch.empty(int(_lib.lib().s3r_render_workspace_bytes(W, H)) // 8, dtype=torch.int64, device=dev)
    depth = torch.empty((len(cams), H, W), dtype=torch.float32, device=dev)
    face = torch.empty((H, W), dtype=torch.int32, device=dev)
    for i, cam in enumerate(cams):
        _lib.call("s3r_render_clear", keys, _lib.ptr(keys), W, H)
        _draw(keys, v, f, cam, near, far, W, H)
        _resolve(keys, W, H, depth[i], face)
    return depth


def render_depth_maps(mesh, poses, K, H, W, near=0.01, far=5.0, device="cuda"):
    """render_dtu.py's `render_depth_maps` with its arguments: mesh ((vertices, faces) or an object with .vertices and
    .faces), poses (c2w, OpenGL convention), K (pyrender IntrinsicsCamera's fx, fy, cx, cy from K[0, 0], K[1, 1],
    K[0, 2], K[1, 2]), image H x W, near / far clip.  The mesh goes to the device once and every pose is drawn against
    it.  Returns a list of fp32 [H, W] numpy depth maps, 0 where nothing was drawn, as pyrender's."""
    W, H = _size(W, H)
    near, far = _planes(near, far)
    cams = [pyrender_camera(p, K) for p in poses]
    _lib.require_device()
    v, f = _to_device_mesh(mesh, device)
    return list(_depth_maps(v, f, cams, H, W, near, far).cpu().numpy())


def load_cam_mvsnet(file, interval_scale=1):
    """render_dtu.py's `load_cam_mvsnet`: an MVSNet camera file (an open text file or a path) -> (intrinsic 4x4, extrinsic
    4x4), float32.  Row 3 of the intrinsic is the depth range (min, interval * interval_scale, count, max): with 29 words
    the count is 192 and max = min + interval * count, with 30 words the count is read and max computed, with 31 words
    both are read, with any other count (at least 27 words) the row is zero."""
    text = open(file).read() if isinstance(file, (str, os.PathLike)) else file.read()
    words = text.split()
    if len(words) < 27:
        raise ValueError(f"camera file: expected at least 27 words, got {len(words)}")
    extrinsic = np.array([float(x) for x in words[1:17]], np.float64).reshape(4, 4)
    intrinsic = np.zeros((4, 4), np.float64)
    intrinsic[:3, :3] = np.array([float(x) for x in words[18:27]], np.float64).reshape(3, 3)
    n = len(words)
    if n in (29, 30, 31):
        lo, step = float(words[27]), float(words[28]) * interval_scale
        count = 192.0 if n == 29 else float(words[29])
        hi = float(words[30]) if n == 31 else lo + step * count
        intrinsic[3] = [lo, step, count, hi]
    return intrinsic.astype(np.float32), extrinsic.astype(np.float32)


def render_dtu_scenes(path_to_scan, method="furu", device="cuda"):
    """render_dtu.py's `render_dtu_scenes`: renders the scan's mesh (`{method}{scan:03d}_l3_surf_11_trim_8.ply`, or
    `{scan:03d}_pcd.ply` for method=None) from every camera in cams/ (one per image in images/, sorted) at the first
    image's size, near 0.01 and far 5000, and writes depths[_method]/<image name with .jpg -> .npy> as float32."""
    import cv2
    cams_dir = os.path.join(path_to_scan, "cams")
    images_dir = os.path.join(path_to_scan, "images")
    scan_id = int("".join(filter(str.isdigit, os.path.basename(os.path.normpath(path_to_scan)))))
    if method is not None:
        depth_dir = os.path.join(path_to_scan, f"depths_{method}")
        mesh_path = os.path.join(path_to_scan, f"{method}{scan_id:03d}_l3_surf_11_trim_8.ply")
    else:
        depth_dir = os.path.join(path_to_scan, "depths")
        mesh_path = os.path.join(path_to_scan, f"{scan_id:03d}_pcd.ply")
    os.makedirs(depth_dir, exist_ok=True)
    frames = sorted(os.listdir(images_dir))
    img = cv2.imread(os.path.join(images_dir, frames[0]))
    if img is None:
        raise ValueError(f"cannot read {os.path.join(images_dir, frames[0])}")
    H, W = img.shape[:2]
    cams = []
    for frame in frames:
        intrinsic, extrinsic = load_cam_mvsnet(os.path.join(cams_dir, frame.replace(".jpg", "_cam.txt")))
        pose = np.linalg.inv(extrinsic)
        pose[:, 1:3] *= -1.0
        cams.append(pyrender_camera(pose, intrinsic))
    _lib.require_device()
    v, f = _to_device_mesh(read_ply_mesh(mesh_path), device)
    depth = _depth_maps(v, f, cams, H, W, 0.01, 5000.0).cpu().numpy()
    for frame, d in zip(frames, depth):
        np.save(os.path.join(depth_dir, frame.replace(".jpg", ".npy")), d)


# ----------------------------------------------------------------------------------------------------------------------
# PLY meshes
# ----------------------------------------------------------------------------------------------------------------------
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _ply_type(t, path):
    if t not in _PLY_TYPES:
        raise ValueError(f"{path}: unknown PLY type {t!r}")
    return _PLY_TYPES[t]


def _ply_header(path: str):
    """-> (file bytes, format, [(element name, count, [property tuples])], offset of the body).  ASCII and binary
    little-endian only; anything else in the header raises ValueError."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.find(b"end_header")
    if not data.startswith(b"ply") or end < 0:
        raise ValueError(f"{path}: not a PLY file")
    body_at = data.index(b"\n", end) + 1 if b"\n" in data[end:] else len(data)
    lines = data[:end].decode("ascii", "replace").splitlines()[1:]
    fmt, elements = None, []
    for line in lines:
        tok = line.split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1] if len(tok) == 3 and tok[2] == "1.0" else None
            if fmt not in ("ascii", "binary_little_endian"):
                raise ValueError(f"{path}: unsupported format {' '.join(tok[1:])!r}")
        elif tok[0] == "element" and len(tok) == 3:
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property" and elements and len(tok) in (3, 5):
            elements[-1][2].append(tuple(tok[1:]))
        else:
            raise ValueError(f"{path}: malformed header line {line!r}")
    if fmt is None:
        raise ValueError(f"{path}: no format line")
    return data, fmt, elements, body_at


def read_ply_mesh(path: str):
    """A triangle mesh PLY (ASCII or binary little-endian) -> (vertices [N, 3] fp32, faces [F, 3] int64).

    The vertex element needs float or double x, y, z; its other scalar properties are skipped by their declared type.
    The optional face element holds one list property `vertex_indices` (or `vertex_index`) of three indices per face.
    Anything else (another format, element or face property, a list on the vertex, a non-triangle, an index out of
    range, a truncated body) raises ValueError."""
    data, fmt, elements, body_at = _ply_header(path)
    names = [e[0] for e in elements]
    if "vertex" not in names or len(set(names)) != len(names) or not set(names) <= {"vertex", "face"}:
        raise ValueError(f"{path}: expected a vertex element and at most a face element, got {names}")
    dtypes = {}
    for name, count, props in elements:
        if count < 0:
            raise ValueError(f"{path}: negative {name} count")
        if name == "vertex":
            if any(p[0] == "list" for p in props):
                raise ValueError(f"{path}: list properties on vertices are not supported")
            pn = [p[1] for p in props]
            if len(set(pn)) != len(pn) or not {"x", "y", "z"} <= set(pn) or \
                    any(_ply_type(p[0], path) not in ("f4", "f8") for p in props if p[1] in "xyz"):
                raise ValueError(f"{path}: vertices need float or double x, y, z")
            dtypes[name] = np.dtype([(p[1], "<" + _ply_type(p[0], path)) for p in props])
        else:
            if len(props) != 1 or props[0][0] != "list" or props[0][3] not in ("vertex_indices", "vertex_index"):
                raise ValueError(f"{path}: the face element must hold exactly one vertex_indices list")
            ct, it = _ply_type(props[0][1], path), _ply_type(props[0][2], path)
            if ct[0] == "f" or it[0] == "f":
                raise ValueError(f"{path}: face indices must be integers")
            dtypes[name] = np.dtype([("n", "<" + ct), ("i", "<" + it, 3)])
    out = {"vertex": None, "face": np.zeros((0, 3), np.int64)}
    if fmt == "binary_little_endian":
        at = body_at
        for name, count, _ in elements:
            dt = dtypes[name]
            if at + count * dt.itemsize > len(data):
                raise ValueError(f"{path}: truncated {name} data")
            rec = np.frombuffer(data, dt, count, at)
            at += count * dt.itemsize
            if name == "face":
                if (rec["n"] != 3).any():
                    raise ValueError(f"{path}: only triangles are supported")
                out["face"] = rec["i"].astype(np.int64)
            else:
                out["vertex"] = np.stack([rec[a].astype(np.float64) for a in "xyz"], 1)
    else:
        rows = data[body_at:].decode("ascii", "replace").splitlines()
        rows = [r.split() for r in rows if r.strip()]
        at = 0
        for name, count, props in elements:
            chunk = rows[at:at + count]
            at += count
            if len(chunk) < count:
                raise ValueError(f"{path}: truncated {name} data")
            try:
                if name == "face":
                    if any(len(r) != 4 or r[0] != "3" for r in chunk):
                        raise ValueError(f"{path}: only triangles are supported")
                    out["face"] = np.array([[int(x) for x in r[1:]] for r in chunk], np.int64).reshape(-1, 3)
                else:
                    if any(len(r) != len(props) for r in chunk):
                        raise ValueError(f"{path}: a vertex row does not have {len(props)} values")
                    cols = [i for a in "xyz" for i, p in enumerate(props) if p[1] == a]
                    out["vertex"] = np.array([[float(r[i]) for i in cols] for r in chunk], np.float64).reshape(-1, 3)
            except (TypeError, ValueError) as ex:
                raise ValueError(f"{path}: malformed {name} data: {ex}")
    v, f = out["vertex"], out["face"]
    if f.size and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError(f"{path}: face indices out of range")
    return v.astype(np.float32), f


def read_point_cloud(path: str):
    """An oriented point cloud PLY (ASCII or binary little-endian), as render_dtu.py's `o3d.io.read_point_cloud` reads
    DTU's stl*_total.ply -> (points [N, 3] fp64, normals [N, 3] fp64), numpy.

    The vertex element comes first and has float or double x, y, z, nx, ny, nz; its other scalar properties are skipped
    by their declared type, and elements after it are not read.  A cloud without normals raises ValueError (Open3D's
    Poisson reconstruction refuses one), as do a list property on the vertex, another format and a truncated body."""
    data, fmt, elements, body_at = _ply_header(path)
    if not elements or elements[0][0] != "vertex" or elements[0][1] < 0:
        raise ValueError(f"{path}: expected the vertex element first, got {[e[0] for e in elements]}")
    _, count, props = elements[0]
    if any(p[0] == "list" for p in props):
        raise ValueError(f"{path}: list properties on vertices are not supported")
    names = [p[1] for p in props]
    if len(set(names)) != len(names) or not {"x", "y", "z"} <= set(names) or \
            any(_ply_type(p[0], path) not in ("f4", "f8") for p in props if p[1] in ("x", "y", "z", "nx", "ny", "nz")):
        raise ValueError(f"{path}: vertices need float or double x, y, z")
    if not {"nx", "ny", "nz"} <= set(names):
        raise ValueError(f"{path}: the point cloud has no normals (nx, ny, nz); Poisson reconstruction needs them")
    cols = ("x", "y", "z", "nx", "ny", "nz")
    if fmt == "binary_little_endian":
        dt = np.dtype([(p[1], "<" + _ply_type(p[0], path)) for p in props])
        if body_at + count * dt.itemsize > len(data):
            raise ValueError(f"{path}: truncated vertex data")
        rec = np.frombuffer(data, dt, count, body_at)
        out = np.stack([rec[a].astype(np.float64) for a in cols], 1) if count else np.zeros((0, 6))
    else:
        rows = [r.split() for r in data[body_at:].decode("ascii", "replace").splitlines() if r.strip()][:count]
        if len(rows) < count or any(len(r) != len(props) for r in rows):
            raise ValueError(f"{path}: truncated or malformed vertex data")
        idx = [names.index(a) for a in cols]
        try:
            out = np.array([[float(r[i]) for i in idx] for r in rows], np.float64).reshape(-1, 6)
        except ValueError as ex:
            raise ValueError(f"{path}: malformed vertex data: {ex}")
    return np.ascontiguousarray(out[:, :3]), np.ascontiguousarray(out[:, 3:])


def write_ply_mesh(path: str, vertices, faces) -> None:
    """Binary little-endian PLY of a triangle mesh: `double x y z` (the layout vis.write_point_cloud writes) and faces
    as `list uchar int vertex_indices`.  read_ply_mesh reads it back exactly.  Tensors on any device or arrays."""
    v = np.ascontiguousarray(_host(vertices, "vertices"), np.float64).reshape(-1, 3)
    f = _host(faces, "faces").reshape(-1, 3)
    if not np.issubdtype(f.dtype, np.integer) or (f.size and (f.min() < 0 or f.max() >= len(v))) or \
            len(v) >= 2 ** 31 or not np.isfinite(v).all():
        raise ValueError(f"write_ply_mesh: expected finite vertices and integer faces indexing them, got "
                         f"{v.shape}, {f.shape} {f.dtype}")
    rec = np.empty(len(f), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    rec["n"] = 3
    rec["i"] = f
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\n"
              + "".join(f"property double {a}\n" for a in "xyz")
              + f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(v.astype("<f8").tobytes())
        fh.write(rec.tobytes())


# ----------------------------------------------------------------------------------------------------------------------
# Screened Poisson reconstruction (render_dtu.py's get_mesh_from_ply)
# ----------------------------------------------------------------------------------------------------------------------
POISSON_TOL = 1e-8          # relative residual |b - A chi| / |b| at which the solve stops
POISSON_MAX_ITER = 500      # conjugate-gradient iterations before the solve raises


class _Poisson:
    """The device workspace of one reconstruction after setup and solve: the screening blocks, b, chi, the iso value
    and the density grid stay on the device for extraction (and for the tests)."""

    def __init__(self, points, normals, depth, scale):
        if isinstance(depth, bool) or not isinstance(depth, (int, np.integer)) or not 1 <= int(depth) <= 10:
            raise ValueError(f"depth: expected an int in 1..10, got {depth!r}")
        scale = float(scale)
        if not (math.isfinite(scale) and scale >= 1.0):
            raise ValueError(f"scale: expected a finite value >= 1, got {scale}")
        p = _cuda(points, "points", (torch.float32, torch.float64), 3, 2)
        n = _cuda(normals, "normals", (torch.float32, torch.float64), 3, 2)
        if n.shape != p.shape or n.device != p.device:
            raise ValueError(f"normals {tuple(n.shape)} on {n.device} must match points {tuple(p.shape)} on {p.device}")
        if p.dtype != n.dtype:
            p, n = p.double(), n.double()
        N = len(p)
        if N < 4 or N >= 2 ** 31:
            raise ValueError(f"points: expected 4 <= N < 2^31 samples, got {N}")
        if not bool(torch.isfinite(p).all()) or not bool(torch.isfinite(n).all()):
            raise ValueError("points / normals: non-finite values")
        if float((p.amax(0) - p.amin(0)).max()) == 0.0:
            raise ValueError("points: the bounding box has zero extent")
        _lib.require_device()
        self.n, self.depth, self.device = N, int(depth), p.device
        self.ws_bytes = int(_lib.lib().s3r_poisson_workspace_bytes(N, self.depth))
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=self.device)
        info = np.zeros(8, np.float64)
        out = np.zeros(3, np.float64)
        _lib.call("s3r_poisson_setup", self.device, _lib.ptr(p), _lib.ptr(n), int(p.dtype == torch.float64), N, self.depth,
                  scale, _lib.ptr(self.ws), self.ws_bytes, C.c_void_p(info.ctypes.data))
        _lib.call("s3r_poisson_solve", self.device, N, self.depth, POISSON_TOL, POISSON_MAX_ITER, _lib.ptr(self.ws),
                  self.ws_bytes, C.c_void_p(out.ctypes.data))
        self.origin, self.L, self.h = info[:3].copy(), float(info[3]), float(info[4])
        self.a, self.beta, self.occupied = float(info[5]), float(info[6]), int(info[7])
        self.iterations, self.residual, self.iso = int(out[0]), float(out[1]), float(out[2])

    def view(self, which: int, dtype, count: int) -> torch.Tensor:
        """One array of the workspace (s3r_poisson_offset's `which`), as a tensor sharing its memory."""
        off = int(_lib.lib().s3r_poisson_offset(self.n, self.depth, which))
        nbytes = count * torch.empty((), dtype=dtype).element_size()
        return self.ws[off:off + nbytes].view(dtype)

    def extract(self):
        sizes = np.zeros(2, np.int64)
        _lib.call("s3r_poisson_extract_count", self.device, self.n, self.depth, _lib.ptr(self.ws), self.ws_bytes,
                  C.c_void_p(sizes.ctypes.data))
        nv, nf = int(sizes[0]), int(sizes[1])
        v = torch.empty((nv, 3), dtype=torch.float32, device=self.device)
        f = torch.empty((nf, 3), dtype=torch.int64, device=self.device)
        d = torch.empty(nv, dtype=torch.float64, device=self.device)
        _lib.call("s3r_poisson_extract", self.device, self.n, self.depth, _lib.ptr(self.ws), self.ws_bytes, _lib.ptr(v),
                  _lib.ptr(f), _lib.ptr(d))
        return v, f, d


def create_from_point_cloud_poisson(points, normals, depth=8, scale=1.1):
    """Open3D's `TriangleMesh.create_from_point_cloud_poisson(pcd, depth, scale=scale)` on the device, as a dense-grid
    screened Poisson reconstruction (the problem: csrc/poisson_math.cuh; differences from Open3D: INTEGRATION.md).

    points, normals: CUDA [N, 3] fp32 or fp64 (N >= 4, finite, a bounding box of non-zero extent); depth: 1..10 (a
    (2^depth + 1)^3 grid); scale >= 1: the cube's side over the bounding box's largest extent.  Returns CUDA tensors
    (vertices [V, 3] fp32, faces [F, 3] int64 wound outward for outward normals, densities [V] fp64: samples per unit
    volume on the depth max(depth - 2, 1) grid, interpolated at each vertex).  Bitwise reproducible."""
    return _Poisson(points, normals, depth, scale).extract()


def remove_vertices_by_mask(vertices, faces, mask):
    """Open3D's `TriangleMesh.remove_vertices_by_mask` on the device: drops the vertices where mask [V] (bool) is true and
    every face that uses one, renumbering the survivors in their order; faces keep theirs.  vertices [V, 3] fp32,
    faces [F, 3] int64 CUDA tensors -> (vertices, faces)."""
    v = _cuda(vertices, "vertices", (torch.float32,), 3, 2)
    f = _cuda(faces, "faces", (torch.int64,), 3, 2)
    if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool or tuple(mask.shape) != (len(v),) or \
            mask.device != v.device or f.device != v.device:
        raise ValueError(f"mask: expected a bool tensor ({len(v)},) on {v.device}")
    if len(v) == 0 or len(v) >= 2 ** 31 or len(f) >= 2 ** 31:
        raise ValueError(f"expected 1 <= V < 2^31 vertices and F < 2^31 faces, got {len(v)}, {len(f)}")
    if len(f) and (int(f.min()) < 0 or int(f.max()) >= len(v)):
        raise ValueError(f"faces: indices must lie in [0, {len(v)})")
    _lib.require_device()
    m = mask.contiguous().view(torch.uint8)
    ws_bytes = int(_lib.lib().s3r_mesh_compact_workspace_bytes(len(v), len(f)))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=v.device)
    sizes = np.zeros(2, np.int64)
    _lib.call("s3r_mesh_compact_count", v, _lib.ptr(m), _lib.ptr(f), len(v), len(f), _lib.ptr(ws), ws_bytes,
              C.c_void_p(sizes.ctypes.data))
    ov = torch.empty((int(sizes[0]), 3), dtype=torch.float32, device=v.device)
    of = torch.empty((int(sizes[1]), 3), dtype=torch.int64, device=v.device)
    _lib.call("s3r_mesh_compact", v, _lib.ptr(v), _lib.ptr(f), len(v), len(f), _lib.ptr(ws), ws_bytes, _lib.ptr(ov),
              _lib.ptr(of))
    return ov, of


def quantile(x, q) -> torch.Tensor:
    """np.quantile(x, q) (method 'linear') of a non-negative fp64 CUDA vector, bit for bit, by two exact order
    statistics on the device -> a 1-element fp64 CUDA tensor."""
    x = _cuda(x, "x", (torch.float64,), None, 1)
    q = float(q)
    if not (0.0 <= q <= 1.0) or len(x) == 0 or len(x) >= 2 ** 31:
        raise ValueError(f"quantile: need 0 <= q <= 1 and 1 <= len(x) < 2^31, got {q}, {len(x)}")
    _lib.require_device()
    ws = torch.empty(int(_lib.lib().s3r_pcl_stats_workspace_bytes()), dtype=torch.uint8, device=x.device)
    out = torch.empty(1, dtype=torch.float64, device=x.device)
    _lib.call("s3r_pcl_quantile", x, _lib.ptr(x), len(x), q, _lib.ptr(ws), _lib.ptr(out))
    return out


def get_mesh_from_ply(path_to_scan, depth=9, density_thresh=0.1, device="cuda"):
    """render_dtu.py's `get_mesh_from_ply`: reads the scan's `stl{scan:03d}_total.ply`, reconstructs it at `depth`,
    removes the vertices whose density is below `np.quantile(densities, density_thresh)` and writes
    `{scan:03d}_pcd.ply`, the mesh `render_dtu_scenes(path_to_scan, method=None)` renders.  Returns (vertices, faces)
    of the trimmed mesh as CUDA tensors."""
    scan_id = int("".join(filter(str.isdigit, os.path.basename(path_to_scan))))
    pts, nrm = read_point_cloud(os.path.join(path_to_scan, f"stl{scan_id:03d}_total.ply"))
    _lib.require_device()
    v, f, dens = create_from_point_cloud_poisson(torch.from_numpy(pts).to(device), torch.from_numpy(nrm).to(device),
                                                 depth=depth)
    if len(v):
        v, f = remove_vertices_by_mask(v, f, dens < quantile(dens, density_thresh))
    write_ply_mesh(os.path.join(path_to_scan, f"{scan_id:03d}_pcd.ply"), v, f)
    return v, f
