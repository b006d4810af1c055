"""ORACLE -- TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/ only; nothing under spann3r_b200/ touches it).

numpy restatement of the triangle mesh kernels (spann3r_b200/mesh.py, csrc/mesh.cu, csrc/mesh_math.cuh): the semantics
stated in include/spann3r_b200.h for s3r_mesh_grid_* and s3r_raster_*, vectorised.

* `grid_faces` builds app.py's face list by enumerating every candidate face in app.py's order and keeping those with
  three valid corners.
* `fragments` / `raster` form every quantity element by element in fp64 in the kernel's operation order (no `@`,
  `einsum` or FMA), so every edge value, depth and key is bit-identical to the device's; the z-buffer is
  `np.minimum.at` on the uint64 keys of the point rasteriser (oracle/render_oracle.py).

Where pyrender samples a pixel (render_dtu.py's `IntrinsicsCamera`; pyrender is not a dependency, so this derivation is
UNVERIFIED against it): pyrender's projection matrix for IntrinsicsCamera(fx, fy, cx, cy) is
    P = [[2 fx / W, 0, 1 - 2 cx / W, 0], [0, 2 fy / H, 2 cy / H - 1, 0], [0, 0, -(f + n) / (f - n), -2 f n / (f - n)],
         [0, 0, -1, 0]]
in GL's camera frame (x right, y up, looking down -z).  An OpenCV camera point (X, Y, Z) is (X, -Y, -Z) there, so
    x_ndc = 2 (fx X / Z + cx) / W - 1,   y_ndc = 1 - 2 (fy Y / Z + cy) / H,
and GL's viewport maps them to window coordinates x_w = u = fx X / Z + cx, y_w = H - v with v = fy Y / Z + cy.  GL
samples window pixel (i, j) at its centre (i + 0.5, j + 0.5), and pyrender flips the rows so that image row r is window
row j = H - 1 - r.  Image pixel (r, c) therefore samples u = c + 0.5, v = H - (H - 1 - r + 0.5) = r + 0.5: with pixel
centres at integer coordinates, as here, the principal point moves to (cx - 0.5, cy - 0.5).
"""
from __future__ import annotations

import numpy as np

from .render_oracle import EMPTY, camera_array  # noqa: F401  (camera_array: the 16 doubles of s3r_raster_triangles)


# ----------------------------------------------------------------------------------------------------------------------
# app.py's pixel-grid mesh
# ----------------------------------------------------------------------------------------------------------------------
def grid_candidates(T: int, H: int, W: int):
    """Every candidate face of a T x H x W grid in app.py's order -> (faces int64 [4 T (H-1)(W-1), 3], colour pixel
    int64 [...]): per frame the blocks [i1,i2,i3], [i3,i2,i1], [i2,i3,i4], [i4,i3,i2] over row-major quads."""
    r, c = np.meshgrid(np.arange(H - 1), np.arange(W - 1), indexing="ij")
    i1 = (r * W + c).reshape(-1)
    i2, i3 = i1 + 1, i1 + W
    i4 = i3 + 1
    blocks = [np.stack(b, 1) for b in ((i1, i2, i3), (i3, i2, i1), (i2, i3, i4), (i4, i3, i2))]
    colour = [i1, i1, i4, i4]
    faces = np.concatenate([np.concatenate(blocks) + t * H * W for t in range(T)]).reshape(-1, 3).astype(np.int64)
    cpix = np.concatenate([np.concatenate(colour) + t * H * W for t in range(T)]).astype(np.int64)
    return faces, cpix


def grid_faces(valid, images):
    """valid [T, H, W] bool, images [T, H, W, 3] -> (faces int64 [F, 3], colours [F, 3] in images' dtype): the faces
    whose three corners are valid, in app.py's order."""
    valid = np.asarray(valid, bool)
    T, H, W = valid.shape
    images = np.asarray(images)
    faces, cpix = grid_candidates(T, H, W)
    keep = valid.reshape(-1)[faces].all(1)
    return faces[keep], images.reshape(-1, 3)[cpix[keep]]


# ----------------------------------------------------------------------------------------------------------------------
# Triangle rasteriser
# ----------------------------------------------------------------------------------------------------------------------
def project_vertices(verts, cam, z_near: float):
    """fp32 vertices [N, 3] -> (u, v, qz fp64 [N], ok bool [N]) as mesh_math.cuh project_vertex."""
    p = np.asarray(verts, np.float32).reshape(-1, 3).astype(np.float64)
    cam = np.asarray(cam, np.float64)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    fx, fy, cx, cy = cam[12:16]
    with np.errstate(all="ignore"):
        q = [((cam[4 * r] * x + cam[4 * r + 1] * y) + cam[4 * r + 2] * z) + cam[4 * r + 3] for r in range(3)]
        ok = np.isfinite(q[0]) & np.isfinite(q[1]) & np.isfinite(q[2]) & (q[2] > z_near)
        u = fx * (q[0] / q[2]) + cx
        v = fy * (q[1] / q[2]) + cy
        ok &= np.isfinite(u) & np.isfinite(v)
    return u, v, q[2], ok


def _less(ax, ay, bx, by):
    return (ax < bx) | ((ax == bx) & (ay < by))


def _edge_raw(ax, ay, bx, by, px, py):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def edge_fn(ax, ay, bx, by, px, py):
    """E(a, b, p) evaluated from the (x, y)-smaller end: exactly antisymmetric in (a, b)."""
    swap = _less(bx, by, ax, ay)
    e = _edge_raw(np.where(swap, bx, ax), np.where(swap, by, ay), np.where(swap, ax, bx), np.where(swap, ay, by), px, py)
    return np.where(swap, -e, e)


def tri_area(x, y):
    """x, y [N, 3] -> signed area (twice it) of the sorted vertices, negated for an odd permutation."""
    x, y = x.copy(), y.copy()
    odd = np.zeros(len(x), bool)
    for i, j in ((0, 1), (1, 2), (0, 1)):
        s = _less(x[:, j], y[:, j], x[:, i], y[:, i])
        x[s, i], x[s, j] = x[s, j], x[s, i].copy()
        y[s, i], y[s, j] = y[s, j], y[s, i].copy()
        odd ^= s
    a = _edge_raw(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
    return np.where(odd, -a, a)


def _top_left(ax, ay, bx, by):
    dx, dy = bx - ax, by - ay
    return (dy > 0) | ((dy == 0) & (dx < 0))


def setup(verts, faces, cam, z_near, w, h):
    """Per face: (x, y, z [F, 3], area, top-left flags [F, 3], box c0, c1, r0, r1 int64, drawn bool [F])."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    inr = ((faces >= 0) & (faces < len(verts))).all(1)
    fi = np.where(inr[:, None], faces, 0)
    u, v, z, ok = project_vertices(verts, cam, z_near)
    X, Y, Z = u[fi], v[fi], z[fi]
    drawn = inr & ok[fi].all(1)
    with np.errstate(all="ignore"):
        area = tri_area(np.where(drawn[:, None], X, 0.0), np.where(drawn[:, None], Y, 0.0))
        drawn &= (area > 0) & np.isfinite(area)
        tl = np.stack([_top_left(X[:, (i + 1) % 3], Y[:, (i + 1) % 3], X[:, (i + 2) % 3], Y[:, (i + 2) % 3])
                       for i in range(3)], 1)
        c0 = np.fmax(np.ceil(X.min(1)), 0.0)
        c1 = np.fmin(np.floor(X.max(1)), w - 1.0)
        r0 = np.fmax(np.ceil(Y.min(1)), 0.0)
        r1 = np.fmin(np.floor(Y.max(1)), h - 1.0)
    drawn &= (c0 <= c1) & (r0 <= r1)
    box = [np.where(drawn, b, 0).astype(np.int64) for b in (c0, c1, r0, r1)]
    return X, Y, Z, area, tl, box, drawn


def fragments(verts, faces, cam, z_near, z_far, w, h, id0=0, chunk=1 << 22):
    """Every covered pixel centre of every drawn face -> (pix int64 [n], face id int64 [n], key uint64 [n]) with the key
    EMPTY where the depth is dropped (not finite or > z_far): the candidates of the z-buffer, before the minimum."""
    X, Y, Z, area, tl, (c0, c1, r0, r1), drawn = setup(verts, faces, cam, z_near, w, h)
    idx = np.flatnonzero(drawn)
    bw, bh = c1[idx] - c0[idx] + 1, r1[idx] - r0[idx] + 1
    n = bw * bh
    out_pix, out_face, out_key = [], [], []
    start = 0
    while start < len(idx):                       # chunks of faces whose boxes hold at most ~chunk pixels
        stop = start + max(1, int(np.searchsorted(np.cumsum(n[start:]), chunk)))
        f = np.repeat(idx[start:stop], n[start:stop])
        k = np.arange(len(f)) - np.repeat(np.cumsum(n[start:stop]) - n[start:stop], n[start:stop])
        col = c0[f] + k % bw[start:stop].repeat(n[start:stop])
        row = r0[f] + k // bw[start:stop].repeat(n[start:stop])
        px, py = col.astype(np.float64), row.astype(np.float64)
        with np.errstate(all="ignore"):
            e = [edge_fn(X[f, (i + 1) % 3], Y[f, (i + 1) % 3], X[f, (i + 2) % 3], Y[f, (i + 2) % 3], px, py)
                 for i in range(3)]
            inside = np.ones(len(f), bool)
            for i in range(3):
                inside &= (e[i] > 0) | ((e[i] == 0) & tl[f, i])
            a = area[f]
            iz = (e[0] / a / Z[f, 0] + e[1] / a / Z[f, 1]) + e[2] / a / Z[f, 2]
            depth = (1.0 / iz).astype(np.float32)
            keep = np.isfinite(depth) & (depth.astype(np.float64) <= z_far)
        bits = depth.view(np.uint32).astype(np.uint64)
        ids = f.astype(np.uint64) + np.uint64(id0)
        key = np.where(keep, (bits << np.uint64(32)) | ids, EMPTY)
        out_pix.append((row * w + col)[inside])
        out_face.append(f[inside] + id0)
        out_key.append(key[inside])
        start = stop
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
    return cat(out_pix, np.int64), cat(out_face, np.int64), cat(out_key, np.uint64)


def raster(zbuf: np.ndarray, verts, faces, cam, z_near, z_far, w, h, id0=0):
    """zbuf [h * w] uint64 <- min(zbuf, keys of the faces' fragments) in place."""
    pix, _, key = fragments(verts, faces, cam, z_near, z_far, w, h, id0)
    np.minimum.at(zbuf, pix, key)


def resolve(zbuf: np.ndarray, w: int, h: int):
    """-> depth [h, w] fp32 (0 where empty), face [h, w] int32 (-1 where empty)."""
    hit = zbuf != EMPTY
    depth = np.zeros(h * w, np.float32)
    depth[hit] = (zbuf[hit] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    face = np.full(h * w, -1, np.int32)
    face[hit] = (zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int32)
    return depth.reshape(h, w), face.reshape(h, w)


def rasterize(verts, faces, cam, w, h, z_near=0.0, z_far=np.inf):
    """One draw from an empty buffer -> (depth, face) as spann3r_b200.mesh.rasterize."""
    zbuf = np.full(h * w, EMPTY, np.uint64)
    raster(zbuf, verts, faces, cam, z_near, z_far, w, h)
    return resolve(zbuf, w, h)
