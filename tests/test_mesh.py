"""Triangle meshes (spann3r_b200.mesh, vis.render_mesh_frames): app.py's pixel-grid mesh and GLB export, and the
z-buffered triangle rasteriser behind render_dtu.py's depth maps.

Checkers:
  * tests/golden/mesh.npz / mesh.json, made by tools/make_golden_mesh.py from the reference's own `pts3d_to_trimesh`,
    `cat_meshes` and `load_cam_mvsnet`;
  * oracle/mesh_oracle.py (numpy, the kernels' fp64 operation order) on hand-built scenes, and bit for bit against the
    host-compiled device math (tests/native/mesh_host_check.cpp) and against every GPU result;
  * analytic depths of planes and boxes; a test-side glTF 2.0 binary parser.
trimesh, pyrender and Open3D are not run.
"""
import ctypes as C
import io
import json
import math
import os
import struct
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import mesh_oracle as mo
from spann3r_b200 import mesh, vis

HERE = os.path.dirname(os.path.abspath(__file__))
EMPTY = mo.EMPTY


def _golden():
    z = np.load(os.path.join(GOLDEN, "mesh.npz"))
    meta = json.load(open(os.path.join(GOLDEN, "mesh.json")))
    return z, meta


def _cam(fx, fy, cx, cy, E=None):
    return mo.camera_array(np.eye(4) if E is None else E, [[fx, 0, cx], [0, fy, cy], [0, 0, 1]])


def _soup(seed, n, w, h, z_lo=1.0, z_hi=4.0, size=0.3):
    """Random triangles in front of an identity camera with focal w: centres in the view, sizes up to `size`."""
    rng = np.random.default_rng(seed)
    c = np.c_[rng.uniform(-0.6, 0.6, (n, 2)), rng.uniform(z_lo, z_hi, n)]
    v = (c[:, None, :] + rng.normal(0, size, (n, 3, 3)) * [1, 1, 0.2]).astype(np.float32)
    return v.reshape(-1, 3), np.arange(3 * n).reshape(n, 3), _cam(w, w, w / 2 - 0.5, h / 2 - 0.5)


def _grid_plane(nx, ny, x0, y0, step, z):
    """A tessellated plane at depth z: (nx + 1)(ny + 1) vertices on an exact grid, both diagonals alternating, every
    triangle counter-clockwise on an identity camera's image."""
    ys, xs = np.meshgrid(np.arange(ny + 1), np.arange(nx + 1), indexing="ij")
    v = np.stack([x0 + xs * step, y0 + ys * step, np.full(xs.shape, z)], -1).reshape(-1, 3).astype(np.float32)
    f = []
    for r in range(ny):
        for c in range(nx):
            a, b, d, e = r * (nx + 1) + c, r * (nx + 1) + c + 1, (r + 1) * (nx + 1) + c, (r + 1) * (nx + 1) + c + 1
            f += [[a, d, e], [a, e, b]] if (r + c) % 2 else [[a, d, b], [b, d, e]]
    return v, np.array(f, np.int64)


# ------------------------------------------------------------------------------------------------------------------
# CPU: goldens and the oracle
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_reproduces_the_reference_grid_mesh():
    z, meta = _golden()
    for case in meta["grid_cases"]:
        n = case["name"]
        faces, colors = mo.grid_faces(z[f"{n}/valid"], z[f"{n}/img"])
        assert faces.shape == z[f"{n}/faces"].shape and np.array_equal(faces, z[f"{n}/faces"]), n
        assert colors.dtype == z[f"{n}/face_colors"].dtype and np.array_equal(colors, z[f"{n}/face_colors"]), n
        assert np.array_equal(z[f"{n}/pts"].reshape(-1, 3), z[f"{n}/vertices"])
        assert len(faces) == case["n_faces"]
    assert {c["n_faces"] == 0 for c in meta["grid_cases"]} == {True, False}


def test_load_cam_mvsnet_equals_the_reference_for_every_word_count(tmp_path):
    _, meta = _golden()
    assert sorted({c["words"] for c in meta["cameras"]}) == [27, 28, 29, 30, 31, 33]
    for c in meta["cameras"]:
        intr, extr = mesh.load_cam_mvsnet(io.StringIO(c["text"]), interval_scale=c["interval_scale"])
        assert intr.dtype == np.float32 and extr.dtype == np.float32
        assert np.array_equal(intr, np.array(c["intrinsic"], np.float32)), c["words"]
        assert np.array_equal(extr, np.array(c["extrinsic"], np.float32)), c["words"]
    p = tmp_path / "00000000_cam.txt"
    p.write_text(meta["cameras"][4]["text"])
    assert np.array_equal(mesh.load_cam_mvsnet(str(p))[0], np.array(meta["cameras"][4]["intrinsic"], np.float32))
    with pytest.raises(ValueError):
        mesh.load_cam_mvsnet(io.StringIO("extrinsic 1 2 3"))


def test_oracle_hand_built_triangle():
    # identity camera, f = 1, c = 0: u = x / z, v = y / z; a counter-clockwise (on the image) triangle at depth 2
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    v = np.array([[0, 0, 2], [0, 8, 2], [8, 0, 2]], np.float32)       # image (0,0), (0,4), (4,0)
    depth, face = mo.rasterize(v, [[0, 1, 2]], cam, 6, 6)
    # covered: u, v >= 0, u + v < 4, plus the top-left edges u = 0 and v = 0; the hypotenuse u + v = 4 is not top-left
    want = np.array([[c + r < 4 for c in range(6)] for r in range(6)])
    assert np.array_equal(face == 0, want) and np.all(depth[want] == 2.0) and np.all(depth[~want] == 0)
    # the reversed winding is a back face
    assert (mo.rasterize(v, [[0, 2, 1]], cam, 6, 6)[1] == -1).all()
    # the hypotenuse belongs to the neighbour across it
    v2 = np.concatenate([v, [[8, 8, 2]]]).astype(np.float32)
    _, face2 = mo.rasterize(v2, [[0, 1, 2], [1, 3, 2]], cam, 6, 6)
    assert np.array_equal(face2[:5, :5] == 1, np.array([[4 <= c + r and c < 4 and r < 4 for c in range(5)] for r in range(5)]))
    assert (face2[:4, :4] >= 0).all()     # the two triangles tile [0, 4)^2 without a gap


def test_oracle_perspective_depth_nearest_and_ties():
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    # the plane z = 2 + x / 4: the pixel at image u sees depth 2 / (1 - u / 4), perspective-correct, not affine
    uv = np.array([[-1.0, -1.0], [-1.0, 3.0], [3.0, -1.0]])
    z = 2.0 / (1.0 - uv[:, 0] / 4)
    v = np.c_[uv * z[:, None], z].astype(np.float32)
    depth, face = mo.rasterize(v, [[0, 1, 2]], cam, 3, 2)
    for u in range(3):
        assert face[0, u] == 0 and abs(depth[0, u] / (2.0 / (1.0 - u / 4)) - 1) < 1e-6
    # equal depths: the smaller id wins whatever the order; nearer wins over id
    flat = np.array([[-1, -1, 2], [-1, 5, 2], [5, -1, 2]], np.float32)
    flat[:, :2] *= 2
    verts = np.concatenate([flat, flat, flat * [1, 1, 0.5]]).astype(np.float32)
    _, face = mo.rasterize(verts, [[3, 4, 5], [0, 1, 2]], cam, 3, 3)
    assert (face[face >= 0] == 0).all()
    _, face = mo.rasterize(verts, [[3, 4, 5], [0, 1, 2], [6, 7, 8]], cam, 3, 3)
    assert (face[face >= 0] == 2).all()


def test_oracle_policy_near_far_degenerate():
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    tri = np.array([[0, 0, 1], [0, 4, 1], [4, 0, 1]], np.float32)
    assert (mo.rasterize(tri, [[0, 1, 2]], cam, 4, 4)[1] == 0).any()
    assert (mo.rasterize(tri, [[0, 1, 2]], cam, 4, 4, z_near=1.0)[1] == -1).all()      # vertex at z_near: skipped
    assert (mo.rasterize(tri, [[0, 1, 2]], cam, 4, 4, z_far=0.999)[1] == -1).all()     # beyond z_far: dropped
    behind = tri.copy()
    behind[2, 2] = -1
    assert (mo.rasterize(behind, [[0, 1, 2]], cam, 4, 4)[1] == -1).all()
    line = np.array([[0, 0, 1], [1, 1, 1], [3, 3, 1]], np.float32)
    assert (mo.rasterize(line, [[0, 1, 2]], cam, 4, 4)[1] == -1).all()


# ------------------------------------------------------------------------------------------------------------------
# CPU: the device math on the host, bit for bit against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("mesh") / "mesh_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "mesh_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.mh_grid_faces.argtypes = [C.c_longlong, C.c_longlong, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.mh_raster.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_longlong, C.c_void_p, C.c_double,
                            C.c_double, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return L


def _host_raster(L, verts, faces, cam, w, h, z_near=0.0, z_far=math.inf, id0=0):
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    f = np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    cam = np.ascontiguousarray(cam, np.float64)
    keys = np.full(w * h, EMPTY, np.uint64)
    cover = np.zeros(w * h, np.int32)
    L.mh_raster(v.ctypes.data, len(v), f.ctypes.data, len(f), id0, cam.ctypes.data, z_near, z_far, w, h,
                keys.ctypes.data, cover.ctypes.data)
    return keys, cover


def _oracle_keys(verts, faces, cam, w, h, z_near=0.0, z_far=math.inf, id0=0):
    z = np.full(w * h, EMPTY, np.uint64)
    mo.raster(z, verts, faces, cam, z_near, z_far, w, h, id0)
    return z


def test_host_grid_faces_match_the_oracle(host_lib):
    for T, H, W in ((2, 5, 7), (3, 7, 9), (1, 2, 2), (2, 9, 5)):
        faces, cpix = mo.grid_candidates(T, H, W)
        n = len(faces)
        hf, hc = np.empty((n, 3), np.int64), np.empty(n, np.int64)
        host_lib.mh_grid_faces(0, n, H, W, hf.ctypes.data, hc.ctypes.data)
        assert np.array_equal(hf, faces) and np.array_equal(hc, cpix)


def test_host_raster_matches_the_oracle_on_random_soups(host_lib):
    drawn = 0
    for seed in range(6):
        w, h = (64, 48) if seed % 2 else (37, 29)
        verts, faces, cam = _soup(seed, 300, w, h)
        if seed >= 3:                                   # a rotated, shifted camera
            rng = np.random.default_rng(seed)
            E = np.eye(4)
            a = rng.uniform(-0.3, 0.3)
            E[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            E[:3, 3] = rng.normal(0, 0.1, 3)
            cam = _cam(w * 0.8, w * 0.9, w / 2 - 0.3, h / 2 - 0.7, E)
        z_near, z_far = [(0.0, math.inf), (1.5, math.inf), (0.0, 2.5)][seed % 3]
        keys, _ = _host_raster(host_lib, verts, faces, cam, w, h, z_near, z_far, id0=seed * 1000)
        want = _oracle_keys(verts, faces, cam, w, h, z_near, z_far, id0=seed * 1000)
        assert np.array_equal(keys, want), seed
        drawn += int((keys != EMPTY).sum())
    assert drawn > 3000


def test_host_raster_matches_the_oracle_on_adversarial_triangles(host_lib):
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    w, h = 9, 7
    tris = [
        [[0, 0, 1], [0, 6, 1], [8, 0, 1]],                 # edges through centres, top and left edges on the border
        [[8, 6, 1], [8, 0, 1], [0, 6, 1]],                 # its partner across the diagonal
        [[-50, -50, 2], [-50, 150, 2], [150, -50, 2]],     # covers the whole image (and beyond)
        [[1, 1, 1], [2, 2, 1], [3, 3, 1]],                 # degenerate
        [[0, 0, 1], [8, 0, 1], [0, 6, 1]],                 # back face
        [[0, 0, 1], [0, 6, -1], [8, 0, 1]],                # a vertex behind the camera
        [[0.5, 0.5, 1], [0.5, 5.5, 1], [7.5, 0.5, 1]],     # half-pixel vertices
        [[2, 2, 3], [2, 4, 3], [4, 2, 3]],                 # equal depth ties below
        [[2, 2, 3], [2, 4, 3], [4, 2, 3]],
    ]
    v = np.array(tris, np.float64)
    v[:, :, :2] *= v[:, :, 2:]
    v = v.astype(np.float32).reshape(-1, 3)
    f = np.arange(len(v)).reshape(-1, 3)
    for z_near, z_far in ((0.0, math.inf), (0.5, 2.0), (1.0, math.inf)):
        keys, _ = _host_raster(host_lib, v, f, cam, w, h, z_near, z_far)
        assert np.array_equal(keys, _oracle_keys(v, f, cam, w, h, z_near, z_far))
    # tiny, huge and sliver triangles with random fp32 coordinates
    rng = np.random.default_rng(7)
    for scale in (1e-3, 1.0, 1e3):
        c = rng.uniform(-0.5, 0.5, (200, 1, 3)) + [0, 0, 2]
        v = (c + rng.normal(0, scale, (200, 3, 3)) * [1, 1, 0.01]).astype(np.float32).reshape(-1, 3)
        v[:, 2] = np.abs(v[:, 2]) + 0.1
        f = np.arange(600).reshape(-1, 3)
        cam2 = _cam(40.0, 40.0, 20.0, 15.0)
        keys, _ = _host_raster(host_lib, v, f, cam2, 41, 31)
        assert np.array_equal(keys, _oracle_keys(v, f, cam2, 41, 31))


@pytest.mark.parametrize("step", [1.0, 0.5, 2.0])
def test_tessellated_grid_covers_every_centre_exactly_once(host_lib, step):
    """Grid vertices on exact pixel centres (or half-pixels): every edge passes through centres, and each centre inside
    the grid is covered by exactly one triangle; outside it, by none."""
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    v, f = _grid_plane(12, 10, 1.0, 2.0, step, 1.0)
    w, h = 40, 30
    keys, cover = _host_raster(host_lib, v, f, cam, w, h)
    pix, _, _ = mo.fragments(v, f, cam, 0.0, math.inf, w, h)
    ocover = np.bincount(pix, minlength=w * h)
    assert np.array_equal(cover, ocover)
    cols, rows = np.meshgrid(np.arange(w), np.arange(h))
    inside = (cols >= 1) & (cols < 1 + 12 * step) & (rows >= 2) & (rows < 2 + 10 * step)
    # the right and bottom borders of the grid are not top-left edges: half-open coverage, as GL draws
    assert np.array_equal(cover.reshape(h, w), inside.astype(np.int32))
    assert np.array_equal(keys, _oracle_keys(v, f, cam, w, h))


def test_app_mesh_covers_each_centre_once_per_winding(host_lib):
    """app.py's mesh on a fronto-parallel grid whose pixels land on pixel centres: one of the two windings of each
    triangle is culled, so every centre of the surface is covered once."""
    H, W = 6, 8
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pts = np.stack([xs + 2.0, ys + 1.0, np.ones_like(xs, float)], -1)[None].astype(np.float32)
    faces, _ = mo.grid_faces(np.ones((1, H, W), bool), pts)
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    _, cover = _host_raster(host_lib, pts.reshape(-1, 3), faces, cam, 12, 9)
    want = np.zeros((9, 12), np.int32)
    want[1:1 + H - 1, 2:2 + W - 1] = 1
    assert np.array_equal(cover.reshape(9, 12), want)


# ------------------------------------------------------------------------------------------------------------------
# CPU: GLB, PLY, ABI
# ------------------------------------------------------------------------------------------------------------------
def _parse_glb(path):
    """A glTF 2.0 binary parser checking the container rules -> (json, arrays by attribute name, indices)."""
    data = open(path, "rb").read()
    magic, version, length = struct.unpack_from("<4sII", data, 0)
    assert magic == b"glTF" and version == 2 and length == len(data)
    jl, jt = struct.unpack_from("<I4s", data, 12)
    assert jt == b"JSON" and jl % 4 == 0
    doc = json.loads(data[20:20 + jl].decode("utf-8"))
    at = 20 + jl
    assert (at % 4) == 0
    bl, bt = struct.unpack_from("<I4s", data, at)
    assert bt == b"BIN\0" and bl % 4 == 0 and at + 8 + bl == len(data)
    binary = data[at + 8:]
    assert doc["asset"]["version"] == "2.0" and doc["buffers"] == [{"byteLength": bl}]
    comp = {5126: np.float32, 5121: np.uint8, 5125: np.uint32}
    width = {"SCALAR": 1, "VEC3": 3, "VEC4": 4}

    def read(i):
        acc = doc["accessors"][i]
        view = doc["bufferViews"][acc["bufferView"]]
        assert view["byteOffset"] % 4 == 0 and view["byteOffset"] + view["byteLength"] <= bl
        dt = np.dtype(comp[acc["componentType"]])
        assert view["byteLength"] == acc["count"] * width[acc["type"]] * dt.itemsize
        a = np.frombuffer(binary, dt, acc["count"] * width[acc["type"]], view["byteOffset"])
        return a.reshape(acc["count"], width[acc["type"]])

    assert len(doc["meshes"]) == 1 and len(doc["meshes"][0]["primitives"]) == 1 and len(doc["nodes"]) == 1
    prim = doc["meshes"][0]["primitives"][0]
    arrays = {k: read(i) for k, i in prim["attributes"].items()}
    pos_acc = doc["accessors"][prim["attributes"]["POSITION"]]
    assert pos_acc["min"] == arrays["POSITION"].min(0).tolist() and pos_acc["max"] == arrays["POSITION"].max(0).tolist()
    if "COLOR_0" in prim["attributes"]:
        assert doc["accessors"][prim["attributes"]["COLOR_0"]]["normalized"] is True
    idx = read(prim["indices"]).reshape(-1, 3) if "indices" in prim else None
    return doc, arrays, idx


def test_write_glb_mesh_and_points(tmp_path):
    z, _ = _golden()
    pts, img, valid = z["random_odd/pts"], z["random_odd/img"], z["random_odd/valid"]
    faces, colors = mo.grid_faces(valid, img)
    path = str(tmp_path / "scene.glb")
    M = mesh.app_scene_matrix()
    mesh.write_glb(path, pts.reshape(-1, 3), faces, img.reshape(-1, 3), matrix=M)
    doc, arrays, idx = _parse_glb(path)
    assert doc["meshes"][0]["primitives"][0]["mode"] == 4
    assert np.array_equal(arrays["POSITION"], pts.reshape(-1, 3)) and np.array_equal(idx, faces)
    rgba = arrays["COLOR_0"]
    assert (rgba[:, 3] == 255).all()
    assert np.array_equal(rgba[:, :3], np.floor(np.clip(img.reshape(-1, 3).astype(np.float64), 0, 1) * 255 + 0.5))
    assert np.array_equal(np.array(doc["nodes"][0]["matrix"]).reshape(4, 4).T, M)
    # app.py's matrix: inv(OPENGL @ R_y(180)) flips x and... y stays, z flips twice
    assert np.allclose(M, np.diag([-1.0, -1.0, 1.0, 1.0]), atol=1e-15)
    # as_pointcloud=True: points with their colours, no indices; odd byte counts are padded
    mesh.write_glb(path, pts[valid][:5], colors=img[valid][:5])
    doc, arrays, idx = _parse_glb(path)
    assert doc["meshes"][0]["primitives"][0]["mode"] == 0 and idx is None and "matrix" not in doc["nodes"][0]
    assert np.array_equal(arrays["POSITION"], pts[valid][:5])
    for bad in (dict(vertices=np.zeros((0, 3))), dict(vertices=np.full((3, 3), np.nan)),
                dict(vertices=np.zeros((3, 3)), faces=np.array([[0, 1, 3]])),
                dict(vertices=np.zeros((3, 3)), colors=np.zeros((2, 3))),
                dict(vertices=np.zeros((3, 3)), matrix=np.eye(3))):
        with pytest.raises(ValueError):
            mesh.write_glb(path, **bad)


def _ply_header(fmt, n_v, n_f, vprops=("float x", "float y", "float z"), fprop="list uchar int vertex_indices"):
    lines = ["ply", f"format {fmt} 1.0", "comment made by a test", f"element vertex {n_v}"]
    lines += [f"property {p}" for p in vprops] + [f"element face {n_f}", f"property {fprop}", "end_header"]
    return ("\n".join(lines) + "\n").encode("ascii")


def test_read_ply_mesh_ascii_binary_and_malformed(tmp_path):
    rng = np.random.default_rng(5)
    v = rng.normal(0, 10, (6, 3))
    f = np.array([[0, 1, 2], [2, 3, 4], [5, 4, 0]])
    # binary: double xyz among other properties (uchar colours, a float before x), uint vertex index lists
    props = ("float quality", "double x", "double y", "double z", "uchar red", "uchar green", "uchar blue")
    rec = np.zeros(6, np.dtype([("q", "<f4"), ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("r", "u1"), ("g", "u1"),
                                ("b", "u1")]))
    rec["x"], rec["y"], rec["z"] = v.T
    frec = np.zeros(3, np.dtype([("n", "u1"), ("i", "<u4", 3)]))
    frec["n"], frec["i"] = 3, f
    p = tmp_path / "b.ply"
    p.write_bytes(_ply_header("binary_little_endian", 6, 3, props, "list uchar uint vertex_indices") + rec.tobytes()
                  + frec.tobytes())
    rv, rf = mesh.read_ply_mesh(str(p))
    assert rv.dtype == np.float32 and np.array_equal(rv, v.astype(np.float32)) and np.array_equal(rf, f)
    # ascii, float xyz
    body = "".join(f"{a:.9g} {b:.9g} {c:.9g}\n" for a, b, c in v.astype(np.float32)) + \
        "".join(f"3 {a} {b} {c}\n" for a, b, c in f)
    p = tmp_path / "a.ply"
    p.write_bytes(_ply_header("ascii", 6, 3) + body.encode())
    rv, rf = mesh.read_ply_mesh(str(p))
    assert np.array_equal(rv, v.astype(np.float32)) and np.array_equal(rf, f)
    good = _ply_header("ascii", 6, 3) + body.encode()
    bad = {
        "big_endian": _ply_header("binary_big_endian", 6, 3) + rec.tobytes(),
        "quad": _ply_header("ascii", 6, 1) + body.encode().split(b"3 0")[0] + b"4 0 1 2 3\n",
        "index": good.replace(b"3 5 4 0", b"3 5 4 9"),
        "int_xyz": _ply_header("ascii", 6, 3, ("int x", "int y", "int z")) + body.encode(),
        "no_z": _ply_header("ascii", 6, 3, ("float x", "float y")) + body.encode(),
        "truncated": _ply_header("binary_little_endian", 6, 3, props) + rec.tobytes()[:-5],
        "not_ply": b"PLY?\n" + good,
        "extra_face_prop": good.replace(b"end_header", b"property uchar red\nend_header"),
        "other_element": good.replace(b"end_header", b"element edge 0\nproperty int vertex1\nend_header"),
        "vertex_list": _ply_header("ascii", 6, 3, ("float x", "float y", "float z", "list uchar int n")) + body.encode(),
    }
    for name, data in bad.items():
        q = tmp_path / f"{name}.ply"
        q.write_bytes(data)
        with pytest.raises(ValueError):
            mesh.read_ply_mesh(str(q))


def test_c_abi_rejects_bad_mesh_arguments():
    """Validation of the s3r_mesh_grid_* and s3r_raster_* entries happens before any CUDA call: status -1 and a
    message, no device needed."""
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_mesh_grid_workspace_bytes(50, 224, 224) == 8 * ((4 * 50 * 223 * 223 + 2047) // 2048 + 1)
    assert L.s3r_mesh_grid_workspace_bytes(1, 1, 1) == 8
    for T, H, W in ((0, 4, 4), (1, 0, 4), (1, 4, -1), (1 << 10, 1 << 11, 1 << 10)):
        assert L.s3r_mesh_grid_workspace_bytes(T, H, W) == 0
    fake, odd = C.c_void_p(64), C.c_void_p(68)
    n = C.c_int64(0)
    count = lambda **kw: L.s3r_mesh_grid_count(*{**dict(valid=fake, T=2, H=4, W=4, ws=fake, wsb=1024,
                                                        n=C.byref(n), stream=None), **kw}.values())
    assert count(T=1 << 10, H=1 << 11, W=1 << 10) == -1 and b"mesh_grid_count" in L.s3r_last_error()
    for kw in (dict(valid=None), dict(ws=None), dict(ws=odd), dict(wsb=8), dict(n=None), dict(T=0), dict(W=0)):
        assert count(**kw) == -1, kw
    faces = lambda **kw: L.s3r_mesh_grid_faces(*{**dict(valid=fake, img=fake, T=2, H=4, W=4, ws=fake, wsb=1024,
                                                        faces=fake, colors=fake, stream=None), **kw}.values())
    for kw in (dict(valid=None), dict(img=None), dict(ws=None), dict(wsb=8), dict(faces=None), dict(colors=None),
               dict(H=-1)):
        assert faces(**kw) == -1 and b"mesh_grid_faces" in L.s3r_last_error(), kw
    cam = (C.c_double * 16)(*([1.0] * 16))
    tri = lambda **kw: L.s3r_raster_triangles(*{**dict(v=fake, nv=3, f=fake, nf=1, id0=0, cam=cam, zn=0.0, zf=math.inf,
                                                       w=4, h=3, keys=fake, stream=None), **kw}.values())
    assert tri(nf=1 << 30, id0=1 << 30) == -1 and b"raster_triangles" in L.s3r_last_error()
    for kw in (dict(v=None), dict(f=None), dict(cam=None), dict(keys=None), dict(keys=odd), dict(nv=-1), dict(nf=-1),
               dict(id0=-1), dict(nv=1 << 31), dict(w=0), dict(h=0), dict(w=1 << 16, h=1 << 15), dict(zn=-1.0),
               dict(zn=math.nan), dict(zn=math.inf), dict(zf=0.0), dict(zn=1.0, zf=1.0), dict(zf=math.nan)):
        assert tri(**kw) == -1, kw
    for i in (0, 11, 12, 15):
        bad = (C.c_double * 16)(*([1.0] * 16))
        bad[i] = math.nan
        assert tri(cam=bad) == -1 and f"camera[{i}]".encode() in L.s3r_last_error()
    assert L.s3r_raster_resolve(None, 4, 3, fake, fake, None) == -1 and b"raster_resolve" in L.s3r_last_error()
    for args in ((odd, 4, 3, fake, fake), (fake, 4, 3, None, fake), (fake, 4, 3, fake, None), (fake, 0, 3, fake, fake)):
        assert L.s3r_raster_resolve(*args, None) == -1


def test_cpu_inputs_are_rejected():
    pts = torch.rand(2, 4, 4, 3)
    with pytest.raises(ValueError):
        mesh.pts3d_to_mesh(pts, pts.clone())
    with pytest.raises(ValueError):
        mesh.rasterize(pts.reshape(-1, 3), torch.zeros(1, 3, dtype=torch.int32), np.ones(16), 4, 4)
    cam = vis.PinholeCameraParameters(vis.PinholeCameraIntrinsic(8, 6, [[4, 0, 4], [0, 4, 3], [0, 0, 1]]), np.eye(4))
    with pytest.raises(ValueError):
        vis.render_mesh_frames(pts, pts.clone(), cam)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _gpu_raster(verts, faces, cam, w, h, z_near=0.0, z_far=math.inf):
    d, f = mesh.rasterize(torch.from_numpy(np.asarray(verts, np.float32)).cuda(),
                          torch.from_numpy(np.asarray(faces, np.int64)).cuda(), cam, w, h, z_near, z_far)
    return d.cpu().numpy(), f.cpu().numpy()


def _check_against_oracle(verts, faces, cam, w, h, z_near=0.0, z_far=math.inf):
    d, f = _gpu_raster(verts, faces, cam, w, h, z_near, z_far)
    od, of = mo.rasterize(verts, faces, cam, w, h, z_near, z_far)
    assert np.array_equal(f, of) and np.array_equal(d.view(np.uint32), od.view(np.uint32))
    return d, f


@pytest.mark.gpu
def test_gpu_grid_mesh_equals_the_golden_and_the_oracle():
    z, meta = _golden()
    for case in meta["grid_cases"]:
        n = case["name"]
        v, f, c = mesh.pts3d_to_mesh(torch.from_numpy(z[f"{n}/pts"]).cuda(), torch.from_numpy(z[f"{n}/img"]).cuda(),
                                     torch.from_numpy(z[f"{n}/valid"]).cuda())
        assert f.dtype == torch.int32 and c.dtype == torch.float32 and v.is_cuda
        assert np.array_equal(v.cpu().numpy(), z[f"{n}/vertices"])
        assert np.array_equal(f.cpu().numpy().astype(np.int64).reshape(-1, 3), z[f"{n}/faces"].reshape(-1, 3)), n
        assert np.array_equal(c.cpu().numpy().reshape(-1, 3), z[f"{n}/face_colors"].reshape(-1, 3)), n


@pytest.mark.gpu
def test_gpu_grid_mesh_at_app_size_equals_the_oracle():
    """app.py's default: 50 frames of 224 x 224, confidence mask ~70 % valid, in clumps and salt."""
    rng = np.random.default_rng(11)
    T, H, W = 50, 224, 224
    pts = torch.randn(T, H, W, 3, generator=torch.Generator().manual_seed(1)).cuda()
    img = torch.rand(T, H, W, 3, generator=torch.Generator().manual_seed(2)).cuda()
    valid = rng.random((T, H, W)) < 0.7
    valid[:, 50:90, 60:120] = False
    valid[7] = True
    valid[8] = False
    v, f, c = mesh.pts3d_to_mesh(pts, img, torch.from_numpy(valid).cuda())
    of, oc = mo.grid_faces(valid, img.cpu().numpy())
    assert np.array_equal(f.cpu().numpy(), of.astype(np.int32)) and np.array_equal(c.cpu().numpy(), oc)
    print(f"app-size mesh: {len(of)} faces of {4 * T * (H - 1) * (W - 1)} candidates")
    again = mesh.pts3d_to_mesh(pts, img, torch.from_numpy(valid).cuda())
    assert torch.equal(again[1], f) and torch.equal(again[2], c)


@pytest.mark.gpu
def test_gpu_raster_random_soup_equals_the_oracle():
    for seed, (w, h, n, size) in enumerate([(64, 48, 2000, 0.2), (160, 120, 5000, 0.05), (97, 61, 300, 1.5)]):
        verts, faces, cam = _soup(100 + seed, n, w, h, size=size)
        for z_near, z_far in ((0.0, math.inf), (1.2, 3.0)):
            d, f = _check_against_oracle(verts, faces, cam, w, h, z_near, z_far)
            assert (f >= 0).sum() > 0.2 * w * h


@pytest.mark.gpu
def test_gpu_raster_adversarial_cases_equal_the_oracle():
    cam = _cam(1.0, 1.0, 0.0, 0.0)
    w, h = 9, 7
    tris = [[[0, 0, 1], [0, 6, 1], [8, 0, 1]], [[8, 6, 1], [8, 0, 1], [0, 6, 1]],       # shared edge through centres
            [[-50, -50, 2], [-50, 150, 2], [150, -50, 2]],                              # whole image
            [[1, 1, 1], [2, 2, 1], [3, 3, 1]],                                          # degenerate
            [[0, 0, 0.5], [8, 0, 0.5], [0, 6, 0.5]],                                    # back face, nearest
            [[0, 0, 0.2], [0, 6, -1], [8, 0, 0.2]],                                     # a vertex behind the camera
            [[2, 2, 0.7], [2, 4, 0.7], [4, 2, 0.7]], [[2, 2, 0.7], [2, 4, 0.7], [4, 2, 0.7]],   # equal-depth ties
            [[0, 0, 9], [0, 6, 9], [8, 0, 9]]]                                          # beyond z_far below
    v = np.array(tris, np.float64)
    v[:, :, :2] *= v[:, :, 2:]
    v = v.astype(np.float32).reshape(-1, 3)
    f = np.arange(len(v)).reshape(-1, 3)
    for z_near, z_far in ((0.0, math.inf), (0.0, 5.0), (0.6, 5.0), (1.0, math.inf)):
        _check_against_oracle(v, f, cam, w, h, z_near, z_far)
    d, face = _check_against_oracle(v, f, cam, w, h)
    assert set(np.unique(face).tolist()) <= {0, 1, 2, 6}            # the tie goes to the smaller id, 6 not 7
    # whole-image triangles at 1600 x 1200, in the second pass, and a few thousand small ones in front of them
    W2, H2 = 1600, 1200
    big = np.array([[-10, -10, 3], [-10, 30, 3], [30, -10, 3], [25, 25, 4], [25, -20, 4], [-20, 25, 4]], np.float32)
    verts, faces, cam2 = _soup(5, 3000, W2, H2, size=0.01)
    allv = np.concatenate([big, verts]).astype(np.float32)
    allf = np.concatenate([[[0, 1, 2], [3, 4, 5]], faces + 6])
    _, face2 = _check_against_oracle(allv, allf, cam2, W2, H2)
    assert (face2 >= 0).all() and (face2 == 0).mean() > 0.5


@pytest.mark.gpu
def test_gpu_raster_is_reproducible_and_independent_of_face_order():
    verts, faces, cam = _soup(42, 20000, 320, 240, size=0.08)
    d1, f1 = _gpu_raster(verts, faces, cam, 320, 240)
    d2, f2 = _gpu_raster(verts, faces, cam, 320, 240)
    assert np.array_equal(d1.view(np.uint32), d2.view(np.uint32)) and np.array_equal(f1, f2)
    perm = np.random.default_rng(0).permutation(len(faces))
    d3, f3 = _gpu_raster(verts, faces[perm], cam, 320, 240)
    assert np.array_equal(d3.view(np.uint32), d1.view(np.uint32))
    hit = f3 >= 0
    # without exact depth ties the winning face is the same; mapped back through the permutation
    assert (perm[f3[hit]] == f1[hit]).mean() > 0.999


@pytest.mark.gpu
def test_gpu_app_mesh_raster_equals_the_oracle():
    z, _ = _golden()
    rng = np.random.default_rng(3)
    T, H, W = 3, 48, 64
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pts = np.stack([(xs - W / 2) / 40, (ys - H / 2) / 40, 1 + 0.3 * np.sin(xs / 7) * np.cos(ys / 5)], -1)
    pts = np.stack([pts + [0.05 * t, 0, 0.1 * t] for t in range(T)]).astype(np.float32)
    valid = rng.random((T, H, W)) < 0.85
    img = rng.uniform(0, 1, (T, H, W, 3)).astype(np.float32)
    v, f, c = mesh.pts3d_to_mesh(torch.from_numpy(pts).cuda(), torch.from_numpy(img).cuda(),
                                 torch.from_numpy(valid).cuda())
    cam = _cam(200.0, 200.0, 159.5, 119.5)
    d, face = mesh.rasterize(v, f, cam, 320, 240)
    od, of = mo.rasterize(pts.reshape(-1, 3), mo.grid_faces(valid, img)[0], cam, 320, 240)
    assert np.array_equal(face.cpu().numpy(), of) and np.array_equal(d.cpu().numpy().view(np.uint32), od.view(np.uint32))
    assert (of >= 0).mean() > 0.5


def _look_at_pose_gl(eye, target):
    """c2w in the OpenGL convention (x right, y up, looking down -z) at `eye` towards `target`, world up = -y."""
    fwd = np.asarray(target, float) - eye
    fwd /= np.linalg.norm(fwd)
    right = np.cross(fwd, [0, -1, 0])
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    P = np.eye(4)
    P[:3, 0], P[:3, 1], P[:3, 2], P[:3, 3] = right, -down, -fwd, eye
    return P


@pytest.mark.gpu
def test_gpu_render_depth_maps_of_a_plane_and_a_box_match_analytic_depth():
    H, W = 120, 160
    K = np.array([[150.0, 0, 80.0], [0, 150.0, 60.0], [0, 0, 1]])
    # a plane z = 5 tessellated 20 x 20 over [-4, 4]^2, seen from the origin looking down +z (OpenCV) -> GL pose
    v, f = _grid_plane(20, 20, -4.0, -4.0, 0.4, 5.0)
    pose = np.diag([1.0, -1.0, -1.0, 1.0])       # OpenCV identity c2w with columns 1, 2 negated
    d = mesh.render_depth_maps((v, f), [pose], K, H, W, near=0.01, far=100.0)[0]
    assert d.dtype == np.float32 and d.shape == (H, W) and (d == np.float32(5.0)).all()
    # tilted view of the plane: depth along pixel (r, c) sampled at (c + 0.5, r + 0.5) in pyrender's intrinsics
    th = 0.3
    R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])     # c2w rotation about y
    c2w = np.eye(4)
    c2w[:3, :3] = R
    c2w[:3, 3] = [0.5, 0.2, 0.0]
    gl = c2w.copy()
    gl[:, 1:3] *= -1
    d = mesh.render_depth_maps((v, f), [gl], K, H, W, near=0.01, far=100.0)[0]
    cols, rows = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    ray = np.stack([(cols - 80.0) / 150.0, (rows - 60.0) / 150.0, np.ones_like(cols)], -1)     # camera frame, z = 1
    world_dir = ray @ R.T
    t = (5.0 - c2w[2, 3]) / world_dir[..., 2]             # camera depth = t (ray z component is 1)
    hit = world_dir[..., 0] * t + 0.5
    hit_y = world_dir[..., 1] * t + 0.2
    inside = (np.abs(hit) < 3.9) & (np.abs(hit_y) < 3.9)
    assert inside.sum() > 0.5 * H * W
    assert np.abs(d[inside] - t[inside]).max() <= 4 * np.spacing(np.float32(t.max())) * 4
    # a box [-1, 1]^2 x [4, 6]: from the origin the visible face is z = 4
    corners = np.array([[x, y, z] for z in (4, 6) for y in (-1, 1) for x in (-1, 1)], np.float32)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    tris = np.array([[q[0], q[1], q[2]] for q in quads] + [[q[0], q[2], q[3]] for q in quads])
    tris = np.concatenate([tris, tris[:, ::-1]])          # both windings: whichever faces the camera is drawn
    d = mesh.render_depth_maps((corners, tris), [pose, _look_at_pose_gl(np.array([0, 0, -1.0]), [0, 0, 5])], K, H, W,
                               near=0.01, far=100.0)
    u = (np.arange(W) + 0.5 - 80.0) / 150.0
    vv = (np.arange(H) + 0.5 - 60.0) / 150.0
    for dm, z0 in zip(d, (4.0, 5.0)):
        inside = (np.abs(vv)[:, None] * z0 < 1) & (np.abs(u)[None, :] * z0 < 1)
        outside = (np.abs(vv)[:, None] * z0 > 1) | (np.abs(u)[None, :] * z0 > 1)
        assert inside.sum() > 1000 and (dm[inside] == np.float32(z0)).all() and (dm[outside] == 0).all()


@pytest.mark.gpu
def test_gpu_render_dtu_scenes_writes_depth_maps(tmp_path):
    import cv2
    scan = tmp_path / "scan24"
    (scan / "images").mkdir(parents=True)
    (scan / "cams").mkdir()
    H, W = 60, 80
    for i in range(3):
        cv2.imwrite(str(scan / "images" / f"{i:08d}.jpg"), np.full((H, W, 3), 128, np.uint8))
        E = np.eye(4)
        E[0, 3] = 0.1 * i
        text = "extrinsic\n" + "\n".join(" ".join(str(x) for x in r) for r in E) + "\n\nintrinsic\n" + \
            "100 0 40\n0 100 30\n0 0 1\n\n425 2.5\n"
        (scan / "cams" / f"{i:08d}_cam.txt").write_text(text)
    v, f = _grid_plane(10, 10, -3.0, -3.0, 0.6, 7.0)
    rec = np.zeros(len(v), np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4")]))
    rec["x"], rec["y"], rec["z"] = v.T
    frec = np.zeros(len(f), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    frec["n"], frec["i"] = 3, f
    header = (f"ply\nformat binary_little_endian 1.0\nelement vertex {len(v)}\nproperty float x\nproperty float y\n"
              f"property float z\nelement face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
    (scan / "furu024_l3_surf_11_trim_8.ply").write_bytes(header.encode() + rec.tobytes() + frec.tobytes())
    mesh.render_dtu_scenes(str(scan))
    out = sorted(os.listdir(scan / "depths_furu"))
    assert out == [f"{i:08d}.npy" for i in range(3)]
    for name in out:
        d = np.load(scan / "depths_furu" / name)
        assert d.dtype == np.float32 and d.shape == (H, W) and (d == np.float32(7.0)).mean() > 0.9


@pytest.mark.gpu
def test_gpu_render_mesh_frames_static_equals_from_scratch(tmp_path):
    rng = np.random.default_rng(9)
    T, H, W = 4, 24, 32
    ys, xs = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    pts = np.stack([np.stack([(xs - W / 2) / 20 + 0.1 * t, (ys - H / 2) / 20, 1.5 + 0.2 * t + 0.1 * np.sin(xs / 3)], -1)
                    for t in range(T)]).astype(np.float32)
    img = rng.uniform(-0.1, 1.1, (T, H, W, 3)).astype(np.float32)
    mask = torch.from_numpy(rng.random((T, H, W)) < 0.9).cuda()
    cam = vis.PinholeCameraParameters(vis.PinholeCameraIntrinsic(96, 72, [[60.0, 0, 47.5], [0, 60.0, 35.5], [0, 0, 1]]),
                                      np.eye(4))
    P, I = torch.from_numpy(pts).cuda(), torch.from_numpy(img).cuda()
    st = vis.render_mesh_frames(P, I, cam, output_dir=str(tmp_path), mask=mask)
    dy = vis.render_mesh_frames(P, I, cam, mask=mask, dynamic=True)
    assert st.dtype == torch.uint8 and tuple(st.shape) == (T, 72, 96, 3)
    assert sorted(os.listdir(tmp_path / "render_frames")) == ["camera.json"] + [f"frame_{i:03d}.png" for i in range(T)]
    v, f, c = mesh.pts3d_to_mesh(P, I, mask)
    c16 = mo.camera_array(cam.extrinsic, cam.intrinsic.intrinsic_matrix)
    from oracle import render_oracle as ro
    for i in range(T):
        # frames 0..i drawn at once from an empty buffer: the same faces with the same ids
        n_i = int((f[:, 0] < (i + 1) * H * W).sum())
        d, face = mesh.rasterize(v, f[:n_i], c16, 96, 72)
        want = np.zeros((72, 96, 3), np.uint8)
        fc = face.cpu().numpy()
        want[fc >= 0] = ro.color_u8(c.cpu().numpy()[fc[fc >= 0]])
        assert np.array_equal(st[i].cpu().numpy(), want), i
        assert int((fc >= 0).sum()) > 500
    assert not torch.equal(st[T - 1], dy[T - 1])


@pytest.mark.gpu
def test_gpu_inputs_are_validated():
    good = torch.rand(2, 4, 4, 3, device="cuda")
    for bad in (good.double(), good[..., :2], good[0]):
        with pytest.raises(ValueError):
            mesh.pts3d_to_mesh(bad, good)
    nan = good.clone()
    nan[0, 1, 1, 0] = math.nan
    with pytest.raises(ValueError):
        mesh.pts3d_to_mesh(nan, good)
    mask = torch.ones(2, 4, 4, dtype=torch.bool, device="cuda")
    mask[0, 1, 1] = False
    assert len(mesh.pts3d_to_mesh(nan, good, mask)[1]) > 0         # non-finite only where invalid: accepted
    v = torch.rand(5, 3, device="cuda")
    f = torch.tensor([[0, 1, 2]], device="cuda")
    cam = np.r_[np.eye(4)[:3].reshape(-1), [4.0, 4.0, 2.0, 2.0]]
    for args in ((v, f + 5, cam, 4, 4), (v.double(), f, cam, 4, 4), (v, f.float(), cam, 4, 4), (v, f, cam[:15], 4, 4),
                 (v, f, cam, 0, 4), (v.cpu(), f, cam, 4, 4)):
        with pytest.raises(ValueError):
            mesh.rasterize(*args)
    vn = v.clone()
    vn[0, 0] = math.inf
    for kw in (dict(vertices=vn), dict(z_near=-1.0), dict(z_far=0.0)):
        a = {**dict(vertices=v, faces=f, camera=cam, w=4, h=4), **kw}
        with pytest.raises(ValueError):
            mesh.rasterize(**a)
