"""Headless rendering and PLY export (spann3r_b200.vis): spann3r/tools/vis.py `render_frames` as a z-buffered point
rasteriser on the device, Open3D's camera.json, and `o3d.io.write_point_cloud`'s binary PLY.

Checkers:
  * oracle/render_oracle.py (numpy, the kernel's operation order, static mode re-rendered from scratch per frame) on
    hand-built scenes, and byte for byte against every frame the GPU renders;
  * the device math header compiled for the host (tests/native/render_host_check.cpp) against the oracle, bit for bit;
  * tests/golden/o3d_camera.json, a hand-written file in Open3D's documented camera format.
Open3D itself is not run.
"""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, get_state_dict
from oracle import render_oracle as ro
from spann3r_b200 import vis

HERE = os.path.dirname(os.path.abspath(__file__))
CAMERA_JSON = os.path.join(GOLDEN, "o3d_camera.json")


def _cam(fx, fy, cx, cy, E=None):
    return ro.camera_array(np.eye(4) if E is None else E, [[fx, 0, cx], [0, fy, cy], [0, 0, 1]])


def _rotation(rng, scale=0.3):
    a = rng.normal(0, scale, 3)
    th = np.linalg.norm(a)
    k = a / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * K @ K


def _extrinsic(rng, t_scale=0.2):
    E = np.eye(4)
    E[:3, :3] = _rotation(rng)
    E[:3, 3] = rng.normal(0, t_scale, 3)
    return E


# ------------------------------------------------------------------------------------------------------------------
# CPU: the oracle on hand-built scenes
# ------------------------------------------------------------------------------------------------------------------
def _render_points(pts, colors, cam, w, h, mask=None, z_near=0.0):
    pts = np.asarray(pts, np.float32).reshape(1, 1, -1, 3)
    colors = np.asarray(colors, np.float32).reshape(1, 1, -1, 3)
    m = None if mask is None else np.asarray(mask, bool).reshape(1, 1, -1)
    return ro.render_frames(pts, colors, cam, w, h, mask=m, z_near=z_near)[0]


def test_oracle_known_pixel_and_colour_rounding():
    cam = _cam(2.0, 2.0, 1.5, 1.0)           # 4 x 3 image; (0, 0, 1) -> u = 1.5, v = 1.0 -> col 2, row 1
    img = _render_points([[0, 0, 1]], [[0.25, 0.5, 1.0]], cam, 4, 3)
    expect = np.zeros((3, 4, 3), np.uint8)
    expect[1, 2] = [64, 128, 255]             # 63.75 -> 64, 127.5 -> 128 (half up), 255
    assert np.array_equal(img, expect)
    assert ro.color_u8([-0.5, 2.0, np.nan, 0.5 / 255, 1.5 / 255]).tolist() == [0, 255, 0, 1, 2]


def test_oracle_nearer_point_wins_in_any_order():
    cam = _cam(2.0, 2.0, 1.5, 1.0)
    for pts, cols, want in (([[0, 0, 2], [0, 0, 1]], [[1, 0, 0], [0, 1, 0]], [0, 255, 0]),
                            ([[0, 0, 1], [0, 0, 2]], [[1, 0, 0], [0, 1, 0]], [255, 0, 0])):
        assert _render_points(pts, cols, cam, 4, 3)[1, 2].tolist() == want


def test_oracle_equal_fp32_depth_goes_to_the_smaller_index():
    E = np.eye(4)
    E[2, 3] = 3 * 2.0 ** -26
    cam = _cam(2.0, 2.0, 1.5, 1.0, E)
    # camera depths 1 + 3 * 2^-26 and 1 - 2^-26 in fp64: the first is farther, both round to 1.0f
    pts = np.array([[0, 0, 1.0], [0, 0, 1.0 - 2.0 ** -24]], np.float32)
    _, _, _, key = ro.project(pts, cam, 0.0, 4, 3)
    assert (key >> np.uint64(32)).tolist() == [int(np.float32(1.0).view(np.uint32))] * 2 and key[0] < key[1]
    assert _render_points(pts, [[1, 0, 0], [0, 0, 1]], cam, 4, 3)[1, 2].tolist() == [255, 0, 0]
    assert _render_points(pts[::-1], [[1, 0, 0], [0, 0, 1]], cam, 4, 3)[1, 2].tolist() == [255, 0, 0]
    # one fp32 step apart: depth decides, not the index
    E[2, 3] = 0.0
    pts = np.array([[0, 0, 1.0 + 2.0 ** -23], [0, 0, 1.0]], np.float32)
    assert _render_points(pts, [[1, 0, 0], [0, 0, 1]], _cam(2.0, 2.0, 1.5, 1.0, E), 4, 3)[1, 2].tolist() == [0, 0, 255]


def test_oracle_drops_behind_outside_nonfinite_and_masked_points():
    cam = _cam(2.0, 2.0, 1.5, 1.0)            # u = 2 x / z + 1.5: col = floor(u + 0.5)
    pts = [[0, 0, -1],                        # behind the camera
           [0, 0, 0],                         # at the camera: q.z > z_near fails for z_near = 0
           [-1.0, 0, 1],                      # u = -0.5 -> col 0: kept
           [-1.0000001, 0, 1],                # u just below -0.5 -> col -1: dropped
           [1.0, 0, 1],                       # u = 3.5 -> col 4 = w: dropped
           [np.nan, 0, 1], [0, np.inf, 1],    # non-finite
           [0, 0, 1]]                         # masked below
    pix, col, row, key = ro.project(pts, cam, 0.0, 4, 3)
    assert pix.tolist() == [-1, -1, 4, -1, -1, -1, -1, 6]
    assert (key[pix < 0] == ro.EMPTY).all() and (key[pix >= 0] != ro.EMPTY).all()
    img = _render_points(pts, np.ones((8, 3)), cam, 4, 3, mask=[1, 1, 1, 1, 1, 1, 1, 0])
    assert np.argwhere(img.any(-1)).tolist() == [[1, 0]]
    # z_near: strictly beyond it
    assert ro.project([[0, 0, 0.5], [0, 0, 0.5000001]], cam, 0.5, 4, 3)[0].tolist() == [-1, 6]


def test_oracle_static_mode_accumulates_and_dynamic_does_not():
    cam = _cam(2.0, 2.0, 1.5, 1.0)
    pts = np.array([[[[0, 0, 1]]], [[[0.5, 0, 1]]], [[[0, 0, 2]]]], np.float32)     # [T=3, 1, 1, 3]
    cols = np.array([[[[1, 0, 0]]], [[[0, 1, 0]]], [[[0, 0, 1]]]], np.float32)
    st = ro.render_frames(pts, cols, cam, 4, 3)
    dy = ro.render_frames(pts, cols, cam, 4, 3, dynamic=True)
    assert [int(f.any(-1).sum()) for f in st] == [1, 2, 2] and [int(f.any(-1).sum()) for f in dy] == [1, 1, 1]
    assert st[2, 1, 2].tolist() == [255, 0, 0] and dy[2, 1, 2].tolist() == [0, 0, 255]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the device math header on the host, bit for bit against the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("render") / "render_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "render_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.rh_project.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_longlong,
                             C.c_void_p, C.c_void_p]
    L.rh_color_u8.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
    return L


def _host_project(L, pts, cam, z_near, w, h, id0):
    pts = np.ascontiguousarray(pts, np.float32)
    cam = np.ascontiguousarray(cam, np.float64)
    pix = np.empty(len(pts), np.int64)
    key = np.empty(len(pts), np.uint64)
    L.rh_project(pts.ctypes.data, len(pts), cam.ctypes.data, z_near, w, h, id0, pix.ctypes.data, key.ctypes.data)
    return pix, key


def test_host_math_matches_oracle_bit_for_bit(host_lib):
    rng = np.random.default_rng(0)
    w, h = 640, 480
    kept = 0
    for trial in range(20):
        cam = ro.camera_array(_extrinsic(rng), [[rng.uniform(50, 800), 0, w / 2 - 0.5], [0, rng.uniform(50, 800), h / 2 - 0.5],
                                                [0, 0, 1]])
        pts = np.c_[rng.uniform(-2, 2, (5000, 2)), rng.uniform(-1, 4, 5000)].astype(np.float32)
        pts[rng.random(5000) < 0.01] = np.nan
        z_near = [0.0, 0.1, 1.0][trial % 3]
        id0 = int(rng.integers(0, 2 ** 32 - 5000))
        pix, key = _host_project(host_lib, pts, cam, z_near, w, h, id0)
        opix, _, _, okey = ro.project(pts, cam, z_near, w, h, id0)
        assert np.array_equal(pix, opix) and np.array_equal(key, okey)
        kept += int((pix >= 0).sum())
    assert kept > 10000
    # the u + 0.5 boundaries: identity camera, q.z = 1, u = fx x + cx lands exactly on k - 0.5 and on its neighbours
    cam = _cam(2.0, 2.0, 1.5, 1.5)
    k = np.arange(-2, 8)
    x = (k - 2.0) / 2.0                      # u = k - 0.5 exactly
    xs = np.concatenate([x, np.nextafter(x.astype(np.float32), np.float32(np.inf)),
                         np.nextafter(x.astype(np.float32), np.float32(-np.inf))]).astype(np.float32)
    pts = np.c_[xs, np.zeros_like(xs), np.ones_like(xs)].astype(np.float32)
    pts = np.concatenate([pts, pts[:, [1, 0, 2]]])     # the same on v
    pix, key = _host_project(host_lib, pts, cam, 0.0, 6, 5, 0)
    opix, col, row, okey = ro.project(pts, cam, 0.0, 6, 5)
    assert np.array_equal(pix, opix) and np.array_equal(key, okey)
    assert col[:10].tolist() == [-1, -1, 0, 1, 2, 3, 4, 5, -1, -1]     # exactly at k - 0.5 -> pixel k
    # colours: every k / 255 step, the exact .5 steps, out of range, NaN
    c = np.concatenate([np.arange(256) / 255.0, (np.arange(255) + 0.5) / 255.0, rng.uniform(-0.5, 1.5, 10000),
                        [np.nan, -np.inf, np.inf, -0.0]]).astype(np.float32)
    out = np.empty(len(c), np.uint8)
    host_lib.rh_color_u8(np.ascontiguousarray(c).ctypes.data, len(c), out.ctypes.data)
    assert np.array_equal(out, ro.color_u8(c))
    assert np.array_equal(out[:256], np.arange(256))


# ------------------------------------------------------------------------------------------------------------------
# CPU: camera files and PLY
# ------------------------------------------------------------------------------------------------------------------
def test_camera_json_round_trip_against_the_open3d_fixture(tmp_path):
    cam = vis.read_pinhole_camera_parameters(CAMERA_JSON)
    assert (cam.intrinsic.width, cam.intrinsic.height) == (1920, 1080)
    assert cam.intrinsic.intrinsic_matrix.tolist() == [[935.5, 0, 959.5], [0, 935.5, 539.5], [0, 0, 1]]
    assert cam.extrinsic.tolist() == [[0.96, 0, 0.28, -0.25], [0, 1, 0, 0.125], [-0.28, 0, 0.96, 2.5], [0, 0, 0, 1]]
    out = tmp_path / "camera.json"
    vis.write_pinhole_camera_parameters(str(out), cam)
    assert json.load(open(out)) == json.load(open(CAMERA_JSON))
    back = vis.read_pinhole_camera_parameters(str(out))
    assert np.array_equal(back.extrinsic, cam.extrinsic) and np.array_equal(back.intrinsic.intrinsic_matrix,
                                                                             cam.intrinsic.intrinsic_matrix)
    # a camera from the inverse pose reproduces the fixture's extrinsic; the principal point is Open3D's
    pose = np.linalg.inv(cam.extrinsic)
    c2 = vis.camera_from_pose(pose, 935.5, 1920, 1080)
    assert np.abs(c2.extrinsic - cam.extrinsic).max() < 1e-15
    assert np.array_equal(c2.intrinsic.intrinsic_matrix, cam.intrinsic.intrinsic_matrix)
    bad = json.load(open(CAMERA_JSON))
    bad["class_name"] = "PinholeCameraIntrinsic"
    (tmp_path / "bad.json").write_text(json.dumps(bad))
    with pytest.raises(ValueError):
        vis.read_pinhole_camera_parameters(str(tmp_path / "bad.json"))


def _read_ply(path):
    data = open(path, "rb").read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    n = int(next(line.split()[2] for line in header if line.startswith("element vertex")))
    props = [line.split()[1:] for line in header if line.startswith("property")]
    dt = np.dtype([(name, {"double": "<f8", "uchar": "u1"}[kind]) for kind, name in props])
    assert len(data) - end == n * dt.itemsize
    return header, np.frombuffer(data[end:], dt)


def test_write_point_cloud_bytes(tmp_path):
    rng = np.random.default_rng(3)
    pts = rng.normal(0, 1, (2, 10, 15, 3)).astype(np.float32)
    # exact .5 steps: c * 255 == k + 0.5 in fp64 (Open3D rounds them up, numpy's round would go to even)
    halves = [c for c in ((np.arange(255) + 0.5) / 255.0) if c * 255.0 == math.floor(c * 255.0) + 0.5]
    assert any(int(c * 255.0) % 2 == 0 for c in halves)
    cols = rng.uniform(-0.2, 1.2, (300, 3))
    cols.reshape(-1)[:len(halves)] = halves
    cols = cols.reshape(2, 10, 15, 3)
    path = tmp_path / "cloud.ply"
    vis.write_point_cloud(str(path), torch.from_numpy(pts), torch.from_numpy(cols))
    header, rec = _read_ply(path)
    assert header == ["ply", "format binary_little_endian 1.0", "element vertex 300", "property double x",
                      "property double y", "property double z", "property uchar red", "property uchar green",
                      "property uchar blue", "end_header"]
    p64 = pts.reshape(-1, 3).astype(np.float64)
    assert np.array_equal(np.c_[rec["x"], rec["y"], rec["z"]], p64)
    rgb = np.c_[rec["red"], rec["green"], rec["blue"]]
    flat = cols.reshape(-1)
    expect = np.floor(np.clip(cols.reshape(-1, 3), 0, 1) * 255 + 0.5).astype(np.uint8)
    assert np.array_equal(rgb, expect)
    assert all(rgb.reshape(-1)[i] == math.floor(flat[i] * 255.0) + 1 for i in range(len(halves)))
    # fp32 colours round exactly like the renderer; no colours -> coordinates only
    vis.write_point_cloud(str(path), pts, cols.astype(np.float32))
    _, rec32 = _read_ply(path)
    assert np.array_equal(np.c_[rec32["red"], rec32["green"], rec32["blue"]], ro.color_u8(cols.reshape(-1, 3)))
    vis.write_point_cloud(str(path), pts.reshape(-1, 3))
    header, rec = _read_ply(path)
    assert rec.dtype.names == ("x", "y", "z") and len(rec) == 300
    with pytest.raises(ValueError):
        vis.write_point_cloud(str(path), pts, cols[:1])
    with pytest.raises(ValueError):
        vis.write_point_cloud(str(path), pts[..., :2])


def test_c_abi_rejects_bad_render_arguments():
    """Validation of the s3r_render_* entries happens before any CUDA call: status -1 and a message, no device needed."""
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_render_workspace_bytes(1920, 1080) == 1920 * 1080 * 8
    assert L.s3r_render_workspace_bytes(0, 10) == 0 and L.s3r_render_workspace_bytes(10, -1) == 0
    assert L.s3r_render_workspace_bytes(1 << 16, 1 << 15) == 0
    fake, odd = C.c_void_p(64), C.c_void_p(68)
    cam = (C.c_double * 16)(*([1.0] * 16))
    assert L.s3r_render_clear(None, 4, 3, None) == -1 and b"render_clear" in L.s3r_last_error()
    assert L.s3r_render_clear(odd, 4, 3, None) == -1 and L.s3r_render_clear(fake, 0, 3, None) == -1
    splat = lambda **kw: L.s3r_render_splat(*{**dict(pts=fake, mask=None, n=10, id0=0, cam=cam, z_near=0.0, w=4, h=3,
                                                     keys=fake, stream=None), **kw}.values())
    assert splat(n=1 << 31, id0=1 << 31) == -1 and b"render_splat" in L.s3r_last_error()      # T H W = 2^32
    for kw in (dict(pts=None), dict(keys=None), dict(keys=odd), dict(cam=None), dict(n=-1), dict(id0=-1), dict(w=0),
               dict(h=0), dict(w=1 << 16, h=1 << 15), dict(z_near=-1.0), dict(z_near=math.nan), dict(z_near=math.inf)):
        assert splat(**kw) == -1, kw
    for i in (0, 5, 11, 12, 15):
        for v in (math.nan, math.inf):
            bad = (C.c_double * 16)(*([1.0] * 16))
            bad[i] = v
            assert splat(cam=bad) == -1 and f"camera[{i}]".encode() in L.s3r_last_error()
    assert L.s3r_render_resolve(None, fake, 4, 3, fake, None) == -1 and b"render_resolve" in L.s3r_last_error()
    assert L.s3r_render_resolve(fake, None, 4, 3, fake, None) == -1
    assert L.s3r_render_resolve(fake, fake, 4, 3, None, None) == -1
    assert L.s3r_render_resolve(fake, fake, 0, 3, fake, None) == -1


def test_cpu_tensors_are_rejected():
    cam = vis.read_pinhole_camera_parameters(CAMERA_JSON)
    pts = torch.rand(2, 4, 4, 3)
    with pytest.raises(ValueError):
        vis.render_frames(pts, pts.clone(), cam)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _scene(seed, T, H, W, nan_frac=0.01):
    """Points in front of an identity camera with quantised depths (many equal fp32 depths across frames) and a few
    non-finite or behind-camera points; colours in [-0.1, 1.1] (clamped by the renderer)."""
    rng = np.random.default_rng(seed)
    pts = np.empty((T, H, W, 3), np.float32)
    pts[..., :2] = rng.uniform(-1, 1, (T, H, W, 2))
    pts[..., 2] = 1.0 + 0.25 * rng.integers(0, 8, (T, H, W))
    bad = rng.random((T, H, W)) < nan_frac
    pts[bad] = np.array([np.nan, 0, 1], np.float32)
    behind = rng.random((T, H, W)) < nan_frac
    pts[behind, 2] = -1.0
    cols = rng.uniform(-0.1, 1.1, (T, H, W, 3)).astype(np.float32)
    mask = rng.random((T, H, W)) < 0.8
    return pts, cols, mask


def _camera(w, h, focal, seed):
    """A roll about the optical axis and a shift: q.z = z + 0.5 exactly, so the quantised depths of _scene tie."""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-0.5, 0.5)
    E = np.eye(4)
    E[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    E[:2, 3] = rng.normal(0, 0.05, 2)
    E[2, 3] = 0.5
    K = [[focal, 0, w / 2 - 0.5], [0, focal, h / 2 - 0.5], [0, 0, 1]]
    return vis.PinholeCameraParameters(vis.PinholeCameraIntrinsic(w, h, K), E)


def _oracle(pts, cols, cam, mask=None, dynamic=False, z_near=0.0):
    c16 = ro.camera_array(cam.extrinsic, cam.intrinsic.intrinsic_matrix)
    return ro.render_frames(pts, cols, c16, cam.intrinsic.width, cam.intrinsic.height, mask=mask, dynamic=dynamic,
                            z_near=z_near)


@pytest.mark.gpu
@pytest.mark.parametrize("dynamic", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_gpu_frames_equal_the_oracle(dynamic, masked):
    pts, cols, mask = _scene(10 + 2 * dynamic + masked, 5, 24, 32)
    cam = _camera(40, 30, 12.0, 1)           # 768 points per frame into ~25 x 25 pixels: heavy collisions
    m = mask if masked else None
    z_near = 0.3 if masked else 0.0
    got = vis.render_frames(torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), cam,
                            mask=None if m is None else torch.from_numpy(m).cuda(), dynamic=dynamic, z_near=z_near)
    assert got.dtype == torch.uint8 and got.is_cuda and tuple(got.shape) == (5, 30, 40, 3)
    want = _oracle(pts, cols, cam, m, dynamic, z_near)
    assert np.array_equal(got.cpu().numpy(), want)
    lit = [int(f.any(-1).sum()) for f in want]
    print(f"dynamic={dynamic} masked={masked}: lit pixels per frame {lit}")
    assert min(lit) > 100


@pytest.mark.gpu
def test_gpu_1080p_static_and_dynamic_equal_the_oracle_and_are_reproducible():
    pts, cols, mask = _scene(20, 3, 160, 160)
    cam = _camera(1920, 1080, 120.0, 2)     # 25.6 k points per frame over ~160 x 160 pixels
    args = (torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), cam)
    mk = torch.from_numpy(mask).cuda()
    for dynamic in (False, True):
        got = vis.render_frames(*args, mask=mk, dynamic=dynamic)
        again = vis.render_frames(*args, mask=mk, dynamic=dynamic)
        assert torch.equal(got, again)
        assert np.array_equal(got.cpu().numpy(), _oracle(pts, cols, cam, mask, dynamic))
    # static frame i == frames 0..i drawn at once (one frame of (i + 1) H rows has the same global point indices)
    st = vis.render_frames(*args)
    for i in range(3):
        once = vis.render_frames(args[0][:i + 1].reshape(1, (i + 1) * 160, 160, 3),
                                 args[1][:i + 1].reshape(1, (i + 1) * 160, 160, 3), cam, dynamic=True)
        assert torch.equal(once[0], st[i])


@pytest.mark.gpu
def test_gpu_writes_the_reference_layout(tmp_path):
    import cv2
    pts, cols, _ = _scene(30, 4, 24, 32)
    cam = _camera(64, 48, 20.0, 3)
    frames = vis.render_frames(torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), cam, output_dir=str(tmp_path))
    for i in range(4):
        png = cv2.imread(str(tmp_path / "render_frames" / f"frame_{i:03d}.png"), cv2.IMREAD_UNCHANGED)
        assert np.array_equal(png[..., ::-1], frames[i].cpu().numpy())
    back = vis.read_pinhole_camera_parameters(str(tmp_path / "render_frames" / "camera.json"))
    assert np.array_equal(back.extrinsic, cam.extrinsic)
    cap = cv2.VideoCapture(str(tmp_path / "render_frame.mp4"))
    n = 0
    while cap.read()[0]:
        n += 1
    cap.release()
    assert n == 4
    # save_video / save_camera off: frames only
    out2 = tmp_path / "plain"
    vis.render_frames(torch.from_numpy(pts).cuda(), torch.from_numpy(cols).cuda(), cam, output_dir=str(out2),
                      save_video=False, save_camera=False)
    assert sorted(os.listdir(out2 / "render_frames")) == [f"frame_{i:03d}.png" for i in range(4)]
    assert not (out2 / "render_frame.mp4").exists()


@pytest.mark.gpu
def test_gpu_pipeline_render_of_a_forward_pass():
    """demo.py's --vis path on a real forward: 3 frames at 224 x 224 through Spann3R on the sharpened synthetic
    checkpoint, masked by (conf - 1) / conf > 1e-3, drawn from the first frame's pose.  Spann3R expresses every
    pointmap in frame 0's camera, so poses_all[0] is the identity; the synthetic weights' clouds are not camera-like
    (no usable focal or PnP pose), so the camera is pulled back along its optical axis and its focal framed to the cloud."""
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().eval()
    frames = synth.make_frames(3, 224, 224)
    with torch.no_grad():
        preds, _ = m(frames)
    pts_all = torch.cat([p["pts3d" if j == 0 else "pts3d_in_other_view"] for j, p in enumerate(preds)]).contiguous()
    conf = torch.cat([p["conf"] for p in preds])
    images_all = torch.cat([(f["img"].cuda().permute(0, 2, 3, 1) + 1.0) / 2.0 for f in frames]).contiguous()
    mask = (conf - 1) / conf > 1e-3
    kept = pts_all[mask].cpu().numpy()
    kept = kept[np.isfinite(kept).all(1)]
    lo, hi = np.percentile(kept, 2, axis=0), np.percentile(kept, 98, axis=0)
    pose = np.eye(4)                                  # poses_all[0]
    pose[:2, 3] = (lo[:2] + hi[:2]) / 2
    pose[2, 3] = lo[2] - (hi[2] - lo[2]) - 1e-3       # behind the cloud
    dist = (hi[2] - lo[2]) * 1.5 + 1e-3
    focal = 0.9 * 540 * dist / max(float(np.max(hi[:2] - lo[:2])) / 2, 1e-6)
    cam = vis.camera_from_pose(pose, focal, 1920, 1080)
    got = vis.render_frames(pts_all, images_all, cam, mask=mask)
    want = _oracle(pts_all.cpu().numpy(), images_all.cpu().numpy(), cam, mask.cpu().numpy())
    lit = [int(f.any(-1).sum()) for f in want]
    print(f"pipeline: focal {focal:.2f}, kept points {int(mask.sum())}, lit pixels per frame {lit}")
    assert np.array_equal(got.cpu().numpy(), want)
    assert lit[0] > 1000


@pytest.mark.gpu
def test_gpu_inputs_are_validated():
    cam = _camera(40, 30, 12.0, 1)
    good = torch.rand(2, 4, 4, 3, device="cuda")
    for bad in (good.cpu(), good.double(), good.half(), good[..., :2], good[0], good.reshape(2, 16, 1, 3)[:, :0],
                good.cpu().numpy()):
        for call in (lambda: vis.render_frames(bad, good, cam), lambda: vis.render_frames(good, bad, cam)):
            with pytest.raises(ValueError):
                call()
    with pytest.raises(ValueError):                     # shapes differ
        vis.render_frames(good, torch.rand(2, 4, 5, 3, device="cuda"), cam)
    for mask in (torch.ones(2, 4, 4, device="cuda"), torch.ones(2, 4, 4, dtype=torch.bool),
                 torch.ones(2, 4, 5, dtype=torch.bool, device="cuda"), np.ones((2, 4, 4), bool)):
        with pytest.raises(ValueError):
            vis.render_frames(good, good, cam, mask=mask)
    for z_near in (-1.0, math.nan, math.inf):
        with pytest.raises(ValueError):
            vis.render_frames(good, good, cam, z_near=z_near)

    def with_(K=None, E=None, w=40, h=30):
        K0 = np.array(cam.intrinsic.intrinsic_matrix)
        return vis.PinholeCameraParameters(vis.PinholeCameraIntrinsic(w, h, K0 if K is None else K),
                                           cam.extrinsic if E is None else E)
    skew = np.array(cam.intrinsic.intrinsic_matrix)
    skew[0, 1] = 0.5
    nan_k = np.array(cam.intrinsic.intrinsic_matrix)
    nan_k[0, 0] = math.nan
    inf_e = np.array(cam.extrinsic)
    inf_e[1, 3] = math.inf
    proj = np.array(cam.extrinsic)
    proj[3, 2] = 1.0
    for bad_cam in (with_(K=skew), with_(K=nan_k), with_(E=inf_e), with_(E=proj), with_(w=0), with_(h=-3),
                    with_(w=1 << 16, h=1 << 15), object()):
        with pytest.raises(ValueError):
            vis.render_frames(good, good, bad_cam)
