"""Dataset views on the GPU (spann3r_b200/views.py over csrc/views.cu) against the reference's loaders.

CPU: the oracle (oracle/views_oracle.py) against the real reference's goldens (tests/golden/views.json, written by
tools/make_golden_views.py); plan_view against the oracle's geometry and RNG state; the nearest-index rule against cv2
itself; plan_frame unchanged; csrc/views_math.cuh compiled for the host against the oracle, bit for bit; the interface
raising without a GPU.
GPU: every output key bit-identical to the goldens; a batched sequence equal to single views; DeviceViews over a
7Scenes-layout scene of PNG files against the oracle, and its DataLoader batch through the model and the criterion.
"""
import ctypes as C
import hashlib
import json
import os
import subprocess

import cv2
import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from spann3r_b200 import synth
from spann3r_b200.synth import SevenScenesLike, write_7scenes_sequence

KEYS = ("img", "depthmap", "pts3d", "valid_mask", "camera_intrinsics", "camera_pose", "true_shape")


def _golden():
    with open(os.path.join(GOLDEN, "views.json")) as f:
        return json.load(f)


def _digest(a) -> str:
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# ------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_reference_golden():
    from oracle import views_oracle as VO
    for c in _golden()["cases"]:
        case = c["case"]
        views = VO.build_item(synth.make_view_case(case), tuple(case["res"]), case["aug"], case["seed"])
        assert len(views) == len(c["views"])
        for v, g in zip(views, c["views"]):
            for k in KEYS:
                assert _digest(v[k]) == g["sha256"][k], (case["name"], k)
            assert v["rng"] == g["rng"]


def test_golden_cases_cover_the_rules():
    """Both square-flip draws, portrait transposes, non-finite points and a view without pose are in the goldens."""
    by = {c["case"]["name"]: c for c in _golden()["cases"]}
    from oracle import views_oracle as VO
    case = by["square_512"]["case"]
    ts = {tuple(v["true_shape"]) for v in VO.build_item(synth.make_view_case(case), tuple(case["res"]), 0, case["seed"])}
    assert ts == {(384, 512), (512, 384)}
    assert all(v["valid"] < 224 * 224 * 0.85 for v in by["extreme_depth"]["views"])
    assert all(v["valid"] == 0 for v in by["no_pose"]["views"])


def test_plan_view_matches_oracle_and_rng():
    from oracle import views_oracle as VO
    from spann3r_b200.views import plan_view
    cases = [c["case"] for c in _golden()["cases"]]
    extra = [dict(h=h, w=w, K=K, res=res, aug=aug) for h, w, K, res, aug in [
        (480, 640, (525.0, 525.0, 320.5, 240.5), (224, 224), 0), (480, 640, (525.0, 525.0, 319.5, 239.5), (512, 384), 0),
        (1200, 1600, (2892.33, 2883.18, 823.205, 619.071), (224, 224), 5), (777, 1031, (900.0, 901.0, 515.2, 388.7),
                                                                           (512, 336), 0),
        (600, 610, (600.0, 600.0, 305.0, 300.0), (512, 384), 16), (1000, 400, (400.0, 400.0, 200.0, 500.0), (512, 384), 3)]]
    for case in cases + extra:
        fx, fy, cx, cy = case["K"]
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32)
        for seed in range(6):
            r1, r2 = np.random.default_rng(seed), np.random.default_rng(seed)
            h, w = case["h"], case["w"]
            dummy = np.zeros((h, w, 3), np.uint8)
            _, _, Ko, go = VO.crop_resize(dummy, np.zeros((h, w), np.float32), K, tuple(case["res"]), case["aug"], r1)
            p = plan_view(h, w, K, tuple(case["res"]), case["aug"], r2)
            for k in ("crop1", "scaled", "crop2", "out", "portrait"):
                assert tuple(np.atleast_1d(p[k])) == tuple(np.atleast_1d(go[k])), (case, k)
            assert p["K"].dtype == np.float32 and p["K"].tobytes() == np.float32(Ko).tobytes()
            assert r1.bit_generator.state == r2.bit_generator.state


def test_plan_view_refuses_what_the_reference_asserts():
    from spann3r_b200.views import plan_view
    K = np.array([[500, 0, 100], [0, 500, 240], [0, 0, 1]], np.float32)
    with pytest.raises(ValueError):
        plan_view(480, 640, K, 224)                               # principal point within a fifth of the border
    with pytest.raises(ValueError):
        plan_view(480, 640, np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1]], np.float32), (384, 512))   # portrait res


def test_nearest_index_is_cv2():
    from spann3r_b200.views import nearest_index
    g = np.random.default_rng(0)
    sizes = [(640, 224), (640, 298), (640, 299), (640, 300), (640, 341), (480, 224), (1600, 512), (1200, 384),
             (333, 517), (17, 3), (3, 17), (480, 480)] + [tuple(int(v) for v in g.integers(2, 2000, 2)) for _ in range(300)]
    for src, dst in sizes:
        a = np.arange(src, dtype=np.float32)[None, :].repeat(2, 0)
        got = cv2.resize(a, (dst, 2), fx=0.37, fy=0.37, interpolation=cv2.INTER_NEAREST)[0].astype(np.int64)
        assert np.array_equal(got, nearest_index(src, dst)), (src, dst)
        col = cv2.resize(a.T.copy(), (2, dst), interpolation=cv2.INTER_NEAREST)[:, 0].astype(np.int64)
        assert np.array_equal(col, nearest_index(src, dst)), (src, dst)


def test_plan_frame_unchanged():
    """The input adapter's pseudo-intrinsics geometry still matches its own golden-checked oracle."""
    from oracle import input_adapter_oracle as O
    from spann3r_b200 import preprocess as P
    with open(os.path.join(GOLDEN, "input_adapter.json")) as f:
        cases = json.load(f)["cases"]
    for c in cases:
        flip = bool(c["square_flip"])
        assert P.plan_frame(c["h"], c["w"], tuple(c["resolution"]), flip) == O.plan_frame(c["h"], c["w"],
                                                                                          tuple(c["resolution"]), flip)


@pytest.fixture(scope="module")
def host_math(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("views") / "views_host_check.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(ROOT, "tests", "native", "views_host_check.cpp"), "-o", so])
    lib = C.CDLL(so)
    lib.vh_points.restype = None
    lib.vh_points.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return lib


def _host_points(lib, depth, K, pose):
    h, w = depth.shape
    depth = np.ascontiguousarray(depth, np.float32)
    intr = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float32)
    rt = np.ascontiguousarray(pose[:3, :4], np.float32)
    cam, world = np.empty((h, w, 3), np.float32), np.empty((h, w, 3), np.float32)
    valid = np.empty((h, w), np.uint8)
    lib.vh_points(depth.ctypes.data, h, w, intr.ctypes.data, rt.ctypes.data, cam.ctypes.data, world.ctypes.data,
                  valid.ctypes.data)
    return cam, world, valid.astype(bool)


def test_views_math_host_matches_oracle(host_math):
    from oracle import views_oracle as VO
    for c in _golden()["cases"]:
        case = c["case"]
        rng = np.random.default_rng(case["seed"])
        for rgb, depth, K, pose in synth.make_view_case(case):
            _, d, Kf, _ = VO.crop_resize(rgb, depth, K, tuple(case["res"]), case["aug"], rng)
            pose = np.full((4, 4), np.nan, np.float32) if pose is None else pose
            cam0, world0, valid0 = VO.unproject(d, Kf, pose)
            cam1, world1, valid1 = _host_points(host_math, d, np.float32(Kf), pose)
            assert cam0.tobytes() == cam1.tobytes(), case["name"]
            assert world0.tobytes() == world1.tobytes(), case["name"]
            assert np.array_equal(valid0, valid1)


def test_interface_needs_gpu():
    from spann3r_b200 import views as V
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(Exception):
        V.ViewBuilder(224)
    with pytest.raises(Exception):
        V.DeviceViews(SevenScenesLike.__new__(SevenScenesLike))


# ------------------------------------------------------------------------------------------------- synthetic scene
def _oracle_scene_views(ds):
    """The same item through the oracle: the dataset's own decoding, then oracle.build_view per frame."""
    from oracle import views_oracle as VO
    calls = []

    def record(image, depthmap, intrinsics, resolution, rng=None, info=None):
        calls.append((image, depthmap, intrinsics))
        return None, None, intrinsics

    ds._crop_resize_if_necessary = record
    rng = np.random.default_rng(ds.seed)
    metas = ds._get_views(0, ds._resolutions[0], rng)
    del ds._crop_resize_if_necessary
    rng = np.random.default_rng(ds.seed)
    views = [VO.build_view(rgb, d, K, m["camera_pose"], ds._resolutions[0], ds.aug_crop, rng)
             for (rgb, d, K), m in zip(calls, metas)]
    for v in views:
        v["rng"] = int.from_bytes(rng.bytes(4), "big")
    return views


def test_device_views_refuse_without_gpu_or_wrong_transform(tmp_path):
    from spann3r_b200 import views as V
    ds = SevenScenesLike(str(tmp_path))
    ds.transform = lambda x: x
    with pytest.raises(Exception):
        V.DeviceViews(ds)


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_views_bit_identical_to_golden():
    from oracle import views_oracle as VO
    from spann3r_b200.views import ViewBuilder
    builders = {}
    for c in _golden()["cases"]:
        case = c["case"]
        key = (tuple(case["res"]), case["aug"])
        vb = builders.setdefault(key, ViewBuilder(key[0], aug_crop=case["aug"]))
        rng = np.random.default_rng(case["seed"])
        views = vb.build_sequence(synth.make_view_case(case), rng)
        torch.cuda.synchronize()
        for v, g in zip(views, c["views"]):
            for k in KEYS:
                assert list(v[k].shape) == g["shapes"][k], (case["name"], k)
                assert _digest(v[k]) == g["sha256"][k], (case["name"], k)     # == the real reference, bit for bit
            assert v["img"].is_cuda and v["pts3d"].is_cuda and v["valid_mask"].dtype == torch.bool
            assert int.from_bytes(rng.bytes(4), "big") == g["rng"]


@pytest.mark.gpu
def test_batched_equals_single():
    """One sequence of mixed geometries (portrait, square flips, aug_crop sizes, several source sizes) in one launch
    per pass equals the views built one at a time."""
    from oracle import views_oracle as VO
    from spann3r_b200.views import ViewBuilder
    cases = {c["case"]["name"]: c["case"] for c in _golden()["cases"]}
    inputs = []
    for name in ("7scenes_512", "dtu_512", "portrait_512", "square_512", "aug16_c"):
        inputs += synth.make_view_case(cases[name])
    vb = ViewBuilder((512, 384), aug_crop=16)
    batched = vb.build_sequence(inputs, np.random.default_rng(3))
    rng = np.random.default_rng(3)
    for inp, b in zip(inputs, batched):
        s = vb.build(*inp, rng=rng)
        for k in KEYS:
            assert torch.equal(b[k], s[k]) or (b[k].is_floating_point() and _digest(b[k]) == _digest(s[k])), k


@pytest.mark.gpu
def test_device_views_match_oracle_and_feed_the_model(tmp_path):
    from conftest import get_state_dict
    from torch.utils.data import DataLoader
    from spann3r_b200 import Spann3R
    from spann3r_b200.loss import L21Loss, Regr3D_t_ScaleShiftInv
    from spann3r_b200.views import DeviceViews
    root = str(tmp_path / "chess" / "seq-01")
    write_7scenes_sequence(root, frames=6)
    ref = _oracle_scene_views(SevenScenesLike(root))
    dv = DeviceViews(SevenScenesLike(root))
    got = dv[0]
    assert len(got) == len(ref) == 3
    for i, (g, r) in enumerate(zip(got, ref)):
        for k in KEYS:
            assert _digest(g[k]) == _digest(r[k]), k
        assert g["rng"] == r["rng"] and g["idx"] == (0, 0, i)
    # eval.py's loader over the wrapper: a batch the forward and the criterion take unchanged
    batch = next(iter(DataLoader(dv, batch_size=1, shuffle=False, num_workers=0)))
    assert batch[0]["img"].shape == (1, 3, 224, 224) and batch[0]["pts3d"].shape == (1, 224, 224, 3)
    for view in batch:
        for name in ("img", "pts3d", "valid_mask", "camera_pose", "camera_intrinsics"):
            view[name] = view[name].to("cuda", non_blocking=True)
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().eval()
    with torch.no_grad():
        preds, preds_all = m.forward(batch)
        gt_pts, pred_pts, *_ = Regr3D_t_ScaleShiftInv(L21Loss(), gt_scale=True).get_all_pts3d_t(batch, preds_all)
    assert len(preds) == 3 and all(torch.isfinite(p).all() for p in gt_pts)


@pytest.mark.gpu
def test_device_views_refuse_depth_readers_and_jitter(tmp_path):
    from spann3r_b200.views import DeviceViews

    class Co3d(SevenScenesLike):
        pass

    with pytest.raises(ValueError, match="ViewBuilder"):
        DeviceViews(Co3d(str(tmp_path)))
    ds = SevenScenesLike(str(tmp_path))
    import torchvision.transforms as tvf
    ds.transform = tvf.Compose([tvf.ColorJitter(0.5, 0.5, 0.5, 0.1), tvf.ToTensor(),
                                tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    with pytest.raises(ValueError, match="ImgNorm"):
        DeviceViews(ds)

    class ReadsDepth(SevenScenesLike):
        def _get_views(self, idx, resolution, rng):
            views = super()._get_views(idx, resolution, rng)
            for v in views:
                v["depthmap"][v["depthmap"] > 5] = 0
            return views

    write_7scenes_sequence(str(tmp_path), frames=2)
    with pytest.raises(TypeError, match="cropped depth"):
        DeviceViews(ReadsDepth(str(tmp_path)))[0]
