"""Training views on the GPU (spann3r_b200/train_views.py over csrc/jitter.cu and csrc/views.cu) against the reference's
training datasets with ColorJitter.

CPU: csrc/jitter_math.cuh compiled for the host against Pillow / torchvision (RGB <-> HSV and L on all 2^24 colours,
every hue shift hue=0.1 can draw and +-0.5, blend on all 65 536 pairs for 1004 factors, the contrast mean against
ImageStat); the host-compiled per-view pipeline against tvf.ColorJitter + ImgNorm for all 24 op orders; the numpy
oracle (oracle/jitter_oracle.py) against both; the worker half of TrainViews over synthetic Co3d, Scannetpp and
BlendMVS trees against the goldens of the real reference (tests/golden/train_views.json, written by
tools/make_golden_train_views.py): cropped depths, numpy / torch RNG states after each item, invalidations and
recursive retries; the oracle against the same goldens; a DataLoader with two workers planning without CUDA; pickling
a patched dataset; the refusal of an edited cropped depth.
GPU: every key of every golden view bit-identical; TrainViews.loader over two workers equal to the oracle's collated
batches; one training step on such a batch through the reference's default criterion.
"""
import ctypes as C
import hashlib
import itertools
import json
import os
import subprocess

import numpy as np
import PIL.Image
import PIL.ImageStat
import pytest
import torch
import torchvision.transforms as tvf
import torchvision.transforms.functional as TF

from conftest import GOLDEN, ROOT
from spann3r_b200 import synth

KEYS = ("img", "depthmap", "pts3d", "valid_mask", "camera_intrinsics", "camera_pose", "true_shape")
P = C.c_void_p


def _golden():
    with open(os.path.join(GOLDEN, "train_views.json")) as f:
        return json.load(f)


def _digest(a) -> str:
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _np_state(rng) -> str:
    return hashlib.sha256(json.dumps(rng.bit_generator.state, sort_keys=True).encode()).hexdigest()


def _torch_state() -> str:
    return hashlib.sha256(torch.get_rng_state().numpy().tobytes()).hexdigest()


CASES = range(4)     # co3d 224, co3d 512x384, scannetpp 224 (recursive retries), blendmvs 512x384 (ImgNorm, max())


def _dataset(root, case):
    kind = case.get("kind", "co3d")
    writer, cls = dict(co3d=(synth.write_co3d_tree, synth.Co3dLike),
                       scannetpp=(synth.write_scannetpp_tree, synth.ScannetppLike),
                       blendmvs=(synth.write_blendmvs_tree, synth.BlendMVSLike))[kind]
    writer(root, **case["tree"])
    d = dict(case["ds"])
    if not isinstance(d["resolution"], int):
        d["resolution"] = tuple(d["resolution"])
    return cls(root, jitter=case.get("jitter", True), **d)


def _count_retries(ds):
    """Wrap the instance's _get_views to count its recursive calls with attempts > 0."""
    n = [0]
    inner = ds._get_views

    def get_views(idx, resolution, rng, attempts=0):
        n[0] += attempts > 0
        return inner(idx, resolution, rng, attempts)

    if "attempts" in inner.__code__.co_varnames:
        ds._get_views = get_views
    return n


def _all_colours() -> np.ndarray:
    a = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(a >> 16) & 255, (a >> 8) & 255, a & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


@pytest.fixture(scope="module")
def jh(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("jitter") / "jitter_host_check.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(ROOT, "tests", "native", "jitter_host_check.cpp"), "-o", so])
    lib = C.CDLL(so)
    for name in ("jh_rgb_to_hsv", "jh_hsv_to_rgb", "jh_luma"):
        getattr(lib, name).argtypes = [P, C.c_longlong, P]
    lib.jh_shift_hue.argtypes = [P, C.c_longlong, C.c_int, P]
    lib.jh_blend.argtypes = [P, P, C.c_longlong, C.c_float, P]
    lib.jh_contrast_mean.argtypes = [C.c_longlong, C.c_longlong]
    lib.jh_contrast_mean.restype = C.c_int
    lib.jh_view.argtypes = [P, C.c_int, C.c_int, P, C.c_int, P, C.c_int, P]
    return lib


def _ptr(a):
    return a.ctypes.data_as(P)


def _host_view(jh, rgb, params) -> np.ndarray:
    from spann3r_b200.views import jitter_fields
    order, skip, facs, shift = jitter_fields(params)
    rgb = np.ascontiguousarray(rgb)
    h, w = rgb.shape[:2]
    out = np.empty((3, h, w), np.float32)
    jh.jh_view(_ptr(rgb), h, w, _ptr(np.array(order, np.int32)), skip, _ptr(np.array(facs, np.float32)), shift, _ptr(out))
    return out


def _tv_view(rgb, params) -> np.ndarray:
    """torchvision's ColorJitter.forward body with the given draw, then ImgNorm."""
    img = PIL.Image.fromarray(rgb)
    fns = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)
    names = ("brightness", "contrast", "saturation", "hue")
    for k in params["order"]:
        if params[names[k]] is not None:
            img = fns[k](img, params[names[k]])
    norm = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    return norm(img).numpy()


# ------------------------------------------------------------------------------------------------------------- CPU
def test_hsv_and_luma_on_every_colour(jh):
    rgb = _all_colours()
    n = C.c_longlong(1 << 24)
    out = np.empty_like(rgb)
    jh.jh_rgb_to_hsv(_ptr(rgb), n, _ptr(out))
    assert np.array_equal(out, np.asarray(PIL.Image.fromarray(rgb).convert("HSV")))
    jh.jh_hsv_to_rgb(_ptr(rgb), n, _ptr(out))           # every (h, s, v) triple
    assert np.array_equal(out, np.asarray(PIL.Image.fromarray(rgb, "HSV").convert("RGB")))
    lum = np.empty(rgb.shape[:2], np.uint8)
    jh.jh_luma(_ptr(rgb), n, _ptr(lum))
    assert np.array_equal(lum, np.asarray(PIL.Image.fromarray(rgb).convert("L")))


def test_hue_shift_every_reachable_shift(jh):
    """hue=0.1 draws factors in [-0.1, 0.1]: shifts -25..25; +-0.5 gives +-127.  1 M colours per shift, against
    torchvision's adjust_hue (which also fixes how the shift is truncated and wrapped)."""
    from spann3r_b200.views import jitter_fields
    g = np.random.default_rng(0)
    rgb = g.integers(0, 256, (1024, 1024, 3), dtype=np.uint8)
    out = np.empty_like(rgb)
    factors = sorted({float(np.float32(s / 255.0)) for s in range(-25, 26)} | {0.1, -0.1, 0.5, -0.5, 0.0999, -0.0999})
    for hue in factors:
        shift = jitter_fields(dict(order=(0, 1, 2, 3), brightness=None, contrast=None, saturation=None, hue=hue))[3]
        jh.jh_shift_hue(_ptr(rgb), C.c_longlong(rgb.shape[0] * rgb.shape[1]), shift, _ptr(out))
        assert np.array_equal(out, np.asarray(TF.adjust_hue(PIL.Image.fromarray(rgb), hue))), hue


def test_blend_all_pairs_for_drawn_factors(jh):
    """All 65 536 (in1, in2) pairs for 1000 factors drawn as torchvision draws them (uniform_ on fp32 over
    [0.5, 1.5]: both Pillow branches), plus 0 and 1 exactly and a few outside [0, 2]."""
    x1, x2 = (np.ascontiguousarray(a) for a in np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8)))
    torch.manual_seed(0)
    facs = [float(torch.empty(1).uniform_(0.5, 1.5)) for _ in range(1000)] + [0.0, 1.0, -0.25, 2.75]
    assert any(f < 1 for f in facs) and any(f > 1 for f in facs)
    out = np.empty_like(x1)
    im1, im2 = PIL.Image.fromarray(x1), PIL.Image.fromarray(x2)
    for a in facs:
        jh.jh_blend(_ptr(x1), _ptr(x2), C.c_longlong(65536), C.c_float(a), _ptr(out))
        assert np.array_equal(out, np.asarray(PIL.Image.blend(im1, im2, a))), a


def test_contrast_mean_against_imagestat(jh):
    g = np.random.default_rng(1)
    cases = [g.integers(0, 256, (h, w), dtype=np.uint8) for h, w in ((224, 224), (384, 512), (7, 3))]
    cases.append(np.array([[10, 11]], np.uint8))                  # mean exactly 10.5 -> 11
    cases.append(np.array([[0, 255, 255, 1]], np.uint8))          # mean exactly 127.75
    cases.append(np.array([[100, 101, 100, 101]], np.uint8))      # 100.5
    for L in cases:
        want = int(PIL.ImageStat.Stat(PIL.Image.fromarray(L)).mean[0] + 0.5)
        assert jh.jh_contrast_mean(int(L.astype(np.int64).sum()), L.size) == want


@pytest.mark.parametrize("shape", [(224, 224), (384, 512)])
def test_host_pipeline_equals_torchvision_for_every_order(jh, shape):
    from oracle import jitter_oracle as JO
    from oracle import views_oracle as VO
    from spann3r_b200.train_views import draw_jitter
    g = np.random.default_rng(sum(shape))
    torch.manual_seed(123)
    cj = tvf.ColorJitter(0.5, 0.5, 0.5, 0.1)
    for order in itertools.permutations(range(4)):
        rgb = g.integers(0, 256, shape + (3,), dtype=np.uint8)
        rgb[: shape[0] // 3] //= 3                               # a dark band: the blends clamp and truncate
        params = dict(draw_jitter(cj), order=order)
        want = _tv_view(rgb, params)
        assert np.array_equal(_host_view(jh, rgb, params), want), order
        assert np.array_equal(VO.img_norm(JO.color_jitter(rgb, params)), want), order


def test_host_pipeline_with_ops_off(jh):
    """ColorJitter(0, 0.3, 0, 0) (None factors skipped) and the None draw (ImgNorm only)."""
    from spann3r_b200.train_views import draw_jitter
    rgb = np.random.default_rng(2).integers(0, 256, (50, 70, 3), dtype=np.uint8)
    torch.manual_seed(4)
    params = draw_jitter(tvf.ColorJitter(0, 0.3, 0, 0))
    assert params["brightness"] is None and params["hue"] is None and params["contrast"] is not None
    assert np.array_equal(_host_view(jh, rgb, params), _tv_view(rgb, params))
    ident = dict(order=(0, 1, 2, 3), brightness=None, contrast=None, saturation=None, hue=None)
    assert np.array_equal(_host_view(jh, rgb, None), _tv_view(rgb, ident))


def test_transform_check():
    from spann3r_b200.train_views import split_transform
    norm = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
    assert split_transform(norm) is None
    cj = tvf.ColorJitter(0.2, 0, 0.4, 0.05)
    assert split_transform(tvf.Compose([cj, norm])) is cj
    for bad in (tvf.Compose([tvf.RandomHorizontalFlip(), norm]), tvf.Compose([norm, cj]), cj,
                tvf.Compose([cj, tvf.ToTensor()]), None):
        with pytest.raises(ValueError):
            split_transform(bad)


@pytest.mark.parametrize("ci", CASES)
def test_worker_half_matches_reference_goldens(tmp_path, ci):
    """The patched dataset's __getitem__ (no GPU, no library): per item the idx / strings / rng of every view, the
    numpy and torch generator states afterwards, Co3d's invalidated frames and the recursive retries of Scannetpp /
    BlendMVS equal the reference's; every cropped depth the dataset saw (BlendMVS reads its max) equals the oracle's
    cv2 crop."""
    from oracle import views_oracle as VO
    from spann3r_b200.train_views import TrainViews, PlannedViews
    c = _golden()["cases"][ci]
    ds = _dataset(str(tmp_path), c["case"])
    TrainViews(ds)
    seen = []
    orig = type(ds)._crop_resize_if_necessary

    def spy(self, image, depthmap, intrinsics, resolution, rng=None, info=None):
        state = rng.bit_generator.state
        out = orig(self, image, depthmap, intrinsics, resolution, rng, info)
        seen.append((np.asarray(image), depthmap, intrinsics, resolution, state, out[1]))
        return out

    ds._crop_resize_if_necessary = spy.__get__(ds)
    retries = _count_retries(ds)
    torch.manual_seed(c["case"]["torch_seed"])
    for item in c["items"]:
        before = retries[0]
        got = ds[item["idx"]]
        assert retries[0] - before == item["retries"]
        assert isinstance(got, PlannedViews) and len(got) == len(item["views"])
        for v, g in zip(got.views, item["views"]):
            assert v["rng"] == g["rng"] and list(v["idx"]) == g["idx"] and v["instance"] == g["instance"]
            assert _digest(v["true_shape"]) == g["sha256"]["true_shape"]
            assert _digest(v["camera_pose"]) == g["sha256"]["camera_pose"]
        assert _np_state(ds._rng) == item["np_state"]
        assert _torch_state() == item["torch_state"]
        assert sorted(i for r in getattr(ds, "invalidate", {}).values() for f in r.values() for i, x in enumerate(f)
                      if x) == item["invalidated"]
    assert len(seen) > sum(len(i["views"]) for i in c["items"])       # retries happened
    assert sum(i["retries"] for i in c["items"]) > 0 or c["case"]["kind"] == "co3d"
    for rgb, depth, K, res, state, cropped in seen:
        rng = np.random.default_rng()
        rng.bit_generator.state = state
        _, want, _, _ = VO.crop_resize(rgb, depth, K, res, 0, rng)
        assert cropped.dtype == want.dtype and np.array_equal(cropped, want)


@pytest.mark.parametrize("ci", CASES)
def test_oracle_matches_reference_goldens(tmp_path, ci):
    from oracle import jitter_oracle as JO
    c = _golden()["cases"][ci]
    ds = _dataset(str(tmp_path), c["case"])
    torch.manual_seed(c["case"]["torch_seed"])
    for item in c["items"]:
        views = JO.getitem(ds, item["idx"])
        for v, g in zip(views, item["views"]):
            for k in KEYS:
                assert _digest(v[k]) == g["sha256"][k], (item["idx"], k)
            assert v["rng"] == g["rng"]
        assert _torch_state() == item["torch_state"]


def test_patched_dataset_pickles(tmp_path):
    """A patched leaf survives pickling (DataLoader workers started with spawn / forkserver) and stays patched."""
    import pickle
    from spann3r_b200.train_views import TrainViews, PlannedViews
    c = _golden()["cases"][0]
    ds = _dataset(str(tmp_path), c["case"])
    TrainViews(ds)
    ds2 = pickle.loads(pickle.dumps(ds))
    assert type(ds2) is type(ds) and type(ds2).__name__ == "Co3dLike"
    torch.manual_seed(c["case"]["torch_seed"])
    item = ds2[0]
    assert isinstance(item, PlannedViews) and item.views[0]["rng"] == c["items"][0]["views"][0]["rng"]


def _collate_with_cuda_state(batch):
    """Runs in the worker after it planned the batch's items: reports whether the worker has initialised CUDA."""
    return batch, torch.cuda.is_initialized()


def test_dataloader_workers_plan_without_cuda(tmp_path):
    from torch.utils.data import DataLoader
    from spann3r_b200.train_views import TrainViews, PlannedViews
    c = _golden()["cases"][0]
    ds = _dataset(str(tmp_path), c["case"])
    TrainViews(ds)
    dl = DataLoader(ds, batch_size=2, num_workers=2, collate_fn=_collate_with_cuda_state)
    batches = [b for _, b in zip(range(3), dl)]
    assert not any(cuda for _, cuda in batches)
    assert all(isinstance(it, PlannedViews) for b, _ in batches for it in b)
    assert [it.views[0]["idx"][0] for b, _ in batches for it in b] == list(range(6))


def test_edited_cropped_depth_raises(tmp_path):
    """The device rebuilds the depth from the source window: a _get_views that edits the cropped depth is refused."""
    from spann3r_b200.train_views import TrainViews

    class Clips(synth.Co3dLike):
        def _get_views(self, idx, resolution, rng):
            views = super()._get_views(idx, resolution, rng)
            views[0]["depthmap"][views[0]["depthmap"] > 3] = 0
            return views

    c = _golden()["cases"][0]
    synth.write_co3d_tree(str(tmp_path), **c["case"]["tree"])
    ds = Clips(str(tmp_path), **c["case"]["ds"])
    TrainViews(ds)
    with pytest.raises(ValueError, match="changed the cropped depth"):
        ds[0]


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("ci", CASES)
def test_device_train_views_match_goldens(tmp_path, ci):
    from spann3r_b200.train_views import TrainViews
    c = _golden()["cases"][ci]
    ds = _dataset(str(tmp_path), c["case"])
    tv = TrainViews(ds)
    torch.manual_seed(c["case"]["torch_seed"])
    items = [ds[item["idx"]] for item in c["items"]]
    batch = tv.build(items)                             # every item of the case in one build_planned call
    for f, view in enumerate(batch):
        for b, item in enumerate(c["items"]):
            g = item["views"][f]
            for k in KEYS:
                got = view[k][b]
                assert _digest(got) == g["sha256"][k], (item["idx"], f, k)
            assert int(view["rng"][b]) == g["rng"]


def _seed_worker(worker_id):
    torch.manual_seed(1000 + worker_id)


def _oracle_batches(ds, idxs, bs):
    from torch.utils.data import default_collate
    from oracle import jitter_oracle as JO
    out = []
    for i in range(0, len(idxs) - bs + 1, bs):
        items = [JO.getitem(ds, j) for j in idxs[i:i + bs]]
        out.append([default_collate([it[f] for it in items]) for f in range(len(items[0]))])
    return out


@pytest.mark.gpu
def test_loader_with_workers_matches_oracle_and_trains(tmp_path):
    from conftest import get_state_dict
    from torch.utils.data import DataLoader, SequentialSampler
    from spann3r_b200 import Spann3R
    from spann3r_b200.loss import ConfLoss_t, L21, Regr3D_t
    from spann3r_b200.train_views import TrainViews
    c = _golden()["cases"][0]
    # a seeded dataset: each item's numpy RNG depends only on its index, and torch's draws in the workers come from
    # each worker's own seed, so the oracle replays them per worker
    ds = _dataset(str(tmp_path / "tv"), c["case"])
    tv = TrainViews(ds)
    base = DataLoader(ds, sampler=SequentialSampler(ds), batch_size=2, num_workers=2, drop_last=True,
                      worker_init_fn=_seed_worker)
    loader = tv.loader(base)
    assert len(loader) == len(base)
    got = [b for _, b in zip(range(2), loader)]
    # worker k serves batch k (items 2k, 2k + 1) with torch seeded 1000 + k and its own copy of the dataset (whose
    # invalidated frames it alone accumulates)
    ref = []
    for k in range(2):
        torch.manual_seed(1000 + k)
        ref.extend(_oracle_batches(_dataset(str(tmp_path / f"ref{k}"), c["case"]), [2 * k, 2 * k + 1], 2))
    for gb, rb in zip(got, ref):
        assert len(gb) == len(rb)
        for gv, rv in zip(gb, rb):
            for k in KEYS:
                assert torch.equal(gv[k].cpu(), torch.as_tensor(rv[k])), k
            assert torch.equal(gv["rng"], rv["rng"]) and gv["instance"] == rv["instance"]
            assert gv["img"].is_cuda and gv["pts3d"].is_cuda
    # one training step on the first batch with the reference's default criterion
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().train()
    crit = ConfLoss_t(Regr3D_t(L21, norm_mode="avg_dis", fix_first=False), alpha=0.4)
    preds, preds_all = m.forward(got[0])
    loss, details, factor_loss = crit.compute_frame_loss(got[0], preds_all)
    (loss + factor_loss).backward()
    assert torch.isfinite(torch.as_tensor(loss)) and torch.isfinite(torch.as_tensor(factor_loss))
    grads = [p.grad for p in m.parameters() if p.grad is not None]
    assert grads and all(torch.isfinite(g).all() for g in grads)
