"""Training views on the GPU: the reference's training datasets (Co3d, BlendMVS, Scannetpp, habitat, Scannet,
ArkitScene) with `transform=ColorJitter` or ImgNorm, file decoding kept in the DataLoader's workers and the pixel work
done in the main process on the device, bit for bit.

The split follows the one the reference's loop needs: a worker runs the dataset's own `_get_views` (file decoding,
masks, frame sampling, the invalidate / retry loops, every numpy RNG draw) and plans each view; the main process builds
a whole batch with one `ViewBuilder.build_planned` call.  Workers never touch CUDA: this module imports and plans
without the library or a GPU.

* `split_transform(t)`: None for ImgNorm, the ColorJitter instance for `Compose([ColorJitter(...), ImgNorm])`;
  anything else raises ValueError.
* `draw_jitter(cj)`: one view's parameters, drawn with the instance's own `get_params` (torch's global RNG), as
  `ColorJitter.forward` draws them.
* `crop_depth(depth, plan)`: the cropped depth map `_crop_resize_if_necessary` returns, as a host array (a gather
  through the depth kernel's own index tables).
* `TrainViews(dataset)`: patches every leaf dataset behind the `@` / `*` / `+` wrappers so that indexing yields
  `PlannedViews`; `TrainViews.loader(data_loader)` turns the reference's DataLoader into one that yields the batches
  `default_collate` makes of the reference's views, with the tensors on the device.
"""
from __future__ import annotations

import numpy as np
import torch

from .views import _is_imgnorm, depth_index, plan_view

# keys the device builds; everything else of a view is collated as default_collate does
DEVICE_KEYS = ("img", "depthmap", "pts3d", "valid_mask", "camera_intrinsics", "camera_pose")


def split_transform(t):
    """ImgNorm -> None; Compose([ColorJitter(...), ImgNorm]) -> the ColorJitter; anything else -> ValueError."""
    if _is_imgnorm(t):
        return None
    ts = getattr(t, "transforms", None)
    if (type(t).__name__ == "Compose" and isinstance(ts, (list, tuple)) and len(ts) == 2
            and type(ts[0]).__name__ == "ColorJitter" and callable(getattr(ts[0], "get_params", None))
            and _is_imgnorm(ts[1])):
        return ts[0]
    raise ValueError("training views reproduce ImgNorm or Compose([ColorJitter(...), ImgNorm]) only; the dataset's "
                     f"transform is {t!r}")


def draw_jitter(cj) -> dict:
    """ColorJitter.get_params on the instance's ranges: torch.randperm(4), then one uniform_ per op that is not None."""
    fn_idx, b, c, s, h = cj.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
    return dict(order=tuple(int(k) for k in fn_idx), brightness=b, contrast=c, saturation=s, hue=h)


def crop_depth(depth: np.ndarray, plan: dict) -> np.ndarray:
    """Crop 1, cv2 INTER_NEAREST rescale and crop 2 of `depth` [h, w] as one gather (the depth kernel's tables)."""
    col_src, row_src = depth_index(plan)
    return depth[row_src[:, None], col_src[None, :]]


class PlannedViews:
    """What a patched dataset's `__getitem__` returns: per view, the uint8 crop-1 window of the image and of the depth
    map, the plan (relative to the window), the jitter parameters and every other key the reference's view carries
    except the ones the device builds.  Picklable, so DataLoader workers can hand it over."""

    def __init__(self, views):
        self.views = views

    def __len__(self):
        return len(self.views)


class _PlannedImage:
    """Stands in for the PIL image `_crop_resize_if_necessary` returns."""

    def __init__(self, rgb, depth, plan):
        self.rgb, self.depth, self.plan = rgb, depth, plan


def _is_good_type(v) -> bool:
    """base_stereo_view_dataset.is_good_type."""
    if isinstance(v, (str, int, tuple)):
        return True
    return getattr(v, "dtype", None) in (np.float32, torch.float32, bool, np.int32, np.int64, np.uint8)


class _Planned:
    """Mixin put in front of a leaf dataset's class: `_crop_resize_if_necessary` only plans and crops the depth on the
    host, `__getitem__` restates the base tail and returns PlannedViews."""

    def _crop_resize_if_necessary(self, image, depthmap, intrinsics, resolution, rng=None, info=None):
        rgb = np.asarray(image)
        if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3:
            raise ValueError(f"expected a uint8 RGB image [H, W, 3] (view {info})")
        depthmap = np.asarray(depthmap)
        if depthmap.shape != rgb.shape[:2]:
            raise ValueError(f"depth map {depthmap.shape} and image {rgb.shape[:2]} differ (view {info})")
        try:
            p = plan_view(rgb.shape[0], rgb.shape[1], intrinsics, resolution, self.aug_crop, rng)
        except ValueError as e:
            raise AssertionError(f"{e} (view {info})") from None
        l, t, r, b = p["crop1"]
        win = dict(p, crop1=(0, 0, r - l, b - t))
        rgb_w = np.ascontiguousarray(rgb[t:b, l:r])
        depth_w = np.ascontiguousarray(depthmap[t:b, l:r])
        return _PlannedImage(rgb_w, depth_w, win), crop_depth(depth_w, win), p["K"]

    def __getitem__(self, idx):
        if isinstance(idx, tuple):
            idx, ar_idx = idx
        else:
            assert len(self._resolutions) == 1
            ar_idx = 0
        if self.seed:
            self._rng = np.random.default_rng(seed=self.seed + idx)
        elif not hasattr(self, "_rng"):
            self._rng = np.random.default_rng(seed=torch.initial_seed())
        resolution = self._resolutions[ar_idx]
        views = self._get_views(idx, resolution, self._rng)
        cj = split_transform(self.transform)
        out = []
        for v, view in enumerate(views):
            assert "pts3d" not in view, "pts3d should not be there"
            raw = view.pop("img")
            if not isinstance(raw, _PlannedImage):
                raise ValueError("a view did not go through _crop_resize_if_necessary")
            view["idx"] = (idx, ar_idx, v)
            W, H = raw.plan["out"]
            view["true_shape"] = np.int32((H, W))
            jit = draw_jitter(cj) if cj is not None else None     # where the reference calls self.transform
            assert "camera_intrinsics" in view
            if "camera_pose" not in view:
                view["camera_pose"] = np.full((4, 4), np.nan, dtype=np.float32)
            else:
                assert np.isfinite(view["camera_pose"]).all(), "NaN in camera pose"
            assert "valid_mask" not in view
            depth = view.pop("depthmap")
            assert np.isfinite(depth).all(), "NaN in depthmap"
            if not np.array_equal(depth, crop_depth(raw.depth, raw.plan)):
                # the device rebuilds depthmap / pts3d / valid_mask from the source window, so an edit would be lost
                raise ValueError(f"_get_views changed the cropped depth map of view {v}; the device cannot reproduce "
                                 "that edit")
            for key, val in view.items():
                assert _is_good_type(val), f"bad type of {key}"
            view["camera_intrinsics"] = np.float32(view["camera_intrinsics"])
            view["camera_pose"] = np.float32(view["camera_pose"])
            view["_raw"] = (raw.rgb, raw.depth, raw.plan)
            view["_jitter"] = jit
            out.append(view)
        for view in out:
            view["rng"] = int.from_bytes(self._rng.bytes(4), "big")
        return PlannedViews(out)

    def __reduce_ex__(self, protocol):
        return _replan, (type(self).__mro__[2], self.__dict__)


_PLANNED_CLASSES = {}


def _planned_class(cls):
    pc = _PLANNED_CLASSES.get(cls)
    if pc is None:
        pc = _PLANNED_CLASSES[cls] = type(cls.__name__, (_Planned, cls), {"__module__": cls.__module__,
                                                                          "__qualname__": cls.__qualname__})
    return pc


def _replan(cls, state):
    obj = cls.__new__(_planned_class(cls))
    obj.__dict__.update(state)
    return obj


def leaves(dataset) -> list:
    """The leaf datasets behind the reference's MulDataset / ResizedDataset (`.dataset`) and CatDataset
    (`.datasets`) wrappers, in order."""
    if hasattr(dataset, "datasets"):
        return [leaf for d in dataset.datasets for leaf in leaves(d)]
    if hasattr(dataset, "dataset"):
        return leaves(dataset.dataset)
    return [dataset]


def _collate_planned(batch):
    """The loader's collate: a batch stays a list of PlannedViews on the host."""
    return batch


class TrainViews:
    """Wraps a training dataset expression of the reference (`10000 @ Co3d(...) + ...`) in place: every leaf's class
    gets a `_Planned` mixin in front of it (same name, same instance state), so its `__getitem__` returns PlannedViews
    and nothing above it is re-wrapped (`set_epoch`, `set_ratio`, `make_sampler` keep working).  A leaf's transform
    must be ImgNorm or Compose([ColorJitter(...), ImgNorm]); a leaf is duck-typed as a BaseStereoViewDataset (it reads
    `_get_views`, `_resolutions`, `seed`, `aug_crop` and `transform`)."""

    def __init__(self, dataset, device="cuda"):
        self.dataset = dataset
        self.device = device
        self._builders = {}
        for leaf in leaves(dataset):
            missing = [a for a in ("_get_views", "_resolutions", "seed", "aug_crop", "transform") if not hasattr(leaf, a)]
            if missing:
                raise ValueError(f"{type(leaf).__name__} is not a BaseStereoViewDataset (it lacks {', '.join(missing)})")
            split_transform(getattr(leaf, "transform", None))
            if not isinstance(leaf, _Planned):
                leaf.__class__ = _planned_class(type(leaf))

    def _builder(self, resolution):
        from .views import ViewBuilder
        key = tuple(resolution)
        b = self._builders.get(key)
        if b is None:
            b = self._builders[key] = ViewBuilder(key, device=self.device)     # plans come from the workers
        return b

    def build(self, items) -> list:
        """A list of B PlannedViews of F views each -> what default_collate makes of the reference's B items: a list of
        F dicts, device tensors [B, ...] for DEVICE_KEYS, host values collated as default_collate does."""
        from torch.utils.data import default_collate
        if not items:
            return []
        F = len(items[0])
        if any(len(it) != F for it in items):
            raise ValueError("items of one batch have different numbers of views")
        flat = [v for it in items for v in it.views]
        planned, jitter = [], []
        for v in flat:
            rgb, depth, plan = v["_raw"]
            planned.append((rgb, depth, v["camera_pose"], dict(plan, K=v["camera_intrinsics"])))
            jitter.append(v["_jitter"])
        res = tuple(int(s) for s in flat[0]["true_shape"][::-1])
        res = (max(res), min(res))
        if any(tuple(sorted((int(s) for s in v["true_shape"]), reverse=True)) != res for v in flat):
            raise ValueError("views of one batch have different resolutions")
        builder = self._builder(res)
        built = builder.build_planned(planned, jitter if any(j is not None for j in jitter) else None)
        B = len(items)
        out = []
        for f in range(F):
            views = [built[b * F + f] for b in range(B)]
            host = [items[b].views[f] for b in range(B)]
            d = {k: torch.stack([v[k] for v in views]) for k in DEVICE_KEYS}
            for k in host[0]:
                if k in ("_raw", "_jitter") or k in DEVICE_KEYS:
                    continue
                d[k] = default_collate([h[k] for h in host])
            out.append(d)
        return out

    def loader(self, data_loader):
        """The DataLoader `get_data_loader` built, rebuilt with the same dataset, sampler, batch size, workers,
        drop_last, generator, worker_init_fn, persistent_workers, prefetch_factor, multiprocessing_context, timeout and
        in_order, but a collate that keeps PlannedViews on the host and no pinning (each batch reaches the device in
        one pinned copy of its own); iterating the result yields device batches.  The original's collate_fn and
        pin_memory_device are not used."""
        from torch.utils.data import DataLoader
        if data_loader.dataset is not self.dataset:
            raise ValueError("the DataLoader serves another dataset than this TrainViews")
        kw = dict(num_workers=data_loader.num_workers, drop_last=data_loader.drop_last, generator=data_loader.generator,
                  worker_init_fn=data_loader.worker_init_fn, timeout=data_loader.timeout,
                  multiprocessing_context=data_loader.multiprocessing_context)
        if hasattr(data_loader, "in_order"):
            kw["in_order"] = data_loader.in_order
        if data_loader.num_workers:
            kw.update(persistent_workers=data_loader.persistent_workers, prefetch_factor=data_loader.prefetch_factor)
        dl = DataLoader(data_loader.dataset, sampler=data_loader.sampler, batch_size=data_loader.batch_size,
                        collate_fn=_collate_planned, pin_memory=False, **kw)
        return _DeviceLoader(self, dl)


class _DeviceLoader:
    def __init__(self, tv, dl):
        self.tv, self.data_loader = tv, dl
        self.dataset, self.sampler = dl.dataset, dl.sampler

    def __len__(self):
        return len(self.data_loader)

    def __iter__(self):
        for items in self.data_loader:
            yield self.tv.build(items)
