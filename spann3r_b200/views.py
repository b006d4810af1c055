"""Dataset views on the GPU: decoded image + depth map + intrinsics + pose -> the view dicts the reference's datasets
yield, bit for bit.

The reference builds every view of its evaluation and training datasets on the CPU
(dust3r/datasets/base/base_stereo_view_dataset.py:63-194 `__getitem__` / `_crop_resize_if_necessary`,
dust3r/datasets/utils/cropping.py, dust3r/utils/geometry.py:165-217): crop on the principal point, Pillow Lanczos
rescale of the image and cv2 INTER_NEAREST rescale of the depth, centred crop, intrinsics moved through both crops and
the rescale, ImgNorm, unprojection of the depth into world points, `valid_mask`, and `transpose_to_landscape` for
portrait views.  Here the host keeps only the geometry and the RNG draws (`plan_view`); the pixels go through three
kernels per sequence in libspann3r_b200.so (csrc/views.cu): the fused depth -> depthmap / pts3d / valid_mask pass and
the input adapter's Lanczos passes with a view index in the grid.

* `plan_view(h, w, K, resolution, aug_crop, rng)`: the crop geometry and final intrinsics, drawing from `rng` exactly
  as the reference does.
* `ViewBuilder(resolution, aug_crop, device)`: views from arrays, one at a time or a sequence per launch.
* `DeviceViews(dataset)`: wraps one of the reference's evaluation datasets (SevenScenes, NRGBD, DTU, Demo) so that
  indexing it yields the same views, built on the device.

File decoding stays on the CPU.  No CPU fallback: without the library or an H100 this raises.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict

import numpy as np
import torch

from . import _lib
from .preprocess import lanczos_coeffs

# Datasets whose `_get_views` reads the depth map after `_crop_resize_if_necessary` (class names of the reference's
# training sets).  DeviceViews cannot hand them the cropped depth, so it refuses them; build their views with
# ViewBuilder directly.
CROPPED_DEPTH_READERS = ("Co3d", "ArkitScene", "Scannet", "Scannetpp", "habitat", "BlendMVS")


def nearest_index(src: int, dst: int) -> np.ndarray:
    """Source index of each of `dst` output positions of cv2.resize(..., dsize, interpolation=INTER_NEAREST) along an
    axis of `src` samples: min(floor(x * (1 / (dst / src))), src - 1) in fp64, OpenCV's resizeNN.  cv2 ignores fx / fy
    when dsize is given, as cropping.py:72 gives both."""
    ifx = 1.0 / (dst / src)
    return np.minimum(np.floor(np.arange(dst, dtype=np.int64) * ifx).astype(np.int64), src - 1)


def depth_index(plan) -> tuple:
    """Source column of every output column and source row of every output row of a planned view's depth map (int32):
    crop 1, cv2 INTER_NEAREST rescale and crop 2 folded into two index tables (what the depth kernel gathers through)."""
    l, t, r, b = plan["crop1"]
    W2, H2 = plan["scaled"]
    l2, t2, r2, b2 = plan["crop2"]
    return ((l + nearest_index(r - l, W2)[l2:r2]).astype(np.int32),
            (t + nearest_index(b - t, H2)[t2:b2]).astype(np.int32))


def _to_colmap_scaled_shifted(K, scaling, offset):
    """camera_matrix_of_crop's arithmetic on a copy of K (cropping.py:82-95): +0.5 on the principal point, rows 0-1
    times `scaling`, principal point minus `offset`, -0.5.  In-place numpy operations on K's dtype, so the float32 /
    float64 promotion of every step is numpy's."""
    K = K.copy()
    K[0, 2] += 0.5
    K[1, 2] += 0.5
    K[:2, :] *= scaling
    K[:2, 2] -= offset
    K[0, 2] -= 0.5
    K[1, 2] -= 0.5
    return K


def plan_view(h: int, w: int, K, resolution, aug_crop=0, rng=None) -> dict:
    """Geometry of `_crop_resize_if_necessary` (base_stereo_view_dataset.py:143-194) for an [h, w] view with
    intrinsics K (3x3), resolution (W, H) with W >= H.  Draws from `rng` (a numpy Generator) where the reference does,
    in the same order: `integers(2)` only for a nearly square crop and a non-square resolution, then
    `integers(0, aug_crop)` only when aug_crop > 1.

    Returns dict(crop1=(l, t, r, b) on the source, scaled=(W2, H2) the rescale target, crop2=(l, t, r, b) on the
    rescaled view, out=(W, H) of the view before any transpose, K=float32 [3, 3] final intrinsics (not transposed),
    portrait=True when W < H, i.e. when the view is stored transposed).  Raises ValueError where the reference asserts."""
    K = np.array(K)
    if K.shape != (3, 3) or K.dtype.kind != "f":
        raise ValueError("K must be a 3x3 floating-point matrix")
    res = (resolution, resolution) if isinstance(resolution, int) else tuple(int(v) for v in resolution)
    if res[0] < res[1]:
        raise ValueError("resolution must be (W, H) with W >= H")
    # crop 1, centred on the rounded principal point (np.round: half to even); numpy int64 like the reference's
    cx, cy = K[:2, 2].round().astype(int)
    mx, my = min(cx, w - cx), min(cy, h - cy)
    if not (mx > w / 5 and my > h / 5):
        raise ValueError(f"principal point ({K[0, 2]}, {K[1, 2]}) too close to the border of a {w}x{h} view")
    l, t = cx - mx, cy - my
    K1 = K.copy()
    K1[0, 2] -= l
    K1[1, 2] -= t
    W1, H1 = int(2 * mx), int(2 * my)
    # portrait / square rule, then the aug_crop draw
    if H1 > 1.1 * W1:
        res = res[::-1]
    elif 0.9 < H1 / W1 < 1.1 and res[0] != res[1]:
        if rng is None:
            raise ValueError("a nearly square view needs `rng` for the reference's orientation draw")
        if rng.integers(2):
            res = res[::-1]
    target = np.array(res)
    if aug_crop > 1:
        if rng is None:
            raise ValueError("aug_crop > 1 needs `rng`")
        target += rng.integers(0, aug_crop)
    # rescale so that the view contains the target (rescale_image_depthmap), intrinsics through it
    size1 = np.array((W1, H1))
    scale_final = max(target / size1) + 1e-8
    size2 = np.floor(size1 * scale_final).astype(int)
    K2 = _to_colmap_scaled_shifted(K1, scale_final, 0.5 * (size1 * scale_final - size2))
    # centred crop to the resolution (camera_matrix_of_crop + bbox_from_intrinsics_in_out), intrinsics through it
    W2, H2 = int(size2[0]), int(size2[1])
    K3 = _to_colmap_scaled_shifted(K2, 1, 0.5 * (np.asarray((W2, H2)) * 1 - res))
    l2, t2 = np.int32(np.round(K2[:2, 2] - K3[:2, 2]))
    Kf = K2.copy()
    Kf[0, 2] -= l2
    Kf[1, 2] -= t2
    l2, t2 = int(l2), int(t2)
    return dict(crop1=(int(l), int(t), int(l) + W1, int(t) + H1), scaled=(W2, H2), crop2=(l2, t2, l2 + res[0], t2 + res[1]),
                out=res, K=Kf.astype(np.float32), portrait=res[0] < res[1])


JITTER_OPS = ("brightness", "contrast", "saturation", "hue")   # torchvision's fn_idx numbering


def jitter_fields(params):
    """One view's ColorJitter draw (None, or dict(order, brightness, contrast, saturation, hue)) -> the descriptor's
    (order, skip mask, (b, c, s) fp32 factors, hue shift).  The shift is np.int32(hue * 255), which adjust_hue adds to
    the uint8 hue (wrapping mod 256)."""
    if params is None:
        return (0, 1, 2, 3), 0xF, (1.0, 1.0, 1.0), 0
    order = tuple(int(k) for k in params["order"])
    if sorted(order) != [0, 1, 2, 3]:
        raise ValueError(f"jitter order {order} is not a permutation of 0..3")
    skip = sum(1 << k for k, name in enumerate(JITTER_OPS) if params.get(name) is None)
    facs = []
    for name in JITTER_OPS[:3]:
        f = params.get(name)
        if f is not None and float(np.float32(f)) != float(f):
            raise ValueError(f"{name} factor {f!r} is not an fp32 value (torchvision draws them in fp32)")
        facs.append(1.0 if f is None else float(f))
    hue = params.get("hue")
    if hue is not None and not -0.5 <= hue <= 0.5:
        raise ValueError(f"hue factor {hue} is not in [-0.5, 0.5]")
    return order, skip, tuple(facs), 0 if hue is None else int(np.int32(hue * 255))


def _as_rgb(rgb) -> np.ndarray:
    if isinstance(rgb, torch.Tensor):
        rgb = rgb.cpu().numpy()
    rgb = np.asarray(rgb)
    if rgb.dtype != np.uint8 or rgb.ndim != 3 or rgb.shape[2] != 3:
        raise ValueError("expected a uint8 RGB image [H, W, 3]")
    return rgb


def _as_depth(depth, h, w) -> np.ndarray:
    if isinstance(depth, torch.Tensor):
        depth = depth.cpu().numpy()
    depth = np.asarray(depth)
    if depth.dtype != np.float32 or depth.shape != (h, w):
        raise ValueError(f"expected a float32 depth map of the image's size ({h}, {w}), got {depth.dtype} {depth.shape}")
    return depth


def _as_pose(pose) -> np.ndarray:
    if pose is None:
        return np.full((4, 4), np.nan, dtype=np.float32)          # a view without pose (base_stereo...:93-94)
    if isinstance(pose, torch.Tensor):
        pose = pose.cpu().numpy()
    pose = np.asarray(pose)
    if pose.dtype != np.float32 or pose.shape != (4, 4):
        raise ValueError("camera_pose must be a float32 4x4 cam-to-world matrix")
    if not np.isfinite(pose).all():
        raise ValueError("NaN in camera pose")
    return pose


def _align(n: int, a: int = 256) -> int:
    return (n + a - 1) // a * a


class ViewBuilder:
    """uint8 RGB [h, w, 3] + float32 depth [h, w] + K + float32 cam-to-world pose (or None) -> the reference's view
    dict on the device: img [3, H, W] f32, depthmap [H, W] f32, pts3d [H, W, 3] f32 (world), valid_mask [H, W] bool,
    camera_intrinsics [3, 3] f32, camera_pose [4, 4] f32, and true_shape int32 (height, width) before the landscape
    transpose (a host tensor, as the reference's collated batch has it).  (H, W) = (resolution[1], resolution[0]):
    portrait views come out transposed, as transpose_to_landscape leaves them.  Coefficient and index tables are
    cached on the device for the MAX_GEOMETRIES most recently used geometries."""

    # Training sets give nearly every frame its own crop geometry (the crop-1 window follows the principal point), so
    # the per-geometry device tables (a few tens of KB each) are kept for the most recently used geometries only.
    MAX_GEOMETRIES = 512

    def __init__(self, resolution, aug_crop=0, device="cuda"):
        _lib.require_device()
        res = (resolution, resolution) if isinstance(resolution, int) else tuple(int(v) for v in resolution)
        if res[0] < res[1]:
            raise ValueError("resolution must be (W, H) with W >= H")
        self.resolution = res
        self.aug_crop = aug_crop
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("ViewBuilder builds views on a CUDA device")
        self._tables = OrderedDict()     # least recently used first; at most MAX_GEOMETRIES entries
        L = _lib.lib()
        if (L.s3r_views_abi_sizeof(0) != C.sizeof(_lib.ViewDepthDesc)
                or L.s3r_views_abi_sizeof(1) != C.sizeof(_lib.ViewImageDesc)
                or L.s3r_views_abi_sizeof(2) != C.sizeof(_lib.ViewJitterDesc)):
            raise _lib.S3RError("libspann3r_b200.so's view descriptors do not match the bindings: rebuild it")

    def plan(self, h: int, w: int, K, rng=None) -> dict:
        return plan_view(h, w, K, self.resolution, self.aug_crop, rng)

    def build(self, rgb, depth, K, pose=None, rng=None) -> dict:
        return self.build_sequence([(rgb, depth, K, pose)], rng)[0]

    def build_sequence(self, views, rng=None) -> list:
        """views: (rgb, depth, K, pose) per view; planned in order, each drawing from `rng` as the reference does."""
        planned = []
        for rgb, depth, K, pose in views:
            rgb = _as_rgb(rgb)
            planned.append((rgb, depth, pose, self.plan(rgb.shape[0], rgb.shape[1], K, rng)))
        return self.build_planned(planned)

    def _geometry(self, h, w, p):
        """Device tables of one view geometry: Lanczos bounds / taps restricted to the kept columns / rows (as
        FrameAdapter), and the depth's source column / row of every output column / row."""
        key = (h, w, p["crop1"], p["scaled"], p["crop2"])
        g = self._tables.get(key)
        if g is not None:
            self._tables.move_to_end(key)
        else:
            l, t, r, b = p["crop1"]
            W1, H1 = r - l, b - t
            W2, H2 = p["scaled"]
            l2, t2, r2, b2 = p["crop2"]
            bh, kh, ksh = lanczos_coeffs(W1, W2)
            bv, kv, ksv = lanczos_coeffs(H1, H2)
            bh, kh = bh[l2:r2], kh[l2:r2]
            bv, kv = bv[t2:b2].copy(), kv[t2:b2]
            row0 = int(bv[0, 0])
            rows = int(bv[-1, 0] + bv[-1, 1]) - row0
            bv[:, 0] -= row0
            n = bh.shape[0]
            span = max(int(bh[min(x0 + 127, n - 1), 0] + bh[min(x0 + 127, n - 1), 1] - bh[x0, 0]) for x0 in range(0, n, 128))
            col_src, row_src = depth_index(p)
            parts = [bh, kh, bv, kv, col_src, row_src]
            offs = np.cumsum([0] + [a.size for a in parts])
            flat = np.concatenate([np.ascontiguousarray(a, dtype=np.int32).ravel() for a in parts])
            dev = torch.from_numpy(flat).to(self.device)
            base = dev.data_ptr()
            ptrs = [base + 4 * int(o) for o in offs[:-1]]
            g = dict(tables=dev, bh=ptrs[0], kh=ptrs[1], bv=ptrs[2], kv=ptrs[3], col_src=ptrs[4], row_src=ptrs[5],
                     ksh=ksh, ksv=ksv, span=span, src_row0=t + row0, src_col0=l, rows=rows)
            self._tables[key] = g
            if len(self._tables) > self.MAX_GEOMETRIES:
                self._tables.popitem(last=False)   # device memory goes back to the stream-ordered caching allocator
        return g

    @torch.no_grad()
    def build_planned(self, planned, jitter=None) -> list:
        """planned: (rgb, depth, pose, plan) per view, `plan` from plan_view (its K may be replaced by the intrinsics
        the caller keeps).  One host-to-device copy and three launches for the whole list.

        jitter: None (ImgNorm only), or one entry per view: None or the parameters torchvision's ColorJitter drew for
        it, dict(order=fn_idx, brightness=, contrast=, saturation=, hue=) with None for an op that does not run (what
        train_views.draw_jitter returns).  Then the vertical Lanczos pass stops at uint8 and a fourth launch applies
        ColorJitter and ImgNorm (csrc/jitter.cu)."""
        n = len(planned)
        if n == 0:
            return []
        if n > 65535:
            raise ValueError("at most 65535 views per call")
        if jitter is not None:
            jitter = list(jitter)
            if len(jitter) != n:
                raise ValueError(f"jitter has {len(jitter)} entries for {n} views")
            jitter = [jitter_fields(j) for j in jitter]
        Wr, Hr = self.resolution
        dev = self.device
        views = []
        for rgb, depth, pose, p in planned:
            rgb = _as_rgb(rgb)
            h, w = rgb.shape[:2]
            depth = _as_depth(depth, h, w)
            K = np.asarray(p["K"], dtype=np.float32)
            if K[0, 1] != 0.0 or K[1, 0] != 0.0:
                raise ValueError("intrinsics with skew are not supported (the reference asserts on them)")
            if (p["out"][0], p["out"][1])[:: -1 if p["portrait"] else 1] != (Wr, Hr):
                raise ValueError(f"plan for resolution {p['out']} does not match the builder's {self.resolution}")
            views.append((rgb, depth, _as_pose(pose), p, K, self._geometry(h, w, p)))
        # one host buffer: images, depths, intrinsics + poses, then the two descriptor arrays (written last, once the
        # device addresses are known)
        off, lay = 0, []
        for rgb, depth, *_ in views:
            lay.append((off, _align(off + rgb.nbytes)))
            off = _align(lay[-1][1] + depth.nbytes)
        kp_off = off
        off = _align(kp_off + n * 25 * 4)
        dd_off = off
        off = _align(dd_off + n * C.sizeof(_lib.ViewDepthDesc))
        id_off = off
        off = _align(id_off + n * C.sizeof(_lib.ViewImageDesc))
        jd_off = off
        total = _align(jd_off + n * C.sizeof(_lib.ViewJitterDesc)) if jitter is not None else off
        host = torch.empty(total, dtype=torch.uint8, pin_memory=True)
        hb = host.numpy()
        buf = torch.empty(total, dtype=torch.uint8, device=dev)
        base = buf.data_ptr()
        tmp_rows = [g["rows"] * p["out"][0] * 3 for (_, _, _, p, _, g) in views]
        tmp = torch.empty(max(1, sum(tmp_rows)), dtype=torch.uint8, device=dev)
        u8_bytes = [_align(p["out"][0] * p["out"][1] * 3) for (_, _, _, p, _, _) in views]
        u8 = torch.empty(sum(u8_bytes) if jitter is not None else 0, dtype=torch.uint8, device=dev)
        img = torch.empty((n, 3, Hr, Wr), dtype=torch.float32, device=dev)
        depthmap = torch.empty((n, Hr, Wr), dtype=torch.float32, device=dev)
        pts3d = torch.empty((n, Hr, Wr, 3), dtype=torch.float32, device=dev)
        valid = torch.empty((n, Hr, Wr), dtype=torch.bool, device=dev)
        nonfinite = torch.zeros(n, dtype=torch.int32, device=dev)
        kp = hb[kp_off:kp_off + n * 100].view(np.float32).reshape(n, 25)
        dds = (_lib.ViewDepthDesc * n)()
        ids = (_lib.ViewImageDesc * n)()
        jds = (_lib.ViewJitterDesc * n)()
        tmp_ptr, u8_ptr = tmp.data_ptr(), u8.data_ptr()
        for i, ((rgb, depth, pose, p, K, g), (ro, do)) in enumerate(zip(views, lay)):
            h, w = rgb.shape[:2]
            hb[ro:ro + rgb.nbytes] = rgb.reshape(-1)
            hb[do:do + depth.nbytes] = np.ascontiguousarray(depth).view(np.uint8).reshape(-1)
            W, H = p["out"]
            tr = int(p["portrait"])
            kp[i, :9] = (K[[1, 0, 2]] if tr else K).reshape(-1)
            kp[i, 9:] = pose.reshape(-1)
            d = dds[i]
            d.depth, d.col_src, d.row_src = base + do, g["col_src"], g["row_src"]
            d.depthmap, d.pts3d, d.valid = depthmap[i].data_ptr(), pts3d[i].data_ptr(), valid[i].data_ptr()
            d.nonfinite = nonfinite.data_ptr() + 4 * i
            d.depth_stride, d.w, d.h, d.transpose = w, W, H, tr
            d.intr[:] = [float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])]
            d.pose[:] = [float(v) for v in pose[:3, :4].reshape(-1)]
            m = ids[i]
            m.src = base + ro + (g["src_row0"] * w + g["src_col0"]) * 3
            m.bh, m.kh, m.bv, m.kv = g["bh"], g["kh"], g["bv"], g["kv"]
            m.tmp, m.img = tmp_ptr, img[i].data_ptr()
            tmp_ptr += tmp_rows[i]
            m.row_stride, m.rows, m.cols, m.out_rows = w * 3, g["rows"], W, H
            m.ksh, m.ksv, m.transpose = g["ksh"], g["ksv"], tr
            if jitter is not None:
                j = jds[i]
                j.u8, j.img = u8_ptr, img[i].data_ptr()
                u8_ptr += u8_bytes[i]
                j.rows, j.cols, j.transpose = H, W, tr
                j.order[:], j.skip, (j.brightness, j.contrast, j.saturation), j.hue_shift = jitter[i]
        hb[dd_off:dd_off + C.sizeof(dds)] = np.frombuffer(bytes(dds), dtype=np.uint8)
        hb[id_off:id_off + C.sizeof(ids)] = np.frombuffer(bytes(ids), dtype=np.uint8)
        if jitter is not None:
            hb[jd_off:jd_off + C.sizeof(jds)] = np.frombuffer(bytes(jds), dtype=np.uint8)
        buf.copy_(host, non_blocking=True)
        max_pix = max(p["out"][0] * p["out"][1] for (_, _, _, p, _, _) in views)
        max_rows = max(g["rows"] for (*_, g) in views)
        max_cols = max(p["out"][0] for (_, _, _, p, _, _) in views)
        max_out_rows = max(p["out"][1] for (_, _, _, p, _, _) in views)
        max_span = max(g["span"] for (*_, g) in views)
        _lib.call("s3r_views_depth", buf, base + dd_off, n, max_pix)
        _lib.call("s3r_views_resample_h", buf, base + id_off, n, max_rows, max_cols, max_span)
        if jitter is None:
            _lib.call("s3r_views_resample_v_norm", buf, base + id_off, n, max_out_rows, max_cols)
        else:
            _lib.call("s3r_views_resample_v_u8", buf, base + id_off, base + jd_off, n, max_out_rows, max_cols)
            _lib.call("s3r_views_color_jitter", buf, base + jd_off, n, max_pix)
        bad = nonfinite.cpu().nonzero().flatten().tolist()     # waits for the launches
        if bad:
            raise ValueError(f"NaN / inf in the cropped depth map of view(s) {bad}")
        kp_dev = buf[kp_off:kp_off + n * 100].view(torch.float32).view(n, 25).clone()   # does not pin `buf`
        out = []
        for i, (rgb, depth, pose, p, K, g) in enumerate(views):
            W, H = p["out"]
            out.append({"img": img[i], "depthmap": depthmap[i], "pts3d": pts3d[i], "valid_mask": valid[i],
                        "camera_intrinsics": kp_dev[i, :9].view(3, 3), "camera_pose": kp_dev[i, 9:].view(4, 4),
                        "true_shape": torch.tensor((H, W), dtype=torch.int32)})
        return out


def _is_imgnorm(t) -> bool:
    """ImgNorm of dust3r/datasets/utils/transforms.py: Compose([ToTensor(), Normalize((0.5,) * 3, (0.5,) * 3)])."""
    ts = getattr(t, "transforms", None)
    if type(t).__name__ != "Compose" or not isinstance(ts, (list, tuple)) or len(ts) != 2:
        return False
    a, b = ts
    try:
        return (type(a).__name__ == "ToTensor" and type(b).__name__ == "Normalize"
                and [float(v) for v in b.mean] == [0.5] * 3 and [float(v) for v in b.std] == [0.5] * 3
                and not getattr(b, "inplace", False))
    except TypeError:
        return False


class _RawView:
    """What the patched `_crop_resize_if_necessary` returns as the image: the decoded arrays and the plan."""

    def __init__(self, rgb, depth, plan):
        self.rgb, self.depth, self.plan = rgb, depth, plan


def _refuse(*_a, **_k):
    raise TypeError("this dataset reads the cropped depth map inside _get_views, which DeviceViews does not provide; "
                    f"build its views with ViewBuilder instead (known such datasets: {', '.join(CROPPED_DEPTH_READERS)})")


class _DeferredDepth:
    """Stands in for the cropped depth map until the device builds it: any use of it inside `_get_views` raises."""
    __slots__ = ()
    __array__ = __getitem__ = __setitem__ = __len__ = __iter__ = _refuse
    __lt__ = __le__ = __gt__ = __ge__ = _refuse
    __add__ = __radd__ = __sub__ = __rsub__ = __mul__ = __rmul__ = __truediv__ = __rtruediv__ = _refuse
    __iadd__ = __isub__ = __imul__ = __itruediv__ = _refuse

    def __getattr__(self, name):
        _refuse()


class DeviceViews:
    """Wraps one of the reference's evaluation datasets (SevenScenes, NRGBD, DTU, Demo; duck-typed: it reads
    `_get_views`, `_resolutions`, `seed`, `aug_crop` and `transform`) so that `wrapper[idx]` returns the views
    `dataset[idx]` returns, with the pixel work on the device.

    The dataset's own `_get_views` still runs on the CPU (file decoding, DTU's mask erosion, frame sampling); its
    `_crop_resize_if_necessary` is replaced on the instance by one that only plans.  The tail of the base
    `__getitem__` (idx, true_shape, ImgNorm, pts3d, valid_mask, transpose_to_landscape, the trailing `rng` bytes) is
    restated here.  `DataLoader(DeviceViews(ds), batch_size=1, num_workers=0)` yields batches `Spann3R.forward` and the
    criteria take unchanged.

    Refused: a `transform` other than ImgNorm (e.g. the training sets' ColorJitter), and datasets whose `_get_views`
    reads the cropped depth map (CROPPED_DEPTH_READERS: Co3d, ARKitScenes, ScanNet, ScanNet++, Habitat, BlendedMVS)."""

    def __init__(self, dataset, device="cuda"):
        _lib.require_device()
        names = {c.__name__ for c in type(dataset).__mro__}
        hit = sorted(names & set(CROPPED_DEPTH_READERS))
        if hit:
            _refuse_dataset = (f"{hit[0]} reads the cropped depth map inside _get_views; DeviceViews cannot serve it. "
                               f"Build its views with ViewBuilder (datasets known to do this: "
                               f"{', '.join(CROPPED_DEPTH_READERS)})")
            raise ValueError(_refuse_dataset)
        if not _is_imgnorm(getattr(dataset, "transform", None)):
            raise ValueError("DeviceViews reproduces ImgNorm only; the dataset's transform is "
                             f"{getattr(dataset, 'transform', None)!r}")
        self.dataset = dataset
        self.device = torch.device(device)
        self._builders = {}
        dataset._crop_resize_if_necessary = self._plan_only

    def __len__(self):
        return len(self.dataset)

    def _builder(self, resolution):
        key = tuple(resolution)
        b = self._builders.get(key)
        if b is None:
            b = self._builders[key] = ViewBuilder(key, aug_crop=self.dataset.aug_crop, device=self.device)
        return b

    def _plan_only(self, image, depthmap, intrinsics, resolution, rng=None, info=None):
        rgb = _as_rgb(np.asarray(image))
        try:
            p = plan_view(rgb.shape[0], rgb.shape[1], intrinsics, resolution, self.dataset.aug_crop, rng)
        except ValueError as e:
            raise ValueError(f"{e} (view {info})") from None
        return _RawView(rgb, depthmap, p), _DeferredDepth(), p["K"]

    def __getitem__(self, idx):
        ds = self.dataset
        if isinstance(idx, tuple):
            idx, ar_idx = idx
        else:
            if len(ds._resolutions) != 1:
                raise ValueError("index with (idx, aspect-ratio idx) for a dataset of several resolutions")
            ar_idx = 0
        if ds.seed:
            ds._rng = np.random.default_rng(seed=ds.seed + idx)
        elif not hasattr(ds, "_rng"):
            ds._rng = np.random.default_rng(seed=torch.initial_seed())
        resolution = ds._resolutions[ar_idx]
        views = ds._get_views(idx, resolution, ds._rng)
        planned = []
        for v, view in enumerate(views):
            raw = view.get("img")
            if not isinstance(raw, _RawView):
                raise ValueError("a view did not go through _crop_resize_if_necessary")
            if "pts3d" in view or "valid_mask" in view or "camera_intrinsics" not in view:
                raise ValueError("a view carries pts3d / valid_mask, or lacks camera_intrinsics")
            view["idx"] = (idx, ar_idx, v)
            plan = dict(raw.plan, K=np.float32(view["camera_intrinsics"]))
            planned.append((raw.rgb, raw.depth, view.get("camera_pose"), plan))
        built = self._builder(resolution).build_planned(planned)
        for view, b in zip(views, built):
            view.update(b)
        for view in views:
            view["rng"] = int.from_bytes(ds._rng.bytes(4), "big")
        return views
