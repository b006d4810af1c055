"""Deterministic synthetic checkpoints in the reference's state-dict layout.

There is no network and no trained checkpoint, so parity and the benchmark run on
random-init weights (BASELINE.json: "random-init ViT-L/Base-dec").  The weights must be
bit-identical here (where the real reference runs on CPU and the golden vectors are made)
and on the GPU box (where /root/reference does not exist), so every tensor is drawn from
its own `torch.Generator` seeded by (seed, crc32(key)): the result depends only on the key
name, the shape and the torch version, not on construction order.

The key/shape inventory is `spann3r_b200/state_dict_spec.json` (package data), dumped from the real
reference model by `tools/make_golden.py` (1101 keys for Spann3R, SURVEY.md §8b).

Init rules follow what the reference constructors do (so activations are conditioned like
the reference's own random init, which SURVEY.md §8d probed finite for 10 frames):
  * nn.Linear weights        xavier-uniform       croco/models/croco.py:111-127
  * conv / conv-transpose    U(+-1/sqrt(fan_in))  (torch default kaiming_uniform(a=sqrt(5)))
  * biases                   small non-zero noise (the reference zeros Linear biases; we do
                             not, so that a dropped bias add cannot hide)
  * LayerNorm gains          1 + 0.1*U(-1,1)      (same reason)
"sharpen=True" multiplies norm_q.weight by 8 (SURVEY.md §7.3-#5): with raw random-init
weights the memory-read attention is near-uniform and the eval-mode 5e-4 threshold
(spann3r/model.py:170-172) zeroes whole rows once the bank is large.
"""
from __future__ import annotations

import json
import math
import os
import re
import zlib

import numpy as np
import torch

_SPEC_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "state_dict_spec.json")


def load_spec(path: str = _SPEC_PATH) -> dict:
    with open(path) as f:
        return json.load(f)


USE_FEAT_DIM = 768   # Spann3R(use_feat=True): the value encoder runs at the decoder's width (spann3r/model.py:225)


def usefeat_spec(spec: dict | None = None) -> dict:
    """The state-dict inventory of `Spann3R(use_feat=True)`, derived from the default one (spann3r/model.py:225-242):
    `pos_patch_embed` is not created, and the value encoder (6 Blocks, 16 heads of 48), `value_norm` and `value_out`'s
    input are 768 wide.  Every other key keeps its shape and its place in the order (1099 keys)."""
    spec = spec or load_spec()
    D = USE_FEAT_DIM
    out = {}
    for key, shape in spec["spann3r"].items():
        if key.startswith("pos_patch_embed."):
            continue
        if key.startswith("value_encoder."):
            shape = [D if s == 1024 else 4 * D if s == 4096 else 3 * D if s == 3072 else s for s in shape]
        elif key.startswith("value_norm."):
            shape = [D]
        elif key == "value_out.weight":
            shape = [shape[0], D]
        out[key] = list(shape)
    return {**{k: v for k, v in spec.items() if k != "spann3r"}, "spann3r": out}


def _gen(seed: int, key: str) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFFFFFFFFFF)
    return g


def _uniform(shape, bound, g):
    return (torch.rand(shape, generator=g, dtype=torch.float32) * 2.0 - 1.0) * bound


def _is_norm_key(key: str) -> bool:
    leaf = key.split(".")[-2]
    return leaf.startswith("norm") or leaf.endswith("_norm") or leaf in ("norm_q", "norm_k", "norm_v")


_ALIAS = re.compile(r"scratch\.layer([1-4])_rn\.")


def canonical_key(key: str) -> str:
    """The DPT head registers each `scratch.layerK_rn` conv twice (also as `scratch.layer_rn.K-1`,
    croco/models/dpt_block.py:59-65); both state-dict keys must carry the same tensor."""
    return _ALIAS.sub(lambda m: f"scratch.layer_rn.{int(m.group(1)) - 1}.", key)


def synth_tensor(key: str, shape, seed: int = 0) -> torch.Tensor:
    key = canonical_key(key)
    g = _gen(seed, key)
    shape = tuple(shape)
    if key.endswith("mask_token"):
        return torch.randn(shape, generator=g, dtype=torch.float32) * 0.02
    if key.endswith(".weight"):
        if len(shape) == 1:
            if _is_norm_key(key):
                return 1.0 + _uniform(shape, 0.1, g)
            raise ValueError(f"unexpected 1-D weight {key}")
        if len(shape) == 2:  # nn.Linear [out, in]
            fan_out, fan_in = shape
            return _uniform(shape, math.sqrt(6.0 / (fan_in + fan_out)), g)
        if len(shape) == 4:
            if key.endswith("patch_embed.proj.weight"):
                # PatchEmbed._init_weights: xavier on w.view(out, -1)   blocks.py:237-239
                fan_out, fan_in = shape[0], shape[1] * shape[2] * shape[3]
                return _uniform(shape, math.sqrt(6.0 / (fan_in + fan_out)), g)
            # Conv2d [out,in,kh,kw] / ConvTranspose2d [in,out,kh,kw]: torch's fan_in = shape[1]*kh*kw
            fan_in = shape[1] * shape[2] * shape[3]
            return _uniform(shape, 1.0 / math.sqrt(fan_in), g)
    if key.endswith(".bias"):
        return _uniform(shape, 0.02, g)
    raise ValueError(f"no init rule for {key} {shape}")


def make_state_dict(spec: dict | None = None, seed: int = 0, sharpen: bool = False,
                    prefix: str | None = None) -> dict:
    """Return {key: fp32 CPU tensor} for every key in the spec (optionally only keys under `prefix`,
    with the prefix stripped -- used to build the DUSt3R-layout checkpoint the ctor consumes)."""
    spec = spec or load_spec()
    out = {}
    for key, shape in spec["spann3r"].items():
        if prefix is not None:
            if not key.startswith(prefix):
                continue
            name = key[len(prefix):]
        else:
            name = key
        t = synth_tensor(key, shape, seed)
        if sharpen and key == "norm_q.weight":
            t = t * 8.0
        out[name] = t
    return out


DUST3R_ARGS = ("AsymmetricCroCo3DStereo(pos_embed='RoPE100', patch_embed_cls='ManyAR_PatchEmbed', "
               "img_size=(512, 512), head_type='dpt', output_mode='pts3d', depth_mode=('exp', -inf, inf), "
               "conf_mode=('exp', 1, inf), enc_embed_dim=1024, enc_depth=24, enc_num_heads=16, "
               "dec_embed_dim=768, dec_depth=12, dec_num_heads=12)")


def make_frames(n_frames: int, height: int, width: int, batch: int = 1, seed0: int = 1):
    """Synthetic frames as SURVEY.md §8d: img_i = rand(B,3,H,W)*2-1 with seed seed0+i."""
    frames = []
    for i in range(n_frames):
        g = torch.Generator(device="cpu")
        g.manual_seed(seed0 + i)
        img = torch.rand((batch, 3, height, width), generator=g, dtype=torch.float32) * 2.0 - 1.0
        frames.append({"img": img})
    return frames


def make_pointmap_case(height: int, width: int, focal: float, rvec, tvec, noise: float, outlier_frac: float, seed: int):
    """A synthetic world-frame pointmap for the post-path geometry tests / bench (numpy): a smooth depth surface seen by a
    pinhole camera (focal, principal point at the image centre) whose pose is x_cam = R(rvec) x_world + tvec, with
    Gaussian noise on the points and a fraction of gross outliers.  Returns (pts3d [H, W, 3] float32, K [3, 3] float64)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    u, v = np.meshgrid(np.arange(width), np.arange(height))
    K = np.array([[focal, 0, width / 2], [0, focal, height / 2], [0, 0, 1]], np.float64)
    d = 2 + 0.5 * np.sin(u / 50.0) + 0.3 * np.cos(v / 40.0)
    xc = np.stack(((u - width / 2) / focal * d, (v - height / 2) / focal * d, d), -1).reshape(-1, 3)
    r = np.asarray(rvec, np.float64)
    th = float(np.linalg.norm(r))
    if th < 1e-12:
        R = np.eye(3)
    else:
        kx, ky, kz = r / th
        Kx = np.array([[0, -kz, ky], [kz, 0, -kx], [-ky, kx, 0]])
        R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    xw = (xc - np.asarray(tvec, np.float64)) @ R          # x_cam = R x_world + t  =>  x_world = R^T (x_cam - t)
    xw += rng.normal(0, noise, xw.shape)
    n_out = int(outlier_frac * len(xw))
    if n_out:
        idx = rng.choice(len(xw), n_out, replace=False)
        xw[idx] += rng.normal(0, 0.5, (n_out, 3))
    return xw.astype(np.float32).reshape(height, width, 3), K


def _rotation(rvec):
    import numpy as np
    r = np.asarray(rvec, np.float64)
    th = float(np.linalg.norm(r))
    if th < 1e-12:
        return np.eye(3)
    kx, ky, kz = r / th
    Kx = np.array([[0, -kz, ky], [kz, 0, -kx], [-ky, kx, 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _surface(kind: str, n: int, rng):
    """n points on a unit-sized surface: 'plane' (z = 0), 'corner' (three faces of a box), 'curved' (a wavy sheet)."""
    import numpy as np
    u = rng.uniform(-1, 1, (n, 2))
    if kind == "plane":
        return np.stack((u[:, 0], u[:, 1], np.zeros(n)), -1)
    if kind == "corner":
        face = rng.integers(0, 3, n)
        p = np.zeros((n, 3))
        for f in range(3):
            sel = face == f
            axes = [a for a in range(3) if a != f]
            p[sel, axes[0]] = (u[sel, 0] + 1) / 2
            p[sel, axes[1]] = (u[sel, 1] + 1) / 2
        return p
    if kind == "curved":
        return np.stack((u[:, 0], u[:, 1], 0.25 * np.sin(2.5 * u[:, 0]) * np.cos(2.0 * u[:, 1])), -1)
    raise ValueError(kind)


def make_recon_case(surface: str, n_gt: int, n_pred: int, scale: float, noise: float, outlier_frac: float,
                    dup_frac: float, rvec, tvec, seed: int):
    """A seeded (ground truth, prediction) pair of clouds for the reconstruction-metric tests (numpy, float32 like the
    network's pointmaps).  Both sample the same surface independently; the prediction gets Gaussian noise (`noise`,
    relative to the scene), `outlier_frac` far outliers (up to 50x the scene scale), `dup_frac` exact duplicates of its
    own points, and is then moved off the ground truth by the rigid x -> R(rvec) x + tvec * scale.  With noise 0 and
    n_pred == n_gt the prediction is exactly the moved ground truth.  Returns (gt [n_gt, 3], pred [n_pred, 3], T [4, 4]
    fp64 with gt ~ T pred)."""
    import numpy as np
    rng = np.random.default_rng(seed)
    gt = _surface(surface, n_gt, rng)
    if noise == 0 and n_pred == n_gt:
        pred = gt.copy()
    else:
        pred = _surface(surface, n_pred, rng) + rng.normal(0, noise, (n_pred, 3))
    n_out = int(round(outlier_frac * n_pred))
    if n_out:
        i = rng.choice(n_pred, n_out, replace=False)
        pred[i] = rng.uniform(-50, 50, (n_out, 3))
    n_dup = int(round(dup_frac * n_pred))
    if n_dup:
        src = rng.choice(n_pred, n_dup, replace=False)
        dst = rng.choice(n_pred, n_dup, replace=False)
        pred[dst] = pred[src]
    gt, pred = gt * scale, pred * scale
    R = _rotation(rvec)
    t = np.asarray(tvec, np.float64) * scale
    pred = pred @ R.T + t                       # moved off the ground truth; gt ~ R^T (pred - t)
    T = np.eye(4)
    T[:3, :3] = R.T
    T[:3, 3] = -R.T @ t
    return gt.astype(np.float32), pred.astype(np.float32), T


# (surface, n_gt, n_pred, scale, noise, outlier_frac, dup_frac, rvec, tvec, seed): tests/golden/recon_eval.json
RECON_CASES = [
    ("plane", 20000, 15000, 1.0, 0.003, 0.01, 0.0, (0.02, -0.01, 0.03), (0.01, 0.02, -0.01), 0),
    ("curved", 50000, 40000, 0.1, 0.004, 0.03, 0.02, (0.01, 0.02, 0.0), (0.0, 0.01, 0.02), 1),
    ("curved", 200000, 180000, 100.0, 0.002, 0.05, 0.01, (-0.03, 0.02, 0.01), (0.02, 0.0, 0.01), 2),
    ("corner", 30000, 30000, 1.0, 0.002, 0.0, 0.05, (0.0, 0.0, 0.02), (0.01, -0.01, 0.0), 3),
    ("curved", 20000, 20000, 1.0, 0.0, 0.0, 0.0, (0.03, -0.02, 0.01), (0.02, 0.01, -0.02), 4),   # clean: ICP recovers T
    ("plane", 1, 7, 1.0, 0.01, 0.0, 0.0, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 5),
    ("plane", 5, 2, 100.0, 0.01, 0.0, 0.5, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 6),
]


def make_eval_scene(n_frames: int = 50, height: int = 224, width: int = 224, seed: int = 0):
    """An eval.py-sized scene (generated, never stored): ground-truth pointmaps [F, H, W, 3] of a wavy surface seen by
    a sweeping camera, the prediction = ground truth + noise + 1 % far outliers, moved by a small rigid transform, and a
    validity mask [F, H, W] (~95 % true).  float32, like eval.py's pts_all / pts_gt_all / masks_all."""
    import numpy as np
    rng = np.random.default_rng(seed)
    v, u = np.meshgrid(np.linspace(-1, 1, height), np.linspace(-1, 1, width), indexing="ij")
    gt = np.empty((n_frames, height, width, 3))
    for f in range(n_frames):
        x = u * 0.6 + 0.04 * f
        y = v * 0.6
        gt[f] = np.stack((x, y, 0.2 * np.sin(3 * x) * np.cos(2 * y) + 1.0), -1)
    pred = gt + rng.normal(0, 0.003, gt.shape)
    flat = pred.reshape(-1, 3)
    n_out = int(0.01 * len(flat))
    flat[rng.choice(len(flat), n_out, replace=False)] = rng.uniform(-50, 50, (n_out, 3))
    R = _rotation((0.01, -0.015, 0.02))
    pred = pred @ R.T + np.array([0.01, -0.02, 0.015])
    masks = rng.random((n_frames, height, width)) < 0.95
    return pred.astype(np.float32), gt.astype(np.float32), masks


# (height, width, focal, rvec, tvec, noise, outlier_frac, seed): the cases of tests/golden/pnp.json
PNP_CASES = [
    (384, 512, 400.0, (0.1, -0.2, 0.05), (0.3, -0.1, 0.2), 0.002, 0.0, 1),
    (384, 512, 450.0, (0.3, 0.2, -0.1), (-0.5, 0.2, 0.4), 0.005, 0.2, 2),
    (224, 224, 250.0, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0.001, 0.1, 3),
    (384, 512, 420.0, (-0.2, 0.4, 0.3), (0.1, 0.6, -0.3), 0.003, 0.3, 4),
    (384, 512, 380.0, (0.05, 1.2, -0.4), (1.0, -0.3, 0.8), 0.004, 0.45, 5),
]


# ---- adversarial inputs of the post-path geometry: tests/test_postprocess_adversarial.py ---------------------------
def _pinhole_map(g, B, H, W, f, noise=0.0):
    """[B, H, W, 3] fp32 pinhole pointmap with focal f and principal point (W / 2, H / 2), depth in [1, 3]."""
    jj, ii = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    z = 1.0 + 2.0 * torch.rand(B, H, W, generator=g, dtype=torch.float64)
    x = (ii - W / 2) * z / f
    y = (jj - H / 2) * z / f
    if noise:
        x = x + noise * torch.randn(B, H, W, generator=g, dtype=torch.float64)
        y = y + noise * torch.randn(B, H, W, generator=g, dtype=torch.float64)
    return torch.stack((x, y, z), -1).float()


def _focal_frame(name: str, g) -> torch.Tensor:
    nan, inf = float("nan"), float("inf")
    if name == "all_z0":                  # every x / z is +-inf or NaN -> a = 0 everywhere, f0 = 0 / 0
        p = _pinhole_map(g, 1, 48, 64, 60.0, 0.01)
        p[..., 2] = 0.0
        return p
    if name == "all_nan":
        return torch.full((1, 48, 64, 3), nan)
    if name == "one_finite":
        p = torch.full((1, 48, 64, 3), nan)
        p[0, 7, 50] = _pinhole_map(g, 1, 48, 64, 60.0, 0.01)[0, 7, 50]
        return p
    if name == "noise_free":              # |p - f a| is fp32 rounding only; 0 at the principal point (weight floor)
        return _pinhole_map(g, 1, 96, 128, 110.0)
    if name == "behind_half":             # half the pixels have z < 0 (x, y kept): their a points the wrong way
        p = _pinhole_map(g, 1, 64, 80, 55.0, 0.01)
        back = torch.rand(1, 64, 80, generator=g) < 0.5
        p[..., 2] = torch.where(back, -p[..., 2], p[..., 2])
        return p
    if name == "inf_lattice":             # x = +-inf on one lattice of pixels, z = 0 on another
        p = _pinhole_map(g, 1, 60, 84, 70.0, 0.01)
        jj, ii = torch.meshgrid(torch.arange(60), torch.arange(84), indexing="ij")
        lat = (jj % 5 == 0) & (ii % 7 == 0)
        p[..., 0] = torch.where(lat, torch.where((ii + jj) % 2 == 0, inf, -inf).float(), p[..., 0])
        p[..., 2] = torch.where((jj % 3 == 1) & (ii % 11 == 3), 0.0, p[..., 2])
        return p
    if name == "h1":
        return _pinhole_map(g, 2, 1, 300, 90.0, 0.01)
    if name == "w1":
        return _pinhole_map(g, 2, 300, 1, 90.0, 0.01)
    if name == "tiny":                    # 120 pixels: fewer than one 256-thread block
        return _pinhole_map(g, 1, 10, 12, 9.0, 0.001)
    if name == "hd":                      # 1080 x 1920: many terms per thread
        return _pinhole_map(g, 1, 1080, 1920, 1400.0, 0.01)
    if name == "scaled":
        return _pinhole_map(g, 1, 64, 80, 55.0, 0.01) * 1e-20
    if name == "underflow":               # a ~ 1e-22: a.a underflows fp32 (subnormal or 0), a.p does not
        p = _pinhole_map(g, 1, 64, 80, 55.0, 0.01)
        p[..., :2] = p[..., :2] * 1e-22
        return p
    if name == "mixed":                   # valid / all-NaN / all-z=0 / valid
        p = _pinhole_map(g, 4, 48, 64, 60.0, 0.01)
        p[1] = nan
        p[2, ..., 2] = 0.0
        return p
    # median-specific frames: votes u z / x and v z / y
    if name == "med_even":                # a few NaN pixels: an even number of non-NaN votes
        p = _pinhole_map(g, 1, 31, 37, 40.0, 0.01)
        p[0, 3:6, 4] = nan
        return p
    if name == "med_odd":                 # one NaN x: an odd number of non-NaN votes
        p = _pinhole_map(g, 1, 31, 37, 40.0, 0.01)
        p[0, 9, 13, 0] = nan
        return p
    if name in ("med_identical", "med_ties"):
        H, W = 24, 32
        jj, ii = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
        u, v = (ii - W / 2).float(), (jj - H / 2).float()
        if name == "med_identical":       # x = u / 64, z = 1: every non-NaN vote is exactly 64
            qx = qy = torch.full((H, W), 64.0)
        else:                             # votes drawn from {16, 32, 64, 128}: long runs of ties around the median
            q = torch.tensor([16.0, 32.0, 64.0, 128.0])
            qx = q[torch.randint(0, 4, (H, W), generator=g)]
            qy = q[torch.randint(0, 4, (H, W), generator=g)]
        return torch.stack((u / qx, v / qy, torch.ones(H, W)), -1)[None]
    if name == "med_inf_mixed":           # x = 0 or y = 0 with u z != 0: +-inf votes among finite ones
        p = _pinhole_map(g, 1, 40, 50, 45.0, 0.01)
        sel = torch.rand(1, 40, 50, generator=g)
        p[..., 0] = torch.where(sel < 0.15, 0.0, p[..., 0])
        p[..., 1] = torch.where(sel > 0.9, -0.0, p[..., 1])
        return p
    if name == "med_plus_inf":            # every x and y is a zero signed like u and v: every non-NaN vote is +inf
        p = _pinhole_map(g, 1, 40, 50, 45.0)
        p[..., 0] = p[..., 0] * 0.0
        p[..., 1] = p[..., 1] * 0.0
        return p
    if name == "med_negative":            # z < 0 everywhere: every vote is about -f
        p = _pinhole_map(g, 1, 40, 50, 45.0, 0.01)
        p[..., 2] = -p[..., 2]
        return p
    if name == "med_one_vote":            # one pixel with a finite x and a NaN y, everything else NaN
        p = torch.full((1, 40, 50, 3), nan)
        p[0, 30, 41] = _pinhole_map(g, 1, 40, 50, 45.0, 0.01)[0, 30, 41]
        p[0, 30, 41, 1] = nan
        return p
    raise ValueError(name)


# name -> seed of the adversarial focal frames; every frame is run in both focal modes.  `underflow`: a.a underflows fp32,
# so the reference's fp32 result is NaN while fp64 is finite (a kernel that keeps a subnormal sum may be either).
FOCAL_ADV_CASES = {name: i + 1 for i, name in enumerate((
    "all_z0", "all_nan", "one_finite", "noise_free", "behind_half", "inf_lattice", "h1", "w1", "tiny", "hd", "scaled",
    "underflow", "mixed", "med_even", "med_odd", "med_identical", "med_ties", "med_inf_mixed", "med_plus_inf",
    "med_negative", "med_one_vote"))}


def make_focal_adv_case(name: str) -> torch.Tensor:
    """Adversarial pointmap `name` of FOCAL_ADV_CASES: [B, H, W, 3] fp32 (CPU); principal point (W / 2, H / 2)."""
    return _focal_frame(name, torch.Generator().manual_seed(FOCAL_ADV_CASES[name])).contiguous()


def _world_from_cam(xc, rvec, tvec):
    return (xc - np.asarray(tvec, np.float64)) @ _rotation(rvec)


def _sparse_exact(rng, n, n_nan, rvec, tvec, K, behind=False):
    """n exact correspondences of random non-coplanar camera-frame points (plus n_nan NaN image points)."""
    u = rng.uniform(20, 2 * K[0, 2] - 20, n)
    v = rng.uniform(20, 2 * K[1, 2] - 20, n)
    d = rng.uniform(1.5, 4.0, n) * (-1.0 if behind else 1.0)
    xc = np.stack(((u - K[0, 2]) / K[0, 0] * d, (v - K[1, 2]) / K[1, 1] * d, d), -1)
    pts = _world_from_cam(xc, rvec, tvec)
    img = np.stack((u, v), -1)
    if n_nan:
        pts = np.concatenate((pts, rng.normal(0, 1, (n_nan, 3))))
        img = np.concatenate((img, np.full((n_nan, 2), np.nan)))
    return pts.astype(np.float32), img.astype(np.float32)


def make_pnp_adv_case(name: str):
    """Adversarial PnP frame `name` of PNP_ADV_CASES -> (pts3d, image_points or None, K).  Dense frames: pts3d
    [H, W, 3] with the pixel grid as image points; sparse frames: pts3d [n, 3], image_points [n, 2].  float32."""
    rng = np.random.default_rng(PNP_ADV_CASES.index(name) + 100)
    if name == "nan_inf":                 # 30 % NaN coordinates, 5 % +-inf coordinates
        pts, K = make_pointmap_case(384, 512, 400.0, (0.1, -0.2, 0.05), (0.3, -0.1, 0.2), 0.002, 0.05, 11)
        flat = pts.reshape(-1, 3)
        n = len(flat)
        bad = rng.choice(n, int(0.35 * n), replace=False)
        flat[bad[: int(0.30 * n)], rng.integers(0, 3, int(0.30 * n))] = np.nan
        k = len(bad) - int(0.30 * n)
        flat[bad[int(0.30 * n):], rng.integers(0, 3, k)] = np.where(rng.random(k) < 0.5, np.inf, -np.inf)
        return pts, None, K
    if name == "behind40":                # 40 % of the points moved behind the camera
        H, W, f, rv, tv = 384, 512, 420.0, (-0.2, 0.4, 0.3), (0.1, 0.6, -0.3)
        pts, K = make_pointmap_case(H, W, f, rv, tv, 0.002, 0.0, 12)
        flat = pts.reshape(-1, 3).astype(np.float64)
        sel = rng.choice(H * W, int(0.4 * H * W), replace=False)
        xc = flat[sel] @ _rotation(rv).T + np.asarray(tv)
        xc *= -rng.uniform(0.3, 2.0, (len(sel), 1))
        flat[sel] = _world_from_cam(xc, rv, tv)
        return flat.astype(np.float32).reshape(H, W, 3), None, K
    if name == "planar":                  # a tilted plane
        H, W, f, rv, tv = 384, 512, 380.0, (0.2, -0.1, 0.3), (-0.2, 0.1, 0.5)
        K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]])
        u, v = np.meshgrid(np.arange(W), np.arange(H))
        ray = np.stack(((u - W / 2) / f, (v - H / 2) / f, np.ones_like(u, np.float64)), -1)
        d = 2.5 / (1.0 + 0.3 * ray[..., 0] - 0.2 * ray[..., 1])        # plane 0.3 x - 0.2 y + z = 2.5
        xc = (ray * d[..., None]).reshape(-1, 3) + rng.normal(0, 0.002, (H * W, 3))
        return _world_from_cam(xc, rv, tv).astype(np.float32).reshape(H, W, 3), None, K
    if name == "collinear":               # a 4 x 512 strip: the points lie close to one line
        pts, K = make_pointmap_case(4, 512, 400.0, (0.05, 0.1, -0.05), (0.1, 0.0, 0.3), 0.001, 0.0, 13)
        return pts, None, K
    if name in ("sparse4", "sparse5", "sparse8"):
        K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
        pts, img = _sparse_exact(rng, int(name[6:]), 3, (0.1, 0.3, -0.2), (0.2, -0.1, 0.4), K)
        return pts, img, K
    if name == "three_finite":            # 3 finite correspondences among 12: no model can have 4 inliers
        K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
        pts, img = _sparse_exact(rng, 3, 0, (0.1, 0.3, -0.2), (0.2, -0.1, 0.4), K)
        pts = np.concatenate((pts, np.full((9, 3), np.nan, np.float32)))
        img = np.concatenate((img, rng.uniform(0, 400, (9, 2)).astype(np.float32)))
        return pts, img, K
    if name == "all_behind":              # 6 correspondences, every point behind the camera
        # A mirror pose (a half turn about the optical axis, then a shift along it) puts behind-camera points of about
        # one depth in front of the camera on their own pixels, so larger such frames do have 4-inlier models.  These 6
        # points have none: 4096 samples (many draws of each of their 20 triples) find no model with 4 inliers.
        K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
        pts, img = _sparse_exact(np.random.default_rng(0), 6, 0, (0.1, 0.3, -0.2), (0.2, -0.1, 0.4), K, behind=True)
        return pts, img, K
    if name == "near_centre":             # identity pose, one exact inlier 2e-3 in front of the camera centre
        pts, K = make_pointmap_case(384, 512, 400.0, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 2e-4, 0.0, 14)
        z = 2e-3
        for r, c in ((100, 300), (250, 120)):
            pts[r, c] = ((c - 256) / 400.0 * z, (r - 192) / 400.0 * z, z)
        return pts, None, K
    if name == "hd":
        pts, K = make_pointmap_case(1080, 1920, 1500.0, (0.1, -0.15, 0.05), (0.2, 0.1, 0.3), 0.002, 0.2, 15)
        return pts, None, K
    if name == "all_nan":
        pts, K = make_pointmap_case(96, 128, 120.0, (0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 0.0, 0.0, 16)
        return np.full_like(pts, np.nan), None, K
    if name == "three_finite_dense":
        pts, K = make_pointmap_case(96, 128, 120.0, (0.1, 0.0, 0.0), (0.0, 0.1, 0.0), 0.001, 0.0, 17)
        keep = pts[[5, 50, 90], [7, 60, 100]].copy()
        pts[:] = np.nan
        pts[[5, 50, 90], [7, 60, 100]] = keep
        return pts, None, K
    if name == "valid_small":
        pts, K = make_pointmap_case(96, 128, 120.0, (0.1, -0.05, 0.02), (0.05, 0.1, 0.2), 0.002, 0.2, 18)
        return pts, None, K
    raise ValueError(name)


# The adversarial PnP frames; `hd` is GPU-only (the host scoring loop would take minutes).  The last three share one
# camera (96 x 128, f = 120) so they can form a mixed batch of solvable and unsolvable frames.
PNP_ADV_CASES = ["nan_inf", "behind40", "planar", "collinear", "sparse4", "sparse5", "sparse8", "three_finite",
                 "all_behind", "near_centre", "hd", "all_nan", "three_finite_dense", "valid_small"]


def make_loss_case(batch: int, frames: int, height: int, width: int, invalid: float = 0.3, seed: int = 0,
                   device="cpu"):
    """Views and `preds_all` for the criteria (spann3r_b200.loss / tests/golden/loss_*.npz): a wavy surface per frame
    in world coordinates seen through a non-identity camera_pose per view; `invalid` of the pixels in irregular blobs
    (0: all valid); predictions = the ground truth in view 0's camera frame, scaled per sequence, plus noise, with the
    keys Spann3R.forward returns (pair 0 left: 'pts3d', every other map: 'pts3d_in_other_view'), conf = 1 + exp(x).
    fp32 CPU tensors (moved to `device`)."""
    g = torch.Generator().manual_seed(seed)
    B, F, H, W = batch, frames, height, width
    v, u = torch.meshgrid(torch.linspace(-1, 1, H), torch.linspace(-1, 1, W), indexing="ij")
    poses = []
    for f in range(F):
        ang = 0.05 * torch.randn(B, 3, generator=g, dtype=torch.float64) + torch.tensor([0.02 * f, -0.01 * f, 0.0],
                                                                                          dtype=torch.float64)
        R = torch.stack([torch.as_tensor(_rotation(a.tolist())) for a in ang])
        P = torch.eye(4, dtype=torch.float64).repeat(B, 1, 1)
        P[:, :3, :3] = R
        P[:, :3, 3] = 0.3 * torch.randn(B, 3, generator=g, dtype=torch.float64) + torch.tensor([0.1 * f, 0.0, 0.05 * f])
        poses.append(P)
    inv0 = torch.linalg.inv(poses[0])
    gts, cam0 = [], []
    for f in range(F):
        z = 2.0 + 0.3 * torch.rand(B, 1, 1, generator=g, dtype=torch.float64) \
            + 0.2 * torch.sin(3 * u + f)[None] * torch.cos(2 * v)[None]
        cam = torch.stack((u[None] * z, v[None] * z * (H / W), z), -1)                   # in camera f
        world = torch.einsum("bij,bhwj->bhwi", poses[f][:, :3, :3], cam) + poses[f][:, None, None, :3, 3]
        if invalid > 0:
            low = torch.rand(B, 1, max(2, H // 24), max(2, W // 24), generator=g)
            blob = torch.nn.functional.interpolate(low, size=(H, W), mode="bicubic", align_corners=False)[:, 0]
            noise = torch.rand(B, H, W, generator=g)
            valid = (blob + 0.15 * noise) > torch.quantile(blob.flatten(1) + 0.15 * noise.flatten(1), invalid, dim=1)[:, None, None]
        else:
            valid = torch.ones(B, H, W, dtype=torch.bool)
        gts.append({"pts3d": world.float(), "valid_mask": valid, "camera_pose": poses[f].float()})
        cam0.append(torch.einsum("bij,bhwj->bhwi", inv0[:, :3, :3], world) + inv0[:, None, None, :3, 3])
    s = 0.5 + torch.rand(B, 1, 1, 1, generator=g, dtype=torch.float64)

    def pred(f):
        return (cam0[f] * s + 0.05 * torch.randn(cam0[f].shape, generator=g, dtype=torch.float64)).float()

    def conf():
        return (1 + torch.exp(0.5 * torch.randn(B, H, W, generator=g))).float()

    preds = []
    for k in range(F - 1):
        left = {("pts3d" if k == 0 else "pts3d_in_other_view"): pred(k), "conf": conf()}
        right = {"pts3d_in_other_view": pred(k + 1), "conf": conf()}
        preds.append((left, right))
    if device != "cpu":
        gts = [{k: t.to(device) for k, t in d.items()} for d in gts]
        preds = [tuple({k: t.to(device) for k, t in d.items()} for d in p) for p in preds]
    return gts, preds


# the cases of tests/golden/loss_<name>.npz: criterion string, call ("loss" = compute_frame_loss, "pts" =
# get_all_pts3d_t), keyword arguments, data (make_loss_case arguments)
LOSS_CASES = {
    "train": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)", "call": "loss",
              "data": {"batch": 2, "frames": 5, "height": 224, "width": 224, "invalid": 0.3, "seed": 1}},
    "test": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=True)", "call": "loss",
             "data": {"batch": 2, "frames": 4, "height": 224, "width": 224, "invalid": 0.3, "seed": 2}},
    "eval": {"criterion": "Regr3D_t_ScaleShiftInv(L21, norm_mode=False, gt_scale=True)", "call": "pts",
             "data": {"batch": 1, "frames": 4, "height": 224, "width": 224, "invalid": 0.2, "seed": 3}},
    "log1p_fixfirst_clip": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_log1p', fix_first=True), alpha=0.2)",
                            "call": "loss", "kw": {"dist_clip": 3.0},
                            "data": {"batch": 2, "frames": 3, "height": 64, "width": 96, "invalid": 0.3, "seed": 4}},
    "scaleinv": {"criterion": "Regr3D_t_ScaleInv(L21, gt_scale=False, fix_first=False)", "call": "loss",
                 "data": {"batch": 3, "frames": 3, "height": 64, "width": 64, "invalid": 0.3, "seed": 5}},
    "regr_mean": {"criterion": "Regr3D_t(L21, norm_mode='avg_dis')", "call": "loss",
                  "data": {"batch": 2, "frames": 3, "height": 48, "width": 64, "invalid": 0.3, "seed": 6}},
    "landscape": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)", "call": "loss",
                  "data": {"batch": 1, "frames": 3, "height": 384, "width": 512, "invalid": 0.3, "seed": 7}},
    "even_pts": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=False)", "call": "pts",
                 "data": {"batch": 2, "frames": 3, "height": 32, "width": 48, "invalid": 0.0, "seed": 8}},
}


def loss_slot(preds, k, side):
    """The pts map of pred slot (pair k, side 0 = left / 1 = right) in `preds_all`."""
    return preds[k][side]["pts3d" if (k == 0 and side == 0) else "pts3d_in_other_view"]


def _adv_empty_b(gts, preds):          # batch element 1 has no valid pixel in any frame
    for g in gts:
        g["valid_mask"][1] = False


def _adv_single_px(gts, preds):        # batch element 0 has exactly one valid pixel, in frame 1
    for g in gts:
        g["valid_mask"][0] = False
    gts[1]["valid_mask"][0, 5, 7] = True


def _adv_planar(gts, preds):
    """Planar steps: every view's depth is 2 (top half) or 3 (bottom half) in one common camera, so half of all values
    tie at each of the two middle ranks; x / y are column / row constant with exact -0.0 and +0.0 columns; predictions
    are column-constant in z.  All pixels valid: an even count, the lower median a real choice."""
    B, H, W, _ = gts[0]["pts3d"].shape
    col = (torch.arange(W, dtype=torch.float32) - W // 2) / 8
    row = (torch.arange(H, dtype=torch.float32) - H // 2) / 8
    z = torch.where(torch.arange(H)[:, None] < H // 2, 2.0, 3.0).expand(H, W)
    for f, g in enumerate(gts):
        x = col.expand(H, W).clone()
        x[:, W // 2] = -0.0 if f % 2 == 0 else 0.0
        g["pts3d"] = torch.stack((x, row[:, None].expand(H, W), z), -1).expand(B, H, W, 3).contiguous()
        g["camera_pose"] = torch.eye(4).repeat(B, 1, 1)
    for k in range(len(preds)):
        for side in (0, 1):
            p = loss_slot(preds, k, side)
            p[..., 2] = (1.0 + torch.arange(W, dtype=torch.float32) / 4).expand(H, W)


def _adv_nan_invalid(gts, preds):      # real depth maps: NaN (and a few +-inf) at the invalid pixels of the ground truth
    for g in gts:
        inv = ~g["valid_mask"]
        g["pts3d"][inv] = float("nan")
        idx = inv.nonzero()[:4]
        for j, (b, i, w) in enumerate(idx.tolist()):
            g["pts3d"][b, i, w] = float("inf") if j % 2 else -float("inf")


def _adv_clipped_factor(gts, preds):   # batch element 0's predictions are so small that its norm factor is clipped
    for k in range(len(preds)):
        for side in (0, 1):
            loss_slot(preds, k, side)[0] *= 1e-10


def _adv_dist_clip_eq(gts, preds):
    """Ground-truth points at exactly dist_clip = 3 from the origin and one ulp either side, forced valid: the clip
    keeps a point at the radius (<=) and drops the next float up."""
    up32 = float(np.nextafter(np.float32(3.0), np.float32(4.0)))
    down32 = float(np.nextafter(np.float32(3.0), np.float32(0.0)))
    pts = [(3, 0, 0), (0, -3, 0), (1, 2, 2), (-2, 1, -2), (up32, 0, 0), (0, 0, -up32), (down32, 0, 0), (0, down32, 0)]
    for f, g in enumerate(gts):
        for j, p in enumerate(pts):
            b, i, w = j % 2, 1 + j, 2 + 2 * j + f
            g["pts3d"][b, i, w] = torch.tensor(p, dtype=torch.float32)
            g["valid_mask"][b, i, w] = True


def _adv_empty_term(gts, preds):       # frame 2 has no valid pixel in any batch element
    gts[2]["valid_mask"][:] = False


def _adv_d_zero(gts, preds):
    """View 0's camera at the identity, so the ground truth reaches the criterion unchanged; on even columns the
    predictions equal it exactly (d == 0); conf exactly 1 on even rows and 1e30 on every fourth odd row."""
    for g in gts:
        g["pts3d"] = g["pts3d"].contiguous()
    gts[0]["camera_pose"] = torch.eye(4).repeat(gts[0]["camera_pose"].shape[0], 1, 1)
    for k in range(len(preds)):
        for side in (0, 1):
            p = loss_slot(preds, k, side)
            p[:, :, 0::2] = gts[k + side]["pts3d"][:, :, 0::2]
            c = preds[k][side]["conf"]
            c[:, 0::2] = 1.0
            c[:, 1::4] = 1e30


# adversarial cases of tests/golden/loss_adv_<name>.npz (tools/make_golden_loss_adv.py): as LOSS_CASES, plus the edit
# applied to make_loss_case's views and predictions (make_loss_adv_case)
LOSS_ADV_CASES = {
    "empty_b": {"criterion": "Regr3D_t(L21, norm_mode='avg_dis', fix_first=False)", "call": "loss", "edit": "empty_b",
                "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 41}},
    "empty_b_ssi": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=False)", "call": "pts", "edit": "empty_b",
                    "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 42}},
    "single_px": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=True)", "call": "loss", "edit": "single_px",
                  "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 43}},
    "planar": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=False)", "call": "pts", "edit": "planar",
               "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.0, "seed": 44}},
    "planar_loss": {"criterion": "Regr3D_t_ScaleShiftInv(L21, gt_scale=True)", "call": "loss", "edit": "planar",
                    "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.0, "seed": 45}},
    "nan_invalid": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)",
                    "call": "loss", "edit": "nan_invalid",
                    "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 46}},
    "clipped_factor": {"criterion": "Regr3D_t(L21, norm_mode='avg_dis', fix_first=False)", "call": "loss",
                       "edit": "clipped_factor",
                       "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 47}},
    "dist_clip_eq": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_log1p', fix_first=True), alpha=0.2)",
                     "call": "loss", "kw": {"dist_clip": 3.0}, "edit": "dist_clip_eq",
                     "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 48}},
    "f2": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)", "call": "loss",
           "edit": None, "data": {"batch": 2, "frames": 2, "height": 16, "width": 24, "invalid": 0.3, "seed": 49}},
    "empty_term": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)",
                   "call": "loss", "edit": "empty_term",
                   "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 50}},
    "d_zero": {"criterion": "ConfLoss_t(Regr3D_t(L21, norm_mode=False), alpha=0.4)", "call": "loss", "edit": "d_zero",
               "data": {"batch": 2, "frames": 3, "height": 16, "width": 24, "invalid": 0.3, "seed": 51}},
}

_ADV_EDITS = {"empty_b": _adv_empty_b, "single_px": _adv_single_px, "planar": _adv_planar,
              "nan_invalid": _adv_nan_invalid, "clipped_factor": _adv_clipped_factor,
              "dist_clip_eq": _adv_dist_clip_eq, "empty_term": _adv_empty_term, "d_zero": _adv_d_zero}


def make_loss_adv_case(name: str, device="cpu"):
    """Views and `preds_all` of LOSS_ADV_CASES[name]: make_loss_case's, edited; fp32 CPU tensors (moved to `device`)."""
    case = LOSS_ADV_CASES[name]
    gts, preds = make_loss_case(**case["data"])
    if case["edit"]:
        _ADV_EDITS[case["edit"]](gts, preds)
    if device != "cpu":
        gts = [{k: t.to(device) for k, t in d.items()} for d in gts]
        preds = [tuple({k: t.to(device) for k, t in d.items()} for d in p) for p in preds]
    return gts, preds


# ---- dataset views (spann3r_b200/views.py): golden cases of tests/golden/views.json (tools/make_golden_views.py),
# regenerated from their parameters by the tests, and a 7Scenes-layout scene on disk for the loader tests / benchmark

_SEVEN_K = (525.0, 525.0, 320.0, 240.0)

VIEW_CASES = [  # name, h, w, (fx, fy, cx, cy), views, resolution, aug_crop, item seed, depth kind, pose kind
    dict(name="7scenes_224", h=480, w=640, K=_SEVEN_K, views=3, res=(224, 224), aug=0, seed=1, depth="std", pose="random"),
    dict(name="7scenes_512", h=480, w=640, K=_SEVEN_K, views=2, res=(512, 384), aug=0, seed=2, depth="std", pose="random"),
    dict(name="dtu_512", h=1200, w=1600, K=(2892.33, 2883.18, 823.205, 619.071), views=1, res=(512, 384), aug=0, seed=3,
         depth="std", pose="random"),
    dict(name="offcentre_224", h=480, w=640, K=(530.5, 529.25, 301.5, 254.5), views=2, res=(224, 224), aug=0, seed=4,
         depth="std", pose="random"),
    dict(name="portrait_512", h=640, w=480, K=(500.0, 500.0, 240.0, 320.0), views=2, res=(512, 384), aug=0, seed=5,
         depth="std", pose="random"),
    dict(name="portrait_224", h=640, w=480, K=(500.0, 500.0, 241.0, 318.0), views=1, res=(224, 224), aug=0, seed=6,
         depth="std", pose="random"),
    dict(name="square_512", h=600, w=600, K=(600.0, 600.0, 300.0, 300.0), views=4, res=(512, 384), aug=0, seed=14,
         depth="std", pose="random"),
    dict(name="aug16_a", h=480, w=640, K=_SEVEN_K, views=2, res=(224, 224), aug=16, seed=8, depth="std", pose="random"),
    dict(name="aug16_b", h=480, w=640, K=_SEVEN_K, views=2, res=(224, 224), aug=16, seed=9, depth="std", pose="random"),
    dict(name="aug16_c", h=480, w=640, K=_SEVEN_K, views=2, res=(512, 384), aug=16, seed=10, depth="std", pose="random"),
    dict(name="extreme_depth", h=480, w=640, K=(150.0, 150.0, 320.0, 240.0), views=1, res=(224, 224), aug=0, seed=11,
         depth="extreme", pose="identity"),
    dict(name="no_pose", h=480, w=640, K=_SEVEN_K, views=1, res=(224, 224), aug=0, seed=12, depth="std", pose="none"),
]


def _random_rotation(g) -> np.ndarray:
    q = g.standard_normal(4)
    a, b, c, d = q / np.linalg.norm(q)
    return np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                     [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                     [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])


def make_view_case(case) -> list:
    """Deterministic [(rgb uint8, depth float32, K float32, pose float32 4x4 or None)] of a VIEW_CASES entry."""
    g = np.random.default_rng(1000 + case["seed"])
    fx, fy, cx, cy = case["K"]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32)
    h, w = case["h"], case["w"]
    out = []
    for _ in range(case["views"]):
        rgb = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
        depth = g.uniform(0.3, 6.0, (h, w)).astype(np.float32)
        depth[g.random((h, w)) < 0.1] = 0.0
        if case["depth"] == "extreme":
            depth[g.random((h, w)) < 0.2] = np.float32(3.0e38)
        if case["pose"] == "random":
            pose = np.eye(4)
            pose[:3, :3] = _random_rotation(g)
            pose[:3, 3] = g.uniform(-2.0, 2.0, 3)
            pose = pose.astype(np.float32)
        elif case["pose"] == "identity":
            pose = np.eye(4, dtype=np.float32)
        else:
            pose = None
        out.append((rgb, depth, K, pose))
    return out


def write_7scenes_sequence(root: str, frames: int = 6, seed: int = 0):
    """A 7Scenes-layout sequence in `root`: frame-XXXXXX.color.png (RGB 640x480, part gradient, part noise),
    .depth.proj.png (uint16 mm, 65535 = missing) and .pose.txt (cam-to-world 4x4).  PNG decodes identically across
    library versions."""
    import cv2
    g = np.random.default_rng(seed)
    os.makedirs(root, exist_ok=True)
    yy, xx = np.mgrid[0:480, 0:640]
    for i in range(frames):
        rgb = np.stack([(xx * (i + 1) // 7) % 256, (yy * 3 + 40 * i) % 256, g.integers(0, 256, (480, 640))], -1)
        cv2.imwrite(os.path.join(root, f"frame-{i:06d}.color.png"), rgb.astype(np.uint8)[..., ::-1])
        depth = g.integers(300, 6000, (480, 640)).astype(np.uint16)
        depth[g.random((480, 640)) < 0.05] = 65535
        depth[g.random((480, 640)) < 0.05] = 0
        cv2.imwrite(os.path.join(root, f"frame-{i:06d}.depth.proj.png"), depth)
        pose = np.eye(4)
        pose[:3, :3] = _random_rotation(g)
        pose[:3, 3] = g.uniform(-1, 1, 3)
        np.savetxt(os.path.join(root, f"frame-{i:06d}.pose.txt"), pose)


class SevenScenesLike:
    """Duck-typed stand-in for the reference's SevenScenes(full_video=True, kf_every=...) over a sequence written by
    write_7scenes_sequence: the same decoding and depth clean-up (spann3r/datasets/seven_scenes.py:87-143), then
    `_crop_resize_if_necessary` per frame, with ImgNorm as transform."""

    def __init__(self, root: str, resolution=224, kf_every: int = 2, seed: int = 7, aug_crop=0):
        import torchvision.transforms as tvf
        self.ROOT, self.kf_every, self.seed, self.aug_crop = root, kf_every, seed, aug_crop
        self._resolutions = [(resolution, resolution) if isinstance(resolution, int) else tuple(resolution)]
        self.transform = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])

    def __len__(self):
        return 1

    def _get_views(self, idx, resolution, rng):
        import cv2
        n = len([f for f in os.listdir(self.ROOT) if "color" in f])
        K = np.array([[525, 0, 320], [0, 525, 240], [0, 0, 1]], dtype=np.float32)
        views = []
        for im_idx in [f"{i:06d}" for i in range(n)][::self.kf_every]:
            rgb = cv2.cvtColor(cv2.imread(os.path.join(self.ROOT, f"frame-{im_idx}.color.png")), cv2.COLOR_BGR2RGB)
            depth = cv2.imread(os.path.join(self.ROOT, f"frame-{im_idx}.depth.proj.png"), cv2.IMREAD_UNCHANGED)
            depth[depth == 65535] = 0
            depth = np.nan_to_num(depth.astype(np.float32), 0.0) / 1000.0
            depth[depth > 10] = 0
            depth[depth < 1e-3] = 0
            pose = np.loadtxt(os.path.join(self.ROOT, f"frame-{im_idx}.pose.txt")).astype(np.float32)
            rgb, depth, Kf = self._crop_resize_if_necessary(rgb, depth, K, resolution, rng=rng, info=im_idx)
            views.append(dict(img=rgb, depthmap=depth, camera_pose=pose, camera_intrinsics=Kf, dataset="7scenes",
                              label=im_idx, instance=im_idx))
        return views


def write_co3d_tree(root: str, frames: int = 10, width: int = 320, height: int = 240, seed: int = 0,
                    zero_frames=(3,), category: str = "apple", instance: str = "110_13051_23361"):
    """A tree in the layout of the reference's preprocessed Co3d (spann3r/datasets/co3d.py): selected_seqs_train.json,
    <cat>/<inst>/images/frameNNNNNN.jpg (+ .npz with camera_pose, camera_intrinsics, maximum_depth),
    depths/frameNNNNNN.jpg.geometric.png (uint16, depth / maximum_depth * 65535) and masks/frameNNNNNN.png (uint8).
    Frames in `zero_frames` have an all-zero depth map, so the dataset's invalidate / retry path fires on them.
    Principal points wander around the centre; some frames are portrait crops."""
    import cv2
    g = np.random.default_rng(seed)
    base = os.path.join(root, category, instance)
    for sub in ("images", "depths", "masks"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    yy, xx = np.mgrid[0:height, 0:width]
    ids = list(range(1, frames + 1))
    for k, fid in enumerate(ids):
        rgb = np.stack([(xx * (k + 2) // 5 + yy) % 256, (yy * 3 + 25 * k) % 256, g.integers(0, 256, (height, width))], -1)
        name = f"frame{fid:06d}"
        cv2.imwrite(os.path.join(base, "images", name + ".jpg"), rgb.astype(np.uint8)[..., ::-1])
        maxd = np.float32(g.uniform(4.0, 6.0))
        depth = g.integers(2000, 65535, (height, width)).astype(np.uint16)
        depth[g.random((height, width)) < 0.1] = 0
        if k in zero_frames:
            depth[:] = 0
        cv2.imwrite(os.path.join(base, "depths", name + ".jpg.geometric.png"), depth)
        mask = np.where(g.random((height, width)) < 0.8, 255, g.integers(0, 40, (height, width))).astype(np.uint8)
        cv2.imwrite(os.path.join(base, "masks", name + ".png"), mask)
        f = g.uniform(0.8, 1.2) * width
        cx, cy = width / 2 + g.uniform(-8, 8), height / 2 + g.uniform(-8, 8)
        if k % 4 == 1:                      # a portrait crop: the principal point near a side
            cx = width * 0.3
        K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], dtype=np.float32)
        pose = np.eye(4, dtype=np.float32)
        pose[:3, :3] = _random_rotation(g)
        pose[:3, 3] = g.uniform(-1, 1, 3)
        np.savez(os.path.join(base, "images", name + ".npz"), camera_pose=pose, camera_intrinsics=K, maximum_depth=maxd)
    with open(os.path.join(root, "selected_seqs_train.json"), "w") as fh:
        json.dump({category: {instance: ids}, "empty": {}}, fh)


def _imread_rgb(path, flags=None):
    import cv2
    img = cv2.imread(path, cv2.IMREAD_COLOR if flags is None else flags)
    if img is None:
        raise IOError(f"could not load image {path}")
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB) if img.ndim == 3 else img


class _ManyViewLike:
    """What the duck-typed training sets below share with the reference's BaseManyViewDataset: the base options, the
    transform (ImgNorm or the reference's Compose([ColorJitter(0.5, 0.5, 0.5, 0.1), ImgNorm])) and sample_frames.
    `_crop_resize_if_necessary` comes from whoever builds the views (TrainViews, or the oracle)."""

    def __init__(self, ROOT, resolution, num_frames, jitter, seed, min_thresh, max_thresh, num_seq, aug_crop, split):
        import torchvision.transforms as tvf
        self.ROOT, self.split, self.num_frames, self.seed = ROOT, split, num_frames, seed
        self.min_thresh, self.max_thresh, self.num_seq, self.aug_crop = min_thresh, max_thresh, num_seq, aug_crop
        self.train_ratio = 0.5
        self._resolutions = [(resolution, resolution) if isinstance(resolution, int) else tuple(resolution)]
        norm = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])
        self.transform = tvf.Compose([tvf.ColorJitter(0.5, 0.5, 0.5, 0.1), norm]) if jitter else norm

    def __len__(self):
        return len(self.scene_list) * self.num_seq

    def sample_frames(self, img_idxs, rng):
        n = self.num_frames
        thresh = int(self.min_thresh + self.train_ratio * (self.max_thresh - self.min_thresh))
        pool = list(range(len(img_idxs)))
        first_span = max(len(pool) // n, len(pool) - thresh * (n - 1))
        cur = rng.choice(pool[:first_span])
        chosen = [cur]
        while len(chosen) < n:
            hi = min(cur + thresh, len(pool) - (n - len(chosen)))
            cand = [i for i in range(cur + 1, hi + 1) if i not in chosen]
            if not cand:
                break
            cur = rng.choice(cand)
            chosen.append(cur)
        if len(chosen) < n:
            return self.sample_frames(img_idxs, rng)
        out = [img_idxs[i] for i in chosen]
        if rng.choice([True, False]):
            out.reverse()
        return out


class Co3dLike(_ManyViewLike):
    """Duck-typed stand-in for the reference's training Co3d(use_comb=False, ...) (spann3r/datasets/co3d.py with
    BaseManyViewDataset.sample_frames) over a tree written by write_co3d_tree, for tests that cannot import the
    reference: the same frame sampling, background masking, invalidate / retry loop and depth-range resampling, with
    the same numpy RNG draws."""

    def __init__(self, ROOT, resolution=224, num_frames=3, mask_bg="rand", jitter=True, seed=None, min_thresh=2,
                 max_thresh=5, num_seq=20, aug_crop=0, split="train"):
        super().__init__(ROOT, resolution, num_frames, jitter, seed, min_thresh, max_thresh, num_seq, aug_crop, split)
        self.mask_bg = mask_bg
        with open(os.path.join(ROOT, f"selected_seqs_{split}.json")) as fh:
            seqs = json.load(fh)
        self.scenes = {(c, i): v for c, insts in seqs.items() if len(insts) > 0 for i, v in insts.items()}
        self.scene_list = list(self.scenes)
        self.invalidate = {s: {} for s in self.scene_list}

    def _get_views(self, idx, resolution, rng):
        import cv2
        from collections import deque
        obj, inst = self.scene_list[idx // self.num_seq]
        pool = self.scenes[obj, inst]
        order = self.sample_frames(range(0, len(pool)), rng)
        bad = self.invalidate[obj, inst].setdefault(resolution, [False] * len(pool))
        mask_bg = (self.mask_bg is True) or (self.mask_bg == "rand" and rng.choice(2))
        queue = deque(order)
        dmin, dmax, dfirst = 1e8, 0.0, None
        views = []
        while queue:
            im = queue.popleft()
            if bad[im]:
                step = 2 * rng.choice(2) - 1
                for off in range(1, len(pool)):
                    alt = (im + step * off) % len(pool)
                    if not bad[alt]:
                        im = alt
                        break
            path = os.path.join(self.ROOT, obj, inst, "images", f"frame{pool[im]:06d}.jpg")
            meta = np.load(path.replace("jpg", "npz"))
            pose = meta["camera_pose"].astype(np.float32)
            K = meta["camera_intrinsics"].astype(np.float32)
            rgb = _imread_rgb(path)
            depth = _imread_rgb(path.replace("images", "depths") + ".geometric.png", cv2.IMREAD_UNCHANGED)
            depth = (depth.astype(np.float32) / 65535) * np.nan_to_num(meta["maximum_depth"])
            if mask_bg:
                m = _imread_rgb(os.path.join(self.ROOT, obj, inst, "masks", f"frame{pool[im]:06d}.png"),
                                cv2.IMREAD_UNCHANGED).astype(np.float32)
                depth *= (m / 255.0) > 0.1
            rgb, depth, K = self._crop_resize_if_necessary(rgb, depth, K, resolution, rng=rng, info=path)
            if (depth > 0.0).sum() == 0:
                bad[im] = True
                queue.appendleft(im)
                continue
            md = meta["maximum_depth"]
            if md > dmax:
                dmax = md
            if md < dmin:
                dmin = md
            if dfirst is None:
                dfirst = md
            views.append(dict(img=rgb, depthmap=depth, camera_pose=pose, camera_intrinsics=K, dataset="Co3d_v2",
                              label=os.path.join(obj, inst), instance=os.path.split(path)[1]))
        if dmax / dmin > 100.0 or dmax / dfirst > 10.0:
            return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
        return views


def _scene_frames(g, k, width, height, zero):
    """One synthetic frame: RGB (part gradient, part noise), depth in metres (10 % holes; all zero when `zero`)."""
    yy, xx = np.mgrid[0:height, 0:width]
    rgb = np.stack([(xx * (k + 3) // 4 + 2 * yy) % 256, (yy * 5 + 31 * k) % 256, g.integers(0, 256, (height, width))], -1)
    depth = g.uniform(0.5, 4.0, (height, width)).astype(np.float32)
    depth[g.random((height, width)) < 0.1] = 0
    if zero:
        depth[:] = 0
    return rgb.astype(np.uint8), depth


def write_scannetpp_tree(root: str, frames: int = 10, width: int = 320, height: int = 240, seed: int = 0,
                         zero_frames=(3,), scene: str = "0a5c013435"):
    """A tree in the layout of the reference's preprocessed ScanNet++ (spann3r/datasets/scannetpp.py):
    splits/nvs_sem_train.txt, data/<scene>/dslr/nerfstudio/transforms_undistorted.json (fl_x, fl_y, cx, cy and a
    cam-to-world OpenGL `transform_matrix` per frame), dslr/train_test_lists.json, dslr/undistorted_images/*.JPG and
    dslr/undistorted_depths/*.png (uint16 mm).  Frames in `zero_frames` have an all-zero depth map, so the dataset's
    recursive retry fires on them."""
    import cv2
    g = np.random.default_rng(seed)
    base = os.path.join(root, "data", scene, "dslr")
    for sub in ("nerfstudio", "undistorted_images", "undistorted_depths"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    os.makedirs(os.path.join(root, "splits"), exist_ok=True)
    names, metas = [], []
    for k in range(frames):
        name = f"DSC{k + 1:05d}.JPG"
        rgb, depth = _scene_frames(g, k, width, height, k in zero_frames)
        cv2.imwrite(os.path.join(base, "undistorted_images", name), rgb[..., ::-1])
        cv2.imwrite(os.path.join(base, "undistorted_depths", name.replace(".JPG", ".png")),
                    np.round(depth * 1000).astype(np.uint16))
        pose = np.eye(4)
        pose[:3, :3] = _random_rotation(g)
        pose[:3, 3] = g.uniform(-1, 1, 3)
        names.append(name)
        metas.append({"file_path": name, "transform_matrix": pose.tolist()})
    f = float(g.uniform(0.8, 1.2) * width)
    cams = {"fl_x": f, "fl_y": f * 1.01, "cx": width / 2 + 3.3, "cy": height / 2 - 2.6, "frames": metas[::-1]}
    with open(os.path.join(base, "nerfstudio", "transforms_undistorted.json"), "w") as fh:
        json.dump(cams, fh)
    with open(os.path.join(base, "train_test_lists.json"), "w") as fh:
        json.dump({"train": names[::-1], "test": []}, fh)
    with open(os.path.join(root, "splits", "nvs_sem_train.txt"), "w") as fh:
        fh.write(scene + "\n")


class ScannetppLike(_ManyViewLike):
    """Duck-typed stand-in for the reference's training Scannetpp (spann3r/datasets/scannetpp.py) over a tree written
    by write_scannetpp_tree: the same frame sampling and the same recursive retry (`attempts`) on a frame without valid
    depth, with the same numpy RNG draws."""

    def __init__(self, ROOT, resolution=224, num_frames=3, jitter=True, seed=None, min_thresh=2, max_thresh=5,
                 num_seq=20, aug_crop=0, split="train"):
        super().__init__(ROOT, resolution, num_frames, jitter, seed, min_thresh, max_thresh, num_seq, aug_crop, split)
        with open(os.path.join(ROOT, "splits", f"nvs_sem_{split}.txt")) as fh:
            self.scene_list = fh.read().splitlines()

    def _get_views(self, idx, resolution, rng, attempts=0):
        import cv2
        scene = self.scene_list[idx // self.num_seq]
        base = os.path.join(self.ROOT, "data", scene, "dslr")
        with open(os.path.join(base, "nerfstudio", "transforms_undistorted.json")) as fh:
            cams = json.load(fh)
        with open(os.path.join(base, "train_test_lists.json")) as fh:
            order = self.sample_frames(sorted(json.load(fh)["train"]), rng)
        by_path = {fr["file_path"]: i for i, fr in enumerate(cams["frames"])}
        K = np.array([[cams["fl_x"], 0, cams["cx"]], [0, cams["fl_y"], cams["cy"]], [0, 0, 1]], dtype=np.float32)
        views = []
        for name in order:
            path = os.path.join(base, "undistorted_images", name)
            rgb = _imread_rgb(path)
            depth = _imread_rgb(os.path.join(base, "undistorted_depths", name.replace(".JPG", ".png")),
                                cv2.IMREAD_UNCHANGED)
            depth = np.nan_to_num(depth.astype(np.float32), 0.0) / 1000.0
            pose = np.array(cams["frames"][by_path[name]]["transform_matrix"], dtype=np.float32)
            pose[:, 1:3] *= -1.0
            rgb, depth, Kf = self._crop_resize_if_necessary(rgb, depth, K, resolution, rng=rng, info=path)
            if (depth > 0.0).sum() == 0 or not np.isfinite(pose).all():
                if attempts >= 5:
                    return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
                return self._get_views(idx, resolution, rng, attempts + 1)
            views.append(dict(img=rgb, depthmap=depth, camera_pose=pose, camera_intrinsics=Kf, dataset="scannetpp",
                              label=os.path.join(scene, name), instance=os.path.split(path)[1]))
        return views


def write_blendmvs_tree(root: str, frames: int = 10, width: int = 320, height: int = 256, seed: int = 0,
                        zero_frames=(3,), scene: str = "5a3ca9cb270f0e3f14d0eddb"):
    """A tree in the layout of the reference's BlendedMVS (spann3r/datasets/blendedmvs.py): train_list.txt,
    <scene>/blended_images/NNNNNNNN.jpg, rendered_depth_maps/NNNNNNNN.pfm (float32), cams/NNNNNNNN_cam.txt (MVSNet
    text: world-to-cam extrinsic, intrinsic) and cams/pair.txt (MVSNet view clusters).  Frames in `zero_frames` have an
    all-zero depth map, so the dataset's recursive retry fires on them."""
    import cv2
    g = np.random.default_rng(seed)
    base = os.path.join(root, scene)
    for sub in ("blended_images", "rendered_depth_maps", "cams"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    for k in range(frames):
        rgb, depth = _scene_frames(g, k, width, height, k in zero_frames)
        cv2.imwrite(os.path.join(base, "blended_images", f"{k:08d}.jpg"), rgb[..., ::-1])
        cv2.imwrite(os.path.join(base, "rendered_depth_maps", f"{k:08d}.pfm"), depth)
        c2w = np.eye(4)
        c2w[:3, :3] = _random_rotation(g)
        c2w[:3, 3] = g.uniform(-1, 1, 3)
        w2c = np.linalg.inv(c2w)
        f = g.uniform(0.8, 1.2) * width
        K = np.array([[f, 0, width / 2 + g.uniform(-6, 6)], [0, f, height / 2 + g.uniform(-6, 6)], [0, 0, 1]])
        with open(os.path.join(base, "cams", f"{k:08d}_cam.txt"), "w") as fh:
            fh.write("extrinsic\n" + "\n".join(" ".join(f"{v:.9g}" for v in row) for row in w2c) + "\n\n")
            fh.write("intrinsic\n" + "\n".join(" ".join(f"{v:.9g}" for v in row) for row in K) + "\n\n")
            fh.write("425.0 2.5\n")
    with open(os.path.join(base, "cams", "pair.txt"), "w") as fh:
        fh.write(f"{frames}\n")
        for k in range(frames):
            others = [j for j in range(frames) if j != k][: frames - 2]
            fh.write(f"{k}\n{len(others)} " + " ".join(f"{j} {100.0 - j:.1f}" for j in others) + "\n")
    with open(os.path.join(root, "train_list.txt"), "w") as fh:
        fh.write(scene + "\n")


class BlendMVSLike(_ManyViewLike):
    """Duck-typed stand-in for the reference's BlendMVS (spann3r/datasets/blendedmvs.py) over a tree written by
    write_blendmvs_tree: the same pair sampling, the margin check, `depthmap.max()` of every cropped depth map for the
    depth-range check, and the same recursive retry (`attempts`) on a frame without valid depth."""

    def __init__(self, ROOT, resolution=224, num_frames=3, jitter=True, seed=None, min_thresh=2, max_thresh=5,
                 num_seq=20, aug_crop=0, split="train"):
        super().__init__(ROOT, resolution, num_frames, jitter, seed, min_thresh, max_thresh, num_seq, aug_crop, split)
        with open(os.path.join(ROOT, f"{split}_list.txt")) as fh:
            self.scene_list = fh.read().splitlines()

    def sample_pairs(self, pairs_path, rng, max_trials=10):
        with open(pairs_path) as fh:
            lines = fh.read().splitlines()
        for _ in range(max_trials):
            s = rng.choice(int(lines[0]))
            ref, cluster = int(lines[2 * s + 1]), lines[2 * s + 2].split()
            n = int(cluster[0])
            if n > self.num_frames - 1:
                names = [f"{ref:08d}.jpg"] + [f"{int(cluster[2 * c + 1]):08d}.jpg"
                                               for c in rng.choice(n, self.num_frames - 1, replace=False)]
                if rng.choice([True, False]):
                    names.reverse()
                return names
        return None

    @staticmethod
    def _read_cam(path):
        with open(path) as fh:
            lines = fh.read().splitlines()
        RT = np.array([row.split() for row in lines[1:5]], dtype=np.float32)
        K = np.array([row.split() for row in lines[7:10]], dtype=np.float32)
        return K, RT

    def _get_views(self, idx, resolution, rng, attempts=0):
        import cv2
        scene = self.scene_list[idx // self.num_seq]
        base = os.path.join(self.ROOT, scene)
        names = self.sample_pairs(os.path.join(base, "cams", "pair.txt"), rng)
        if names is None:
            return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
        dmin, dmax, dfirst = 1e8, 0.0, None
        views = []
        for name in names:
            path = os.path.join(base, "blended_images", name)
            rgb = _imread_rgb(path)
            depth = _imread_rgb(os.path.join(base, "rendered_depth_maps", name.replace(".jpg", ".pfm")),
                                cv2.IMREAD_UNCHANGED)
            depth = np.nan_to_num(depth.astype(np.float32), 0.0)
            K, RT = self._read_cam(os.path.join(base, "cams", name.replace(".jpg", "_cam.txt")))
            K = K[:3, :3]
            pose = np.linalg.inv(RT)
            H, W = rgb.shape[:2]
            cx, cy = K[:2, 2].round().astype(int)
            if min(cx, W - cx) <= W / 5 or min(cy, H - cy) <= H / 5:
                return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
            rgb, depth, Kf = self._crop_resize_if_necessary(rgb, depth, K, resolution, rng=rng, info=path)
            dm = depth.max()
            if dm > dmax:
                dmax = dm
            if dm < dmin:
                dmin = dm
            if dfirst is None:
                dfirst = dm
            if (depth > 0.0).sum() == 0 or not np.isfinite(pose).all():
                if attempts >= 5:
                    return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
                return self._get_views(idx, resolution, rng, attempts + 1)
            views.append(dict(img=rgb, depthmap=depth, camera_pose=pose, camera_intrinsics=Kf, dataset="blendmvs",
                              label=os.path.join(scene, name), instance=os.path.split(path)[1]))
        if dmax / dmin > 100.0 or dmax / dfirst > 10.0:
            return self._get_views(rng.integers(0, len(self) - 1), resolution, rng)
        return views
