"""Offline reconstruction's pair graph on the CUDA engine, without the reference's Python.

The reference's offline mode (demo.py / eval.py `--offline`) builds a scene graph with `dust3r.image_pairs.make_pairs`,
runs `dust3r.inference.inference` over it (every pair forward re-encodes both images; every batch is symmetrised a
second time) and hands the result to `Spann3R.offline_reconstruction`, which reads one number per pair from it.  This
module provides:

* `make_pairs`: the reference's scene graphs and prefilters, same pairs in the same order.
* `inference`: a drop-in for `dust3r.inference.inference(pairs, model.dust3r, ...)` that encodes each distinct image once
  and decodes each distinct ordered pair once, batched.  Same dict, same entry order, results on the CPU.
* `pair_scores`: only what `find_initial_pair` reads -- the [F, F] matrix of summed per-head means of (c-1)/c -- kept on
  the device, from batched decodes and one batched score kernel (`s3r_conf_score_batched`) per batch.

`Spann3R.offline_reconstruction(frames)` (no graph) uses `pair_scores` for its initial pair and `next_best_view` to score
the next-best-view candidates in batches.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import conf_score_batched


# ------------------------------------------------------------------------------------------------
# scene graphs (dust3r/image_pairs.py semantics)
# ------------------------------------------------------------------------------------------------
def make_pairs(imgs, scene_graph="complete", prefilter=None, symmetrize=True):
    """List of (view_a, view_b) over `imgs`, in the reference's order.

    scene_graph: 'complete' (every (i, j) with j < i), 'swin' / 'swin-k' (each frame with its next k, default 3, wrapping
    around; each unordered edge once, in the order of a Python set of (low, high) tuples, as the reference iterates it),
    'oneref' / 'oneref-k' (frame k, default 0, with every other frame), 'prev' (every (j, i) with j < i).
    symmetrize appends the reversed pairs.  prefilter 'seqN' keeps pairs whose 'idx' values are at most N apart, 'cycN'
    the same with wrap-around distance over n = 1 + the largest idx.  As in the reference, 'oneref-k' with k past the
    end raises IndexError and a prefilter over no pairs raises ValueError."""
    n = len(imgs)
    if scene_graph == "complete":
        ids = [(i, j) for i in range(n) for j in range(i)]
    elif scene_graph.startswith("swin"):
        win = int(scene_graph.split("-")[1]) if "-" in scene_graph else 3
        edges = set()
        for i in range(n):
            for d in range(1, win + 1):
                k = (i + d) % n
                edges.add((min(i, k), max(i, k)))
        ids = list(edges)
    elif scene_graph.startswith("oneref"):
        ref = int(scene_graph.split("-")[1]) if "-" in scene_graph else 0
        ids = [(ref, j) for j in range(n) if j != ref]
    elif scene_graph.startswith("prev"):
        ids = [(j, i) for i in range(1, n) for j in range(i)]
    else:
        raise ValueError(f"unknown scene graph {scene_graph!r} (complete, swin[-k], oneref[-k], prev)")
    pairs = [(imgs[i], imgs[j]) for i, j in ids]
    if symmetrize:
        pairs += [(b, a) for a, b in pairs]
    if isinstance(prefilter, str) and prefilter.startswith("seq"):
        pairs = _filter_seq(pairs, int(prefilter[3:]), cyclic=False)
    if isinstance(prefilter, str) and prefilter.startswith("cyc"):
        pairs = _filter_seq(pairs, int(prefilter[3:]), cyclic=True)
    return pairs


def _filter_seq(pairs, max_dist, cyclic):
    edges = [(a["idx"], b["idx"]) for a, b in pairs]
    n = 1 + max(max(e) for e in edges)          # ValueError on an empty graph, as in the reference
    kept = []
    for p, (i, j) in zip(pairs, edges):
        d = abs(i - j)
        if cyclic:
            d = min(d, abs(i + n - j), abs(i - n - j))
        if d <= max_dist:
            kept.append(p)
    return kept


# ------------------------------------------------------------------------------------------------
# batched pair decodes
# ------------------------------------------------------------------------------------------------
def _spann3r(model):
    """`model.dust3r` or the Spann3R model itself -> the Spann3R model that owns the engines."""
    owner = getattr(model, "_owner", None)
    return owner if owner is not None else model


def _host(t: torch.Tensor):
    """The one device-to-host read of a scoring step."""
    return t.tolist()


def _pad(chunk, k):
    """A short last chunk repeats its last entry up to the engine's batch k (one engine serves every chunk)."""
    return list(chunk) + [chunk[-1]] * (k - len(chunk))


def decode_scores(eng, f1, f2) -> torch.Tensor:
    """Decode + heads of one batch of pairs on `eng`, then one batched score: per pair the fp64 sum of the two heads'
    means of (c-1)/c (what the host computes as float(m1) + float(m2)), as a [eng.B] device tensor."""
    eng.decode(f1, f2)
    _, conf = eng.heads()
    s = conf_score_batched(conf)
    return s[0].double() + s[1].double()


def score_matrix(m, feats, H, W, scene_graph="complete", prefilter=None, max_batch=8) -> torch.Tensor:
    """fp32 [F, F] device matrix of pair scores over the graph's distinct ordered pairs (zero elsewhere, like the
    reference's conf_matrix); feats: the F encoded single views [1, N, 1024]."""
    if max_batch < 1:
        raise ValueError(f"max_batch must be >= 1, got {max_batch}")
    F_ = len(feats)
    views = [{"idx": i} for i in range(F_)]
    pairs = list(dict.fromkeys((a["idx"], b["idx"]) for a, b in make_pairs(views, scene_graph, prefilter, symmetrize=True)))
    if not pairs:
        raise ValueError(f"the scene graph {scene_graph!r} has no pairs over {F_} frame(s)")
    eng = m._engine_for(min(max_batch, len(pairs)), H, W)
    out = torch.zeros(F_, F_, dtype=torch.float32, device=eng.device)
    for s in range(0, len(pairs), eng.B):
        chunk = pairs[s: s + eng.B]
        padded = _pad(chunk, eng.B)
        tot = decode_scores(eng, torch.cat([feats[i] for i, _ in padded]), torch.cat([feats[j] for _, j in padded]))
        i1 = torch.tensor([i for i, _ in chunk], device=eng.device)
        i2 = torch.tensor([j for _, j in chunk], device=eng.device)
        out[i1, i2] = tot[: len(chunk)].float()
    return out


def initial_pair(m, feats, H, W, scene_graph="complete", prefilter=None, max_batch=8):
    """find_initial_pair over `score_matrix`: the flattened argmax (first maximum), with one host read."""
    M = score_matrix(m, feats, H, W, scene_graph, prefilter, max_batch)
    flat, best = _host(torch.stack((M.view(-1).argmax().double(), M.max().double())))
    pair_idx = (int(flat) // M.shape[0], int(flat) % M.shape[0])
    print(f"init pair:{pair_idx}, conf: {best}")
    return pair_idx


def next_best_view(eng, feat_fuse, feats, idx_todo):
    """find_next_best_view over the candidates idx_todo, eng.B at a time against the same fused feature [1, N, 1024].
    Totals and their argmax stay on the device; returns (frame index, fp64 score) from one host read.  The argmax is the
    first maximum in idx_todo order: the reference's strict `>` scan from 0.0."""
    K = eng.B
    fuse = feat_fuse.expand(K, -1, -1).contiguous()
    totals = []
    for s in range(0, len(idx_todo), K):
        chunk = idx_todo[s: s + K]
        totals.append(decode_scores(eng, fuse, torch.cat([feats[i] for i in _pad(chunk, K)]))[: len(chunk)])
    totals = torch.cat(totals)
    pos = totals.argmax()
    pos, best = _host(torch.stack((pos.double(), totals[pos])))
    if not best > 0.0:
        raise RuntimeError(f"find_next_best_view: no candidate scored above 0 (best {best})")
    return idx_todo[int(pos)], best


def _single_views(imgs):
    shapes = {tuple(t.shape) for t in imgs}
    if len(shapes) != 1:
        raise ValueError(f"all images must have one shape; got {sorted(shapes)} (mixed shapes are not supported)")
    shape = shapes.pop()
    if len(shape) != 4 or shape[0] != 1:
        raise ValueError(f"images must be single views [1, 3, H, W], got {shape}")
    return shape[-2], shape[-1]


def pair_scores(model, frames, scene_graph="complete", prefilter=None, max_batch=8) -> torch.Tensor:
    """The [F, F] fp32 matrix find_initial_pair builds from `inference(make_pairs(frames, ...))`, computed on the device
    without materialising the graph: every frame encoded once, the distinct ordered pairs decoded max_batch at a time.
    frames: list of view dicts {'img': [1, 3, H, W]}; returns a CUDA tensor (matrix[i, j]: pair (i, j) or 0 if absent)."""
    m = _spann3r(model)
    H, W = _single_views([f["img"] for f in frames])
    m._check_true_shape(frames, H, W)
    with torch.no_grad():
        feats = m._encode_frames(m._engine_for(1, H, W, n_frames=len(frames)), [m._dev(f["img"]) for f in frames])
        return score_matrix(m, feats, H, W, scene_graph, prefilter, max_batch)


# ------------------------------------------------------------------------------------------------
# drop-in for dust3r.inference.inference
# ------------------------------------------------------------------------------------------------
def _collate(vals):
    """collate_with_cat of one key over the entries: tensors / arrays concatenated on the CPU, anything else listed."""
    v0 = vals[0]
    if v0 is None:
        return None
    if isinstance(v0, torch.Tensor):
        return torch.cat([v.cpu() for v in vals])
    if isinstance(v0, np.ndarray):
        return torch.cat([torch.from_numpy(v) for v in vals])
    return list(vals)


@torch.no_grad()
def inference(pairs, model, device=None, batch_size=8, verbose=True):
    """Drop-in for `dust3r.inference.inference(pairs, model.dust3r, device, batch_size)` (model: `model.dust3r` or the
    Spann3R model).  Returns the reference's dict {view1, view2, pred1 {pts3d, conf}, pred2 {pts3d_in_other_view, conf},
    loss=None} on the CPU, with the reference's entries in its order: every pair (a, b) followed by its mirror (b, a)
    (the reference's symmetrised batches interleave them, whatever the batch size).

    Each distinct image (by tensor identity: device, data_ptr, shape, stride) is encoded once and each distinct ordered
    pair decoded once, `batch_size` pairs per engine call; duplicates are copies.  Images must share one shape
    [1, 3, H, W] (the reference falls back to per-pair lists there, which offline reconstruction cannot use).  Portrait
    maps are returned landscape, as `model.dust3r` returns them.  `device` is accepted for the signature: the model's
    device is used."""
    m = _spann3r(model)
    if verbose:
        print(f">> Inference with model on {len(pairs)} image pairs")
    if not pairs:
        raise ValueError("inference needs at least one pair")
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    H, W = _single_views([v["img"] for p in pairs for v in p])

    def key(t):
        return (t.device, t.data_ptr(), tuple(t.shape), t.stride())

    slot, imgs = {}, []
    for p in pairs:
        for v in p:
            k = key(v["img"])
            if k not in slot:
                slot[k] = len(imgs)
                imgs.append(v["img"])
    entries = [e for a, b in pairs for e in ((a, b), (b, a))]
    ekeys = [(slot[key(a["img"])], slot[key(b["img"])]) for a, b in entries]
    distinct = list(dict.fromkeys(ekeys))
    where = {k: n for n, k in enumerate(distinct)}

    eng = m._engine_for(min(batch_size, len(distinct)), H, W)
    feats = m._encode_frames(eng, [m._dev(t) for t in imgs])
    pts_parts, conf_parts = [], []
    for s in range(0, len(distinct), eng.B):
        chunk = distinct[s: s + eng.B]
        padded = _pad(chunk, eng.B)
        eng.decode(torch.cat([feats[i] for i, _ in padded]), torch.cat([feats[j] for _, j in padded]))
        pts, conf = eng.heads()
        pts_parts.append(pts[:, : len(chunk)].cpu())
        conf_parts.append(conf[:, : len(chunk)].cpu())
    pts, conf = torch.cat(pts_parts, dim=1), torch.cat(conf_parts, dim=1)
    sel = torch.tensor([where[k] for k in ekeys])

    def out(t):   # [D, H, W, ...] per distinct pair -> landscape per entry (contiguous, as the reference's collated maps)
        return (t.swapaxes(1, 2) if H > W else t).index_select(0, sel)

    view1 = {k: _collate([a[k] for a, _ in entries]) for k in entries[0][0]}
    view2 = {k: _collate([b[k] for _, b in entries]) for k in entries[0][1]}
    return {"view1": view1, "view2": view2,
            "pred1": {"pts3d": out(pts[0]), "conf": out(conf[0])},
            "pred2": {"pts3d_in_other_view": out(pts[1]), "conf": out(conf[1])},
            "loss": None}
