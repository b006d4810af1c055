"""Offline reconstruction's pair graph without a GPU: `offline.make_pairs` against the reference's recorded graphs, and the
host control flow of `offline.inference` / `offline_reconstruction(frames)` (no graph) on a fake engine whose outputs
name the pair they came from."""
import json
import math
import os
import re

import pytest
import torch

from conftest import GOLDEN, ROOT

PAIRS = json.load(open(os.path.join(GOLDEN, "pairs.json")))


def _views(n):
    return [{"img": torch.full((1, 3, 32, 32), float(i)), "idx": i, "instance": str(i)} for i in range(n)]


@pytest.mark.parametrize("case", PAIRS["graphs"], ids=lambda c: f"{c['n']}-{c['scene_graph']}-{c['symmetrize']}-{c['prefilter']}")
def test_make_pairs_matches_the_reference(case):
    from spann3r_b200 import offline
    args = (_views(case["n"]), case["scene_graph"], case["prefilter"], case["symmetrize"])
    if "raises" in case:
        with pytest.raises({"IndexError": IndexError, "ValueError": ValueError}[case["raises"]]):
            offline.make_pairs(*args)
        return
    got = [[a["idx"], b["idx"]] for a, b in offline.make_pairs(*args)]
    assert got == case["pairs"]


def test_make_pairs_rejects_unknown_graphs():
    from spann3r_b200 import offline
    with pytest.raises(ValueError, match="scene graph"):
        offline.make_pairs(_views(3), "star")


# ------------------------------------------------------------------------------------------------------------------
# a fake engine: a frame's features hold its index, every map of a decoded pair holds the pair's code
# (first stream's value * 1000 + second's); a batch column that repeats the previous one (padding) gets code -1
# ------------------------------------------------------------------------------------------------------------------
class _FakeEngine:
    def __init__(self, B, H, W, log):
        self.B, self.H, self.W, self.N = B, H, W, (H // 16) * (W // 16)
        self.device, self.max_images, self.log = torch.device("cpu"), 2 * B, log
        self.codes = None

    def encode(self, img):
        assert img.shape[0] <= self.max_images
        self.log.append((self.B, "encode", img.shape[0]))
        return img[:, 0, 0, 0].view(-1, 1, 1).expand(-1, self.N, 1024).clone()

    def decode(self, f1, f2, want_all=False):
        assert f1.shape == f2.shape == (self.B, self.N, 1024) and f1.is_contiguous() and f2.is_contiguous()
        a, c = f1[:, 0, 0].tolist(), f2[:, 0, 0].tolist()
        self.codes = [-1.0 if b and (a[b], c[b]) == (a[b - 1], c[b - 1]) else a[b] * 1000 + c[b] for b in range(self.B)]
        self.log.append((self.B, "decode", a, c))

    def keyheads(self, f1, f2):
        self.log.append((self.B, "keyheads"))
        return f1 + 100, f2 + 100

    def heads(self):
        code = torch.tensor(self.codes).view(1, self.B, 1, 1)
        pts = (code + torch.tensor([0.0, 0.5]).view(2, 1, 1, 1)).unsqueeze(-1).expand(2, self.B, self.H, self.W, 3)
        conf = code.expand(2, self.B, self.H, self.W)
        return pts.contiguous(), conf.contiguous()

    def value(self, pts3d, feat_k1, transposed=False, rope=False):
        self.log.append((self.B, "value"))
        return feat_k1 * 0

    def memory_read(self, bank, feat, thresh):
        return feat

    def memory_append(self, bank, k, v):
        bank.len += self.N

    def check_sim(self, bank, feat_k, wm):
        return torch.zeros(self.B, wm)


def _plant(code):
    """A planted score for a decoded pair (small integers: exact sums and plenty of ties); padding would always win."""
    return 1e6 if code < 0 else float((int(code) * 2654435761) % 97 % 13 + 1)


def _fake_scores(conf):
    s = torch.tensor([_plant(c) for c in conf[0, :, 0, 0].tolist()], dtype=torch.float32)
    return torch.stack((s * 0.5, s * 0.5))


def _fake_model(monkeypatch):
    from spann3r_b200 import Spann3R, offline
    from spann3r_b200 import model as M
    m = Spann3R(dus3r_name=None).eval()
    engines, log = {}, []
    monkeypatch.setattr(m, "_engine_for", lambda B, H, W, n_frames=2, encode_only=False:
                        engines.setdefault((B, H, W), _FakeEngine(B, H, W, log)))
    monkeypatch.setattr(M.SpatialMemory, "check_sim_async", lambda self, feat_k, thresh=0.7: None)
    monkeypatch.setattr(offline, "conf_score_batched", _fake_scores)
    return m, engines, log


@pytest.mark.parametrize("n,H,W", [(4, 64, 96), (5, 96, 64)])
@pytest.mark.parametrize("bs", [2, 3, 8])
def test_inference_order_counts_and_copies(monkeypatch, n, H, W, bs):
    from spann3r_b200 import offline
    m, engines, log = _fake_model(monkeypatch)
    views = [{"img": torch.full((1, 3, H, W), float(i)), "true_shape": torch.tensor([[H, W]]), "idx": i, "instance": str(i)}
             for i in range(n)]
    pairs = offline.make_pairs(views, "complete", None, True)
    out = offline.inference(pairs, m.dust3r, "cuda", batch_size=bs, verbose=False)
    gold = [e for e in PAIRS["entries"] if e["n"] == n]
    assert all(e["view1_idx"] == gold[0]["view1_idx"] for e in gold)        # the reference's order ignores batch_size
    E = len(gold[0]["view1_idx"])
    assert out["view1"]["idx"] == gold[0]["view1_idx"] and out["view2"]["idx"] == gold[0]["view2_idx"]
    assert out["view1"]["instance"] == [str(i) for i in gold[0]["view1_idx"]]
    assert set(out) == {"view1", "view2", "pred1", "pred2", "loss"} and out["loss"] is None
    assert set(out["pred1"]) == {"pts3d", "conf"} and set(out["pred2"]) == {"pts3d_in_other_view", "conf"}
    lh, lw = min(H, W), max(H, W)
    assert out["view1"]["img"].shape == (E, 3, H, W) and out["view1"]["true_shape"].shape == (E, 2)
    assert out["pred1"]["pts3d"].shape == (E, lh, lw, 3) and out["pred2"]["conf"].shape == (E, lh, lw)
    assert all(t.device.type == "cpu" for t in (out["pred1"]["pts3d"], out["pred2"]["conf"], out["view1"]["img"]))
    assert torch.equal(out["view1"]["img"][:, 0, 0, 0], torch.tensor(gold[0]["view1_idx"], dtype=torch.float32))
    # every entry carries its own pair's maps (duplicates are copies of one decode)
    code = torch.tensor([a * 1000 + c for a, c in zip(gold[0]["view1_idx"], gold[0]["view2_idx"])], dtype=torch.float32)
    assert torch.equal(out["pred1"]["conf"][:, -1, -1], code) and torch.equal(out["pred2"]["conf"][:, 0, 0], code)
    assert torch.equal(out["pred2"]["pts3d_in_other_view"][:, 1, 2, 0], code + 0.5)
    # n images encoded in all; one decode per batch of distinct ordered pairs, on one engine
    P = min(bs, n * (n - 1))
    assert list(engines) == [(P, H, W)]
    assert sum(c[2] for c in log if c[1] == "encode") == n
    assert sum(1 for c in log if c[1] == "decode") == math.ceil(n * (n - 1) / P)


def test_inference_rejects_mixed_shapes(monkeypatch):
    from spann3r_b200 import offline
    m, _, _ = _fake_model(monkeypatch)
    a = {"img": torch.zeros(1, 3, 64, 96), "idx": 0}
    b = {"img": torch.zeros(1, 3, 96, 64), "idx": 1}
    with pytest.raises(ValueError, match="shape"):
        offline.inference([(a, b)], m, batch_size=2, verbose=False)


def _brute_force(n):
    """find_initial_pair over the complete symmetrised graph + the reference's strict `>` next-best-view scan."""
    best, pair = -1.0, None
    for i in range(n):
        for j in range(n):
            s = _plant(i * 1000 + j) if i != j else 0.0
            if s > best:                                    # flattened argmax: the first maximum
                best, pair = s, (i, j)
    used, todo = list(pair), [k for k in range(n) if k not in pair]
    while todo:
        best, bid = 0.0, None
        for c in todo:
            s = _plant((used[-1] + 100) * 1000 + c)       # the fused feature: memory_read(feat_k2) = last frame + 100
            if s > best:
                best, bid = s, c
        used.append(bid)
        todo.remove(bid)
    return used


@pytest.mark.parametrize("n,max_batch", [(7, None), (7, 3), (9, 8), (3, 8)])
def test_offline_without_graph_picks_the_brute_force_order(monkeypatch, n, max_batch):
    from spann3r_b200 import offline
    m, engines, log = _fake_model(monkeypatch)
    reads = []
    monkeypatch.setattr(offline, "_host", lambda t: reads.append(t.numel()) or t.tolist())
    H, W = 64, 96
    frames = [{"img": torch.full((1, 3, H, W), float(i))} for i in range(n)]
    kw = {} if max_batch is None else {"max_batch": max_batch}
    preds, preds_all, idx_used = m.offline_reconstruction(frames, **kw)
    assert idx_used == _brute_force(n)
    assert len(preds) == n and len(preds_all) == n - 1 and set(preds[0]) == {"pts3d", "conf"}
    # one host read for the initial pair, then one per next-best-view step
    assert reads == [2] * (1 + n - 2)
    K = min(max_batch or 8, n - 2)
    assert (K, H, W) in engines
    # the frames are encoded once, on the main engine
    assert sum(c[2] for c in log if c[1] == "encode") == n and all(c[0] == 1 for c in log if c[1] == "encode")
    # the main (batch-1) engine decodes the initial pair, then each winner, each time before keyheads and value
    main = [c for c in log if c[0] == 1 and c[1] in ("decode", "keyheads", "value")]
    if K == 1:    # the candidate engine is the main engine: drop the candidate decodes (those right before another decode)
        main = [c for i, c in enumerate(main) if not (c[1] == "decode" and i + 1 < len(main) and main[i + 1][1] == "decode")]
    assert [c[1] for c in main] == ["decode", "keyheads", "value"] * (n - 1)
    decs = [c for c in main if c[1] == "decode"]
    assert [c[3] for c in decs] == [[float(i)] for i in idx_used[1:]]
    assert [c[2] for c in decs] == [[float(idx_used[0])]] + [[float(i + 100)] for i in idx_used[1:-1]]


def test_offline_without_graph_rejects_lockstep_batches(monkeypatch):
    m, _, _ = _fake_model(monkeypatch)
    frames = [{"img": torch.zeros(2, 3, 64, 64)} for _ in range(3)]
    with pytest.raises(ValueError, match="single views"):
        m.offline_reconstruction(frames)
    with pytest.raises(ValueError, match="max_batch"):
        m.offline_reconstruction([{"img": torch.zeros(1, 3, 64, 64)}] * 3, max_batch=0)


def test_conf_score_batched_prototype_and_argument_checks():
    """s3r_conf_score_batched: the header's prototype, its ctypes binding, and the argument checks (which run before
    any device work, so they are checked here without a GPU)."""
    import ctypes as C
    from spann3r_b200 import _lib
    header = open(os.path.join(ROOT, "include", "spann3r_b200.h")).read()
    m = re.search(r"int\s+s3r_conf_score_batched\s*\(([^)]*)\)\s*;", header)
    assert m is not None
    kinds = [a.strip().rsplit(" ", 1)[0].replace("const ", "") for a in m.group(1).split(",")]
    assert kinds == ["float*", "int", "int64_t", "float*", "float*", "void*"]
    assert _lib._PROTOS["s3r_conf_score_batched"] == (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_void_p,
                                                                C.c_void_p])
    L = _lib.lib()
    p = C.c_void_p(16)
    for args, msg in (((p, 0, 4, p, p, None), b"batch"), ((p, 32768, 4, p, p, None), b"batch"),
                      ((p, 1, 0, p, p, None), b"H*W"), ((None, 1, 4, p, p, None), b"null"),
                      ((p, 1, 4, None, p, None), b"null"), ((p, 1, 4, p, None, None), b"null")):
        assert L.s3r_conf_score_batched(*args) == -1, args
        assert msg in L.s3r_last_error()
