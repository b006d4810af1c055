"""Offline reconstruction's pair graph on the GPU: the batched confidence score (bitwise against the single-image kernel),
`offline.pair_scores` / `offline.inference` against `model.dust3r` pair by pair, `offline_reconstruction(frames)` without a
graph against the real reference's goldens, and batched next-best-view scoring against the serial loop."""
import contextlib
import io
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, get_state_dict, rel_l2

pytestmark = pytest.mark.gpu

TOL = 1e-3
SCORE_TOL = 1e-5


@pytest.fixture(scope="module")
def model():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(get_state_dict(True), strict=True)
    return m.cuda().eval()


def _quiet():
    return contextlib.redirect_stdout(io.StringIO())


# ------------------------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("H,W", [(224, 224), (384, 512), (288, 224), (17, 23)])
def test_conf_score_batched_is_bitwise_the_single_image_score(B, H, W):
    from spann3r_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H + W)
    conf = 1.0 + torch.rand(2, B, H, W, device="cuda", generator=g).mul_(6.0).exp_()
    got = _lib.conf_score_batched(conf)
    assert got.shape == (2, B)
    ref64 = ((conf.double() - 1) / conf.double()).mean(dim=(2, 3))
    for h in range(2):
        for b in range(B):
            single = _lib.conf_score(conf[h, b].contiguous())
            assert torch.equal(got[h, b].view(1), single), (h, b, float(got[h, b]), float(single))
    assert float(((got.double() - ref64).abs() / ref64).max()) < 1e-5


def test_conf_score_batched_rejects_bad_arguments():
    from spann3r_b200 import _lib
    conf = torch.full((2, 2, 8, 8), 2.0, device="cuda")
    scratch = torch.empty(2 * 2 * 256, device="cuda")
    out = torch.empty(4, device="cuda")
    L, p = _lib.lib(), _lib.ptr
    st = _lib.stream_ptr()
    assert L.s3r_conf_score_batched(p(conf), 0, 64, p(scratch), p(out), st) == -1
    assert L.s3r_conf_score_batched(p(conf), 2, 0, p(scratch), p(out), st) == -1
    assert L.s3r_conf_score_batched(p(conf), 2, 64, None, p(out), st) == -1
    assert L.s3r_conf_score_batched(p(conf), 2, 64, p(scratch), p(out), st) == 0
    torch.cuda.synchronize()
    assert torch.equal(out, torch.full((4,), 0.5, device="cuda"))
    with pytest.raises(AssertionError):
        _lib.conf_score_batched(conf[0])                     # not [2, B, H, W]
    with pytest.raises(_lib.S3RError, match="H\\*W"):
        _lib.conf_score_batched(torch.empty(2, 1, 0, 4, device="cuda"))


# ------------------------------------------------------------------------------------------------------------------
# pair scores and the drop-in inference
# ------------------------------------------------------------------------------------------------------------------
def _pairwise_scores(m, frames):
    """fp64 sum of conf_score over model.dust3r(a, b) at batch 1, for every ordered pair."""
    from spann3r_b200._lib import conf_score
    n = len(frames)
    out = torch.zeros(n, n, dtype=torch.float64)
    for i in range(n):
        for j in range(n):
            if i != j:
                r1, r2 = m.dust3r(frames[i], frames[j])
                out[i, j] = float(conf_score(r1["conf"].contiguous())) + float(conf_score(r2["conf"].contiguous()))
    return out


def test_pair_scores_match_the_pairwise_forward(model):
    from spann3r_b200 import offline, synth
    g = np.load(os.path.join(GOLDEN, "offline_224_4f_sharp.npz"))
    frames = synth.make_frames(4, 224, 224)
    with torch.no_grad():
        M = offline.pair_scores(model, frames)
        ref = _pairwise_scores(model, frames)
    assert M.is_cuda and M.dtype == torch.float32 and M.shape == (4, 4)
    off = ~torch.eye(4, dtype=torch.bool)
    err = float(((M.cpu().double() - ref).abs()[off] / ref[off].abs()).max())
    print("pair_scores max rel err vs model.dust3r at batch 1: %.2e" % err)
    assert err < SCORE_TOL
    flat = int(M.view(-1).argmax())
    assert [flat // 4, flat % 4] == list(g["idx_used"][:2])


def test_drop_in_inference_matches_the_pairwise_forward(model):
    from spann3r_b200 import offline, synth
    g = np.load(os.path.join(GOLDEN, "offline_224_4f_sharp.npz"))
    frames = synth.make_frames(4, 224, 224)
    views = [{"img": f["img"].cuda(), "true_shape": torch.tensor([[224, 224]]), "idx": i, "instance": str(i)}
             for i, f in enumerate(frames)]
    pairs = offline.make_pairs(views, "complete", None, True)
    with torch.no_grad(), _quiet():
        out = offline.inference(pairs, model.dust3r, "cuda", batch_size=2)
    assert out["view1"]["idx"] == list(g["graph/view1_idx"]) and out["view2"]["idx"] == list(g["graph/view2_idx"])
    errs = []
    with torch.no_grad():
        for e, (i, j) in enumerate(zip(out["view1"]["idx"], out["view2"]["idx"])):
            r1, r2 = model.dust3r(views[i], views[j])
            errs += [rel_l2(out["pred1"]["pts3d"][e], r1["pts3d"][0].cpu()), rel_l2(out["pred1"]["conf"][e], r1["conf"][0].cpu()),
                     rel_l2(out["pred2"]["pts3d_in_other_view"][e], r2["pts3d_in_other_view"][0].cpu()),
                     rel_l2(out["pred2"]["conf"][e], r2["conf"][0].cpu())]
    print("drop-in inference worst rel-L2 vs model.dust3r: %.2e" % max(errs))
    assert max(errs) < TOL
    with torch.no_grad(), _quiet():
        _, _, idx_used = model.offline_reconstruction(frames, out)
    assert list(idx_used) == list(g["idx_used"])


# ------------------------------------------------------------------------------------------------------------------
# offline_reconstruction without a graph
# ------------------------------------------------------------------------------------------------------------------
def _check_against_golden(m, fname):
    from spann3r_b200 import synth
    g = np.load(os.path.join(GOLDEN, fname))
    frames = synth.make_frames(4, 224, 224)
    with _quiet():
        preds, _, idx_used = m.offline_reconstruction(frames)
    assert list(idx_used) == list(g["idx_used"])
    s = int(g["meta/px_stride"])
    errs = {f"{i}/{k}": rel_l2(v[:, ::s, ::s].cpu(), g[f"preds/{i}/{k}"]) for i, p in enumerate(preds) for k, v in p.items()}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


def test_offline_without_graph_matches_reference_golden(model):
    _check_against_golden(model, "offline_224_4f_sharp.npz")


def test_offline_without_graph_matches_reference_golden_use_feat():
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None, use_feat=True)
    m.load_state_dict(synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True), strict=True)
    _check_against_golden(m.cuda().eval(), "offline_224_4f_sharp_usefeat.npz")


def test_offline_without_graph_runs_in_bf16(model):
    from spann3r_b200 import synth
    model.set_precision("bf16")
    try:
        with _quiet():
            preds, _, idx_used = model.offline_reconstruction(synth.make_frames(5, 224, 224))
        assert (5 - 2, 224, 224, "bf16") in model._engines
    finally:
        model.set_precision("fp32")
    assert sorted(idx_used) == list(range(5))
    assert all(bool(torch.isfinite(v).all()) for p in preds for v in p.values())


def _run_recording(m, frames, max_batch, monkeypatch):
    """offline_reconstruction(frames, max_batch=...) -> (preds, idx_used, per-step {candidate: fp64 score})."""
    from spann3r_b200 import model as M
    from spann3r_b200 import offline
    steps = []
    if max_batch > 1:
        rec = {"cur": None}
        orig_scores, orig_nbv = offline.decode_scores, offline.next_best_view

        def scores(eng, f1, f2):
            t = orig_scores(eng, f1, f2)
            if rec["cur"] is not None:
                rec["cur"].append(t.clone())
            return t

        def nbv(eng, fuse, feats, todo):
            rec["cur"] = []
            r = orig_nbv(eng, fuse, feats, todo)
            vals = []
            for c, s in zip(rec["cur"], range(0, len(todo), eng.B)):
                vals += c[: len(todo[s: s + eng.B])].tolist()
            steps.append(dict(zip(todo, vals)))
            rec["cur"] = None
            return r
        monkeypatch.setattr(offline, "decode_scores", scores)
        monkeypatch.setattr(offline, "next_best_view", nbv)
    else:
        calls = []
        orig = M._conf_score
        monkeypatch.setattr(M, "_conf_score", lambda c: calls.append(float(orig(c))) or orig(c))
    with torch.no_grad(), _quiet():
        preds, _, idx_used = m.offline_reconstruction(frames, max_batch=max_batch)
    preds = [{k: v.clone() for k, v in p.items()} for p in preds]
    monkeypatch.undo()
    if max_batch == 1:
        todo, pos = [i for i in range(len(frames)) if i not in idx_used[:2]], 0
        for used in idx_used[2:]:
            steps.append({c: calls[pos + 2 * k] + calls[pos + 2 * k + 1] for k, c in enumerate(todo)})
            pos += 2 * len(todo)
            todo.remove(used)
    return preds, idx_used, steps


@pytest.mark.parametrize("n,H,W", [(10, 224, 224), (6, 384, 512)])
def test_batched_next_best_view_agrees_with_the_serial_loop(model, monkeypatch, n, H, W):
    from spann3r_b200 import synth
    frames = synth.make_frames(n, H, W)
    pb, ub, sb = _run_recording(model, frames, 8, monkeypatch)
    ps, us, ss = _run_recording(model, frames, 1, monkeypatch)
    assert len(sb) == len(ss) == n - 2
    same_so_far = ub[:2] == us[:2]
    for k, (b, s) in enumerate(zip(sb, ss)):
        if not same_so_far:
            break
        assert set(b) == set(s)
        err = max(abs(b[c] - s[c]) / abs(s[c]) for c in s)
        top = sorted(b.values(), reverse=True)
        margin = (top[0] - top[1]) / top[0] if len(top) > 1 else float("inf")
        print(f"step {k}: {len(s)} candidates, max rel score diff {err:.1e}, top-two margin {margin:.1e}")
        assert err < SCORE_TOL
        if margin > SCORE_TOL:
            assert ub[2 + k] == us[2 + k]
        same_so_far = ub[2 + k] == us[2 + k]
    print("visiting order batched", ub, "serial", us)
    if ub == us:
        worst = max(rel_l2(a[key].cpu(), c[key].cpu()) for a, c in zip(pb, ps) for key in a)
        print("batched vs serial outputs, worst rel-L2: %.1e" % worst)
        assert worst < TOL
