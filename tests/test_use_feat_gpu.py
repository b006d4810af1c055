"""`Spann3R(use_feat=True)` on the GPU: the 768-wide value encoder (16 heads of 48 in 64-wide slots) fed with the decoder
tokens, in eval, offline and training modes, against the real reference's goldens (tools/make_golden.py --only usefeat) and
the use_feat oracle (oracle/usefeat_oracle.py).  Tolerance: the 1e-3 relative L2 of test_model_gpu.py; gradients: the
3e-3 / cosine 0.99999 bar of test_train_gpu.py."""
import contextlib
import ctypes
import io
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu

TOL = 1e-3


def _sd():
    from spann3r_b200 import synth
    return synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True)


@pytest.fixture(scope="module")
def sd():
    return _sd()


@pytest.fixture(scope="module")
def model(sd):
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, use_feat=True)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def _strict_fp32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.parametrize("fname,nf,H,W,mem_pos_enc", [
    ("seq_224_3f_sharp_usefeat.npz", 3, 224, 224, False),
    ("seq_288x224_3f_sharp_usefeat_mempos.npz", 3, 288, 224, True),
])
def test_eval_forward_matches_reference_golden(model, sd, fname, nf, H, W, mem_pos_enc):
    from spann3r_b200 import Spann3R, synth
    g = np.load(os.path.join(GOLDEN, fname))
    m = model
    if mem_pos_enc:
        m = Spann3R(dus3r_name=None, use_feat=True, mem_pos_enc=True)
        m.load_state_dict(sd, strict=True)
        m = m.cuda().eval()
    frames = synth.make_frames(nf, H, W)
    preds, preds_all, mem = m(frames, return_memory=True)
    torch.cuda.synchronize()
    s = int(g["meta/px_stride"])
    errs = {}
    for i, p in enumerate(preds):
        assert set(p.keys()) == {k.split("/")[-1] for k in g.files if k.startswith(f"preds/{i}/")}
        for k, v in p.items():
            assert v.shape[1:3] == (min(H, W), max(H, W))
            errs[f"preds/{i}/{k}"] = rel_l2(v[:, ::s, ::s].cpu(), g[f"preds/{i}/{k}"])
    for i, (_, r2) in enumerate(preds_all):
        for k, v in r2.items():
            errs[f"preds_all/{i}/res2/{k}"] = rel_l2(v[:, ::s, ::s].cpu(), g[f"preds_all/{i}/res2/{k}"])
    errs["mem_k"] = rel_l2(mem.mem_k[:, ::7, ::8].cpu(), g["mem/mem_k_sub"])
    errs["mem_v"] = rel_l2(mem.mem_v[:, ::7, ::8].cpu(), g["mem/mem_v_sub"])
    errs["mem_attn"] = rel_l2(mem.mem_attn.cpu(), g["mem/mem_attn"])
    assert np.array_equal(mem.mem_count.cpu().numpy(), g["mem/mem_count"])
    if "act/value_out#0" in g.files:
        # value_out of step 0 alone: the engine's value stage on its own decode of frames 0, 1, with feat_k1 = 0
        eng = m._engine_for(1, H, W)
        img = torch.cat([f["img"] for f in frames[:2]]).cuda()
        feats = eng.encode(img)
        eng.decode(feats[:1].contiguous(), feats[1:].contiguous())
        cur_v = eng.value(None, torch.zeros(1, eng.N, 1024, device="cuda"), tokens=True)
        errs["value_out"] = rel_l2(cur_v[:, ::7, ::8].cpu(), g["act/value_out#0"])
    print({k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


def test_value_stage_vs_oracle_with_explicit_tokens(model, sd):
    """s3r_engine_value with S3R_VALUE_DEC_TOKENS on given tokens (and NULL = the engine's own dec_norm output) against the
    use_feat oracle's encode_cur_value + feat_k1 in strict fp32, with and without RoPE, at a landscape grid."""
    from oracle import spann3r_oracle as orc
    from oracle import usefeat_oracle as ufo
    from spann3r_b200 import Spann3R, synth
    _strict_fp32()
    sdc = {k: v.cuda() for k, v in sd.items()}
    H, W = 224, 320
    for rope in (False, True):
        m = model
        if rope:
            m = Spann3R(dus3r_name=None, use_feat=True, mem_pos_enc=True)
            m.load_state_dict(sd, strict=True)
            m = m.cuda().eval()
        eng = m._engine_for(1, H, W)
        img = torch.cat([f["img"] for f in synth.make_frames(2, H, W)]).cuda()
        feats, pos = orc.encode_image(sdc, img)
        f1, f2 = feats[:1].contiguous(), feats[1:].contiguous()
        d1, _ = orc.decoder(sdc, f1, pos[:1], f2, pos[1:])
        k1 = orc.key_head(sdc, 1, f1, d1[-1]).contiguous()
        ref = ufo.encode_cur_value(sdc, d1[-1], pos[:1], mem_pos_enc=rope) + k1
        got = eng.value(d1[-1].contiguous(), k1, rope=rope, tokens=True)
        assert rel_l2(got.cpu(), ref.cpu()) < 2e-4, (rope, rel_l2(got.cpu(), ref.cpu()))
        eng.decode(f1, f2)
        own = eng.value(None, k1, rope=rope, tokens=True)
        assert rel_l2(own.cpu(), ref.cpu()) < 3e-4, (rope, rel_l2(own.cpu(), ref.cpu()))


def test_offline_reconstruction_matches_reference_golden(model):
    from spann3r_b200 import synth
    from test_oracle_vs_golden import _pair_graph
    g = np.load(os.path.join(GOLDEN, "offline_224_4f_sharp_usefeat.npz"))
    frames = synth.make_frames(4, 224, 224)

    def fwd(a, b):
        r1, r2 = model.dust3r(a, b)
        return {k: v.clone() for k, v in r1.items()}, {k: v.clone() for k, v in r2.items()}

    graph = _pair_graph(fwd, frames)
    with contextlib.redirect_stdout(io.StringIO()):
        preds, _, idx_used = model.offline_reconstruction(frames, graph)
    assert list(idx_used) == list(g["idx_used"])
    s = int(g["meta/px_stride"])
    errs = {f"{i}/{k}": rel_l2(v[:, ::s, ::s].cpu(), g[f"preds/{i}/{k}"]) for i, p in enumerate(preds) for k, v in p.items()}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < TOL, errs


def test_invalid_flag_and_width_combinations_launch_nothing(model):
    """Each invalid flag / width combination returns an error through s3r_last_error() before any launch."""
    from spann3r_b200 import Spann3R, _lib, synth
    from spann3r_b200.engine import VALUE_DEC_TOKENS, VALUE_PTS_TRANSPOSED, VALUE_ROPE
    L = _lib.lib()
    default = Spann3R(dus3r_name=None)
    default.load_state_dict(synth.make_state_dict(seed=0, sharpen=True), strict=True)
    default = default.cuda().eval()
    for m, flags, what in ((model, 0, "768 wide"), (model, VALUE_ROPE, "768 wide"),
                           (model, VALUE_DEC_TOKENS | VALUE_PTS_TRANSPOSED, "PTS_TRANSPOSED"),
                           (default, VALUE_DEC_TOKENS, "1024 wide"), (default, VALUE_DEC_TOKENS | VALUE_ROPE, "1024 wide"),
                           (model, 8, "unknown flags")):
        eng = m._engine_for(1, 224, 224)
        k1 = torch.zeros(1, eng.N, 1024, device="cuda")
        out = torch.full((1, eng.N, 1024), 7.0, device="cuda")
        pts = torch.zeros(1, 224, 224, 3, device="cuda")
        eng.take_launches()
        torch.cuda.synchronize()
        r = L.s3r_engine_value(eng._h, ctypes.c_void_p(pts.data_ptr()), ctypes.c_void_p(k1.data_ptr()), flags,
                               ctypes.c_void_p(out.data_ptr()), _lib.stream_ptr())
        torch.cuda.synchronize()
        assert r < 0, (what, flags)
        assert what in L.s3r_last_error().decode(), (what, L.s3r_last_error())
        assert eng.take_launches() == 0 and bool((out == 7.0).all()), what


def _loss_of(preds, wts):
    tot = 0.0
    for p, w in zip(preds, wts):
        k = "pts3d" if "pts3d" in p else "pts3d_in_other_view"
        tot = tot + (p[k] * w).sum() + 0.1 * p["conf"].log().sum()
    return tot


@pytest.fixture(scope="module")
def train_model(sd):
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, use_feat=True, memory_dropout=0.0)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def test_training_forward_matches_oracle_training_branches(train_model, sd):
    from oracle import usefeat_oracle as ufo
    from spann3r_b200 import synth
    _strict_fp32()
    frames = synth.make_frames(4, 224, 224)
    train_model.train()
    try:
        preds, _ = train_model(frames)
        assert preds[1]["pts3d_in_other_view"].requires_grad
        sdc = {k: v.cuda() for k, v in sd.items()}
        ref, _ = ufo.forward(sdc, [{"img": f["img"].cuda()} for f in frames], attn_thresh=0, sim_thresh=1.0)
        for p, r in zip(preds, ref):
            assert set(p) == set(r)
            for k in r:
                assert rel_l2(p[k].detach().cpu(), r[k].cpu()) < TOL, k
    finally:
        train_model.eval()


WATCH = ["value_encoder.0.attn.qkv.weight", "value_encoder.3.attn.qkv.weight", "value_encoder.1.attn.proj.weight",
         "value_encoder.5.attn.proj.weight", "value_out.weight", "dust3r.dec_norm.weight",
         "dust3r.dec_blocks.11.mlp.fc2.weight", "value_encoder.4.mlp.fc1.bias", "norm_v.weight"]


@pytest.mark.parametrize("native_linear", [False, True])
def test_backward_gradients_vs_oracle_autograd(train_model, sd, native_linear):
    """Gradients through the training forward (native forward, PyTorch recompute backward; Linears of the backward on the
    GEMM engine when native_linear) against autograd through the use_feat oracle in strict fp32.  The watch list includes
    dec_norm and a last-layer decoder weight, which the memory values now reach through the value encoder's input."""
    from oracle import usefeat_oracle as ufo
    from spann3r_b200 import synth, train
    _strict_fp32()
    frames = synth.make_frames(3, 224, 224)
    g = torch.Generator().manual_seed(5)
    wts = [torch.randn(1, 224, 224, 3, generator=g).cuda() for _ in range(3)]
    named = dict(train_model.named_parameters())
    try:
        train.set_native_linear(native_linear)
        train_model.train()
        train_model.zero_grad(set_to_none=True)
        preds, _ = train_model(frames)
        loss = _loss_of(preds, wts)
        loss.backward()
        got = {k: named[k].grad.detach().clone() for k in WATCH}
    finally:
        train.set_native_linear(False)
        train_model.zero_grad(set_to_none=True)
        train_model.eval()
    sdc = {k: v.cuda().requires_grad_(k in WATCH) for k, v in sd.items()}
    ref_preds, _ = ufo.forward.__wrapped__(sdc, [{"img": f["img"].cuda()} for f in frames], attn_thresh=0, sim_thresh=1.0)
    ref_loss = _loss_of(ref_preds, wts)
    grads = torch.autograd.grad(ref_loss, [sdc[k] for k in WATCH])
    assert abs(float(loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss))
    errs = {k: rel_l2(got[k].cpu(), gr.cpu()) for k, gr in zip(WATCH, grads)}
    cos = {k: float(torch.nn.functional.cosine_similarity(got[k].flatten().double().cpu(), gr.flatten().double().cpu(), dim=0))
           for k, gr in zip(WATCH, grads)}
    print(native_linear, {k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < 3e-3, errs
    assert min(cos.values()) > 0.99999, cos
