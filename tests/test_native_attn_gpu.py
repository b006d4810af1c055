"""The attention of the training backward on the library's split-bf16 flash kernels (`_native_attn`,
`train.set_native_attention`): the operator against fp64 autograd of `_sdpa` on every shape the recompute issues plus
ragged tails, bitwise reproducibility, O(N) memory, routing, and whole training steps against the PyTorch backward."""
import ctypes as C

import pytest
import torch

from conftest import get_state_dict, rel_l2

pytestmark = pytest.mark.gpu

# (images, heads, nq, nk, dh): every attention of a 224 x 224 step (N = 196; B = 4, F = 10 encodes 40 images at once),
# a 224 x 288 grid (N = 252), the 512 x 384 encoder (N = 768), cross-attention with nq != nk, and tails around a tile
SHAPES = [
    (40, 16, 196, 196, 64),    # encoder, 224^2, B = 4, F = 10
    (4, 12, 196, 196, 64),     # decoder self / cross
    (4, 16, 196, 196, 64),     # value encoder
    (4, 16, 196, 196, 48),     # use_feat value encoder
    (2, 16, 252, 252, 64),
    (2, 12, 252, 252, 64),
    (3, 16, 252, 252, 48),
    (2, 16, 768, 768, 64),     # encoder, 512 x 384
    (1, 12, 768, 768, 64),
    (2, 12, 196, 252, 64),     # nq != nk
    (2, 16, 252, 196, 48),
    (1, 4, 1, 1, 64),
    (1, 4, 17, 129, 64),
    (1, 4, 127, 17, 48),
    (1, 4, 129, 127, 64),
    (2, 3, 1, 129, 48),
    (2, 3, 129, 1, 64),
]


def _inputs(B, H, nq, nk, dh, seed, peak=1.0):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(B, H, nq, dh, generator=g) * peak).cuda()
    k = torch.randn(B, H, nk, dh, generator=g).cuda()
    v = torch.randn(B, H, nk, dh, generator=g).cuda()
    go = torch.randn(B, nq, H * dh, generator=g).cuda()
    return q, k, v, go


def _check(B, H, nq, nk, dh, seed, peak=1.0):
    from spann3r_b200 import _native_attn as NA, _recompute as R
    q, k, v, go = _inputs(B, H, nq, nk, dh, seed, peak)
    qn, kn, vn = (t.clone().requires_grad_(True) for t in (q, k, v))
    o = NA.attention(qn, kn, vn, dh ** -0.5)
    dq, dk, dv = torch.autograd.grad(o, (qn, kn, vn), go)
    _, lse = NA.attention_with_lse(q, k, v, dh ** -0.5)
    qd, kd, vd = (t.double().requires_grad_(True) for t in (q, k, v))
    od = R._sdpa(qd, kd, vd).transpose(1, 2).reshape(B, nq, H * dh)
    rq, rk, rv = torch.autograd.grad(od, (qd, kd, vd), go.double())
    lse_ref = torch.logsumexp((qd @ kd.transpose(-2, -1)) * dh ** -0.5, dim=-1).reshape(B * H, nq)
    errs = {"O": rel_l2(o.detach().cpu(), od.detach().cpu()), "LSE": rel_l2(lse.cpu(), lse_ref.detach().cpu()),
            "dQ": rel_l2(dq.cpu(), rq.cpu()), "dK": rel_l2(dk.cpu(), rk.cpu()), "dV": rel_l2(dv.cpu(), rv.cpu())}
    if nk == 1:
        # one key: the softmax is constant, dQ = dK = 0 exactly (dS = P (dP - D) with dP = D), so the relative error of
        # the rounding left by that cancellation is measured against the size of the cancelling term, scale dP K
        dp = go.double().view(B, nq, H, dh).transpose(1, 2) @ vd.detach().transpose(-2, -1)
        errs["dQ"] = float(dq.double().norm().cpu() / (dp @ kd.detach() * dh ** -0.5).norm().cpu())
        errs["dK"] = float(dk.double().norm().cpu() / (dp.transpose(-2, -1) @ qd.detach() * dh ** -0.5).norm().cpu())
    print((B, H, nq, nk, dh, peak), {k_: "%.1e" % e for k_, e in errs.items()})
    assert errs["O"] < 3e-5 and errs["LSE"] < 3e-5, errs
    assert max(errs["dQ"], errs["dK"], errs["dV"]) < 1e-4, errs


@pytest.mark.parametrize("B,H,nq,nk,dh", SHAPES)
def test_attention_forward_backward_vs_fp64(B, H, nq, nk, dh):
    _check(B, H, nq, nk, dh, seed=nq * 7 + nk + dh)


def test_attention_peaked_softmax_vs_fp64():
    """q x 8: nearly one-hot rows, where the running max and the rebuilt probabilities matter most."""
    _check(4, 16, 196, 196, 64, seed=11, peak=8.0)
    _check(2, 16, 129, 127, 48, seed=12, peak=8.0)


def test_strided_views_of_qkv_match_contiguous_operands():
    """The recompute hands the kernels views of the qkv Linear's output ([B, N, 3, heads, dh] permuted): the strided read
    gives the same bits as contiguous copies."""
    from spann3r_b200 import _native_attn as NA
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(3, 196, 3, 16, 48, generator=g).cuda().permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    a = NA.attention_with_lse(q, k, v, 48 ** -0.5)
    b = NA.attention_with_lse(q.contiguous(), k.contiguous(), v.contiguous(), 48 ** -0.5)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_attention_is_bitwise_reproducible():
    from spann3r_b200 import _native_attn as NA
    q, k, v, go = _inputs(8, 16, 252, 196, 64, seed=3)
    outs = []
    for _ in range(2):
        qn, kn, vn = (t.clone().requires_grad_(True) for t in (q, k, v))
        o = NA.attention(qn, kn, vn, 0.125)
        outs.append((o.detach(), NA.attention_with_lse(q, k, v, 0.125)[1]) + torch.autograd.grad(o, (qn, kn, vn), go))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_attention_memory_is_linear_in_n():
    """Forward + backward at 40 images x 16 heads x N = 768 raises peak allocated memory by less than 1 GB; the fp32
    probabilities autograd keeps for `_sdpa` would be 1.5 GB on their own."""
    from spann3r_b200 import _native_attn as NA
    q, k, v, go = _inputs(40, 16, 768, 768, 64, seed=1)
    q.requires_grad_(True)
    k.requires_grad_(True)
    v.requires_grad_(True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    o = NA.attention(q, k, v, 0.125)
    grads = torch.autograd.grad(o, (q, k, v), go)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("peak above inputs: %.0f MB" % (peak / 2 ** 20))
    assert peak < 2 ** 30, peak
    del grads, o


def test_invalid_calls_return_an_error_and_launch_nothing():
    """Every invalid call returns -1 before any CUDA call: the output buffers keep their sentinel."""
    from spann3r_b200 import _lib, _native_attn as NA
    L = _lib.lib()
    q, k, v, go = _inputs(2, 4, 33, 33, 64, seed=2)
    o = torch.full((2, 33, 256), 7.0, device="cuda")
    lse = torch.full((8, 33), 7.0, device="cuda")
    dq, dk, dv = (torch.full_like(t, 7.0) for t in (q, k, v))

    def backward(d, ws_bytes):
        ws = torch.empty(max(ws_bytes, 256) // 4, device="cuda")
        return L.s3r_attn_train_backward(C.byref(d), _lib.ptr(o), _lib.ptr(lse), _lib.ptr(go), _lib.ptr(ws), ws_bytes,
                                         _lib.ptr(dq), _lib.ptr(dk), _lib.ptr(dv), _lib.stream_ptr())

    def call(d):
        r1 = L.s3r_attn_train_forward(C.byref(d), _lib.ptr(o), _lib.ptr(lse), _lib.stream_ptr())
        return r1, backward(d, L.s3r_attn_train_workspace_bytes(C.byref(d)))

    for field, val in (("dh", 32), ("nq", 0), ("nk", 0), ("batch", 0), ("scale", -1.0)):
        d = NA._desc(q, k, v, 0.125)
        setattr(d, field, val)
        assert call(d) == (-1, -1), field
    d = NA._desc(q, k, v, 0.125)
    d.q_stride[2] = 66
    assert call(d) == (-1, -1)
    d = NA._desc(q, k, v, 0.125)
    assert backward(d, 16) == -1
    torch.cuda.synchronize()
    for t in (o, lse, dq, dk, dv):
        assert bool((t == 7.0).all())


@pytest.fixture(scope="module")
def model():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(get_state_dict(True), strict=True)
    return m.cuda()


def _step_grads(model, frames, watch, lin=False, conv=False, attn=False):
    from spann3r_b200 import train
    named = dict(model.named_parameters())
    try:
        train.set_native_linear(lin)
        train.set_native_conv(conv)
        train.set_native_attention(attn)
        model.train()
        model.zero_grad(set_to_none=True)
        preds, _ = model(frames)
        loss = sum(p[k].square().mean() + p["conf"].log().mean() for p in preds for k in p if k != "conf")
        loss.backward()
        return {k: named[k].grad.detach().clone() for k in watch}
    finally:
        train.set_native_linear(False)
        train.set_native_conv(False)
        train.set_native_attention(False)
        model.zero_grad(set_to_none=True)
        model.eval()


def _compare(a, b, bar):
    errs = {k: rel_l2(a[k].cpu(), b[k].cpu()) for k in a}
    cos = {k: float(torch.nn.functional.cosine_similarity(a[k].flatten().double().cpu(), b[k].flatten().double().cpu(),
                                                           dim=0)) for k in a}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < bar, errs
    assert min(cos.values()) >= 0.99999, cos


WATCH = ["dust3r.enc_blocks.3.attn.qkv.weight", "dust3r.enc_blocks.20.attn.qkv.bias",
         "dust3r.dec_blocks.7.cross_attn.projq.weight", "dust3r.dec_blocks.7.cross_attn.projk.weight",
         "dust3r.dec_blocks2.2.attn.qkv.weight", "value_encoder.4.attn.qkv.weight", "norm_k.weight"]


def test_training_step_never_reaches_sdpa_with_the_switch_on(model, monkeypatch):
    from spann3r_b200 import _recompute as R, synth
    calls = []
    orig = R._sdpa
    monkeypatch.setattr(R, "_sdpa", lambda *a: (calls.append(1), orig(*a))[1])
    frames = synth.make_frames(3, 224, 224)
    _step_grads(model, frames, WATCH[:1], attn=True)
    assert calls == []
    _step_grads(model, frames, WATCH[:1], attn=False)
    assert len(calls) >= 24 + 2 * 12 * 2 * 2, len(calls)             # the off arm does count: encoder + 2 frame steps


def test_training_step_with_native_attention_matches_the_torch_backward(model):
    """Switch on against off (the off arm in strict fp32): relative L2 < 5e-4 and cosine >= 0.99999 on the attention
    parameters of every stage and on norm_k (the memory keys' gradient runs through the decoder's cross-attention);
    all three switches on against all off: < 1e-3."""
    from spann3r_b200 import synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = synth.make_frames(3, 224, 224)
    off = _step_grads(model, frames, WATCH)
    on = _step_grads(model, frames, WATCH, attn=True)
    _compare(on, off, 5e-4)
    every = _step_grads(model, frames, WATCH, lin=True, conv=True, attn=True)
    _compare(every, off, 1e-3)


def test_use_feat_training_step_with_native_attention_matches_the_torch_backward():
    """The use_feat model (16 heads of 48 in the value encoder): switch on against off, relative L2 < 5e-4."""
    from spann3r_b200 import Spann3R, synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    m = Spann3R(dus3r_name=None, use_feat=True, memory_dropout=0.0)
    m.load_state_dict(synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True), strict=True)
    m = m.cuda()
    watch = ["value_encoder.0.attn.qkv.weight", "value_encoder.5.attn.qkv.weight", "value_encoder.2.attn.proj.weight",
             "dust3r.dec_norm.weight", "dust3r.dec_blocks.11.attn.qkv.weight", "dust3r.enc_blocks.5.attn.qkv.weight"]
    frames = synth.make_frames(3, 224, 224)
    off = _step_grads(m, frames, watch)
    on = _step_grads(m, frames, watch, attn=True)
    _compare(on, off, 5e-4)
