"""Training mode on the GPU (SURVEY.md §8f rank 1 / §8e-train, staged): the CUDA forward with the reference's training
branches against the oracle, the Philox dropout mask against its host restatement, and the PyTorch-recompute backward
against autograd through the oracle."""
import numpy as np
import pytest
import torch

from conftest import get_state_dict, rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(get_state_dict(True), strict=True)
    return m.cuda()


def test_dropout_mask_kernel_equals_host_philox():
    from spann3r_b200 import _lib
    from test_train_cpu import philox_keep_scale_numpy
    for seed, n, p in ((1234567890123, 4099, 0.15), (7, 1000, 0.5), ((1 << 61) + 12345, 777, 0.15)):
        got = _lib.dropout_mask((n,), seed, p, "cuda").cpu().numpy()
        assert np.array_equal(got, philox_keep_scale_numpy(seed, n, p)), (seed, n, p)


def test_training_mode_read_with_dropout_vs_torch(model):
    """s3r_engine_memory_read_train: softmax -> dropout(p) -> (no cut) -> . V + feat, mask = the Philox keep-scale."""
    from spann3r_b200 import _lib, _recompute as R
    from spann3r_b200.engine import MemoryBank
    model.eval()
    eng = model._engine_for(1, 224, 224)
    g = torch.Generator().manual_seed(11)
    bank = MemoryBank(1, 4000 + 8 * eng.N, "cuda")
    ks = [torch.randn(1, eng.N, 1024, generator=g).cuda() for _ in range(3)]
    vs = [torch.randn(1, eng.N, 1024, generator=g).cuda() for _ in range(3)]
    for k, v in zip(ks, vs):
        eng.memory_append(bank, k, v)
    q = (4 * torch.randn(1, eng.N, 1024, generator=g)).cuda()
    P = {k: v.cuda() for k, v in get_state_dict(True).items() if k.startswith("norm_")}
    for p, seed in ((0.0, 0), (0.15, 99), (0.15, 100)):
        out = eng.memory_read(bank, q, 0.0, drop_p=p, seed=seed)
        mask = _lib.dropout_mask((1, eng.N, 3 * eng.N), seed, p, "cuda") if p > 0 else None
        ref = R.memory_read(P, q, torch.cat(ks, 1), torch.cat(vs, 1), mask)
        assert rel_l2(out.cpu(), ref.cpu()) < 2e-4, (p, seed)
    a = eng.memory_read(bank, q, 0.0, drop_p=0.15, seed=99)
    b = eng.memory_read(bank, q, 0.0, drop_p=0.15, seed=100)
    assert rel_l2(a.cpu(), b.cpu()) > 1e-3          # a different seed is a different mask


def test_training_forward_matches_oracle_training_branches(model):
    """model.train() forward (CUDA kernels; attn_thresh = 0, ungated add_mem, dropout p = 0 here) == the oracle run with the
    same branches (attn_thresh=0, sim_thresh=1.0 disables the gate), 4 frames at 224 x 224, <= 1e-3."""
    from oracle import spann3r_oracle as orc
    from spann3r_b200 import synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = synth.make_frames(4, 224, 224)
    model.train()
    preds, preds_all = model(frames)
    assert preds[1]["pts3d_in_other_view"].requires_grad and preds[0]["conf"].grad_fn is not None
    sd = {k: v.cuda() for k, v in get_state_dict(True).items()}
    ref, _ = orc.forward(sd, [{"img": f["img"].cuda()} for f in frames], attn_thresh=0, sim_thresh=1.0)
    for p, r in zip(preds, ref):
        assert set(p) == set(r)
        for k in r:
            assert rel_l2(p[k].detach().cpu(), r[k].cpu()) < 1e-3, k
    model.eval()
    with torch.no_grad():
        pe, _ = model(frames)                         # eval after train: weights re-packed, the gated / cut path again
    assert not pe[0]["pts3d"].requires_grad


def test_backward_gradients_vs_oracle_autograd(model):
    """Gradients of a scalar loss through the training forward (native kernels forward, PyTorch recompute backward) vs
    gradients of the same loss through the oracle differentiated by autograd (strict fp32), on a sample of parameters from
    every stage.  The backward itself is exact (tests/test_train_cpu.py: <= 2e-4 when it is fed fp32-exact activations);
    here it is fed the CUDA forward's activations (<= 3e-4 from fp32: bf16x3 / tf32), and the random-sign loss below makes
    the parameter gradients sums of cancelling contributions, which amplifies that.  Bar: 3e-3 relative and cosine
    similarity >= 0.99999."""
    from oracle import spann3r_oracle as orc
    from spann3r_b200 import synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = synth.make_frames(3, 224, 224)
    g = torch.Generator().manual_seed(5)
    wts = [torch.randn(1, 224, 224, 3, generator=g).cuda() for _ in range(3)]

    def loss_of(preds):
        tot = 0.0
        for p, w in zip(preds, wts):
            k = "pts3d" if "pts3d" in p else "pts3d_in_other_view"
            tot = tot + (p[k] * w).sum() + 0.1 * p["conf"].log().sum()
        return tot

    watch = ["dust3r.enc_blocks.3.attn.qkv.weight", "dust3r.enc_norm.weight", "dust3r.dec_blocks.7.cross_attn.projk.weight",
             "dust3r.dec_blocks2.2.mlp.fc1.bias", "attn_head_2.0.weight", "norm_k.weight", "value_encoder.4.mlp.fc2.weight",
             "value_out.bias", "dust3r.downstream_head1.dpt.scratch.refinenet2.resConfUnit1.conv1.weight",
             "dust3r.downstream_head2.dpt.head.4.weight", "pos_patch_embed.proj.weight"]
    model.train()
    model.zero_grad(set_to_none=True)
    preds, _ = model(frames)
    loss = loss_of(preds)
    loss.backward()
    named = dict(model.named_parameters())
    got = {k: named[k].grad.detach().clone() for k in watch}
    model.zero_grad(set_to_none=True)
    model.eval()

    sd = {k: v.cuda().requires_grad_(k in watch) for k, v in get_state_dict(True).items()}
    ref_preds, _ = orc.forward.__wrapped__(sd, [{"img": f["img"].cuda()} for f in frames], attn_thresh=0, sim_thresh=1.0)
    ref_loss = loss_of(ref_preds)
    grads = torch.autograd.grad(ref_loss, [sd[k] for k in watch])
    assert abs(float(loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss))
    errs = {k: rel_l2(got[k].cpu(), gr.cpu()) for k, gr in zip(watch, grads)}
    cos = {k: float(torch.nn.functional.cosine_similarity(got[k].flatten().double().cpu(), gr.flatten().double().cpu(), dim=0))
           for k, gr in zip(watch, grads)}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < 3e-3, errs
    assert min(cos.values()) > 0.99999, cos


def test_native_linear_forward_dgrad_wgrad_vs_torch():
    """`_native_linear`: y = x W^T + b, dx = dy W, dW = dy^T x, db on the wgmma GEMM engine (bf16x3) against torch fp64,
    incl. a row count that is not a multiple of 8 (the wgrad contraction is zero-padded) and the 1792-wide key head."""
    from spann3r_b200 import _native_linear as NL
    g = torch.Generator().manual_seed(3)
    for lead, K, N in (((2, 196), 768, 3072), ((1, 588), 1024, 1024), ((3, 50), 1792, 1792), ((784,), 3072, 768)):
        x = torch.randn(*lead, K, generator=g).cuda().requires_grad_(True)
        w = (torch.randn(N, K, generator=g) * K ** -0.5).cuda().requires_grad_(True)
        b = torch.randn(N, generator=g).cuda().requires_grad_(True)
        gy = torch.randn(*lead, N, generator=g).cuda()
        y = NL._NativeLinear.apply(x, w, b)
        gx, gw, gb = torch.autograd.grad(y, (x, w, b), gy)
        xd, wd, bd = (t.detach().double().requires_grad_(True) for t in (x, w, b))
        yr = torch.nn.functional.linear(xd, wd, bd)
        rx, rw, rb = torch.autograd.grad(yr, (xd, wd, bd), gy.double())
        for name, a, r in (("y", y, yr), ("dx", gx, rx), ("dW", gw, rw), ("db", gb, rb)):
            assert a.shape == r.shape, name
            assert rel_l2(a.detach().cpu(), r.detach().cpu()) < 3e-5, (lead, K, N, name, rel_l2(a.detach().cpu(), r.detach().cpu()))


def test_backward_with_native_linear_matches_the_torch_backward(model):
    """The same training step differentiated with the Linear layers of the backward on the GEMM engine (`set_native_linear`)
    and with PyTorch's: the gradients agree to bf16x3 accuracy (each GEMM differs from cuBLAS fp32 by ~1e-5, the parameter
    gradients are sums of cancelling terms; the op itself is held to 3e-5 against fp64 above)."""
    from spann3r_b200 import synth, train
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = synth.make_frames(3, 224, 224)
    watch = ["dust3r.enc_blocks.3.attn.qkv.weight", "dust3r.dec_blocks.7.cross_attn.projk.weight", "dust3r.dec_blocks2.2.mlp.fc1.bias",
             "attn_head_2.0.weight", "value_encoder.4.mlp.fc2.weight", "value_out.bias", "norm_k.weight",
             "dust3r.downstream_head1.dpt.scratch.refinenet2.resConfUnit1.conv1.weight"]
    named = dict(model.named_parameters())
    grads = {}
    try:
        for native in (False, True):
            train.set_native_linear(native)
            model.train()
            model.zero_grad(set_to_none=True)
            preds, _ = model(frames)
            loss = sum(p[k].square().mean() + p["conf"].log().mean() for p in preds for k in p if k != "conf")
            loss.backward()
            grads[native] = {k: named[k].grad.detach().clone() for k in watch}
    finally:
        train.set_native_linear(False)
        model.zero_grad(set_to_none=True)
        model.eval()
    errs = {k: rel_l2(grads[True][k].cpu(), grads[False][k].cpu()) for k in watch}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < 5e-4, errs
