"""The convolutions of the training backward on the library's kernels (`_native_conv`, `train.set_native_conv`): every conv
the DPT heads and the patch embeddings issue, forward / dx / dW / db against torch fp64 autograd; the weight-gradient
kernel's bitwise reproducibility; and a full training step with the switch on against it off."""
import zlib

import pytest
import torch

from conftest import get_state_dict, rel_l2

pytestmark = pytest.mark.gpu


def _convs(H, W):
    """(name, kind, Cin, Cout, map h, map w) of one DPT head + the patch embeddings for an H x W frame (`_recompute._dpt`)."""
    gh, gw = H // 16, W // 16
    h3, w3 = (gh + 1) // 2, (gw + 1) // 2
    return [
        ("act_postprocess.0.0", "1x1", 1024, 96, gh, gw),
        ("act_postprocess.1.0", "1x1", 768, 192, gh, gw),
        ("act_postprocess.2.0", "1x1", 768, 384, gh, gw),
        ("act_postprocess.3.0", "1x1", 768, 768, gh, gw),
        ("act_postprocess.0.1", "convT4", 96, 96, gh, gw),
        ("act_postprocess.1.1", "convT2", 192, 192, gh, gw),
        ("act_postprocess.3.1", "3x3s2", 768, 768, gh, gw),
        ("layer_rn.0", "3x3nb", 96, 256, 4 * gh, 4 * gw),
        ("layer_rn.1", "3x3nb", 192, 256, 2 * gh, 2 * gw),
        ("layer_rn.2", "3x3nb", 384, 256, gh, gw),
        ("layer_rn.3", "3x3nb", 768, 256, h3, w3),
        ("refinenet4.rcu", "3x3", 256, 256, h3, w3),
        ("refinenet3.rcu", "3x3", 256, 256, gh, gw),
        ("refinenet2.rcu", "3x3", 256, 256, 2 * gh, 2 * gw),
        ("refinenet1.rcu", "3x3", 256, 256, 4 * gh, 4 * gw),
        ("refinenet4.out_conv", "1x1", 256, 256, gh, gw),
        ("refinenet3.out_conv", "1x1", 256, 256, 2 * gh, 2 * gw),
        ("refinenet2.out_conv", "1x1", 256, 256, 4 * gh, 4 * gw),
        ("refinenet1.out_conv", "1x1", 256, 256, 8 * gh, 8 * gw),
        ("head.0", "3x3", 256, 128, H // 2, W // 2),
        ("head.2", "3x3", 128, 128, H, W),
        ("patch_embed", "patch", 3, 1024, H, W),
        ("pos_patch_embed", "patch_dx", 3, 1024, H, W),
    ]


_CASES = ([(n, k, ci, co, h, w, 1) for n, k, ci, co, h, w in _convs(224, 224)] +
          [(n, k, ci, co, h, w, 4) for n, k, ci, co, h, w in _convs(224, 224)] +
          [(n, k, ci, co, h, w, 1) for n, k, ci, co, h, w in _convs(288, 224)] +
          [(n, k, ci, co, h, w, 1) for n, k, ci, co, h, w in _convs(512, 384) if n in ("head.0", "head.2", "refinenet1.rcu",
                                                                                       "refinenet1.out_conv")])


def _torch_call(kind, x, w, b):
    F = torch.nn.functional
    if kind in ("1x1",):
        return F.conv2d(x, w, b)
    if kind in ("3x3", "3x3nb"):
        return F.conv2d(x, w, b, padding=1)
    if kind == "3x3s2":
        return F.conv2d(x, w, b, stride=2, padding=1)
    if kind.startswith("patch"):
        return F.conv2d(x, w, b, stride=16)
    return F.conv_transpose2d(x, w, b, stride=int(kind[-1]))


def _native_call(kind, x, w, b):
    from spann3r_b200 import _native_conv as NC
    if kind in ("1x1",):
        return NC._Conv1x1.apply(x, w, b)
    if kind in ("3x3", "3x3nb"):
        return NC._Conv3x3.apply(x, w, b)
    if kind == "3x3s2":
        return NC._Conv3x3s2.apply(x, w, b)
    if kind.startswith("patch"):
        return NC._PatchConv.apply(x, w, b)
    return NC._ConvT.apply(x, w, b, int(kind[-1]))


@pytest.mark.parametrize("name,kind,cin,cout,h,w,nb", _CASES,
                         ids=[f"{c[0]}-{c[6]}x{c[4]}x{c[5]}" for c in _CASES])
def test_native_conv_forward_dgrad_wgrad_vs_torch_fp64(name, kind, cin, cout, h, w, nb):
    """y, dx, dW, db of the native Function against F.conv2d / F.conv_transpose2d in fp64 autograd: relative L2 < 3e-5 (the
    bar of the native Linear).  The image input of `patch_embed` needs no gradient, so its dgrad is skipped."""
    g = torch.Generator().manual_seed(zlib.crc32(f"{name}-{nb}-{h}-{w}".encode()))
    if kind.startswith("convT"):
        s = int(kind[-1])
        wt = torch.randn(cin, cout, s, s, generator=g) * cin ** -0.5
    else:
        k = {"1x1": 1, "patch": 16, "patch_dx": 16}.get(kind, 3)
        wt = torch.randn(cout, cin, k, k, generator=g) * (cin * k * k) ** -0.5
    x = torch.randn(nb, cin, h, w, generator=g)
    if kind == "patch_dx":   # pos_patch_embed: the input is pts3d [B, H, W, 3] seen as NCHW (a strided view)
        x = torch.randn(nb, h, w, 3, generator=g).cuda().permute(0, 3, 1, 2)
    else:
        x = x.cuda()
    bias = None if kind == "3x3nb" else torch.randn(cout, generator=g).cuda().requires_grad_(True)
    wt = wt.cuda().requires_grad_(True)
    x = x.requires_grad_(kind != "patch")
    y = _native_call(kind, x, wt, bias)
    gy = torch.randn(y.shape, generator=g).cuda()
    wrt = [t for t in (x, wt, bias) if t is not None and t.requires_grad]
    got = torch.autograd.grad(y, wrt, gy)
    ref_in = [t.detach().double().requires_grad_(t.requires_grad) if t is not None else None for t in (x, wt, bias)]
    yr = _torch_call(kind, *ref_in)
    ref = torch.autograd.grad(yr, [t for t in ref_in if t is not None and t.requires_grad], gy.double())
    names = [n for n, t in zip(("dx", "dW", "db"), (x, wt, bias)) if t is not None and t.requires_grad]
    assert y.shape == yr.shape
    errs = {"y": rel_l2(y.detach().cpu(), yr.detach().cpu())}
    for n, a, r in zip(names, got, ref):
        assert a.shape == r.shape, n
        errs[n] = rel_l2(a.cpu(), r.cpu())
    assert max(errs.values()) < 3e-5, (name, nb, h, w, errs)


@pytest.mark.parametrize("nb,h,w,n,kc,taps", [(1, 7, 7, 256, 768, 9), (2, 37, 53, 128, 96, 9), (3, 19, 23, 192, 256, 1),
                                              (4, 224, 224, 128, 128, 9)])
def test_conv_wgrad_is_bitwise_reproducible(nb, h, w, n, kc, taps):
    """Two calls on the same planes give identical bits: a 7 x 7 map, pixel counts that are not a multiple of the 64-pixel
    k-block, channel counts that leave part of a 128-wide tile empty, and the longest contraction of the 224 x 224 path."""
    from spann3r_b200 import _lib
    g = torch.Generator().manual_seed(nb * 1000 + h)
    dy = _lib.split(torch.randn(nb, h, w, n, generator=g).cuda())
    x = _lib.split(torch.randn(nb, h, w, kc, generator=g).cuda())
    a = _lib.conv_wgrad(dy, x, taps)
    b = _lib.conv_wgrad(dy, x, taps)
    assert torch.equal(a, b)
    # and it is the weight gradient: against fp64 on the same split-bf16 operands' fp32 values
    yd = (dy[0].double() + dy[1].double()).permute(0, 3, 1, 2)
    xd = (x[0].double() + x[1].double()).permute(0, 3, 1, 2)
    ref = torch.nn.grad.conv2d_weight(xd, (n, kc, 3, 3) if taps == 9 else (n, kc, 1, 1), yd, padding=1 if taps == 9 else 0)
    got = a.view(n, 3, 3, kc).permute(0, 3, 1, 2) if taps == 9 else a.view(n, kc, 1, 1)
    assert rel_l2(got.cpu(), ref.cpu()) < 3e-5


def test_col2im_is_the_adjoint_of_im2col():
    """<col2im(G), X> == <G, im2col(X)> for the 3x3 stride-2 pad-1 conv, odd and even maps."""
    from spann3r_b200 import _lib
    g = torch.Generator().manual_seed(1)
    for nb, h, w, c in ((2, 14, 14, 64), (1, 7, 9, 32)):
        ho, wo = (h + 1) // 2, (w + 1) // 2
        cols = torch.randn(nb * ho * wo, 9 * c, generator=g).cuda()
        got = _lib.col2im_3x3s2(cols, nb, h, w, c)
        # F.unfold's column index is c * 9 + tap; the engine's is tap * C + c
        gu = cols.double().view(nb, ho * wo, 9, c).permute(0, 3, 2, 1).reshape(nb, c * 9, ho * wo)
        x = torch.zeros(nb, c, h, w, dtype=torch.float64, device="cuda", requires_grad=True)
        (gx,) = torch.autograd.grad(torch.nn.functional.unfold(x, 3, padding=1, stride=2), x, gu)
        assert rel_l2(got.permute(0, 3, 1, 2).cpu(), gx.cpu()) < 1e-6


@pytest.fixture(scope="module")
def model():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, memory_dropout=0.0)
    m.load_state_dict(get_state_dict(True), strict=True)
    return m.cuda()


def test_training_step_with_native_conv_matches_the_torch_backward(model):
    """A training step's gradients with the convolutions of the backward native (`set_native_conv`) and in PyTorch agree to
    relative L2 < 5e-4 on a parameter of every conv kind and their biases (measured on an H100: at most 2.2e-4).  With both
    native switches on against both off the bar is 1e-3: the worst parameter, refinenet4.resConfUnit2.conv1.weight (the
    7 x 7 map, a sum of cancelling terms), measured 6.0e-4 there."""
    from spann3r_b200 import synth, train
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    frames = synth.make_frames(3, 224, 224)
    h1 = "dust3r.downstream_head1.dpt."
    watch = [h1 + "act_postprocess.0.1.weight", h1 + "act_postprocess.3.1.weight", h1 + "scratch.layer_rn.0.weight",
             h1 + "scratch.refinenet4.resConfUnit2.conv1.weight", h1 + "head.2.weight", "pos_patch_embed.proj.weight",
             "dust3r.patch_embed.proj.weight", h1 + "act_postprocess.0.1.bias", h1 + "act_postprocess.3.1.bias",
             h1 + "head.2.bias", "dust3r.downstream_head2.dpt.scratch.refinenet1.out_conv.bias",
             "dust3r.downstream_head2.dpt.act_postprocess.1.0.weight", "pos_patch_embed.proj.bias",
             "dust3r.patch_embed.proj.bias"]
    named = dict(model.named_parameters(remove_duplicate=False))   # scratch.layer_rn.K aliases scratch.layerK+1_rn
    grads = {}
    try:
        for lin, conv in ((False, False), (False, True), (True, True)):
            train.set_native_linear(lin)
            train.set_native_conv(conv)
            model.train()
            model.zero_grad(set_to_none=True)
            preds, _ = model(frames)
            loss = sum(p[k].square().mean() + p["conf"].log().mean() for p in preds for k in p if k != "conf")
            loss.backward()
            grads[(lin, conv)] = {k: named[k].grad.detach().clone() for k in watch}
    finally:
        train.set_native_linear(False)
        train.set_native_conv(False)
        model.zero_grad(set_to_none=True)
        model.eval()
    for key, bar in (((False, True), 5e-4), ((True, True), 1e-3)):
        errs = {k: rel_l2(grads[key][k].cpu(), grads[(False, False)][k].cpu()) for k in watch}
        print(key, {k: "%.1e" % v for k, v in errs.items()})
        assert max(errs.values()) < bar, (key, errs)
