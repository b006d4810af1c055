"""`spann3r_b200.curope`: drop-in for the reference's pybind module `curope` / `cuRoPE2D`
(croco/models/curope/curope.cpp:49-69, curope2d.py:12-40) -- argument checks, in-place + autograd wiring (CPU, the kernel
replaced by the oracle's rotation), and the CUDA kernel through the C ABI (GPU)."""
import pytest
import torch

from conftest import rel_l2


def _qkv_views(B=2, N=50, H=4, D=64, seed=0, device="cpu", requires_grad=False):
    """q, k as croco/models/blocks.py:96-97 makes them: views of the qkv projection output."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, N, 3, H, D, generator=g).to(device)
    if requires_grad:
        x.requires_grad_(True)
    qkv = (x * 1.0).transpose(1, 3)                     # [B, H, 3, N, D], non-leaf
    pos = torch.randint(0, 32, (B, N, 2), generator=g).to(device)
    return x, qkv[:, :, 0], qkv[:, :, 1], pos


def test_argument_checks_match_the_pybind_module():
    from spann3r_b200 import curope
    tok, pos = torch.zeros(2, 5, 4, 64), torch.zeros(2, 5, 2, dtype=torch.int64)
    for bad_tok, bad_pos, msg in [
        (tok[0], pos, "tokens must have 4 dimensions"),
        (tok, pos[0], "positions must have 3 dimensions"),
        (tok, pos[:1], "batch size differs"),
        (tok, pos[:, :4], "seq_length differs"),
        (tok, torch.zeros(2, 5, 3, dtype=torch.int64), r"positions.shape\[2\] must be equal to 2"),
        (tok, pos, "no CPU path"),
    ]:
        with pytest.raises(RuntimeError, match=msg):
            curope.rope_2d(bad_tok, bad_pos, 100.0, 1.0)


def test_inplace_and_autograd_wiring_with_the_oracle_rotation(monkeypatch):
    """The Function / Module plumbing on the CPU: the kernel launch is replaced by the pinned oracle's rope2d, everything
    else (views, mark_dirty, the -F0 backward) is the module's own code."""
    from oracle.spann3r_oracle import rope2d
    from spann3r_b200 import curope

    def fake_rope_2d(tokens, positions, base, fwd):     # tokens [B, N, H, D] view, rotated in place
        pos = positions if fwd > 0 else positions       # inverse rotation = rotate by -angle: swap the sin sign
        t = tokens.detach().transpose(1, 2)
        if fwd > 0:
            out = rope2d(t, pos, base)
        else:                                           # R(-a) x: conjugate trick, rope2d(x with v negated) negated back
            D = t.shape[-1]
            sgn = torch.ones(D)
            q = D // 4
            sgn[q: 2 * q] = -1
            sgn[3 * q:] = -1
            out = rope2d(t * sgn, pos, base) * sgn
        with torch.no_grad():
            tokens.copy_(out.transpose(1, 2))

    monkeypatch.setattr(curope, "rope_2d", fake_rope_2d)
    x, q, k, pos = _qkv_views(requires_grad=True)
    ref_x = x.detach().clone().double().requires_grad_(True)
    ref_q = rope2d((ref_x * 1.0).transpose(1, 3)[:, :, 0], pos)
    rope = curope.cuRoPE2D(freq=100.0)
    out = rope(q, pos)
    assert out is q and rel_l2(out.detach(), ref_q.detach()) < 1e-6          # rotated in place, same object back
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(3))
    (out * w).sum().backward()
    (ref_q * w.double()).sum().backward()
    assert rel_l2(x.grad, ref_x.grad) < 1e-6


@pytest.mark.gpu
@pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")
def test_cuda_rope_matches_the_oracle_forward_and_backward():
    from oracle.spann3r_oracle import rope2d
    from spann3r_b200 import curope
    x, q, k, pos = _qkv_views(device="cuda", requires_grad=True)
    ref_x = x.detach().clone().double().requires_grad_(True)
    rq = rope2d((ref_x * 1.0).transpose(1, 3)[:, :, 0], pos)
    rope = curope.cuRoPE2D(freq=100.0)
    out = rope(q, pos)
    assert out is q and rel_l2(out.detach().cpu(), rq.detach().cpu()) < 1e-5
    w = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).cuda()
    (out * w).sum().backward()
    (rq * w.double()).sum().backward()
    assert rel_l2(x.grad.cpu(), ref_x.grad.cpu()) < 1e-5
    # direct call on a [B, N, H, D] tensor (the pybind signature), per-batch launches when the batch stride is irregular
    tok = torch.randn(3, 20, 4, 64, device="cuda")
    big = torch.zeros(3, 25, 4, 64, device="cuda")
    view = big[:, :20]                                   # stride(0) != N * stride(1)
    view.copy_(tok)
    p = torch.randint(0, 32, (3, 20, 2), device="cuda")
    exp = rope2d(tok.transpose(1, 2).double(), p).transpose(1, 2)
    curope.rope_2d(tok, p, 100.0, 1.0)
    curope.rope_2d(view, p, 100.0, 1.0)
    torch.cuda.synchronize()
    assert rel_l2(tok.cpu(), exp.cpu()) < 1e-5 and rel_l2(view.cpu(), exp.cpu()) < 1e-5
    with pytest.raises(RuntimeError, match="tokens are not contiguous"):
        curope.rope_2d(torch.zeros(2, 4, 20, 64, device="cuda").transpose(1, 2), p[:2], 100.0, 1.0)
