"""The training attention bit for bit: s3r_attn_train_forward / s3r_attn_train_backward and the autograd Function of
`_native_attn`, on inputs where every step is exact in fp32 (attn_train_exact.py), against the one correct answer
computed in fp64 on the GPU.

O, dQ, dK and dV are compared with `torch.equal`, with the wrong elements reported per slice and 64-row tile.  LSE is
compared the same way on rows that keep one key, and within 1 ulp of fp32(s max + ln k) on rows that keep k > 1 (logf's
documented error).  The backward runs on a given LSE and O, so that P has several ones per row and D = rowsum(dO o O) is
far from dP.  Each case runs on three layouts of q / k / v: contiguous; the permuted view of a [B, N, 3, heads, dh] qkv
buffer (nq = nk); views into a NaN-filled buffer with a padded token stride, a head stride of 64 at dh = 48, a start
offset and NaN past the end.  Every output is followed by a sentinel that must survive, every input by NaN that must not
reach an output, and the workspace starts as NaN."""
import ctypes as C
import functools

import pytest
import torch

import attn_train_exact as A

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs an H100")]

SENT = -7.0e30
LAYOUTS = ("contiguous", "qkv", "padded")


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


@functools.lru_cache(maxsize=2)
def _case(case: A.Case):
    c = A.make(case)
    fwd = A.forward_ref(c, "cuda")
    bwd = A.backward_ref(c, "cuda")
    return c, fwd, bwd


def _guarded(t: torch.Tensor) -> torch.Tensor:
    """A device copy of t followed by NaN."""
    buf = torch.full((t.numel() + 1024,), float("nan"), dtype=t.dtype, device="cuda")
    v = buf[:t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _out(shape):
    """(buffer, view): an output of `shape` followed by 1024 sentinels."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + 1024,), SENT, device="cuda")
    return buf, buf[:n].view(shape)


def _tail_intact(name, buf, n):
    bad = buf[n:] != SENT
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} sentinels past the end overwritten"


def _operands(c, layout):
    """q, k, v on the device in the given layout."""
    q, k, v = c["q"], c["k"], c["v"]
    B, H, nq, dh = q.shape
    if layout == "contiguous":
        return tuple(_guarded(x) for x in (q, k, v))
    if layout == "qkv":
        buf = torch.full((B, nq, 3, H, dh), float("nan"), device="cuda")
        for i, x in enumerate((q, k, v)):
            buf[:, :, i] = x.transpose(1, 2).cuda()
        qkv = buf.permute(2, 0, 3, 1, 4)
        return qkv[0], qkv[1], qkv[2]
    out = []
    hs = 64 if dh == 48 else dh + 4
    for x in (q, k, v):
        n = x.shape[2]
        ts = H * hs + 8
        bs = n * ts + 16
        buf = torch.full((8 + B * bs + 64,), float("nan"), device="cuda")
        view = buf.as_strided((B, H, n, dh), (bs, hs, ts, 1), 8)
        view.copy_(x)
        out.append(view)
    return tuple(out)


def _layouts(case):
    return [lay for lay in LAYOUTS if lay != "qkv" or case.nq == case.nk]


def _params(cases):
    return [pytest.param(case, lay, id=f"{case.id}-{lay}") for case in cases for lay in _layouts(case)]


def _no_nan(name, x):
    assert not bool(torch.isnan(x).any()), f"{name}: NaN in the output"


@pytest.mark.parametrize("case,layout", _params(A.cases()))
def test_forward_is_exact(L, case, layout):
    from spann3r_b200 import _native_attn as NA
    c, (o_ref, lse_ref, k), _ = _case(case)
    q, k_, v = _operands(c, layout)
    B, H, nq, dh = q.shape
    d = NA._desc(q, k_, v, A.SCALE)
    ob, o = _out((B, nq, H * dh))
    lb, lse = _out((B * H, nq))
    L.check(L.lib().s3r_attn_train_forward(C.byref(d), L.ptr(o), L.ptr(lse), L.stream_ptr()), "forward")
    torch.cuda.synchronize()
    for name, x, buf in (("O", o, ob), ("LSE", lse, lb)):
        _no_nan(name, x)
        _tail_intact(name, buf, x.numel())
    tiles = A.row_tiles(c, nq)
    A.tile_report("O", A.slices(o, B, H), A.slices(o_ref, B, H), tiles)
    one = k == 1
    A.tile_report("LSE (k = 1)", torch.where(one, lse, 0.0)[..., None], torch.where(one, lse_ref, 0.0)[..., None],
                  tiles)
    inf = torch.full_like(lse_ref, float("inf"))
    ulp = torch.nextafter(lse_ref.abs(), inf) - lse_ref.abs()
    off = (lse - lse_ref).abs() > ulp
    assert not bool(off.any()), f"LSE (k > 1): {int(off.sum())} rows off by more than 1 ulp, first at " \
                                f"{off.nonzero()[0].tolist()}: {float(lse[off][0])!r} vs {float(lse_ref[off][0])!r}"


def _backward(L, c, q, k, v, lse, o, go):
    """s3r_attn_train_backward on the given operands; (dq, dk, dv) after checking their sentinels."""
    from spann3r_b200 import _native_attn as NA
    d = NA._desc(q, k, v, A.SCALE)
    lib = L.lib()
    ws_bytes = lib.s3r_attn_train_workspace_bytes(C.byref(d))
    ws = torch.full((ws_bytes // 4,), float("nan"), device="cuda")
    outs = [_out(x.shape) for x in (c["q"], c["k"], c["v"])]
    (qb, dq), (kb, dk), (vb, dv) = outs
    o, lse, go = _guarded(o), _guarded(lse), _guarded(go)   # held until the kernels have run
    L.check(lib.s3r_attn_train_backward(C.byref(d), L.ptr(o), L.ptr(lse), L.ptr(go), L.ptr(ws), ws_bytes, L.ptr(dq),
                                        L.ptr(dk), L.ptr(dv), L.stream_ptr()), "backward")
    torch.cuda.synchronize()
    for name, (buf, x) in zip(("dQ", "dK", "dV"), outs):
        _no_nan(name, x)
        _tail_intact(name, buf, x.numel())
    return dq, dk, dv


@pytest.mark.parametrize("case,layout", _params(A.cases()))
def test_backward_with_given_lse_is_exact(L, case, layout):
    c, _, (dq_ref, dk_ref, dv_ref) = _case(case)
    q, k, v = _operands(c, layout)
    dq, dk, dv = _backward(L, c, q, k, v, c["lse"], c["o"], c["go"])
    B, H = case.B, case.H
    A.tile_report("dQ", A.slices(dq, B, H), A.slices(dq_ref, B, H), A.row_tiles(c, case.nq))
    A.tile_report("dK", A.slices(dk, B, H), A.slices(dk_ref, B, H), A.row_tiles(c, case.nk))
    A.tile_report("dV", A.slices(dv, B, H), A.slices(dv_ref, B, H), A.row_tiles(c, case.nk))


@pytest.mark.parametrize("case", A.e2e_cases(), ids=lambda c: c.id)
def test_autograd_forward_then_backward_is_exact(L, case):
    """Every row keeps one key: O and LSE are exact, D equals dP on the kept key, so dQ = dK = 0 and dV = P^T dO."""
    from spann3r_b200 import _native_attn as NA
    c = A.make(case)
    o_ref, lse_ref, k = A.forward_ref(c, "cuda")
    assert bool((k == 1).all())
    dq_ref, dk_ref, dv_ref = A.backward_ref(c, "cuda", lse=lse_ref, o=o_ref)
    q, k_, v = (c[n].cuda().requires_grad_(True) for n in ("q", "k", "v"))
    o = NA.attention(q, k_, v, A.SCALE)
    dq, dk, dv = torch.autograd.grad(o, (q, k_, v), c["go"].cuda())
    _, lse = NA.attention_with_lse(q.detach(), k_.detach(), v.detach(), A.SCALE)
    B, H = case.B, case.H
    tq, tk = A.row_tiles(c, case.nq), A.row_tiles(c, case.nk)
    A.tile_report("O", A.slices(o.detach(), B, H), A.slices(o_ref, B, H), tq)
    A.tile_report("LSE", lse[..., None], lse_ref[..., None], tq)
    for name, got, exp, t in (("dQ", dq, dq_ref, tq), ("dK", dk, dk_ref, tk), ("dV", dv, dv_ref, tk)):
        A.tile_report(name, A.slices(got, B, H), A.slices(exp, B, H), t)
    assert not bool(dq.any()) and not bool(dk.any())
