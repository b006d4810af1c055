"""The native-convolution switch and its C entry points, without a GPU: argument validation happens before any CUDA call,
and on CPU tensors the recompute keeps the PyTorch convolutions whatever the switch says."""
import ctypes as C

import pytest
import torch

from conftest import get_state_dict

_P = C.c_void_p(1 << 20)   # a 16-byte aligned address that is never dereferenced: validation must reject first


def _wgrad(L, nb=1, h=14, w=14, n=256, kc=256, taps=9, ldy=None, ldx=None, ptrs=(_P,) * 4, ws=_P, ws_bytes=None, dw=_P):
    if ws_bytes is None:
        ws_bytes = L.s3r_conv_wgrad_workspace_bytes(nb, h, w, n, kc, taps)
    return L.s3r_conv_wgrad(ptrs[0], ptrs[1], n if ldy is None else ldy, ptrs[2], ptrs[3], kc if ldx is None else ldx, nb, h,
                            w, n, kc, taps, ws, ws_bytes, dw, None)


def test_conv_wgrad_and_col2im_reject_bad_arguments_without_touching_the_device():
    from spann3r_b200 import _lib
    L = _lib.lib()
    need = L.s3r_conv_wgrad_workspace_bytes(4, 224, 224, 128, 128, 9)
    assert need >= 128 * 9 * 128 * 4 and need % 16 == 0
    assert L.s3r_conv_wgrad_workspace_bytes(1, 14, 14, 256, 256, 3) == 0          # taps not in {1, 9}
    assert L.s3r_conv_wgrad_workspace_bytes(0, 14, 14, 256, 256, 9) == 0          # no image
    assert L.s3r_conv_wgrad_workspace_bytes(1, 14, 14, 100, 256, 9) == 0          # n not a multiple of 8
    cases = [
        (dict(taps=4), b"taps"),
        (dict(h=0), b"unsupported shape"),
        (dict(kc=30), b"unsupported shape"),
        (dict(ldy=260), b"multiples of 8"),
        (dict(ldx=250), b"multiples of 8"),
        (dict(ldy=128), b"multiples of 8"),                                      # row stride shorter than the row
        (dict(ptrs=(_P, None, _P, _P)), b"pointer"),
        (dict(ptrs=(_P, _P, C.c_void_p((1 << 20) + 8), _P)), b"aligned"),
        (dict(dw=None), b"pointer"),
        (dict(ws=None), b"pointer"),
        (dict(ws_bytes=L.s3r_conv_wgrad_workspace_bytes(1, 14, 14, 256, 256, 9) - 4), b"workspace"),
    ]
    for kw, msg in cases:
        assert _wgrad(L, **kw) == -1, kw
        assert msg in L.s3r_last_error(), (kw, L.s3r_last_error())
    assert L.s3r_col2im_3x3s2(_P, 1, 14, 14, 768, 7, 7, None, None) == -1
    assert b"pointer" in L.s3r_last_error()
    assert L.s3r_col2im_3x3s2(_P, 1, 14, 14, 768, 8, 7, _P, None) == -1          # ho != (h + 1) / 2
    assert b"ho = (h+1)/2" in L.s3r_last_error()
    assert L.s3r_col2im_3x3s2(_P, 1, 14, 14, 20, 7, 7, _P, None) == -1           # c not a multiple of 8
    assert L.s3r_col2im_3x3s2(_P, 0, 14, 14, 768, 7, 7, _P, None) == -1


def test_recompute_on_cpu_keeps_the_torch_convolutions_with_the_switch_on(monkeypatch):
    """With the switch on, a DPT head and the value encoder's patch embedding recomputed on CPU tensors go through
    F.conv2d / F.conv_transpose2d (no native Function is built) and give the same bits as with it off."""
    from spann3r_b200 import _native_conv as NC, _recompute as R, train
    sd = get_state_dict(True)
    P = {k: v for k, v in sd.items() if k.startswith(("dust3r.downstream_head1.", "pos_patch_embed."))}
    g = torch.Generator().manual_seed(0)
    gh = gw = 2
    hooks = [torch.randn(1, gh * gw, 1024, generator=g)] + [torch.randn(1, gh * gw, 768, generator=g) for _ in range(3)]
    pts = torch.randn(1, 32, 32, 3, generator=g)

    def run():
        with torch.no_grad():
            p, c = R._dpt(P, "dust3r.downstream_head1.dpt", hooks, gh, gw)
            v = R._conv(P, "pos_patch_embed.proj", pts.permute(0, 3, 1, 2), stride=16)
        return p, c, v

    off = run()
    for cls in (NC._Conv1x1, NC._Conv3x3, NC._Conv3x3s2, NC._PatchConv, NC._ConvT):
        monkeypatch.setattr(cls, "apply", staticmethod(lambda *a: pytest.fail("native conv on CPU tensors")))
    try:
        train.set_native_conv(True)
        on = run()
    finally:
        train.set_native_conv(False)
    for a, b in zip(off, on):
        assert torch.equal(a, b)
