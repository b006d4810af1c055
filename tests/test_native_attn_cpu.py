"""The native-attention switch of the training backward and its C entry points, without a GPU: the sm_90a build of
csrc/attention_train.cu has no spills, argument validation happens before any CUDA call, and on CPU tensors the recompute
keeps the PyTorch attention whatever the switch says."""
import ctypes as C
import os
import re
import subprocess

import pytest
import torch

from conftest import get_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_P = 1 << 20   # a 16-byte aligned address that is never dereferenced: validation must reject first


def test_attention_train_cu_builds_without_spills(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "spann3r_b200", "csrc", "attention_train.cu"), "-o",
                        str(tmp_path / "attention_train.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == 4 and all(s == ("0", "0") for s in spills), spills


def _desc(**kw):
    from spann3r_b200 import _lib
    d = _lib.AttnTrainDesc()
    d.batch, d.heads, d.nq, d.nk, d.dh, d.scale = 2, 16, 196, 196, 64, 0.125
    d.q, d.k, d.v = _P, _P, _P
    for name in ("q_stride", "k_stride", "v_stride"):
        getattr(d, name)[:] = [16 * 196 * 64, 196 * 64, 64]
    for k, v in kw.items():
        if k.endswith("_stride"):
            getattr(d, k)[:] = v
        else:
            setattr(d, k, v)
    return d


def test_attn_train_abi_rejects_bad_arguments_without_touching_the_device():
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_abi_sizeof(4) == C.sizeof(_lib.AttnTrainDesc)
    ok = _desc()
    need = L.s3r_attn_train_workspace_bytes(C.byref(ok))
    assert need >= 2 * 16 * 196 * 4 and need % 256 == 0
    assert L.s3r_attn_train_workspace_bytes(None) == 0
    assert b"null descriptor" in L.s3r_last_error()
    cases = [
        (dict(dh=32), b"48 or 64"),
        (dict(dh=80), b"48 or 64"),
        (dict(batch=0), b">= 1"),
        (dict(heads=0), b">= 1"),
        (dict(nq=0), b">= 1"),
        (dict(nk=-3), b">= 1"),
        (dict(batch=5000, heads=16), b"65535"),
        (dict(scale=0.0), b"scale"),
        (dict(scale=float("nan")), b"scale"),
        (dict(q=None), b"aligned"),
        (dict(k=_P + 4), b"aligned"),
        (dict(v=None), b"aligned"),
        (dict(q_stride=[16 * 196 * 64, 196 * 64, 66]), b"multiples of 4"),
        (dict(v_stride=[-64, 196 * 64, 64]), b"multiples of 4"),
    ]
    for kw, msg in cases:
        d = _desc(**kw)
        assert L.s3r_attn_train_workspace_bytes(C.byref(d)) == 0, kw
        assert msg in L.s3r_last_error(), (kw, L.s3r_last_error())
        assert L.s3r_attn_train_forward(C.byref(d), _P, _P, None) == -1, kw
        assert msg in L.s3r_last_error(), (kw, L.s3r_last_error())
        assert L.s3r_attn_train_backward(C.byref(d), _P, _P, _P, _P, need, _P, _P, _P, None) == -1, kw
        assert msg in L.s3r_last_error(), (kw, L.s3r_last_error())
    assert L.s3r_attn_train_forward(None, _P, _P, None) == -1
    assert b"null descriptor" in L.s3r_last_error()
    for o, lse in ((None, _P), (_P, None), (_P + 8, _P)):
        assert L.s3r_attn_train_forward(C.byref(ok), o, lse, None) == -1
        assert b"aligned" in L.s3r_last_error()
    ptrs = [_P] * 7                                       # o, lse, d_o, workspace, dq, dk, dv
    for i in range(7):
        bad = list(ptrs)
        bad[i] = None if i % 2 else _P + 4
        args = bad[:4] + [need] + bad[4:]
        assert L.s3r_attn_train_backward(C.byref(ok), *args, None) == -1, i
        assert b"aligned" in L.s3r_last_error(), i
    assert L.s3r_attn_train_backward(C.byref(ok), _P, _P, _P, _P, need - 256, _P, _P, _P, None) == -1
    assert b"workspace" in L.s3r_last_error()


def test_recompute_on_cpu_keeps_the_torch_attention_with_the_switch_on(monkeypatch):
    """With the switch on, an encoder block, a decoder block (self + cross) and a 48-wide use_feat value block recomputed
    on CPU tensors go through `_sdpa` (the native Function is never built) and give the same bits as with it off."""
    from spann3r_b200 import _native_attn as NA, _recompute as R, synth, train
    sd = get_state_dict(True)
    uf = synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True)
    g = torch.Generator().manual_seed(0)
    gh, gw = 2, 3
    cs = R._rope_cs(gh, gw, "cpu")
    cs48 = R._rope_cs(gh, gw, "cpu", head_dim=48)
    x = torch.randn(2, gh * gw, 1024, generator=g)
    y = torch.randn(2, gh * gw, 768, generator=g)
    z = torch.randn(2, gh * gw, 768, generator=g)

    def run():
        with torch.no_grad():
            return (R._block(sd, "dust3r.enc_blocks.0", x, R.ENC_HEADS, cs),
                    R._dec_block(sd, "dust3r.dec_blocks.0", y, z, cs),
                    R._block(uf, "value_encoder.0", y, R.VAL_HEADS, cs48))

    off = run()
    monkeypatch.setattr(NA._Attention, "apply", staticmethod(lambda *a: pytest.fail("native attention on CPU tensors")))
    try:
        train.set_native_attention(True)
        on = run()
    finally:
        train.set_native_attention(False)
    for a, b in zip(off, on):
        assert torch.equal(a, b)
