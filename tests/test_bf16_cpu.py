"""The opt-in bf16 precision without a GPU: the public switch, engine keying, the descriptor check, the cs_hi column sums
and the fp64 emulation oracle (oracle/bf16_oracle.py) that the GPU results are held to."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import GOLDEN, get_state_dict, rel_l2

FAKE = 0x7F0000000000   # never dereferenced: a rejected descriptor must not reach the driver


# ------------------------------------------------------------------------------------------------
# public switch
# ------------------------------------------------------------------------------------------------
def test_precision_kwarg_and_set_precision():
    from spann3r_b200 import Spann3R
    assert Spann3R(dus3r_name=None).precision == "fp32"
    m = Spann3R(dus3r_name=None, precision="bf16")
    assert m.precision == "bf16"
    m.set_precision("fp32")
    assert m.precision == "fp32"
    for bad in ("fp16", "BF16", "tf32", None, 1):
        with pytest.raises(ValueError, match="precision"):
            Spann3R(dus3r_name=None, precision=bad)
        with pytest.raises(ValueError, match="precision"):
            m.set_precision(bad)
    assert m.precision == "fp32"


def test_bf16_refuses_training_mode():
    """The PyTorch-recompute backward differentiates the fp32-grade forward, not the bf16 one."""
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None, precision="bf16").train()
    with pytest.raises(NotImplementedError, match="inference only"):
        m(synth.make_frames(2, 224, 224))
    with pytest.raises(NotImplementedError, match="inference only"):
        m._engine_for(1, 224, 224, training=True)


def test_engines_are_keyed_by_precision_and_share_the_packed_weights(monkeypatch):
    from spann3r_b200 import model as M
    made = []

    class _FakeEngine:
        def __init__(self, w, B, H, W, max_images=0, precision="fp32"):
            self.w, self.B, self.H, self.W, self.max_images, self.precision = w, B, H, W, max(max_images, 2 * B), precision
            made.append(self)

    packed = object()
    monkeypatch.setattr(M, "Engine", _FakeEngine)
    m = M.Spann3R(dus3r_name=None)
    monkeypatch.setattr(m, "_weights", lambda: packed)
    e32 = m._engine_for(1, 224, 224)
    assert e32.precision == "fp32" and m._engine_for(1, 224, 224) is e32
    m.set_precision("bf16")
    e16 = m._engine_for(1, 224, 224)
    assert e16 is not e32 and e16.precision == "bf16" and m._engine_for(1, 224, 224) is e16
    assert e16.w is packed and e32.w is packed
    m.set_precision("fp32")
    assert m._engine_for(1, 224, 224) is e32        # switching back reuses the fp32 engine
    assert set(m._engines) == {(1, 224, 224, "fp32"), (1, 224, 224, "bf16")}
    assert len(made) == 2


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
def _desc(L, precision):
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = FAKE, FAKE + 0x100000, FAKE + 0x200000, FAKE + 0x300000
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = 1, 1, 1, 196, 768, 1, 768
    d.out_f32, d.ldo = FAKE + 0x400000, 768
    d.precision = precision
    return d


@pytest.mark.parametrize("precision", [-1, 2, 3, 1 << 30])
def test_s3r_gemm_rejects_bad_precision_before_the_driver(precision):
    from spann3r_b200 import _lib as L
    d = _desc(L, precision)
    assert L.lib().s3r_gemm(C.byref(d), None) == -1
    assert b"precision" in L.lib().s3r_last_error()
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) == -1


def test_s3r_gemm_bf16_rejects_the_head_tail():
    from spann3r_b200 import _lib as L
    d = _desc(L, 1)
    d.n, d.epi = 128, L.EPI_HEADTAIL
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) == -1
    assert b"EPI_HEADTAIL" in L.lib().s3r_last_error()


def test_abi_mirrors_match():
    from spann3r_b200 import _lib as L
    from spann3r_b200.engine import ModelW
    assert L.lib().s3r_abi_sizeof(0) == C.sizeof(L.GemmDesc)
    assert L.lib().s3r_abi_sizeof(1) == C.sizeof(ModelW)


def test_engine_create_ex_rejects_bad_precision():
    from spann3r_b200 import _lib as L
    from spann3r_b200 import engine as E   # noqa: F401  (registers the engine prototypes)
    w = E.ModelW()
    assert not L.lib().s3r_engine_create_ex(C.byref(w), 1, 224, 224, 2, 7)
    assert b"precision" in L.lib().s3r_last_error()


# ------------------------------------------------------------------------------------------------
# cs_hi
# ------------------------------------------------------------------------------------------------
def _cpu_packed(monkeypatch, sd, host_math):
    """PackedWeights on the CPU: the library's split kernel replaced by the same round-to-nearest-even split in torch."""
    from spann3r_b200 import _lib, engine as E

    def split(x, relu=False, out=None):
        hi = x.to(torch.bfloat16)
        lo = (x - hi.float()).to(torch.bfloat16)
        if out is None:
            return hi, lo
        out[0].copy_(hi)
        out[1].copy_(lo)
        return out

    monkeypatch.setattr(_lib, "split", split)
    monkeypatch.setattr(_lib, "require_device", lambda: None)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    return E.PackedWeights(sd, device="cpu", host_math=host_math)


def _folded_lins(s):
    yield s.enc[0].qkv
    yield s.enc[23].fc1
    yield s.dec[0].qkv
    yield s.dec[11].q
    yield s.dec[5].fc1
    yield s.val[0].qkv
    yield s.val[5].fc1


@pytest.mark.parametrize("host_math", [True, False], ids=["host", "device_refresh"])
def test_cs_hi_is_the_row_sum_of_the_packed_hi_plane(monkeypatch, host_math):
    sd = get_state_dict(True)
    pw = _cpu_packed(monkeypatch, sd, host_math)
    if not host_math:    # the training path re-packs in place: check the refreshed buffers
        sd2 = {k: (v * 1.01 if k.endswith("norm1.weight") else v) for k, v in sd.items()}
        pw.refresh(sd2)
    by_ptr = {t.data_ptr(): t for t in pw._keep}
    for lin in _folded_lins(pw.struct):
        hi, cs, cs_hi = by_ptr[lin.w.hi], by_ptr[lin.cs], by_ptr[lin.cs_hi]
        hi2 = hi.reshape(cs.numel(), -1).double()
        lo2 = by_ptr[lin.w.lo].reshape(cs.numel(), -1).double()
        assert torch.equal(cs_hi, hi2.sum(dim=1).float())
        assert torch.equal(cs, (hi2 + lo2).sum(dim=1).float())
        assert not torch.equal(cs, cs_hi)


# ------------------------------------------------------------------------------------------------
# emulation oracle
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cfg1():
    from spann3r_b200 import synth
    sd = {k: v.double() for k, v in get_state_dict(False).items()}
    frames = [{"img": f["img"].double()} for f in synth.make_frames(2, 224, 224)]
    return sd, frames


def test_emulation_without_rounding_is_the_fp64_oracle(cfg1):
    from oracle import bf16_oracle, spann3r_oracle as orc
    sd, frames = cfg1
    ref, ref_all = orc.forward(sd, frames)
    got, got_all = bf16_oracle.forward(sd, frames, rounding=False)
    worst = 0.0
    for a, b in zip(got + [r2 for _, r2 in got_all], ref + [r2 for _, r2 in ref_all]):
        assert a.keys() == b.keys()
        for k in a:
            worst = max(worst, rel_l2(a[k], b[k]))
    print(f"emulation without rounding vs fp64 oracle: {worst:.2e}")
    assert worst < 1e-12


def test_emulation_with_rounding_shows_the_format_error(cfg1):
    """The bf16 emulation against the reference's own outputs (cfg1_224_2f_raw): the error is the format's, well above
    the fp32-grade 2e-5 of the default path."""
    from oracle import bf16_oracle
    sd, frames = cfg1
    g = np.load(f"{GOLDEN}/cfg1_224_2f_raw.npz")
    s = int(g["meta/px_stride"])
    preds, preds_all = bf16_oracle.forward(sd, frames, rounding=True)
    errs = {}
    for i, p in enumerate(preds):
        for k, v in p.items():
            errs[f"preds/{i}/{k}"] = rel_l2(v[:, ::s, ::s], g[f"preds/{i}/{k}"])
    for i, (_, r2) in enumerate(preds_all):
        for k, v in r2.items():
            errs[f"preds_all/{i}/res2/{k}"] = rel_l2(v[:, ::s, ::s], g[f"preds_all/{i}/res2/{k}"])
    for k, e in errs.items():
        print(f"bf16 emulation vs cfg1_224_2f_raw {k}: {e:.2e}")
    assert all(np.isfinite(e) for e in errs.values())
    assert max(e for k, e in errs.items() if "pts3d" in k) > 1e-4


def test_bf16_rounds_from_fp32_to_nearest_even():
    from oracle.bf16_oracle import bf16
    x = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 1.0 + 2 ** -8 + 2 ** -30], dtype=torch.float64)
    # ties to even; the fp64 excess below fp32 precision is dropped first (fp32 -> bf16, as the planes are written)
    assert bf16(x).tolist() == [1.0, 1.0 + 2 ** -6, 1.0]
