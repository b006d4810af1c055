"""CPU-side checks: state-dict layout of the drop-in module, C-ABI symbol table, host logic."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT


def test_state_dict_keys_match_reference(spec):
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None)
    sd = m.state_dict()
    assert list(sd.keys()) == list(spec["spann3r"].keys())          # same keys, same order as the reference
    for k, shape in spec["spann3r"].items():
        assert list(sd[k].shape) == shape, k
    # aliased DPT convs share storage, like the reference (dpt_block.py:59-65)
    a = sd["dust3r.downstream_head1.dpt.scratch.layer1_rn.weight"]
    b = sd["dust3r.downstream_head1.dpt.scratch.layer_rn.0.weight"]
    assert a.data_ptr() == b.data_ptr()


def test_strict_load_and_roundtrip(spec):
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None)
    sd = synth.make_state_dict(spec)
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    out = m.state_dict()
    for k in ("dust3r.enc_blocks.3.attn.qkv.weight", "norm_q.bias", "attn_head_2.2.weight"):
        assert torch.equal(out[k], sd[k])


def test_dust3r_checkpoint_ctor(tmp_path, spec):
    """Constructor path of the reference: Spann3R(dus3r_name=<DUSt3R ckpt file>) (spann3r/model.py:222)."""
    import argparse
    from spann3r_b200 import Spann3R, synth
    sd = synth.make_state_dict(spec, prefix="dust3r.")
    sd = {k: v for k, v in sd.items() if not k.startswith("dec_blocks2")}   # released ckpts lack dec_blocks2
    path = tmp_path / "fake_dust3r.pth"
    torch.save({"args": argparse.Namespace(model=synth.DUST3R_ARGS), "model": sd}, path)
    m = Spann3R(dus3r_name=str(path))
    assert torch.equal(m.dust3r.dec_blocks2._modules["0"].attn.qkv.weight, m.dust3r.dec_blocks._modules["0"].attn.qkv.weight)
    assert torch.equal(m.pos_patch_embed.proj.weight, m.dust3r.patch_embed.proj.weight)


def test_no_cpu_fallback(spec):
    from spann3r_b200 import Spann3R, synth
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    m = Spann3R(dus3r_name=None).eval()
    with pytest.raises(Exception):
        m(synth.make_frames(2, 64, 64))


def test_library_exports_every_declared_symbol():
    from spann3r_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "spann3r_b200.h")).read()
    declared = set(re.findall(r"\b(s3r_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 24
    for name in declared:
        assert hasattr(L, name), f"{name} declared in include/spann3r_b200.h but not exported"
    assert declared == set(_lib.declared_symbols()), declared ^ set(_lib.declared_symbols())
    assert L.s3r_version() == 100


def test_header_is_plain_c(tmp_path):
    """include/spann3r_b200.h is the drop-in boundary: it must compile as C99 on its own (cgo / JNI / ctypes-gen users)."""
    import subprocess
    src = tmp_path / "h.c"
    src.write_text('#include "spann3r_b200.h"\nint (*probe)(void) = s3r_version;\nint main(void) { return probe == 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)])


def test_rope_table_matches_reference_fallback():
    """engine.rope_cs_table == cos/sin of croco/models/pos_embed.py:120-129 (through the pinned oracle)."""
    from oracle.spann3r_oracle import rope_tables
    from spann3r_b200.engine import rope_cs_table
    cs = rope_cs_table(64)
    cos, sin = rope_tables(32, 64)
    assert torch.equal(cs[..., 0], cos[:, :16]) and torch.equal(cs[..., 1], sin[:, :16])


def test_ctypes_mirrors_match_the_compiled_structs():
    """The ctypes mirrors of s3r_gemm_desc / s3r_model_w / s3r_bank have the sizes the library was compiled with."""
    from spann3r_b200 import _lib, engine
    L = _lib.lib()
    assert L.s3r_abi_sizeof(0) == ctypes.sizeof(_lib.GemmDesc)
    assert L.s3r_abi_sizeof(1) == ctypes.sizeof(engine.ModelW)
    assert L.s3r_abi_sizeof(2) == ctypes.sizeof(engine.Bank)


def test_layernorm_fold_algebra():
    """engine.fold_layernorm + the epilogue formula of the folded LayerNorm (gemm_epilogue.cuh: per-row statistics
    from 32-column chunk sums, rstd * (acc - mean * colsum) + bias') reproduce Linear(LayerNorm(x)) of
    croco/models/blocks.py:127-130 -- restated here in fp64 / fp32 on the CPU."""
    from spann3r_b200.engine import fold_layernorm
    g = torch.Generator().manual_seed(0)
    C_, N_, R_ = 768, 96, 40
    x = torch.randn(R_, C_, generator=g) * 3 + 0.7          # non-zero mean: exercises the mean * colsum term
    w = torch.randn(N_, C_, generator=g) * C_ ** -0.5
    b = torch.randn(N_, generator=g)
    gamma = 1 + 0.2 * torch.randn(C_, generator=g)
    beta = 0.1 * torch.randn(C_, generator=g)
    ref = torch.nn.functional.linear(torch.nn.functional.layer_norm(x.double(), (C_,), gamma.double(), beta.double(), 1e-6),
                                     w.double(), b.double())
    wf, bf = fold_layernorm(w, b, gamma, beta)
    # producer epilogue: (sum, sum of squares) per 32-column chunk, fp32
    ch = x.view(R_, C_ // 32, 32)
    s1, s2 = ch.sum(-1), (ch * ch).sum(-1)
    mean = s1.sum(-1) / C_
    var = (s2.sum(-1) / C_ - mean * mean).clamp_min(0)
    rstd = torch.rsqrt(var + 1e-6)
    acc = x @ wf.t()                                        # the tensor-core GEMM on the raw stream (fp32 here)
    cs = wf.sum(dim=1)
    out = rstd[:, None] * acc - (rstd * mean)[:, None] * cs[None, :] + bf[None, :]
    err = float((out.double() - ref).norm() / ref.norm())
    assert err < 2e-6, err


# ------------------------------------------------------------------------------------------------------------------
# Host control flow of Spann3R.forward / offline_reconstruction over a FAKE engine (shapes only, no arithmetic): the
# frame loop, the dict keys / shapes of spann3r/model.py:473-539, the landscape views of portrait frames, which pointmap
# the value stage is handed, and the memory bookkeeping -- everything the Python layer decides, checked without a GPU.
# ------------------------------------------------------------------------------------------------------------------
class _FakeEngine:
    def __init__(self, B, H, W):
        self.B, self.H, self.W, self.N = B, H, W, (H // 16) * (W // 16)
        self.device, self.max_images, self.calls = torch.device("cpu"), 64, []

    def encode(self, img):
        self.calls.append(("encode", img.shape[0]))
        return torch.full((img.shape[0], self.N, 1024), 1.0) * img.mean(dim=(1, 2, 3))[:, None, None]

    def decode(self, f1, f2, want_all=False):
        assert f1.shape == f2.shape == (self.B, self.N, 1024)
        self.calls.append(("decode",))
        return torch.zeros(12, 2, self.B, self.N, 768) if want_all else None

    def keyheads(self, f1, f2):
        return f1 + 1, f2 + 2

    def heads(self):
        self.calls.append(("heads",))
        pts = torch.arange(2 * self.B * self.H * self.W * 3, dtype=torch.float32).view(2, self.B, self.H, self.W, 3)
        return pts, torch.ones(2, self.B, self.H, self.W) * 2

    def value(self, pts3d, feat_k1, transposed=False, rope=False):
        assert pts3d.is_contiguous() and pts3d.shape == (self.B, self.H, self.W, 3)     # head layout, never the view
        self.calls.append(("value", transposed, rope))
        return feat_k1 * 0

    def memory_read(self, bank, feat, thresh):
        self.calls.append(("read", bank.len))
        return feat

    def memory_append(self, bank, k, v):
        bank.len += self.N

    def check_sim(self, bank, feat_k, wm):
        return torch.zeros(self.B, wm)


def _fake_model(monkeypatch, mem_pos_enc=False):
    from spann3r_b200 import Spann3R
    from spann3r_b200 import model as M
    m = Spann3R(dus3r_name=None, mem_pos_enc=mem_pos_enc).eval()
    engines = {}

    def engine_for(B, H, W, n_frames=2, encode_only=False):
        return engines.setdefault((B, H, W), _FakeEngine(B, H, W))

    monkeypatch.setattr(m, "_engine_for", engine_for)
    monkeypatch.setattr(M.SpatialMemory, "check_sim_async", lambda self, feat_k, thresh=0.7: None)
    return m, engines


@pytest.mark.parametrize("H,W", [(64, 96), (96, 64)])
def test_forward_control_flow_on_a_fake_engine(monkeypatch, H, W):
    from spann3r_b200 import synth
    m, engines = _fake_model(monkeypatch, mem_pos_enc=(H > W))
    F_ = 5
    frames = synth.make_frames(F_, H, W)
    frames[0]["true_shape"] = torch.tensor([[H, W]], dtype=torch.int32)
    preds, preds_all, mem = m(frames, return_memory=True)
    eng = engines[(1, H, W)]
    lh, lw = min(H, W), max(H, W)
    assert len(preds) == F_ and len(preds_all) == F_ - 1
    assert set(preds[0]) == {"pts3d", "conf"}
    for p in preds[1:]:
        assert set(p) == {"pts3d_in_other_view", "conf"}
    for p in preds:
        for k, v in p.items():
            assert v.shape[:3] == (1, lh, lw), (k, v.shape)                      # always landscape (misc.py:66-94)
    # a portrait output is the axis-swapped VIEW of what the head wrote
    raw = eng.heads()[0]
    exp = raw[0].swapaxes(1, 2) if H > W else raw[0]
    assert torch.equal(preds[0]["pts3d"], exp)
    assert torch.equal(preds[-1]["pts3d_in_other_view"], raw[1].swapaxes(1, 2) if H > W else raw[1])
    assert preds_all[0][0] is preds[0] and preds_all[-1][1] is preds[-1]
    # one batched encode, then per step: (read from step 1 on) decode, heads, value with the right flags
    assert eng.calls[0] == ("encode", F_)
    steps = [c for c in eng.calls if c[0] in ("read", "decode", "value")]
    assert [c[0] for c in steps[:3]] == ["decode", "value", "read"]
    assert all(c == ("value", H > W, H > W) for c in steps if c[0] == "value")   # transposed read; rope = mem_pos_enc
    assert [c[1] for c in steps if c[0] == "read"] == [eng.N * i for i in range(1, F_ - 1)]
    assert mem.wm == F_ - 1 and mem.bank.len == eng.N * (F_ - 1) and mem.lm == 0
    assert mem.mem_k.shape == (1, eng.N * (F_ - 1), 1024) and mem.mem_count.shape == (1, eng.N * (F_ - 1), 1)
    # inconsistent inputs are rejected, not silently reshaped
    bad = synth.make_frames(2, H, W)
    bad[1]["true_shape"] = torch.tensor([[W, H]])
    with pytest.raises(NotImplementedError):
        m(bad)
    with pytest.raises(ValueError):
        m([synth.make_frames(1, H, W)[0], synth.make_frames(1, W, H)[0]])


def test_pairwise_and_offline_control_flow_on_a_fake_engine(monkeypatch):
    from spann3r_b200 import synth
    from spann3r_b200 import model as M
    H, W = 96, 64
    m, engines = _fake_model(monkeypatch)
    monkeypatch.setattr(M, "_conf_score", lambda c: c.mean())
    fr = synth.make_frames(4, H, W)
    r1, r2 = m.dust3r(fr[0], fr[1])
    assert set(r1) == {"pts3d", "conf"} and set(r2) == {"pts3d_in_other_view", "conf"}
    assert r1["pts3d"].shape == (1, W, H, 3) and r2["conf"].shape == (1, W, H)
    graph = {"view1": {"idx": [0, 1, 2, 3]}, "view2": {"idx": [1, 2, 3, 0]},
             "pred1": {"conf": torch.tensor([2.0, 5.0, 3.0, 2.5]).view(4, 1, 1).expand(4, 4, 4).contiguous()},
             "pred2": {"conf": torch.ones(4, 4, 4) * 2}}
    preds, preds_all, idx_used = m.offline_reconstruction(fr, graph)
    assert idx_used[:2] == [1, 2] and sorted(idx_used) == [0, 1, 2, 3]
    assert len(preds) == 4 and set(preds[0]) == {"pts3d", "conf"} and all("_raw" not in p for p in preds)
    assert all(v.shape[1:3] == (W, H) for p in preds for v in p.values())
    eng = engines[(1, H, W)]
    assert all(c == ("value", True, False) for c in eng.calls if c[0] == "value")


def test_prototype_table_matches_the_header():
    """Every function declared in include/spann3r_b200.h is bound in Python with the same number of arguments and the same
    scalar kinds (pointer / int / int64 / uint64 / float / double / size_t) -- guards the ctypes layer against ABI drift."""
    import ctypes as C
    from spann3r_b200 import _lib
    header = open(os.path.join(ROOT, "include", "spann3r_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", " ", header, flags=re.S)
    header = re.sub(r"^\s*#.*$", " ", header, flags=re.M)
    protos = _lib._PROTOS

    def kind_c(t):
        t = t.strip()
        if "*" in t:
            return "ptr"
        t = re.sub(r"\bconst\b", "", t).split()
        t = " ".join(t[:-1]) if len(t) > 1 else t[0]          # drop the parameter name
        return {"int": "i32", "int32_t": "i32", "int64_t": "i64", "long long": "i64", "uint64_t": "u64", "float": "f32",
                "double": "f64", "size_t": "u64", "void": "void", "unsigned": "u32", "uint32_t": "u32"}[t]

    def kind_py(t):
        if t is None:
            return "void"
        if t in (C.c_void_p, C.c_char_p) or (isinstance(t, type) and issubclass(t, (C._Pointer,))):
            return "ptr"
        return {C.c_int: "i32", C.c_int64: "i64", C.c_longlong: "i64", C.c_uint64: "u64", C.c_float: "f32",
                C.c_double: "f64", C.c_size_t: "u64", C.c_uint: "u32"}[t]      # LP64: size_t is uint64

    found = 0
    for m in re.finditer(r"([A-Za-z_][\w\s\*]*?)\b(s3r_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", header):
        ret, name, args = m.group(1), m.group(2), m.group(3)
        assert name in protos, name
        res, argtypes = protos[name]
        c_args = [] if args.strip() in ("", "void") else [kind_c(a) for a in args.split(",")]
        assert len(c_args) == len(argtypes), (name, c_args, argtypes)
        assert c_args == [kind_py(t) for t in argtypes], (name, c_args, [kind_py(t) for t in argtypes])
        rk = "ptr" if "*" in ret else kind_c(ret.strip() + " x")
        assert rk == kind_py(res), (name, rk, res)
        found += 1
    assert found == len(protos), (found, len(protos))


def test_c_abi_rejects_bad_arguments_without_touching_the_device():
    """Argument validation of the C ABI happens before any CUDA call: status < 0 (or NULL / 0) plus a message from
    s3r_last_error(), no exception, no crash -- checked here without a GPU."""
    import ctypes as C
    from spann3r_b200 import _lib, engine
    L = _lib.lib()
    assert L.s3r_pnp_workspace_bytes(0, 100) == 0 and L.s3r_pnp_workspace_bytes(2, 100) > 2 * 400 * 96
    assert L.s3r_pnp_ransac(None, None, 1, 100, 10, 1.0, 1.0, 0.0, 0.0, 8.0, 100, 15, 0, None, None, None, None) == -1
    assert b"pnp_ransac" in L.s3r_last_error()
    assert L.s3r_focal_median(None, 1, 8, 8, 4.0, 4.0, 0.0, 1.0, None, None, None) == -1
    assert L.s3r_focal_weiszfeld(None, 0, 8, 8, 4.0, 4.0, 10, 0.0, 1.0, None, None, None) == -1
    assert not L.s3r_engine_create(None, 1, 224, 224, 2)
    w = engine.ModelW()
    assert not L.s3r_engine_create(C.byref(w), 1, 100, 224, 2)            # height not a multiple of 16
    assert b"multiples of 16" in L.s3r_last_error()
    assert not L.s3r_engine_create(C.byref(w), 0, 224, 224, 2)


def test_only_checkers_touch_the_oracle():
    """oracle/ is test infrastructure: nothing in the product package or in tools/ may import it; bench.py may, in its
    baseline legs only (run_reference, cpu_baseline, reference_eager_gpu), and __graft_entry__.smoke() as the checker."""
    import glob
    pat = re.compile(r"^\s*(from\s+oracle\b|import\s+oracle\b)", re.M)
    for path in glob.glob(os.path.join(ROOT, "spann3r_b200", "**", "*.py"), recursive=True) + glob.glob(os.path.join(ROOT, "tools", "*.py")):
        assert not pat.search(open(path).read()), f"{path} imports the oracle"
    for path in glob.glob(os.path.join(ROOT, "spann3r_b200", "csrc", "*")):
        assert "oracle" not in open(path).read(), path
    bench = open(os.path.join(ROOT, "bench.py")).read()
    timed = bench[bench.index("# ---- timed: inputs resident in HBM"): bench.index("# ---- roofline leg")]
    assert "oracle" not in timed and "orc." not in timed           # never inside the measured regions
    # the two port fallbacks of the baseline legs (CPU leg, eager-GPU leg) when the staged reference is absent
    assert len(pat.findall(bench)) == 2
    for path in glob.glob(os.path.join(ROOT, "baseline", "*.py")):
        assert not pat.search(open(path).read()), f"{path} imports the oracle"
    entry = open(os.path.join(ROOT, "__graft_entry__.py")).read()
    assert pat.search(entry[entry.index("def smoke"):])
    # build() runs the reference peer's build recipe (oracle/stage_reference.py) and nothing else of oracle/
    head = entry[: entry.index("def smoke")]
    assert re.findall(r"^\s*((?:from|import)\s+oracle\b.*)$", head, re.M) == ["from oracle import stage_reference as sr"]


def test_reference_style_init_and_zero_fill(tmp_path, spec):
    """ADVICE r1: parameters are never uninitialised memory.  Without a DUSt3R checkpoint they are zero-filled (the
    caller loads a full Spann3R state dict); with one, the keys it does not cover get the reference constructors' default
    init (LayerNorm 1 / 0, Linear kaiming-uniform), as spann3r/model.py:228-261 leaves them."""
    import argparse
    from spann3r_b200 import Spann3R, synth
    m0 = Spann3R(dus3r_name=None)
    assert all(float(p.abs().max()) == 0.0 for p in m0.parameters())
    sd = synth.make_state_dict(spec, prefix="dust3r.")
    path = tmp_path / "dust3r.pth"
    torch.save({"args": argparse.Namespace(model=synth.DUST3R_ARGS), "model": sd}, path)
    m = Spann3R(dus3r_name=str(path))
    assert torch.all(m.norm_q.weight == 1) and torch.all(m.norm_q.bias == 0)
    assert torch.all(m.value_norm.weight == 1) and torch.all(getattr(m.value_encoder, "0").norm1.bias == 0)
    w = getattr(m.attn_head_1, "0").weight
    assert float(w.std()) > 0 and float(w.abs().max()) <= 1.0 / (1792 ** 0.5) + 1e-6      # kaiming_uniform(a=sqrt 5): +-1/sqrt(fan_in)
    assert float(m.value_out.bias.abs().max()) <= 1.0 / (1024 ** 0.5) + 1e-6 and float(m.value_out.bias.std()) > 0
    assert torch.equal(m.pos_patch_embed.proj.weight, m.dust3r.patch_embed.proj.weight)   # spann3r/model.py:240-241


def test_packed_weights_are_invalidated_by_loads_and_moves(spec):
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None)
    assert m._packed_dirty
    m._packed_dirty = False
    m.load_state_dict(synth.make_state_dict(spec), strict=True)
    assert m._packed_dirty
    m._packed_dirty = False
    m.float()
    assert m._packed_dirty
    m._packed_dirty = False
    m.dust3r.load_state_dict({k[len("dust3r."):]: v for k, v in m.state_dict().items() if k.startswith("dust3r.")})
    assert m._packed_dirty
    m._packed_dirty = False
    m.invalidate_packed()
    assert m._packed_dirty


def test_decoder_takes_the_grid_from_the_positions(monkeypatch):
    """ADVICE r1: `_decoder(f1, pos1, f2, pos2)` used hidden state for (H, W); 768 tokens are 24 x 32 or 32 x 24 and only
    the positions tell which (the reference's RoPE is position-driven, croco/models/blocks.py:94-112)."""
    m, engines = _fake_model(monkeypatch)

    class _Dec(_FakeEngine):
        def decode(self, f1, f2, want_all=False):
            return torch.zeros(12, 2, self.B, self.N, 768)
    eng_for = m._engine_for
    monkeypatch.setattr(m, "_engine_for", lambda B, H, W, **k: engines.setdefault((B, H, W), _Dec(B, H, W)))
    for gh, gw in ((4, 6), (6, 4)):
        pos = torch.cartesian_prod(torch.arange(gh), torch.arange(gw))[None]
        f = torch.zeros(1, gh * gw, 1024)
        m.dust3r._decoder(f, pos, f, pos)
        assert (1, 16 * gh, 16 * gw) in engines
    with pytest.raises(RuntimeError, match="positions"):
        m.dust3r._decoder(f, None, f, None)
    with pytest.raises(RuntimeError, match="patch grids"):
        m.dust3r._decoder(torch.zeros(1, 20, 1024), pos, torch.zeros(1, 20, 1024), pos)


def test_dropout_mask_rejects_a_null_output_without_a_device():
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_dropout_mask(None, 4, 1, 0.15, None) == -1 and b"dropout_mask" in L.s3r_last_error()
