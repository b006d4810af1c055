"""The opt-in bf16 precision on the GPU: one tensor-core product per GEMM in encode, decode, keyheads and value.

Op level: s3r_gemm with precision = 1 (a_lo / b_lo NULL) against fp64 hi(A) hi(B)^T with the same epilogue -- held to the
split kernel's bar against its own fp64 product (3e-5; 3e-4 for the tf32-rounded EPI_QKV outputs) -- and more than 1e-4 away
from fp64 A B^T, which shows that one product is what ran.  Repeated calls are bitwise equal.

Stage level: each stage of a bf16 engine on the fp64 oracle's stage input rounded to fp32 (as test_stages_gpu.py builds
them), against the fp64 truth (oracle.spann3r_oracle) and the fp64 emulation of the format (oracle.bf16_oracle):
    |GPU - truth| <= 1.25 |emulation - truth|,   |GPU - emulation| <= 0.75 |emulation - truth|.
The first bar was fixed from the rounding analysis before any run and holds (measured 0.999-1.001 on an H100).  The
second bar was fixed at 0.25 on the assumption that the kernel's own error (fp32 accumulation order, one-pass LayerNorm
statistics, the tf32 attention cores: 1e-5 to 1e-4, test_stages_gpu.py) simply adds to the emulation's.  That analysis
was wrong: bf16 rounding is discontinuous, so a relative perturbation d of an operand the engine rounds does not move the
rounded value by d but flips about a fraction 2 d / u of the roundings by one ulp u = 2^-8, an RMS change of
sqrt(2 d / u) u against the rounding's own u / sqrt(12).  With d ~ 1e-4 (the tf32 attention output proj rounds) that is
0.2-0.8 of the format's error per operand, and the flips compound over the layers.  Measured on an H100 80GB HBM3 (700 W)
over the four geometries: decode 0.19-0.31, key heads 0.51-0.54, encode 0.52-0.56; value 0.46-0.55 and use_feat value
0.55-0.60 (512 x 384, 208 x 240).
Independent errors of equal size would give sqrt(2) = 1.41; a kernel that mis-rounded or dropped a product would give
|GPU - truth| well above the first bar, which is the one that bounds the accuracy.  The op-level tests hold the kernel
itself to 3e-5 of fp64 hi(A) hi(B)^T.
End to end: every frame's error against the reference's golden output is at most 1.5 times the emulation's (run in fp64 on
the GPU on the same frames).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, get_state_dict, rel_l2

pytestmark = pytest.mark.gpu

TOL_GEMM, TOL_QKV = 3e-5, 3e-4
ENGAGED = 1e-4


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _hi(t):
    return t.to(torch.bfloat16).double()


def _desc(L, ah, bh, groups, NB, H, W, kc, taps, n, **kw):
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = ah.data_ptr(), None, bh.data_ptr(), None   # the lo planes are never read
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, NB, H, W, kc, taps, n
    d.precision = L.PRECISION_BF16
    for k, v in kw.items():
        setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return d


def _conv(x, w, taps):
    """x [NB, H, W, K], w [N, taps, K] -> [NB, H, W, N] in fp64 (3x3 pad 1 for 9 taps)."""
    if taps == 1:
        return torch.einsum("bhwk,nk->bhwn", x, w[:, 0])
    N, K = w.shape[0], w.shape[2]
    return F.conv2d(x.permute(0, 3, 1, 2), w.view(N, 3, 3, K).permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1)


def _check(got, ref_hi, ref_full, tol, what):
    e_hi, e_full = rel_l2(got, ref_hi), rel_l2(got, ref_full)
    print(f"OP {what:40s} vs hi*hi {e_hi:.2e}  vs fp64 A*B {e_full:.2e}")
    assert e_hi < tol, (what, e_hi)
    assert e_full > ENGAGED, (what, e_full)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("act", ["none", "gelu", "relu"])
@pytest.mark.parametrize("G,NB,H,W,kc,taps,n", [
    (1, 1, 1, 700, 1024, 1, 1024),     # linear
    (2, 1, 1, 300, 200, 1, 96),        # ragged K (200 = 6 k-blocks + 8) and N (96: a partial tile at either width)
    (2, 2, 9, 13, 40, 9, 64),          # 3x3 conv, ragged K per tap
    (1, 1, 16, 16, 256, 9, 256),
])
def test_plain(L, bn, act, G, NB, H, W, kc, taps, n):
    x = _rand(G * NB, H, W, kc, seed=1)
    w = _rand(G * n, taps, kc, seed=2, scale=(taps * kc) ** -0.5)
    b = _rand(G * n, seed=3, scale=0.1)
    r = _rand(G * NB, H, W, n, seed=4, scale=0.1)
    xh = x.to(torch.bfloat16).contiguous()
    wh = w.reshape(G * n, taps * kc).to(torch.bfloat16).contiguous()
    out = torch.empty(G * NB, H, W, n, device="cuda")
    oh = torch.empty(out.shape, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    A = {"none": L.ACT_NONE, "gelu": L.ACT_GELU, "relu": L.ACT_RELU}[act]
    if act != "none":     # the engine's activated launches (fc1, key fc1, RCU conv1) take no residual
        r = torch.zeros_like(r)
    d = _desc(L, xh, wh, G, NB, H, W, kc, taps, n, epi=L.EPI_PLAIN, act=A, force_bn=bn, bias=b, out_f32=out, ldo=n,
              out_hi=oh, out_lo=ol, ldp=n, **({"res1": r, "ldr1": n} if act == "none" else {}))
    assert L.lib().s3r_gemm_tile_n(d) == bn
    L.gemm(d)
    first = out.clone()
    L.gemm(d)
    torch.cuda.synchronize()
    assert torch.equal(first, out), "repeated bf16 launches differ"
    fa = {"none": lambda t: t, "gelu": F.gelu, "relu": F.relu}[act]

    def ref(xd, wd):
        y = torch.stack([_conv(xd.view(G, NB, H, W, kc)[g], wd.view(G, n, taps, kc)[g], taps) for g in range(G)])
        return fa(y + b.double().view(G, 1, 1, 1, n)).reshape(out.shape) + r.double()

    r_hi, r_full = ref(_hi(x), _hi(w)), ref(x.double(), w.double())
    _check(out, r_hi, r_full, TOL_GEMM, f"plain {act} bn{bn} G{G} {H}x{W} k{kc} t{taps} n{n}")
    assert rel_l2(oh.double() + ol.double(), r_hi) < TOL_GEMM      # producers still write both planes


@pytest.mark.parametrize("bn", [64, 128])
def test_pixshuf(L, bn):
    """ConvTranspose2d(k = s = 2) as the DPT's act2_up launch: col (i, j, co) -> pixel (2h + i, 2w + j)."""
    G, NB, H, W, kc, s, cout = 2, 1, 6, 10, 192, 2, 96
    n = s * s * cout
    x = _rand(G * NB, H, W, kc, seed=11)
    w = _rand(G * n, 1, kc, seed=12, scale=kc ** -0.5)
    b = _rand(G * cout, seed=13, scale=0.1)
    oh = torch.empty(G * NB, H * s, W * s, cout, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    xh, wh = x.to(torch.bfloat16).contiguous(), w.reshape(G * n, kc).to(torch.bfloat16).contiguous()
    L.gemm(_desc(L, xh, wh, G, NB, H, W, kc, 1, n, epi=L.EPI_PIXSHUF, ps_s=s, ps_cout=cout, force_bn=bn, bias=b, out_hi=oh,
                 out_lo=ol, ldp=cout))
    torch.cuda.synchronize()

    def ref(xd, wd):
        y = torch.einsum("gbhwk,gnk->gbhwn", xd.view(G, NB, H, W, kc), wd.view(G, n, kc)).view(G, NB, H, W, s, s, cout)
        y = y + b.double().view(G, 1, 1, 1, 1, 1, cout)
        return y.permute(0, 1, 2, 4, 3, 5, 6).reshape(G * NB, H * s, W * s, cout)

    _check(oh.double() + ol.double(), ref(_hi(x), _hi(w)), ref(x.double(), w.double()), TOL_GEMM, f"pixshuf bn{bn}")


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("nb,ntok", [(1, 196), (2, 195)])
def test_qkv(L, bn, nb, ntok):
    """The encoder's qkv launch without RoPE: q scaled, k, V^T (padded to a multiple of 4), tf32-rounded."""
    C, heads, kc = 256, 4, 256
    pad = (ntok + 3) // 4 * 4
    x = _rand(nb * ntok, kc, seed=21)
    w = _rand(3 * C, kc, seed=22, scale=kc ** -0.5)
    b = _rand(3 * C, seed=23, scale=0.1)
    q = torch.empty(nb, heads, ntok, 64, device="cuda")
    k = torch.empty_like(q)
    vt = torch.zeros(nb, heads, 64, pad, device="cuda")
    L.gemm(_desc(L, x.to(torch.bfloat16).contiguous(), w.to(torch.bfloat16).contiguous(), 1, 1, 1, nb * ntok, kc, 1, 3 * C,
                 epi=L.EPI_QKV, force_bn=bn, bias=b, q_c=C, q_role_base=0, q_ntok=ntok, q_ntok_pad=pad, q_rope=0, q_nb=nb,
                 q_out=q, k_out=k, vt_out=vt, q_scale=0.125))
    torch.cuda.synchronize()

    def ref(xd, wd):
        y = (xd @ wd.T + b.double()).view(nb, ntok, 3, heads, 64)
        return y[:, :, 0].transpose(1, 2) * 0.125, y[:, :, 1].transpose(1, 2), y[:, :, 2].permute(0, 2, 3, 1)

    for name, got, rh, rf in zip("q k vt".split(), (q, k, vt[..., :ntok]), ref(_hi(x), _hi(w)), ref(x.double(), w.double())):
        _check(got, rh, rf, TOL_QKV, f"qkv {name} bn{bn} nb{nb} ntok{ntok}")


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("kc", [64, 128, 256, 768, 1024])
def test_folded_layernorm_uses_hi_column_sums(L, kc, bn):
    """rstd (acc - mean cs_hi) + b' with acc = hi(x) hi(W')^T: the column sums of the hi plane alone."""
    from spann3r_b200.engine import bf16_hi_rowsum, fold_layernorm
    from test_epilogue_gpu import _producer
    rows, n = 300, 512
    x, (xh, _), stats = _producer(L, 1, rows, kc, seed=31)
    w = _rand(n, kc, seed=32, scale=kc ** -0.5)
    b0 = _rand(n, seed=33, scale=0.1)
    gamma = 1 + _rand(kc, seed=34, scale=0.2)
    beta = _rand(kc, seed=35, scale=0.2)
    wf, bf = fold_layernorm(w, b0, gamma, beta)
    wh = wf.to(torch.bfloat16).contiguous()
    cs_hi = bf16_hi_rowsum(wf).contiguous()
    out = torch.empty(rows, n, device="cuda")
    L.gemm(_desc(L, xh, wh, 1, 1, 1, rows, kc, 1, n, epi=L.EPI_PLAIN, force_bn=bn, bias=bf, out_f32=out, ldo=n,
                 ln_stats=stats, ln_np=kc // 32, ln_eps=1e-6, ln_cs=cs_hi))
    torch.cuda.synchronize()
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = torch.rsqrt(xd.var(-1, unbiased=False, keepdim=True) + 1e-6)
    r_hi = rstd * (_hi(x) @ _hi(wf).T - mean * _hi(wf).sum(1)) + bf.double()
    r_full = F.layer_norm(xd, (kc,), gamma.double(), beta.double(), 1e-6) @ w.double().T + b0.double()
    _check(out, r_hi, r_full, TOL_GEMM, f"folded LN kc{kc} bn{bn}")


# ------------------------------------------------------------------------------------------------
# stage level
# ------------------------------------------------------------------------------------------------
GEOMS = [("224", 1, 224, 224), ("224_b2", 2, 224, 224), ("512x384", 1, 512, 384), ("208x240", 1, 208, 240)]
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    _MODELS.clear()
    torch.cuda.empty_cache()


def _model(use_feat=False):
    from spann3r_b200 import Spann3R, synth
    if use_feat not in _MODELS:
        m = Spann3R(dus3r_name=None, use_feat=use_feat)
        sd = synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True) if use_feat else get_state_dict(True)
        m.load_state_dict(sd, strict=True)
        _MODELS[use_feat] = (m.cuda().eval(), {k: v.double().cuda() for k, v in sd.items()})
    return _MODELS[use_feat]


def _ratio_check(gid, name, got, emu, truth):
    fmt = rel_l2(emu, truth)
    kern = rel_l2(got, emu)
    tot = rel_l2(got, truth)
    print(f"STAGE {gid:8s} {name:22s} |emu-truth| {fmt:.2e}  |gpu-emu| {kern:.2e} ({kern / fmt:.3f})  "
          f"|gpu-truth| {tot:.2e} ({tot / fmt:.3f})")
    assert bool(torch.isfinite(got).all()), (gid, name)
    assert tot <= 1.25 * fmt, (gid, name, tot, fmt)
    assert kern <= 0.75 * fmt, (gid, name, kern, fmt)


class Case:
    def __init__(self, gid, B, H, W):
        from oracle import spann3r_oracle as orc
        from oracle.bf16_oracle import Emu
        from spann3r_b200 import synth
        from spann3r_b200.engine import Engine
        self.gid, self.B, self.H, self.W = gid, B, H, W
        self.model, sd = _model()
        self.sd, self.emu = sd, Emu(sd)
        nimg = 2 * B + 1
        self.eng = Engine(self.model._weights(), B, H, W, max_images=nimg, precision="bf16")
        self.img = torch.cat([f["img"] for f in synth.make_frames(nimg, H, W, seed0=7)]).cuda().contiguous()
        with torch.no_grad():
            feats, pos = orc.encode_image(sd, self.img.double())
            self.ref_feats = feats
            self.f1, self.f2 = feats[:B].float().contiguous(), feats[B:2 * B].float().contiguous()
            self.p1, self.p2 = pos[:B], pos[B:2 * B]
            self.rdec1, self.rdec2 = orc.decoder(sd, self.f1.double(), self.p1, self.f2.double(), self.p2)
            self.edec1, self.edec2 = self.emu.decoder(self.f1.double(), self.p1, self.f2.double(), self.p2)
            self.r1 = orc.dpt_head(sd, "dust3r.downstream_head1", self.rdec1, H, W)
            self.rk1 = orc.key_head(sd, 1, self.f1.double(), self.rdec1[-1])


@pytest.fixture(scope="module", params=GEOMS, ids=[g[0] for g in GEOMS])
def case(request):
    c = Case(*request.param)
    yield c
    del c.eng
    torch.cuda.empty_cache()


def test_encode(case):
    feats = case.eng.encode(case.img)
    with torch.no_grad():
        emu, _ = case.emu.encode_image(case.img.double())
    for i in range(feats.shape[0]):
        _ratio_check(case.gid, f"encode img{i}", feats[i], emu[i], case.ref_feats[i])


def test_decode(case):
    dec = case.eng.decode(case.f1, case.f2, want_all=True)
    for l in range(12):
        for s, (edec, rdec) in enumerate(((case.edec1, case.rdec1), (case.edec2, case.rdec2))):
            _ratio_check(case.gid, f"decode l{l} s{s}", dec[l, s], edec[l + 1], rdec[l + 1])


def test_keyheads(case):
    from oracle import spann3r_oracle as orc
    case.eng.decode(case.f1, case.f2)
    k1, k2 = case.eng.keyheads(case.f1, case.f2)
    with torch.no_grad():
        e1 = case.emu.key_head(1, case.f1.double(), case.edec1[-1])
        e2 = case.emu.key_head(2, case.f2.double(), case.edec2[-1])
        r2 = orc.key_head(case.sd, 2, case.f2.double(), case.rdec2[-1])
    _ratio_check(case.gid, "keyheads head1", k1, e1, case.rk1)
    _ratio_check(case.gid, "keyheads head2", k2, e2, r2)


@pytest.mark.parametrize("rope", [False, True], ids=["norope", "rope"])
def test_value(case, rope):
    from oracle import spann3r_oracle as orc
    portrait = case.H > case.W
    pts = case.r1["pts3d"].float().contiguous()
    k1 = case.rk1.float().contiguous()
    got = case.eng.value(pts, k1, transposed=portrait, rope=rope)
    land = pts.double().swapaxes(1, 2) if portrait else pts.double()
    with torch.no_grad():
        truth = orc.encode_cur_value(case.sd, land, mem_pos_enc=rope) + k1.double()
        emu = case.emu.encode_cur_value(land, mem_pos_enc=rope) + k1.double()
    _ratio_check(case.gid, f"value {'rope' if rope else 'norope'}", got, emu, truth)


@pytest.mark.parametrize("rope", [False, True], ids=["norope", "rope"])
def test_value_usefeat(case, rope):
    from oracle import usefeat_oracle as ufo
    from oracle.bf16_oracle import Emu
    from spann3r_b200.engine import Engine
    m, sdu = _model(use_feat=True)
    eng = Engine(m._weights(), case.B, case.H, case.W, precision="bf16")
    tok = case.rdec1[-1].float().contiguous()
    k1 = case.rk1.float().contiguous()
    got = eng.value(tok, k1, rope=rope, tokens=True)
    with torch.no_grad():
        truth = ufo.encode_cur_value(sdu, tok.double(), case.p1, mem_pos_enc=rope) + k1.double()
        emu = Emu(sdu).encode_cur_value_usefeat(tok.double(), case.p1, mem_pos_enc=rope) + k1.double()
    del eng
    _ratio_check(case.gid, f"value_usefeat {'rope' if rope else 'norope'}", got, emu, truth)


# ------------------------------------------------------------------------------------------------
# isolation: which launches run at one product
# ------------------------------------------------------------------------------------------------
def _kinds(eng, fn):
    eng.profile(True)
    try:
        fn()
        kinds = [k for _, _, k in eng.profile_list()]
        eng.profile_read()
    finally:
        eng.profile(False)
    return kinds


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_only_the_four_stages_run_at_one_product(precision):
    from spann3r_b200 import synth
    from spann3r_b200.engine import Engine, MemoryBank
    m, _ = _model()
    B, H, W = 1, 224, 224
    eng = Engine(m._weights(), B, H, W, max_images=2, precision=precision)
    img = torch.cat([f["img"] for f in synth.make_frames(2, H, W)]).cuda().contiguous()
    one = 2 if precision == "bf16" else 0
    feats = None
    out = {}

    def enc():
        nonlocal feats
        feats = eng.encode(img)
    out["encode"] = _kinds(eng, enc)
    f1, f2 = feats[:1].contiguous(), feats[1:].contiguous()
    out["decode"] = _kinds(eng, lambda: eng.decode(f1, f2))
    ks = {}
    out["keyheads"] = _kinds(eng, lambda: ks.update(k=eng.keyheads(f1, f2)))
    hs = {}
    out["heads"] = _kinds(eng, lambda: hs.update(h=eng.heads()))
    k1 = ks["k"][0]
    pts = hs["h"][0][0].contiguous()
    v = {}
    out["value"] = _kinds(eng, lambda: v.update(v=eng.value(pts, k1)))
    bank = MemoryBank(B, 4 * eng.N, eng.device)
    eng.memory_append(bank, k1, v["v"])
    out["memory_read"] = _kinds(eng, lambda: eng.memory_read(bank, ks["k"][1], 5e-4))
    for stage, kinds in out.items():
        gemms = [k for k in kinds if k != 1]
        assert gemms, stage
        want = one if stage in ("encode", "decode", "keyheads", "value") else 0
        assert all(k == want for k in gemms), (precision, stage, kinds)
    print(precision, {s: sum(k == 2 for k in ks_) for s, ks_ in out.items()})


# ------------------------------------------------------------------------------------------------
# end to end
# ------------------------------------------------------------------------------------------------
E2E = [
    # golden, frames, H, W, use_feat
    ("cfg2_384x512_10f_sharp.npz", 10, 384, 512, False),
    ("seq_512x384_3f_sharp.npz", 3, 512, 384, False),
    ("seq_224_3f_sharp_usefeat.npz", 3, 224, 224, True),
]


def _frame_errs(preds, g):
    s = int(g["meta/px_stride"])
    errs = []
    for i, p in enumerate(preds):
        k = "pts3d" if "pts3d" in p else "pts3d_in_other_view"
        errs.append(rel_l2(p[k][:, ::s, ::s].float().cpu(), g[f"preds/{i}/{k}"]))
    return errs


@pytest.mark.parametrize("fname,nf,H,W,use_feat", E2E, ids=[e[0][:-4] for e in E2E])
def test_forward_vs_golden_within_the_format_error(fname, nf, H, W, use_feat):
    from oracle import bf16_oracle
    from spann3r_b200 import synth
    g = np.load(os.path.join(GOLDEN, fname))
    m, sd = _model(use_feat)
    frames = synth.make_frames(nf, H, W)
    m.set_precision("bf16")
    try:
        with torch.no_grad():
            preds, _ = m([{"img": f["img"].cuda()} for f in frames])
    finally:
        m.set_precision("fp32")
    got = _frame_errs(preds, g)
    emu_preds, _ = bf16_oracle.forward(sd, [{"img": f["img"].double().cuda()} for f in frames], use_feat=use_feat)
    emu = _frame_errs(emu_preds, g)
    for i, (a, b) in enumerate(zip(got, emu)):
        print(f"E2E {fname:32s} frame {i}: gpu bf16 {a:.2e}  emulation {b:.2e}  ratio {a / b:.3f}")
    assert all(np.isfinite(got))
    assert all(a <= 1.5 * b for a, b in zip(got, emu)), list(zip(got, emu))


def test_batch_lockstep_equals_single_runs():
    from spann3r_b200 import synth
    m, _ = _model()
    fa, fb = synth.make_frames(3, 224, 224, seed0=0), synth.make_frames(3, 224, 224, seed0=50)
    m.set_precision("bf16")
    try:
        with torch.no_grad():
            both, _ = m([{"img": torch.cat((a["img"], b["img"])).cuda()} for a, b in zip(fa, fb)])
            both = [{k: v.clone() for k, v in p.items()} for p in both]
            one_a, _ = m([{"img": a["img"].cuda()} for a in fa])
            one_a = [{k: v.clone() for k, v in p.items()} for p in one_a]
            one_b, _ = m([{"img": b["img"].cuda()} for b in fb])
    finally:
        m.set_precision("fp32")
    # Not bit-equal, as in fp32 mode (test_model_gpu.py): B = 2 and B = 1 pick different tiles, so fp32 sums differ in
    # the last bits -- and here a last-bit change can move a value across a bf16 rounding boundary (2^-8 relative for
    # that element), so the bar is the fp32 one's 1e-4 times 10.
    worst = 0.0
    for p2, pa, pb in zip(both, one_a, one_b):
        for k in p2:
            worst = max(worst, rel_l2(p2[k][0:1], pa[k]), rel_l2(p2[k][1:2], pb[k]))
    print(f"bf16 batched-vs-single worst rel-L2: {worst:.2e}")
    assert worst < 1e-3


def test_long_sequence_with_prunes_stays_finite():
    from spann3r_b200 import synth
    m, _ = _model()
    frames = synth.make_frames(30, 224, 224)
    m.set_precision("bf16")
    try:
        with torch.no_grad():
            preds, _, mem = m([{"img": f["img"].cuda()} for f in frames], return_memory=True)
    finally:
        m.set_precision("fp32")
    assert len(preds) == 30
    assert all(bool(torch.isfinite(v).all()) for p in preds for v in p.values())
    print("30-frame bf16 run: bank length", mem.bank.len)


def test_offline_and_pairwise_run_in_bf16():
    from spann3r_b200 import synth
    m, _ = _model()
    frames = [{"img": f["img"].cuda(), "idx": i} for i, f in enumerate(synth.make_frames(4, 224, 224))]
    m.set_precision("bf16")
    try:
        with torch.no_grad():
            r1, r2 = m.dust3r({"img": frames[0]["img"]}, {"img": frames[1]["img"]})
            assert (1, 224, 224, "bf16") in m._engines
            pairs = [(i, j) for i in range(4) for j in range(4) if i != j]
            p1, p2 = [], []
            for i, j in pairs:
                a, b = m.dust3r(frames[i], frames[j])
                p1.append(a["conf"][0].clone()); p2.append(b["conf"][0].clone())
            graph = {"view1": {"idx": [i for i, _ in pairs]}, "view2": {"idx": [j for _, j in pairs]},
                     "pred1": {"conf": p1}, "pred2": {"conf": p2}}
            preds, _, idx_used = m.offline_reconstruction(frames, graph)
    finally:
        m.set_precision("fp32")
    assert all(bool(torch.isfinite(v).all()) for v in list(r1.values()) + list(r2.values()))
    assert sorted(idx_used) == [0, 1, 2, 3]
    assert all(bool(torch.isfinite(v).all()) for p in preds for v in p.values())
