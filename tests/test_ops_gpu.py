"""GPU parity of the op-level C ABI (s3r_gemm / s3r_attention / elementwise) against fp64 PyTorch math.

Tolerances: the split-bf16 scheme carries ~16 mantissa bits per operand, so a K-long dot product is
good to ~2^-16/sqrt-ish relative; we hold every GEMM-like op to 3e-5 relative L2 (SURVEY.md §7.3-#1
measured 2-5e-5 end to end) and tf32 attention to 5e-4 (measured <= 2e-4 in the survey).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu

TOL_GEMM = 3e-5
TOL_ATTN = 5e-4


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def test_split_roundtrip(L):
    x = _rand(1000, 768, seed=1)
    hi, lo = L.split(x)
    torch.cuda.synchronize()
    assert rel_l2(hi.double() + lo.double(), x.double()) < 1e-5
    assert torch.equal(hi, x.to(torch.bfloat16))


@pytest.mark.parametrize("rows,K,N,groups,bn", [
    (768, 1024, 3072, 1, 0), (768, 1024, 1024, 1, 0), (768, 4096, 1024, 1, 0), (196, 768, 2304, 1, 0),
    (300, 96, 1536, 1, 0), (768, 768, 768, 2, 0), (768, 1792, 1792, 2, 0),
    (1000, 512, 512, 1, 64), (1000, 512, 512, 1, 96), (1000, 512, 512, 1, 128), (7680, 1024, 1024, 1, 0),
    (130, 64, 32, 1, 0),
    # forced widths on the model's shapes
    (768, 1024, 3072, 1, 128), (768, 1024, 3072, 1, 64), (768, 768, 768, 2, 128), (7680, 1024, 1024, 1, 128),
    (1536, 768, 96, 1, 128), (768, 4096, 1024, 1, 128),
    (768, 768, 768, 2, 64), (768, 3072, 768, 2, 64), (768, 1024, 1024, 1, 64), (768, 4096, 1024, 1, 64),
    (1536, 768, 96, 1, 64), (512, 96, 1536, 1, 64),
    # K-heavy shapes with few tiles (value-encoder fc2, decoder fc2, tiny-M long-K)
    (768, 4096, 1024, 1, 0), (768, 3072, 768, 2, 0), (256, 6912, 768, 2, 0), (196, 1024, 1024, 1, 0),
])
def test_linear_bias_gelu_residual(L, rows, K, N, groups, bn):
    x = _rand(groups * rows, K, seed=2)
    w = _rand(groups * N, K, seed=3, scale=K ** -0.5)
    b = _rand(groups * N, seed=4, scale=0.1)
    r = _rand(groups * rows, N, seed=5)
    xp, wp = L.split(x), L.split(w)
    out, oh, ol = L.linear(xp, wp, bias=b, act=L.ACT_GELU, res=r, want_f32=True, want_planes=True, groups=groups,
                           force_bn=bn)
    torch.cuda.synchronize()
    xd, wd = x.double().view(groups, rows, K), w.double().view(groups, N, K)
    ref = F.gelu(torch.einsum("grk,gnk->grn", xd, wd) + b.double().view(groups, 1, N)) + r.double().view(groups, rows, N)
    ref = ref.reshape(groups * rows, N)
    assert rel_l2(out, ref) < TOL_GEMM, rel_l2(out, ref)
    assert rel_l2(oh.double() + ol.double(), ref) < TOL_GEMM


@pytest.mark.parametrize("NB,H,W,Cin,Cout,groups,bn", [
    (1, 12, 16, 256, 256, 2, 0), (1, 24, 32, 96, 256, 1, 0), (2, 7, 7, 256, 256, 1, 0), (1, 96, 128, 256, 128, 2, 0),
    (1, 14, 14, 384, 256, 1, 0), (1, 48, 64, 192, 256, 1, 0), (1, 12, 16, 768, 256, 2, 0),
    # forced widths on a 3x3 conv
    (1, 96, 128, 256, 256, 2, 128), (1, 96, 128, 256, 128, 1, 128), (2, 24, 32, 96, 256, 1, 128),
    (1, 24, 32, 96, 256, 1, 64), (1, 96, 128, 256, 128, 2, 64),
])
def test_conv3x3(L, NB, H, W, Cin, Cout, groups, bn):
    x = _rand(groups * NB, Cin, H, W, seed=6)
    w = _rand(groups * Cout, Cin, 3, 3, seed=7, scale=(9 * Cin) ** -0.5)
    b = _rand(groups * Cout, seed=8, scale=0.1)
    res = _rand(groups * NB, H, W, Cout, seed=9)
    xh, xl = L.split(x.permute(0, 2, 3, 1).contiguous())                    # NHWC planes
    wh, wl = L.split(w.permute(0, 2, 3, 1).contiguous().view(groups * Cout, 9 * Cin))  # [N, tap, Cin]
    out = torch.empty(groups * NB, H, W, Cout, device="cuda")
    oh = torch.empty(out.shape, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, NB, H, W, Cin, 9, Cout
    d.epi, d.act, d.plane_relu, d.force_bn = L.EPI_PLAIN, L.ACT_NONE, 1, bn
    d.bias = b.data_ptr()
    d.res1, d.ldr1 = res.data_ptr(), Cout
    d.out_f32, d.ldo = out.data_ptr(), Cout
    d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), Cout
    L.gemm(d)
    torch.cuda.synchronize()
    xd = x.double().view(groups, NB, Cin, H, W)
    wd = w.double().view(groups, Cout, Cin, 3, 3)
    bd = b.double().view(groups, Cout)
    ref = torch.stack([F.conv2d(xd[g], wd[g], bd[g], padding=1) for g in range(groups)]).reshape(groups * NB, Cout, H, W)
    ref = ref.permute(0, 2, 3, 1) + res.double()
    assert rel_l2(out, ref) < TOL_GEMM, rel_l2(out, ref)
    assert rel_l2(oh.double() + ol.double(), ref.clamp_min(0)) < TOL_GEMM


@pytest.mark.parametrize("H,W,C,s", [(24, 32, 96, 4), (24, 32, 192, 2), (14, 14, 96, 4)])
def test_conv_transpose_pixshuf(L, H, W, C, s):
    groups, NB = 2, 1
    x = _rand(groups * NB, C, H, W, seed=10)
    w = _rand(groups, C, C, s, s, seed=11, scale=C ** -0.5)   # ConvTranspose2d weight [in, out, kh, kw]
    b = _rand(groups * C, seed=12, scale=0.1)
    xh, xl = L.split(x.permute(0, 2, 3, 1).contiguous())
    # B[(i, j, co), ci] = w[ci, co, i, j]
    wb = w.permute(0, 3, 4, 2, 1).contiguous().view(groups * s * s * C, C)
    wh, wl = L.split(wb)
    out = torch.empty(groups * NB, H * s, W * s, C, device="cuda")
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, NB, H, W, C, 1, s * s * C
    d.epi, d.ps_s, d.ps_cout = L.EPI_PIXSHUF, s, C
    d.bias = b.data_ptr()
    d.out_f32, d.ldo = out.data_ptr(), C
    L.gemm(d)
    torch.cuda.synchronize()
    xd = x.double().view(groups, NB, C, H, W)
    ref = torch.stack([F.conv_transpose2d(xd[g], w[g].double(), b.double().view(groups, C)[g], stride=s)
                       for g in range(groups)]).reshape(groups * NB, C, H * s, W * s).permute(0, 2, 3, 1)
    assert rel_l2(out, ref) < TOL_GEMM, rel_l2(out, ref)


def _cs_table(maxpos=64):
    from oracle.spann3r_oracle import rope_tables
    cos, sin = rope_tables(32, maxpos)           # [maxpos, 32] (two identical halves)
    return torch.stack((cos[:, :16], sin[:, :16]), dim=-1).contiguous().cuda()  # [maxpos,16,2]


@pytest.mark.parametrize("B,gh,gw,heads,groups", [(1, 24, 32, 16, 1), (2, 14, 14, 12, 1), (1, 24, 32, 12, 2), (1, 5, 9, 2, 1)])
def test_qkv_rope_attention(L, B, gh, gw, heads, groups):
    """QKV projection with the fused RoPE/head-split epilogue, then the wgmma attention core,
    against croco/models/blocks.py:94-112 evaluated in fp64 (through the pinned oracle's rope2d)."""
    from oracle.spann3r_oracle import rope2d
    C = heads * 64
    N = gh * gw
    npad = (N + 3) // 4 * 4
    x = _rand(groups * B * N, C, seed=13)
    w = _rand(groups * 3 * C, C, seed=14, scale=C ** -0.5)
    b = _rand(groups * 3 * C, seed=15, scale=0.1)
    pos = torch.cartesian_prod(torch.arange(gh), torch.arange(gw)).view(1, N, 2).expand(groups * B, N, 2).contiguous()
    pos32 = pos.to(torch.int32).cuda()
    cs = _cs_table()
    xp, wp = L.split(x), L.split(w)
    q = torch.empty(groups * B, heads, N, 64, device="cuda")
    k = torch.empty_like(q)
    vt = torch.zeros(groups * B, heads, 64, npad, device="cuda")
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, 1, 1, B * N, C, 1, 3 * C
    d.epi = L.EPI_QKV
    d.bias = b.data_ptr()
    d.q_c, d.q_role_base, d.q_ntok, d.q_ntok_pad, d.q_rope, d.q_nb = C, 0, N, npad, 1, B
    d.q_pos, d.q_cs = pos32.data_ptr(), cs.data_ptr()
    d.q_out, d.k_out, d.vt_out, d.q_scale = q.data_ptr(), k.data_ptr(), vt.data_ptr(), 0.125
    L.gemm(d)
    o = torch.empty(groups * B * N, C, device="cuda")
    oh = torch.empty(o.shape, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    L.check(L.lib().s3r_attention(L.ptr(q), L.ptr(k), L.ptr(vt), groups * B * heads, heads, N, N, npad, L.ptr(oh),
                                  L.ptr(ol), L.ptr(o), C, L.stream_ptr()), "s3r_attention")
    torch.cuda.synchronize()
    # fp64 reference
    xd = x.double().view(groups, B, N, C)
    wd = w.double().view(groups, 3 * C, C)
    qkv = torch.einsum("gbnc,gkc->gbnk", xd, wd) + b.double().view(groups, 1, 1, 3 * C)
    qkv = qkv.reshape(groups * B, N, 3, heads, 64).transpose(1, 3)
    qr, kr, vr = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    posd = pos.cuda()
    qr, kr = rope2d(qr, posd), rope2d(kr, posd)
    assert rel_l2(q, qr * 0.125) < 3e-4   # tf32-rounded
    assert rel_l2(k, kr) < 3e-4
    assert rel_l2(vt[..., :N], vr.transpose(-1, -2)) < 3e-4
    att = ((qr @ kr.transpose(-2, -1)) * 0.125).softmax(-1)
    ref = (att @ vr).transpose(1, 2).reshape(groups * B * N, C)
    assert rel_l2(o, ref) < TOL_ATTN, rel_l2(o, ref)
    assert rel_l2(oh.double() + ol.double(), ref) < TOL_ATTN


@pytest.mark.parametrize("BH,heads,nq,nk", [
    (6, 3, 196, 300),
    # many-wave launches (one CTA per 128-query tile and head): full / ragged key blocks, ragged last query tile, a
    # single key block.  tests/test_attention_core_gpu.py holds the kernel to a per-element bound.
    (96, 16, 768, 768), (128, 16, 512, 300), (160, 16, 700, 768), (256, 16, 256, 100),
])
def test_cross_attention_shapes(L, BH, heads, nq, nk):
    """nq != nk and non-multiple-of-128 sizes through the attention core alone."""
    def tf32(x):  # the kernel's contract: operands already rounded to tf32 (done by the QKV epilogue)
        return ((x.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    q = tf32(_rand(BH, nq, 64, seed=20, scale=0.3))
    k = tf32(_rand(BH, nk, 64, seed=21))
    v = tf32(_rand(BH, nk, 64, seed=22))
    vt = v.transpose(1, 2).contiguous()
    o = torch.empty(BH // heads * nq, heads * 64, device="cuda")
    L.check(L.lib().s3r_attention(L.ptr(q), L.ptr(k), L.ptr(vt), BH, heads, nq, nk, nk, None, None, L.ptr(o),
                                  heads * 64, L.stream_ptr()), "s3r_attention")
    torch.cuda.synchronize()
    att = (q.double() @ k.double().transpose(1, 2)).softmax(-1) @ v.double()          # [BH, nq, 64]
    ref = att.view(BH // heads, heads, nq, 64).transpose(1, 2).reshape(-1, heads * 64)
    assert rel_l2(o, ref) < TOL_ATTN, rel_l2(o, ref)


@pytest.mark.parametrize("H,W,bn", [(48, 64, 0), (48, 64, 128), (24, 40, 0), (96, 128, 0)])
def test_head_tail(L, H, W, bn):
    """The DPT head tail runs 128 wide whatever force_bn asks (the two column halves' partial dot products meet in
    shared memory): bn 0 and 128 give the same launch."""
    groups, NB, Cin = 2, 1, 128
    x = _rand(groups * NB, Cin, H, W, seed=30)
    w = _rand(groups * 128, Cin, 3, 3, seed=31, scale=(9 * Cin) ** -0.5)
    b = _rand(groups * 128, seed=32, scale=0.1)
    w4 = _rand(groups, 4, 128, seed=33, scale=128 ** -0.5)
    b4 = _rand(groups, 4, seed=34, scale=0.1)
    xh, xl = L.split(x.permute(0, 2, 3, 1).contiguous())
    wh, wl = L.split(w.permute(0, 2, 3, 1).contiguous().view(groups * 128, 9 * Cin))
    pts = torch.empty(groups * NB, H, W, 3, device="cuda")
    conf = torch.empty(groups * NB, H, W, device="cuda")
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, NB, H, W, Cin, 9, 128
    d.epi, d.act, d.force_bn = L.EPI_HEADTAIL, L.ACT_RELU, bn
    d.bias = b.data_ptr()
    d.ht_w, d.ht_b, d.ht_pts, d.ht_conf = w4.data_ptr(), b4.data_ptr(), pts.data_ptr(), conf.data_ptr()
    L.gemm(d)
    torch.cuda.synchronize()
    from oracle.spann3r_oracle import postprocess
    for g in range(groups):
        y = F.conv2d(x[g:g + 1].double(), w[g * 128:(g + 1) * 128].double(), b[g * 128:(g + 1) * 128].double(), padding=1)
        y = F.conv2d(F.relu(y), w4[g].double().view(4, 128, 1, 1), b4[g].double())
        ref = postprocess(y)
        assert rel_l2(pts[g], ref["pts3d"][0]) < TOL_GEMM * 2
        assert rel_l2(conf[g], ref["conf"][0]) < TOL_GEMM


def test_layernorm_upsample_im2col_rope(L):
    x = _rand(500, 1024, seed=40)
    w, b = _rand(1024, seed=41), _rand(1024, seed=42)
    out, hi, lo = L.layernorm(x, w, b, 1e-6, want_f32=True, want_planes=True)
    ref = F.layer_norm(x.double(), (1024,), w.double(), b.double(), 1e-6)
    torch.cuda.synchronize()
    assert rel_l2(out, ref) < 2e-6
    assert rel_l2(hi.double() + lo.double(), ref) < 1e-5
    x7 = _rand(77, 768, seed=43)
    out7, _, _ = L.layernorm(x7, w[:768].contiguous(), b[:768].contiguous(), 1e-5)
    assert rel_l2(out7, F.layer_norm(x7.double(), (768,), w[:768].double(), b[:768].double(), 1e-5)) < 2e-6
    # upsample
    f = _rand(2, 12, 16, 256, seed=44)
    up = torch.empty(2, 24, 32, 256, device="cuda")
    L.check(L.lib().s3r_upsample2x(L.ptr(f), 2, 12, 16, 256, L.ptr(up), None, None, L.stream_ptr()), "upsample")
    ref = F.interpolate(f.permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    assert rel_l2(up, ref) < 1e-6
    # patch im2col (NCHW image)
    img = _rand(2, 3, 32, 48, seed=45)
    hi = torch.empty(2 * 2 * 3, 768, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty_like(hi)
    s = img.stride()
    L.check(L.lib().s3r_im2col_patch16(L.ptr(img), s[0], s[1], s[2], s[3], 2, 2, 3, L.ptr(hi), L.ptr(lo), L.stream_ptr()),
            "im2col")
    ref = F.unfold(img, kernel_size=16, stride=16).transpose(1, 2).reshape(-1, 768)
    torch.cuda.synchronize()
    assert rel_l2(hi.double() + lo.double(), ref) < 1e-5
    # rope shim == oracle rope2d
    from oracle.spann3r_oracle import rope2d
    tok = _rand(2, 50, 4, 64, seed=46)          # [B, N, H, D] as curope sees it
    pos = torch.randint(0, 32, (2, 50, 2), generator=torch.Generator().manual_seed(1)).cuda()
    exp = rope2d(tok.transpose(1, 2).double(), pos).transpose(1, 2)
    L.check(L.lib().s3r_rope2d_inplace(L.ptr(tok), L.ptr(pos), 100, 4, 64, 256, 64, 100.0, 1.0, L.stream_ptr()), "rope")
    torch.cuda.synchronize()
    assert rel_l2(tok, exp) < 1e-5


@pytest.mark.parametrize("rows,C,N,groups,swap,bn", [
    (768, 768, 2304, 2, 0, 0), (768, 768, 1536, 2, 1, 0), (768, 1024, 4096, 1, 0, 0), (196, 1024, 3072, 1, 0, 0),
    (7680, 1024, 3072, 1, 0, 0), (768, 768, 768, 2, 1, 128), (1000, 768, 768, 1, 0, 64),
    (768, 768, 768, 2, 1, 64), (768, 768, 2304, 2, 0, 64), (1024, 768, 768, 1, 0, 64),
])
def test_folded_layernorm_chain(L, rows, C, N, groups, swap, bn):
    """Producer GEMM (x = r + a W0^T + b0: writes x fp32, planes(x) and the per-row chunk statistics) followed by a
    consumer GEMM with the LayerNorm folded in (engine.fold_layernorm) == Linear(LayerNorm(x)) of
    croco/models/blocks.py:127-130 / :186-191 (a_swap: norm_y of the other stream, dust3r/model.py:197-199)."""
    from spann3r_b200.engine import fold_layernorm
    K0 = 256
    a = _rand(groups * rows, K0, seed=21)
    w0 = _rand(C, K0, seed=22, scale=K0 ** -0.5).repeat(groups, 1)
    b0 = _rand(groups * C, seed=23, scale=0.5) + 0.3
    r = _rand(groups * rows, C, seed=24, scale=2.0)
    x = torch.empty(groups * rows, C, device="cuda")
    xh = torch.empty(x.shape, dtype=torch.bfloat16, device="cuda")
    xl = torch.empty_like(xh)
    stats = torch.zeros(groups * rows, C // 32, 2, device="cuda")
    ap, w0p = L.split(a), L.split(w0.contiguous())
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = ap[0].data_ptr(), ap[1].data_ptr(), w0p[0].data_ptr(), w0p[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, 1, 1, rows, K0, 1, C
    d.epi = L.EPI_PLAIN
    d.bias = b0.data_ptr()
    d.res1, d.ldr1 = r.data_ptr(), C
    d.out_f32, d.ldo = x.data_ptr(), C
    d.out_hi, d.out_lo, d.ldp = xh.data_ptr(), xl.data_ptr(), C
    d.stats_out = stats.data_ptr()
    L.gemm(d)
    torch.cuda.synchronize()
    xd = x.double()
    ch = xd.view(groups * rows, C // 32, 32)
    assert rel_l2(stats[..., 0], ch.sum(-1)) < 1e-5
    assert rel_l2(stats[..., 1], (ch * ch).sum(-1)) < 1e-5

    w = _rand(groups * N, C, seed=25, scale=C ** -0.5)
    b = _rand(groups * N, seed=26, scale=0.1)
    gamma = 1 + 0.2 * _rand(groups, C, seed=27)
    beta = 0.1 * _rand(groups, C, seed=28)
    wf, bf = [], []
    for g in range(groups):
        f = fold_layernorm(w[g * N:(g + 1) * N], b[g * N:(g + 1) * N], gamma[g], beta[g])
        wf.append(f[0]); bf.append(f[1])
    wf, bf = torch.cat(wf).contiguous(), torch.cat(bf).contiguous()
    wp = L.split(wf)
    cs = (wp[0].double() + wp[1].double()).sum(1).float().contiguous()
    out = torch.empty(groups * rows, N, device="cuda")
    d2 = L.GemmDesc()
    d2.a_hi, d2.a_lo, d2.b_hi, d2.b_lo = xh.data_ptr(), xl.data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d2.groups, d2.nb, d2.h, d2.w, d2.kc, d2.taps, d2.n = groups, 1, 1, rows, C, 1, N
    d2.epi, d2.force_bn = L.EPI_PLAIN, bn
    d2.bias = bf.data_ptr()
    d2.out_f32, d2.ldo = out.data_ptr(), N
    d2.ln_stats, d2.ln_np, d2.ln_eps, d2.ln_cs, d2.a_swap = stats.data_ptr(), C // 32, 1e-6, cs.data_ptr(), swap
    L.gemm(d2)
    torch.cuda.synchronize()
    xg = xd.view(groups, rows, C)
    if swap:
        xg = xg.flip(0)
    ref = torch.stack([F.linear(F.layer_norm(xg[g], (C,), gamma[g].double(), beta[g].double(), 1e-6),
                                w[g * N:(g + 1) * N].double(), b[g * N:(g + 1) * N].double()) for g in range(groups)])
    ref = ref.reshape(groups * rows, N)
    assert rel_l2(out, ref) < TOL_GEMM, rel_l2(out, ref)
