"""The s3r_gemm epilogue modes and layout kernels the engine launches, each against fp64 PyTorch at op level.

Every grouped case gives the two groups different A rows, weights, biases, LayerNorm affines and RoPE positions, so that a
swapped group, a wrong role or positions read for the wrong group change the answer.  Tolerances: TOL_GEMM / TOL_ATTN
of test_ops_gpu.py, 3e-4 for the tf32-rounded q / k / V^T outputs of EPI_QKV."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2
from test_ops_gpu import TOL_ATTN, TOL_GEMM, _cs_table, _rand

pytestmark = pytest.mark.gpu

TOL_QKV = 3e-4


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _desc(L, a, w, groups, rows, kc, n, **kw):
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = a[0].data_ptr(), a[1].data_ptr(), w[0].data_ptr(), w[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, 1, 1, rows, kc, 1, n
    for k, v in kw.items():
        setattr(d, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return d


def _producer(L, groups, rows, C, seed, offset=None):
    """x = a W0^T + b0 + r (per-group W0, b0) through an EPI_PLAIN launch that writes x, planes(x) and the chunk
    statistics, as the engine's proj / cproj / fc2 launches do.  offset [groups*rows]: added to every column of a row."""
    K0 = 64
    a = _rand(groups * rows, K0, seed=seed)
    w0 = _rand(groups * C, K0, seed=seed + 1, scale=K0 ** -0.5)
    b0 = _rand(groups * C, seed=seed + 2, scale=0.5)
    r = _rand(groups * rows, C, seed=seed + 3)
    if offset is not None:
        r = r + offset[:, None]
    x = torch.empty(groups * rows, C, device="cuda")
    xh = torch.empty(x.shape, dtype=torch.bfloat16, device="cuda")
    xl = torch.empty_like(xh)
    stats = torch.empty(groups * rows, C // 32, 2, device="cuda")
    L.gemm(_desc(L, L.split(a), L.split(w0), groups, rows, K0, C, epi=L.EPI_PLAIN, bias=b0, res1=r, ldr1=C,
                 out_f32=x, ldo=C, out_hi=xh, out_lo=xl, ldp=C, stats_out=stats))
    return x, (xh, xl), stats


def _folded(L, parts):
    """parts: per group, a list of (w [n_i, C], b [n_i], gamma [C], beta [C]) -> planes of the folded weights [G*N, C],
    folded bias [G*N] and ln_cs [G*N] (engine.fold_layernorm)."""
    from spann3r_b200.engine import fold_layernorm
    ws, bs = [], []
    for group in parts:
        for w, b, gamma, beta in group:
            f = fold_layernorm(w, b, gamma, beta)
            ws.append(f[0]); bs.append(f[1])
    wp = L.split(torch.cat(ws).contiguous())
    cs = (wp[0].double() + wp[1].double()).sum(1).float().contiguous()
    return wp, torch.cat(bs).contiguous(), cs


def _ln(x, gamma, beta):
    return F.layer_norm(x, (x.shape[-1],), gamma.double(), beta.double(), 1e-6)


def _heads(t, B, N, heads):   # [B*N, heads*64] -> [B, heads, N, 64]
    return t.reshape(B, N, heads, 64).transpose(1, 2)


def _grid_pos(gh, gw, B, flip):
    """[B, N, 2] (y, x) patch positions; flip: the grid mirrored in both axes (a second, different position set)."""
    p = torch.cartesian_prod(torch.arange(gh), torch.arange(gw))
    if flip:
        p = torch.stack((gh - 1 - p[:, 0], gw - 1 - p[:, 1]), 1)
    return p.view(1, gh * gw, 2).expand(B, gh * gw, 2).contiguous()


def _attn_ref(q, k, v):
    return (q @ k.transpose(-2, -1)).softmax(-1) @ v


@pytest.mark.parametrize("B,gh,gw", [(1, 14, 14), (2, 14, 14), (1, 24, 32)])
def test_decoder_merged_projection(L, B, gh, gw):
    """The decoder's qkv launch (engine.cu qkv_launch): one EPI_QKV GEMM writes self-attention q, k, V^T (norm1 of the
    stream folded) and, in columns >= 2304 with the groups swapped, the cross-attention k2, V2^T of the OTHER stream
    (norm_y folded, rotated by that stream's positions).  Then both attentions over those outputs."""
    from oracle.spann3r_oracle import rope2d
    G, C, heads = 2, 768, 12
    N = gh * gw
    R = B * N
    npad = (N // 64 + 1) * 64          # V^T padding columns the kernel must neither write nor read
    x, xp, stats = _producer(L, G, R, C, seed=100)
    w = _rand(G * 5 * C, C, seed=110, scale=C ** -0.5)
    b = _rand(G * 5 * C, seed=111, scale=0.1)
    g1, be1 = 1 + 0.2 * _rand(G, C, seed=112), 0.1 * _rand(G, C, seed=113)
    gy, bey = 1 + 0.2 * _rand(G, C, seed=114), 0.1 * _rand(G, C, seed=115)
    W = lambda g, lo, hi: (w[g * 5 * C + lo:g * 5 * C + hi], b[g * 5 * C + lo:g * 5 * C + hi])   # noqa: E731
    wp, bf, cs = _folded(L, [[(*W(g, 0, 3 * C), g1[g], be1[g]), (*W(g, 3 * C, 5 * C), gy[g], bey[g])] for g in range(G)])
    pos = [_grid_pos(gh, gw, B, flip=g == 1) for g in range(G)]
    pos32 = torch.cat([p.reshape(R, 2) for p in pos]).to(torch.int32).cuda()
    q = torch.empty(G * B, heads, N, 64, device="cuda")
    k, k2 = torch.empty_like(q), torch.empty_like(q)
    vt = torch.full((G * B, heads, 64, npad), float("nan"), device="cuda")
    vt2 = torch.full_like(vt, float("nan"))
    L.gemm(_desc(L, xp, wp, G, R, C, 5 * C, epi=L.EPI_QKV, bias=bf, q_c=C, q_role_base=0, q_ntok=N, q_ntok_pad=npad,
                 q_rope=1, q_nb=B, q_pos=pos32, q_cs=_cs_table(), q_out=q, k_out=k, vt_out=vt, k2_out=k2, vt2_out=vt2,
                 q_scale=0.125, ln_stats=stats, ln_np=C // 32, ln_eps=1e-6, ln_cs=cs, a_swap=1, swap_col0=3 * C))
    o = torch.empty(G * R, C, device="cuda")
    o2 = torch.empty_like(o)
    for qq, kk, vv, oo in ((q, k, vt, o), (q, k2, vt2, o2)):
        L.check(L.lib().s3r_attention(L.ptr(qq), L.ptr(kk), L.ptr(vv), G * B * heads, heads, N, N, npad, None, None,
                                      L.ptr(oo), C, L.stream_ptr()), "s3r_attention")
    torch.cuda.synchronize()
    assert torch.isnan(vt[..., N:]).all() and torch.isnan(vt2[..., N:]).all()   # padding untouched
    xd = x.double().view(G, R, C)
    refs = {n: [] for n in ("q", "k", "v", "k2", "v2")}
    for g in range(G):
        h1 = F.linear(_ln(xd[g], g1[g], be1[g]), *[t.double() for t in W(g, 0, 3 * C)])
        h2 = F.linear(_ln(xd[1 - g], gy[g], bey[g]), *[t.double() for t in W(g, 3 * C, 5 * C)])
        p_self, p_other = pos[g].cuda(), pos[1 - g].cuda()
        refs["q"].append(rope2d(_heads(h1[:, :C], B, N, heads), p_self) * 0.125)
        refs["k"].append(rope2d(_heads(h1[:, C:2 * C], B, N, heads), p_self))
        refs["v"].append(_heads(h1[:, 2 * C:], B, N, heads))
        refs["k2"].append(rope2d(_heads(h2[:, :C], B, N, heads), p_other))
        refs["v2"].append(_heads(h2[:, C:], B, N, heads))
    refs = {n: torch.cat(t) for n, t in refs.items()}
    errs = {"q": rel_l2(q, refs["q"]), "k": rel_l2(k, refs["k"]), "k2": rel_l2(k2, refs["k2"]),
            "vt": rel_l2(vt[..., :N], refs["v"].transpose(-1, -2)), "vt2": rel_l2(vt2[..., :N], refs["v2"].transpose(-1, -2))}
    for name, (oo, kk, vv) in {"self": (o, refs["k"], refs["v"]), "cross": (o2, refs["k2"], refs["v2"])}.items():
        ref = _attn_ref(refs["q"], kk, vv).transpose(1, 2).reshape(G * R, C)
        assert torch.isfinite(oo).all(), name
        errs[name] = rel_l2(oo, ref)
    print(f"merged qkv B={B} N={N}:", {k_: f"{v_:.2e}" for k_, v_ in errs.items()})
    for name, e in errs.items():
        assert e < (TOL_ATTN if name in ("self", "cross") else TOL_QKV), (name, e)


@pytest.mark.parametrize("B,gh,gw", [(1, 14, 14), (2, 14, 14)])
def test_cross_attention_q_launch(L, B, gh, gw):
    """engine.cu's cross-attention q: EPI_QKV with n == q_c (role 0 only), norm2 folded: only q_out is written."""
    from oracle.spann3r_oracle import rope2d
    G, C, heads = 2, 768, 12
    N = gh * gw
    R = B * N
    x, xp, stats = _producer(L, G, R, C, seed=200)
    w = _rand(G * C, C, seed=210, scale=C ** -0.5)
    b = _rand(G * C, seed=211, scale=0.1)
    g2, be2 = 1 + 0.2 * _rand(G, C, seed=212), 0.1 * _rand(G, C, seed=213)
    wp, bf, cs = _folded(L, [[(w[g * C:(g + 1) * C], b[g * C:(g + 1) * C], g2[g], be2[g])] for g in range(G)])
    pos = [_grid_pos(gh, gw, B, flip=g == 1) for g in range(G)]
    pos32 = torch.cat([p.reshape(R, 2) for p in pos]).to(torch.int32).cuda()
    q = torch.empty(G * B, heads, N, 64, device="cuda")
    k = torch.full_like(q, 7.0)
    vt = torch.full((G * B, heads, 64, N), -7.0, device="cuda")
    L.gemm(_desc(L, xp, wp, G, R, C, C, epi=L.EPI_QKV, bias=bf, q_c=C, q_role_base=0, q_ntok=N, q_ntok_pad=N, q_rope=1,
                 q_nb=B, q_pos=pos32, q_cs=_cs_table(), q_out=q, k_out=k, vt_out=vt, q_scale=0.125, ln_stats=stats,
                 ln_np=C // 32, ln_eps=1e-6, ln_cs=cs))
    torch.cuda.synchronize()
    assert (k == 7.0).all() and (vt == -7.0).all()
    xd = x.double().view(G, R, C)
    ref = torch.cat([rope2d(_heads(F.linear(_ln(xd[g], g2[g], be2[g]), w[g * C:(g + 1) * C].double(),
                                            b[g * C:(g + 1) * C].double()), B, N, heads), pos[g].cuda()) * 0.125
                     for g in range(G)])
    e = rel_l2(q, ref)
    print(f"cross q B={B} N={N}: {e:.2e}")
    assert e < TOL_QKV, e


# DPT level sizes (engine.cu LH / LW): 224 x 224 (14 x 14 patches) and 512 x 384 (W x H: 24 x 32 patches)
_LEVELS = [(56, 56), (28, 28), (14, 14), (7, 7), (96, 128), (48, 64), (24, 32), (12, 16)]


@pytest.mark.parametrize("H,W", _LEVELS)
@pytest.mark.parametrize("mode", ["relu_planes", "res_res_plane_relu"])
def test_rcu_epilogues(L, H, W, mode):
    """The residual conv units of the DPT refinenets (engine.cu, refinenet loop): conv1 = ReLU with only planes out;
    conv2 = + layer + path (res1 + res2) with the fp32 sum out and its ReLU as planes.  3x3 convs, two groups."""
    G, C = 2, 256
    x = _rand(G, C, H, W, seed=300)
    w = _rand(G * C, C, 3, 3, seed=301, scale=(9 * C) ** -0.5)
    b = _rand(G * C, seed=302, scale=0.1)
    r1, r2 = _rand(G, H, W, C, seed=303), _rand(G, H, W, C, seed=304)
    xp = L.split(x.permute(0, 2, 3, 1).contiguous())
    wp = L.split(w.permute(0, 2, 3, 1).contiguous().view(G * C, 9 * C))
    oh = torch.empty(G, H, W, C, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xp[0].data_ptr(), xp[1].data_ptr(), wp[0].data_ptr(), wp[1].data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, 1, H, W, C, 9, C
    d.epi, d.bias = L.EPI_PLAIN, b.data_ptr()
    d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), C
    out = None
    if mode == "relu_planes":
        d.act = L.ACT_RELU
    else:
        out = torch.empty(G, H, W, C, device="cuda")
        d.res1, d.ldr1, d.res2, d.ldr2 = r1.data_ptr(), C, r2.data_ptr(), C
        d.out_f32, d.ldo, d.plane_relu = out.data_ptr(), C, 1
    L.gemm(d)
    torch.cuda.synchronize()
    y = torch.cat([F.conv2d(x[g:g + 1].double(), w[g * C:(g + 1) * C].double(), b[g * C:(g + 1) * C].double(), padding=1)
                   for g in range(G)]).permute(0, 2, 3, 1)
    if mode == "relu_planes":
        y = y.clamp_min(0)
    else:
        y = y + r1.double() + r2.double()
        e = rel_l2(out, y)
        assert e < TOL_GEMM, e
    ep = rel_l2(oh.double() + ol.double(), y.clamp_min(0))
    assert ep < TOL_GEMM, ep


@pytest.mark.parametrize("rows", [1000, 333])
@pytest.mark.parametrize("bn", [64, 128])
def test_inplace_residual(L, rows, bn):
    """res1 == out_f32 (the proj / cproj / fc2 launches) with stats_out: bitwise the out-of-place result."""
    K, N = 768, 768
    a, w = L.split(_rand(rows, K, seed=400)), L.split(_rand(N, K, seed=401, scale=K ** -0.5))
    b = _rand(N, seed=402, scale=0.1)
    r = _rand(rows, N, seed=403)
    outs = []
    for inplace in (False, True):
        o = r.clone() if inplace else torch.empty_like(r)
        oh = torch.empty(rows, N, dtype=torch.bfloat16, device="cuda")
        ol = torch.empty_like(oh)
        st = torch.empty(rows, N // 32, 2, device="cuda")
        L.gemm(_desc(L, a, w, 1, rows, K, N, epi=L.EPI_PLAIN, force_bn=bn, bias=b, res1=o if inplace else r, ldr1=N,
                     out_f32=o, ldo=N, out_hi=oh, out_lo=ol, ldp=N, stats_out=st))
        outs.append((o, oh, ol, st))
    torch.cuda.synchronize()
    for u, v in zip(*outs):
        assert torch.equal(u, v)
    ref = F.linear(a[0].double() + a[1].double(), w[0].double() + w[1].double(), b.double()) + r.double()
    assert rel_l2(outs[1][0], ref) < TOL_GEMM


@pytest.mark.parametrize("kc", [64, 256, 768, 1024])
def test_folded_layernorm_chunk_counts_and_offsets(L, kc):
    """Folded LayerNorm with ln_np = kc/32 from 2 to 32 (the edge of the 16-lane statistics read), on rows whose mean is
    0, 3 and 30 times their standard deviation.  The epilogue forms var = E[x^2] - mean^2 in fp32 from the chunk sums, which
    cancels as mean/std grows: 0 and 3 are held to TOL_GEMM, 30 to a bound measured for it."""
    band, N = 200, 256
    ratios = (0.0, 3.0, 30.0)
    offset = torch.cat([torch.full((band,), rt) for rt in ratios]).cuda()
    rows = band * len(ratios)
    x, xp, stats = _producer(L, 1, rows, kc, seed=500, offset=offset * 1.5)   # x - offset: std ~1.5 (a W0^T + b0 + r)
    w = _rand(N, kc, seed=510, scale=kc ** -0.5)
    b = _rand(N, seed=511, scale=0.1)
    gamma, beta = 1 + 0.2 * _rand(kc, seed=512), 0.1 * _rand(kc, seed=513)
    wp, bf, cs = _folded(L, [[(w, b, gamma, beta)]])
    out = torch.empty(rows, N, device="cuda")
    L.gemm(_desc(L, xp, wp, 1, rows, kc, N, epi=L.EPI_PLAIN, bias=bf, out_f32=out, ldo=N, ln_stats=stats, ln_np=kc // 32,
                 ln_eps=1e-6, ln_cs=cs))
    torch.cuda.synchronize()
    xd = x.double()
    ref = F.linear(_ln(xd, gamma, beta), w.double(), b.double())
    ratio = (xd.mean(-1).abs() / xd.std(-1, unbiased=False)).view(len(ratios), band).max(-1).values
    errs = [rel_l2(out[i * band:(i + 1) * band], ref[i * band:(i + 1) * band]) for i in range(len(ratios))]
    print(f"folded LN kc={kc}: " + ", ".join(f"mean/std<={float(rt):.1f}: {e:.2e}" for rt, e in zip(ratio, errs)))
    assert errs[0] < TOL_GEMM and errs[1] < TOL_GEMM, errs
    # mean/std ~30: the raw-x GEMM and the one-pass variance lose ~log2(30) bits (1.2-1.5e-4 measured on an H100)
    assert errs[2] < 10 * TOL_GEMM, errs


@pytest.mark.parametrize("C", [768, 1024])
@pytest.mark.parametrize("swap", [False, True])
def test_layernorm_groups_swap_and_plane_window(L, C, swap):
    """s3r_layernorm with two weight sets (wb_group_stride, rows_per_group), optionally swap_rows (norm_y of the twin
    decoders), planes written at column col0 of a wider buffer (ldp), as the key-head input cat(feat, dec[-1])."""
    S, col0, ldp = 150, 1024, C + 1024
    x = _rand(2 * S, C, seed=600)
    wt, bt = 1 + 0.2 * _rand(2, C, seed=601), 0.1 * _rand(2, C, seed=602)
    out = torch.empty(2 * S, C, device="cuda")
    hi = torch.full((2 * S, ldp), 3.0, dtype=torch.bfloat16, device="cuda")
    lo = torch.full_like(hi, -3.0)
    L.check(L.lib().s3r_layernorm(L.ptr(x), C, L.ptr(wt), L.ptr(bt), C, S, 1e-6, 2 * S, C, L.ptr(out), C, L.ptr(hi),
                                  L.ptr(lo), ldp, col0, S if swap else 0, L.stream_ptr()), "s3r_layernorm")
    torch.cuda.synchronize()
    xd = x.double().view(2, S, C)
    ref = torch.stack([_ln(xd[g], wt[1 - g if swap else g], bt[1 - g if swap else g]) for g in range(2)])
    if swap:
        ref = ref.flip(0)
    ref = ref.reshape(2 * S, C)
    assert rel_l2(out, ref) < 2e-6
    ph, pl = hi[:, col0:col0 + C], lo[:, col0:col0 + C]
    assert rel_l2(ph.double() + pl.double(), ref) < 1e-5
    assert torch.equal(ph, out.to(torch.bfloat16))
    assert (hi[:, :col0] == 3.0).all() and (lo[:, :col0] == -3.0).all()


def test_split_relu_window(L):
    """s3r_split with ReLU from a strided fp32 source into a column window of wider planes: bitwise hi = bf16(x),
    lo = bf16(x - hi); everything outside the window untouched."""
    rows, C, ldx, ldp, col0 = 333, 512, 776, 1024, 256
    src = _rand(rows, ldx, seed=700)
    hi = torch.full((rows, ldp), 3.0, dtype=torch.bfloat16, device="cuda")
    lo = torch.full_like(hi, -3.0)
    L.check(L.lib().s3r_split(L.ptr(src), ldx, L.ptr(hi), L.ptr(lo), ldp, col0, rows, C, 1, L.stream_ptr()), "s3r_split")
    torch.cuda.synchronize()
    x = src[:, :C].clamp_min(0)
    h = x.to(torch.bfloat16)
    assert torch.equal(hi[:, col0:col0 + C], h)
    assert torch.equal(lo[:, col0:col0 + C], (x - h.float()).to(torch.bfloat16))
    outside = torch.ones(ldp, dtype=torch.bool)
    outside[col0:col0 + C] = False
    assert (hi[:, outside] == 3.0).all() and (lo[:, outside] == -3.0).all()


@pytest.mark.parametrize("H,W", [(7, 9), (13, 13)])
@pytest.mark.parametrize("c", [8, 768])
def test_im2col_3x3s2(L, H, W, c):
    """Planes [nb, h, w, c] -> [nb*ho*wo, 9c] (k = tap*c + channel), bitwise F.unfold(3, padding=1, stride=2)."""
    nb = 2
    ho, wo = (H + 1) // 2, (W + 1) // 2
    xh, xl = L.split(_rand(nb, H, W, c, seed=800))
    oh = torch.empty(nb * ho * wo, 9 * c, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    L.check(L.lib().s3r_im2col_3x3s2(L.ptr(xh), L.ptr(xl), nb, H, W, c, ho, wo, L.ptr(oh), L.ptr(ol), L.stream_ptr()),
            "s3r_im2col_3x3s2")
    torch.cuda.synchronize()
    for got, p in ((oh, xh), (ol, xl)):
        ref = F.unfold(p.float().permute(0, 3, 1, 2), 3, padding=1, stride=2)        # [nb, c*9, ho*wo]
        ref = ref.view(nb, c, 9, ho * wo).permute(0, 3, 2, 1).reshape(nb * ho * wo, 9 * c)
        assert torch.equal(got.float(), ref)


@pytest.mark.parametrize("nb,H,W,C", [(2, 12, 16, 256), (4, 7, 9, 128)])
def test_upsample2x_planes(L, nb, H, W, C):
    """Planes mode of s3r_upsample2x == s3r_split of its fp32 mode, bitwise."""
    f = _rand(nb, H, W, C, seed=900)
    up = torch.empty(nb, 2 * H, 2 * W, C, device="cuda")
    hi = torch.empty(up.shape, dtype=torch.bfloat16, device="cuda")
    lo = torch.empty_like(hi)
    L.check(L.lib().s3r_upsample2x(L.ptr(f), nb, H, W, C, L.ptr(up), None, None, L.stream_ptr()), "upsample")
    L.check(L.lib().s3r_upsample2x(L.ptr(f), nb, H, W, C, None, L.ptr(hi), L.ptr(lo), L.stream_ptr()), "upsample")
    sh, sl = L.split(up)
    torch.cuda.synchronize()
    assert torch.equal(hi, sh) and torch.equal(lo, sl)
    ref = F.interpolate(f.double().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    assert rel_l2(up, ref.permute(0, 2, 3, 1)) < 1e-6


@pytest.mark.parametrize("n", [1, 255, 196608, 2 * 196608 + 3])
def test_conf_score(L, n):
    """mean((conf - 1) / conf) against fp64; a fixed reduction order: two calls give the same bits."""
    conf = 1 + torch.exp(_rand(n, seed=1000))
    a, b = L.conf_score(conf), L.conf_score(conf)
    torch.cuda.synchronize()
    ref = ((conf.double() - 1) / conf.double()).mean()
    assert torch.equal(a, b)
    assert abs(float(a) - float(ref)) <= 1e-6 * abs(float(ref)), (float(a), float(ref))
