"""The GEMM engine's 128 x 96 tile.

A tile width changes which CTA computes an output element, never how: the same k16 steps, the same hi*lo, lo*hi, hi*hi
product order and the same epilogue arithmetic per element.  So on random operands, whose products and sums round,
force_bn 64, 96 and 128 must give the same bits.  Held here for every epilogue the planner gives the 96-wide tile: PLAIN
with a folded LayerNorm, an in-place residual and stats_out; QKV with RoPE at q_c 768 (the decoder's five merged roles,
a_swap from column 2304) and q_c 1024 (a 96-wide tile spans the q | k boundary); PIXSHUF at ps_cout 96 and 192 (a tile
splits a sub-pixel); the one-product precision; rings that wrap at 6 (split) and 13 (one product) stages.

The 96-wide tile is also held to the exact answer (gemm_exact.py), to fp64, and to the one-product bars of
test_bf16_gpu.py on the op-level cases the 64 / 128 widths are held to there."""
import math

import pytest
import torch

import gemm_exact as E
from test_bf16_gpu import test_folded_layernorm_uses_hi_column_sums as _bf16_lnfold
from test_bf16_gpu import test_pixshuf as _bf16_pixshuf
from test_bf16_gpu import test_plain as _bf16_plain
from test_bf16_gpu import test_qkv as _bf16_qkv
from test_gemm_exact_gpu import _gemm
from test_gemm_ring_gpu import KCS, _run

pytestmark = pytest.mark.gpu

WIDTHS = (64, 96, 128)


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _same_at_every_width(L, build):
    """build(bn) -> (desc, outputs, keep); runs the launch at each width and compares every output bitwise."""
    ref = None
    for bn in WIDTHS:
        d, outs, keep = build(bn)
        assert L.lib().s3r_gemm_tile_n(d) == bn
        L.gemm(d)
        torch.cuda.synchronize()
        got = [o.clone() for o in outs]
        del keep
        for o in got:
            assert bool(torch.isfinite(o.float()).all())
        if ref is None:
            ref = got
            continue
        for i, (a, b) in enumerate(zip(ref, got)):
            if not torch.equal(a, b):
                bad = (a != b).nonzero()
                pytest.fail(f"output {i}: bn {bn} differs from bn {WIDTHS[0]} at {int(bad.shape[0])} elements, "
                            f"first {bad[0].tolist()}")


def _planes_desc(L, x, w, G, NB, H, W, Kc, taps, N, precision):
    xh, xl = L.split(x)
    wh, wl = L.split(w)
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n, d.precision = G, NB, H, W, Kc, taps, N, precision
    return d, [xh, xl, wh, wl]


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("rows,K,N", [(768, 768, 768), (768, 1024, 3072), (300, 768, 1056)])
def test_plain_lnfold_inplace_residual_stats(L, rows, K, N, precision):
    """The decoder's proj / fc2 pattern on two groups: folded LayerNorm, bias, GELU-free, residual read and written in
    place, split-bf16 planes and stats_out.  N = 1056 ends in a partial 96-wide tile (11 x 96) and a partial 128 one."""
    G = 2
    x = _rand(G * rows, K, seed=1)
    w = _rand(G * N, K, seed=2, scale=K ** -0.5)
    b = _rand(G * N, seed=3, scale=0.1)
    cs = _rand(G * N, seed=4)
    st = torch.stack((x.view(G * rows, K // 32, 32).sum(-1), x.view(G * rows, K // 32, 32).pow(2).sum(-1)), -1)
    res0 = _rand(G * rows, N, seed=5)

    def build(bn):
        d, keep = _planes_desc(L, x, w, G, 1, 1, rows, K, 1, N, precision)
        out = res0.clone()
        oh = torch.full((G * rows, N), float("nan"), dtype=torch.bfloat16, device="cuda")
        ol = torch.full_like(oh, float("nan"))
        sto = torch.full((G * rows, N // 32, 2), float("nan"), device="cuda")
        d.force_bn, d.bias = bn, b.data_ptr()
        d.res1, d.ldr1, d.out_f32, d.ldo = out.data_ptr(), N, out.data_ptr(), N
        d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), N
        d.stats_out = sto.data_ptr()
        d.ln_stats, d.ln_np, d.ln_eps, d.ln_cs = st.data_ptr(), K // 32, 1e-6, cs.data_ptr()
        return d, [out, oh, ol, sto], keep
    _same_at_every_width(L, build)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("case", ["dec-merged-q768-swap2304", "val-qkv-q1024"])
def test_qkv_rope(L, case, precision):
    """EPI_QKV with RoPE (random angles) and a folded LayerNorm: the decoder's merged projection (five 768-wide roles on
    two groups, a_swap from column 2304 = 24 x 96) and the value encoder's qkv (q_c 1024: the tile at columns 960..1055
    holds q and k chunks)."""
    if case.startswith("dec"):
        G, qc, nroles, base, swap, swap_col0 = 2, 768, 5, 0, 1, 2304
    else:
        G, qc, nroles, base, swap, swap_col0 = 1, 1024, 3, 0, 0, 0
    rows, K, heads = 300, 768, qc // 64
    N = nroles * qc
    x = _rand(G * rows, K, seed=11)
    w = _rand(G * N, K, seed=12, scale=K ** -0.5)
    b = _rand(G * N, seed=13, scale=0.1)
    cs = _rand(G * N, seed=14)
    st = torch.stack((x.view(G * rows, K // 32, 32).sum(-1), x.view(G * rows, K // 32, 32).pow(2).sum(-1)), -1)
    maxpos = 40
    pos = torch.randint(0, maxpos, (G * rows, 2), generator=torch.Generator().manual_seed(15)).to(torch.int32).cuda()
    ang = torch.rand(maxpos, 16, generator=torch.Generator().manual_seed(16)) * 2 * math.pi
    qcs = torch.stack((ang.cos(), ang.sin()), -1).contiguous().cuda()
    npad = rows + 4

    def build(bn):
        d, keep = _planes_desc(L, x, w, G, 1, 1, rows, K, 1, N, precision)
        outs = [torch.full((G * heads * (npad if r in (2, 4) else rows) * 64,), -7.0, device="cuda") for r in range(nroles)]
        d.force_bn, d.epi, d.bias = bn, L.EPI_QKV, b.data_ptr()
        d.q_c, d.q_role_base, d.q_ntok, d.q_ntok_pad, d.q_rope, d.q_nb = qc, base, rows, npad, 1, 1
        d.q_pos, d.q_cs, d.q_scale = pos.data_ptr(), qcs.data_ptr(), 0.125
        ptrs = [o.data_ptr() for o in outs] + [None] * (5 - nroles)
        d.q_out, d.k_out, d.vt_out, d.k2_out, d.vt2_out = ptrs
        d.ln_stats, d.ln_np, d.ln_eps, d.ln_cs = st.data_ptr(), K // 32, 1e-6, cs.data_ptr()
        d.a_swap, d.swap_col0 = swap, swap_col0
        return d, outs, keep
    _same_at_every_width(L, build)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("s,cout,Kc", [(4, 96, 96), (2, 192, 192)])
def test_pixshuf(L, s, cout, Kc, precision):
    """EPI_PIXSHUF as the DPT's act1_up / act2_up at 512 x 384 (a 24 x 32 patch grid, two heads as groups): with
    ps_cout 96 a 96-wide tile is one sub-pixel, with 192 it holds half of one and half of the next."""
    G, NB, H, W = 2, 1, 24, 32
    N = s * s * cout
    x = _rand(G * NB, H, W, Kc, seed=21)
    w = _rand(G * N, Kc, seed=22, scale=Kc ** -0.5)
    b = _rand(G * cout, seed=23, scale=0.1)
    orows = G * NB * H * s * W * s

    def build(bn):
        d, keep = _planes_desc(L, x, w, G, NB, H, W, Kc, 1, N, precision)
        out = torch.full((orows, cout), float("nan"), device="cuda")   # a chunk left unwritten fails the finite check
        oh = torch.full((orows, cout), float("nan"), dtype=torch.bfloat16, device="cuda")
        ol = torch.full_like(oh, float("nan"))
        d.force_bn, d.epi, d.ps_s, d.ps_cout, d.bias = bn, L.EPI_PIXSHUF, s, cout, b.data_ptr()
        d.out_f32, d.ldo = out.data_ptr(), cout
        d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), cout
        return d, [out, oh, ol], keep
    _same_at_every_width(L, build)


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("rows,Kc,N", [(7680, 1024, 768), (1536, 3072, 768), (300, 160, 96), (300, 416, 96)])
def test_ring_wrap(L, rows, Kc, N, precision):
    """Rings of 6 (split) and 13 (one product) stages: 5 and 13 k-blocks per tile (one ring pass, and one short of or
    exactly one), 32 and 96 k-blocks per tile, and persistent CTAs that take several tiles (7680 rows: 480 tiles)."""
    x = _rand(rows, Kc, seed=31)
    w = _rand(N, Kc, seed=32, scale=Kc ** -0.5)
    b = _rand(N, seed=33, scale=0.1)
    r = _rand(rows, N, seed=34)

    def build(bn):
        d, keep = _planes_desc(L, x, w, 1, 1, 1, rows, Kc, 1, N, precision)
        out = torch.full((rows, N), float("nan"), device="cuda")
        d.force_bn, d.act, d.bias = bn, L.ACT_GELU, b.data_ptr()
        d.res1, d.ldr1, d.out_f32, d.ldo = r.data_ptr(), N, out.data_ptr(), N
        return d, [out], keep
    _same_at_every_width(L, build)


# ------------------------------------------------------------------------------------------------ exact and fp64
@pytest.mark.parametrize("precision,lo", [(0, "planes"), (1, "nan")], ids=["split", "bf16-nan-lo"])
@pytest.mark.parametrize("geom", E.GEOMETRY, ids=["x".join(map(str, g)) for g in E.GEOMETRY])
def test_exact_geometry_bn96(L, geom, precision, lo):
    """test_gemm_exact_gpu.test_gemm_geometry at force_bn 96."""
    _gemm(L, *geom, precision=precision, lo=lo, force_bn=96, seed=sum(geom))


@pytest.mark.parametrize("swap_col0", [0, 768])
@pytest.mark.parametrize("geom", [(2, 1, 1, 300, 96, 1, 1056), (2, 2, 13, 19, 40, 9, 960)], ids=["linear", "3x3"])
def test_exact_groups_a_swap_bn96(L, geom, swap_col0):
    """groups = 2, a_swap from column swap_col0 on (a multiple of 96), at force_bn 96."""
    _gemm(L, *geom, force_bn=96, a_swap=True, swap_col0=swap_col0, seed=7 + swap_col0)


@pytest.mark.parametrize("Kc", KCS)
def test_fp64_linear_k_blocks_bn96(L, Kc):
    """test_gemm_ring_gpu.test_linear_k_blocks at force_bn 96 (N = 160: one full 96-wide tile and a 64-wide tail)."""
    _run(L, 1, 1, 1, 300, Kc, 1, 160, 96, 0)


@pytest.mark.parametrize("Kc", [8, 24, 40, 96])
def test_fp64_conv3x3_k_blocks_bn96(L, Kc):
    _run(L, 1, 2, 13, 19, Kc, 9, 96, 96, 0)


@pytest.mark.parametrize("act", ["none", "gelu", "relu"])
@pytest.mark.parametrize("G,NB,H,W,kc,taps,n", [(1, 1, 1, 700, 1024, 1, 1024), (2, 1, 1, 300, 200, 1, 96),
                                                (2, 2, 9, 13, 40, 9, 64), (1, 1, 16, 16, 256, 9, 256)])
def test_bf16_plain_bn96(L, act, G, NB, H, W, kc, taps, n):
    """test_bf16_gpu.test_plain at force_bn 96."""
    _bf16_plain(L, 96, act, G, NB, H, W, kc, taps, n)


def test_bf16_pixshuf_bn96(L):
    """test_bf16_gpu.test_pixshuf (the DPT's act2_up at ps_cout 96) at force_bn 96."""
    _bf16_pixshuf(L, 96)


@pytest.mark.parametrize("nb,ntok", [(1, 196), (2, 195)])
def test_bf16_qkv_bn96(L, nb, ntok):
    """test_bf16_gpu.test_qkv at force_bn 96 (q_c 256: the tiles at columns 192 and 480 hold two roles)."""
    _bf16_qkv(L, 96, nb, ntok)


@pytest.mark.parametrize("kc", [64, 128, 256, 768, 1024])
def test_bf16_folded_layernorm_bn96(L, kc):
    """test_bf16_gpu.test_folded_layernorm_uses_hi_column_sums at force_bn 96."""
    _bf16_lnfold(L, kc, 96)
