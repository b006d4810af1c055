"""The GEMM engine's operand ring: 32-channel k-blocks in a 64-byte swizzle, 5 stages at BN = 128 and 7 at BN = 64.

Covers what the k-block geometry decides: channel counts that are not a multiple of the k-block (zero-filled tails),
one and nine taps, both tile widths, k-block counts below, equal to and above the ring depth (the weight prefetch
before the dependency wait covers min(k-blocks, stages)), ragged M and N, persistent CTAs that wrap the ring over
several tiles, and groups = 2 with a_swap.  Every case is held to fp64 at the tolerance of test_ops_gpu.py.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_l2

pytestmark = pytest.mark.gpu

TOL_GEMM = 3e-5


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def _run(L, groups, NB, H, W, Kc, taps, N, bn, swap):
    """A [G*NB, H, W, Kc] NHWC, Wt [G*N, taps, Kc]; out = A (*) Wt + bias + res, fp32 and split-bf16 planes."""
    x = _rand(groups * NB, H, W, Kc, seed=31)
    w = _rand(groups * N, taps, Kc, seed=32, scale=(taps * Kc) ** -0.5)
    b = _rand(groups * N, seed=33, scale=0.1)
    res = _rand(groups * NB, H, W, N, seed=34)
    xh, xl = L.split(x)
    wh, wl = L.split(w.view(groups * N, taps * Kc))
    out = torch.empty(groups * NB, H, W, N, device="cuda")
    oh = torch.empty(out.shape, dtype=torch.bfloat16, device="cuda")
    ol = torch.empty_like(oh)
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr()
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = groups, NB, H, W, Kc, taps, N
    d.epi, d.act, d.force_bn, d.a_swap = L.EPI_PLAIN, L.ACT_NONE, bn, swap
    d.bias = b.data_ptr()
    d.res1, d.ldr1 = res.data_ptr(), N
    d.out_f32, d.ldo = out.data_ptr(), N
    d.out_hi, d.out_lo, d.ldp = oh.data_ptr(), ol.data_ptr(), N
    L.gemm(d)
    torch.cuda.synchronize()

    xd = x.double().view(groups, NB, H, W, Kc)
    if swap:
        xd = xd.flip(0)
    wd = w.double().view(groups, N, taps, Kc)
    bd = b.double().view(groups, N)
    ref = []
    for g in range(groups):
        if taps == 1:
            y = torch.einsum("bhwk,nk->bhwn", xd[g], wd[g, :, 0]) + bd[g]
        else:
            wc = wd[g].view(N, 3, 3, Kc).permute(0, 3, 1, 2)
            y = F.conv2d(xd[g].permute(0, 3, 1, 2), wc, bd[g], padding=1).permute(0, 2, 3, 1)
        ref.append(y)
    ref = torch.stack(ref).reshape(out.shape) + res.double()
    assert rel_l2(out, ref) < TOL_GEMM, rel_l2(out, ref)
    assert rel_l2(oh.double() + ol.double(), ref) < TOL_GEMM


KCS = [8, 24, 32, 40, 96, 160, 224, 1024, 3072, 4096]


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("Kc", KCS)
def test_linear_k_blocks(L, Kc, bn):
    """300 rows (128-row tiles: 2 full + 44) x N = 160 (BN = 128: 128 + 32; BN = 64: 64 + 64 + 32).  Kc = 160 is exactly
    the 5-stage ring at BN = 128 and Kc = 224 the 7-stage ring at BN = 64."""
    _run(L, 1, 1, 1, 300, Kc, 1, 160, bn, 0)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("Kc", [8, 24, 32, 40, 96])
def test_conv3x3_k_blocks(L, Kc, bn):
    """9 taps of ceil(Kc / 32) k-blocks; a 13 x 19 map (32 x 4 pixel tiles, ragged in both directions), N = 96."""
    _run(L, 1, 2, 13, 19, Kc, 9, 96, bn, 0)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("Kc,taps", [(96, 1), (1024, 1), (40, 9)])
def test_groups_a_swap(L, Kc, taps, bn):
    """Group g reads the A rows of group 1 - g for every output column."""
    if taps == 1:
        _run(L, 2, 1, 1, 300, Kc, 1, 160, bn, 1)
    else:
        _run(L, 2, 1, 13, 19, Kc, 9, 96, bn, 1)


@pytest.mark.parametrize("rows,Kc,N,bn", [
    (7680, 4096, 1024, 0),   # enc.fc2 (the planner picks BN = 128): 480 tiles of 128 k-blocks over at most 132 CTAs
    (7680, 1024, 3072, 64),  # enc.qkv at BN = 64: 2880 tiles of 32 k-blocks, ~22 per CTA
    (7700, 160, 1056, 128),  # 5 k-blocks per tile = one ring pass per tile; ragged M (60 x 128 + 20) and N (8 x 128 + 32)
])
def test_persistent_ring_wrap(L, rows, Kc, N, bn):
    _run(L, 1, 1, 1, rows, Kc, 1, N, bn, 0)
