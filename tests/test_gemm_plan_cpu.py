"""The GEMM tile planner without a GPU: s3r_gemm_plan_bn is the rule gemm_plan applies (waves x bytes staged per
k-block, 24 / 28 / 32 KB at 64 / 96 / 128 columns), checked on the launches of a 512 x 384 sequence at 132 SMs, and the
rule that no tile may straddle a_swap's swap_col0."""
import ctypes as C

import pytest

from test_gemm_contract_cpu import _qkv

SMS = 132


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    return _lib


def _plan(L, m_tiles, n, col_align=0, force_bn=0, sms=SMS):
    return L.lib().s3r_gemm_plan_bn(m_tiles, n, sms, col_align, force_bn)


# (launch, 128-row tiles, N, width): 768 tokens per group are 6 row tiles; the decoder and key heads run two groups
PLAN = [
    ("dec.proj / q / cproj / fc2, decoder_embed", 12, 768, 96),
    ("dec.fc1", 12, 3072, 96),
    ("dec.qkv + cross kv", 12, 3840, 128),
    ("key.fc1", 12, 1792, 96),
    ("key.fc2", 12, 1024, 96),
    ("val.qkv", 6, 3072, 96),
    ("val.fc1", 6, 4096, 96),
    ("memory read score, bank of 3072", 6, 3072, 96),
    ("val.proj / fc2 / out", 6, 1024, 64),
    ("enc.qkv", 60, 3072, 128),
    ("enc.proj", 60, 1024, 128),
    ("enc.fc1", 60, 4096, 128),
    ("enc.fc2", 60, 1024, 128),
    # DPT head at 512 x 384 (24 x 32 patches, 32 x 4 pixel tiles, the two heads as groups): act1_up, act2_up and
    # act4_conv move from 128 to 96; every other conv keeps its width
    ("dpt act1_up (PIXSHUF, ps_cout 96)", 12, 1536, 96),
    ("dpt act2_up (PIXSHUF, ps_cout 192)", 12, 768, 96),
    ("dpt act4_conv", 12, 768, 96),
    ("dpt act1_conv", 12, 96, 64),
    ("dpt act2_conv", 12, 192, 64),
    ("dpt act3_conv", 12, 384, 64),
    ("dpt act4_down", 4, 768, 64),
    ("dpt layer_rn / refinenet, 96 x 128", 192, 256, 128),
    ("dpt layer_rn / refinenet, 48 x 64", 48, 256, 128),
    ("dpt layer_rn / refinenet, 24 x 32", 12, 256, 64),
    ("dpt layer_rn / refinenet, 12 x 16", 4, 256, 64),
    ("dpt head0", 768, 128, 128),
]


@pytest.mark.parametrize("name,m_tiles,n,bn", PLAN, ids=[p[0] for p in PLAN])
def test_planner_widths_at_132_sms(L, name, m_tiles, n, bn):
    assert _plan(L, m_tiles, n) == bn


def test_decoder_merged_projection_keeps_its_alignment(L):
    """The merged qkv + cross kv launch swaps A from column 2304 = 24 x 96 = 18 x 128 on: every width fits it."""
    for bn in (64, 96, 128):
        assert _plan(L, 12, 3840, col_align=2304, force_bn=bn) == bn
    assert _plan(L, 12, 3840, col_align=2304) == 128


@pytest.mark.parametrize("col_align", [256, 512, 1280])
def test_width_that_straddles_swap_col0_is_never_chosen(L, col_align):
    """N = 768 on 12 row tiles picks 96 without a constraint; with swap_col0 not a multiple of 96 it must not."""
    assert _plan(L, 12, 768) == 96
    assert _plan(L, 12, 768, col_align=col_align) in (64, 128)
    for m_tiles in (1, 6, 12, 60, 400):
        for n in (256, 768, 1024, 1792, 3072, 3840):
            assert _plan(L, m_tiles, n, col_align=col_align) != 96


def test_forced_width_that_straddles_swap_col0_is_rejected(L):
    assert _plan(L, 12, 768, col_align=256, force_bn=96) == -1
    assert b"swap_col0" in L.lib().s3r_last_error()
    d = _qkv(L)                      # the decoder's merged projection descriptor, with a_swap moved to column 2560
    d.force_bn, d.swap_col0 = 96, 2560
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) == -1
    assert b"swap_col0" in L.lib().s3r_last_error()


def test_forced_widths_are_the_kernels_own(L):
    """force_bn takes 64, 96 or 128 (0 = the planner's choice); any other value, the CTA-pair widths of other
    architectures included, is rejected."""
    for fb in (64, 96, 128):
        assert _plan(L, 12, 768, force_bn=fb) == fb
    for fb in (32, 2096, 256, 1128, 2064, 2128, 2256):
        assert _plan(L, 12, 768, force_bn=fb) == -1
        assert b"force_bn" in L.lib().s3r_last_error()
