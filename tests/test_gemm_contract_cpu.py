"""Descriptor rules of the op-level C ABI, checked without a GPU: every s3r_gemm descriptor the epilogue cannot execute is
rejected by the planner (s3r_gemm_tile_n runs it and never launches) before the driver is touched, with the offending field
named in s3r_last_error(); the layout and attention entry points reject their bad arguments before any CUDA call.
Pointers are fake non-null addresses: nothing here may reach a launch."""
import ctypes as C

import pytest

FAKE = 0x7F0000000000   # 256-byte aligned, never dereferenced


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    return _lib


def _p(i):
    return FAKE + 0x100000 * i


def _plain(L):
    """A well-formed folded-LayerNorm producer / consumer descriptor (768 -> 768, two groups, every output)."""
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = _p(1), _p(2), _p(3), _p(4)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = 2, 1, 1, 196, 768, 1, 768
    d.epi = L.EPI_PLAIN
    d.bias = _p(5)
    d.res1, d.ldr1 = _p(6), 768
    d.res2, d.ldr2 = _p(7), 768
    d.out_f32, d.ldo = _p(8), 768
    d.out_hi, d.out_lo, d.ldp = _p(9), _p(10), 768
    d.ln_stats, d.ln_np, d.ln_eps, d.ln_cs = _p(11), 24, 1e-6, _p(12)
    return d


def _qkv(L):
    """The decoder's merged projection as the engine builds it: five 768-wide roles, norm1 / norm_y folded, a_swap."""
    d = L.GemmDesc()
    d.a_hi, d.a_lo, d.b_hi, d.b_lo = _p(1), _p(2), _p(3), _p(4)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = 2, 1, 1, 196, 768, 1, 3840
    d.epi = L.EPI_QKV
    d.bias = _p(5)
    d.q_c, d.q_role_base, d.q_ntok, d.q_ntok_pad, d.q_rope, d.q_nb = 768, 0, 196, 196, 1, 1
    d.q_pos, d.q_cs = _p(6), _p(7)
    d.q_out, d.k_out, d.vt_out, d.k2_out, d.vt2_out, d.q_scale = _p(8), _p(9), _p(10), _p(11), _p(12), 0.125
    d.ln_stats, d.ln_np, d.ln_eps, d.ln_cs, d.a_swap, d.swap_col0 = _p(13), 24, 1e-6, _p(14), 1, 2304
    return d


def _rejects(L, d, field):
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) == -1
    msg = L.lib().s3r_last_error()
    assert field.encode() in msg, msg


@pytest.mark.parametrize("kc,ln_np", [(800, 25), (1088, 34), (2048, 64), (32, 1)])
def test_folded_layernorm_needs_an_even_chunk_count_up_to_32(L, kc, ln_np):
    """The statistics are read as float4 pairs by 16 lanes: an odd count misaligns them, more than 32 are dropped."""
    d = _plain(L)
    d.kc, d.ln_np = kc, ln_np
    _rejects(L, d, "ln_np")


@pytest.mark.parametrize("n", [100, 16, 784])
def test_n_must_be_whole_32_column_chunks(L, n):
    d = _plain(L)
    d.n = n
    d.ln_stats = None
    _rejects(L, d, f"n={n}")


@pytest.mark.parametrize("change", [dict(ldo=96), dict(res1=_p(6)), dict(res2=_p(7)), dict(out_hi=_p(9)),
                                    dict(stats_out=_p(13))])
def test_only_a_bare_wide_enough_fp32_output_takes_a_chunk_tail(L, change):
    """The memory read's scores (n = bank length, out_f32 alone, ldo >= n rounded up to 32) are the one launch whose n
    is not whole chunks: anything else the tail chunk would touch past n rejects it."""
    d = _plain(L)
    d.n, d.ln_stats, d.res1, d.res2, d.out_hi, d.out_lo, d.ldo = 100, None, None, None, None, None, 128
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) != -1, L.lib().s3r_last_error()   # accepted (-3 without a driver)
    for k, v in change.items():
        setattr(d, k, v)
    _rejects(L, d, "n=100")


@pytest.mark.parametrize("field,value", [
    ("ldr1", 770), ("ldr2", 6), ("ldo", 770), ("ldp", 2), ("plane_col0", 2), ("ldo", 1 << 32), ("ldp", -768),
])
def test_strides_and_offsets_are_vector_aligned_ints(L, field, value):
    d = _plain(L)
    setattr(d, field, value)
    _rejects(L, d, field)


@pytest.mark.parametrize("field,value", [
    ("lda", 772), ("lda", -768), ("ldb", 6), ("ldb", -8), ("b_group_rows", -1), ("b_group_rows", 1 << 31),
    ("kc", 100),   # the dense lda / ldb of kc = 100 are not 16-byte strides
    ("taps", 3),
])
def test_operand_layout_is_tma_aligned(L, field, value):
    """lda / ldb are TMA row strides (multiples of 16 bytes); b_group_rows fits the kernel's int; taps is 1 or 9."""
    d = _plain(L)
    d.ln_stats = None
    d.lda, d.ldb, d.b_group_rows, d.b_static = 1024, 776, 800, 1   # a memory-read-like layout is accepted
    assert L.lib().s3r_gemm_tile_n(C.byref(d)) != -1, L.lib().s3r_last_error()
    d.lda, d.ldb = 0, 0
    setattr(d, field, value)
    _rejects(L, d, {"kc": "lda"}.get(field, field))


@pytest.mark.parametrize("change,field", [
    (dict(n=3840 - 256), "q_c"),                         # not a whole number of roles
    (dict(q_role_base=1), "q_role_base"),                # roles 1..5: there is no sixth
    (dict(n=3072, k2_out=None, vt2_out=None), "k2_out"),   # role 3 reached without its output
    (dict(vt2_out=None), "vt2_out"),
    (dict(n=768, q_role_base=2, vt_out=None), "vt_out"),
    (dict(q_out=None), "q_out"),
    (dict(q_ntok_pad=192), "q_ntok_pad"),                # shorter than q_ntok
    (dict(q_ntok_pad=198), "q_ntok_pad"),                # not a multiple of 4
    (dict(q_pos=None), "q_pos"),
    (dict(q_cs=None), "q_cs"),
])
def test_qkv_roles_outputs_padding_and_rope_inputs(L, change, field):
    d = _qkv(L)
    for k, v in change.items():
        setattr(d, k, v)
    _rejects(L, d, field)


def test_layout_kernels_reject_before_any_launch(L):
    lib = L.lib()
    # s3r_layernorm: swap_rows must split the rows into exactly two groups of swap_rows rows ...
    assert lib.s3r_layernorm(_p(1), 768, _p(2), _p(3), 768, 100, 1e-6, 150, 768, _p(4), 768, None, None, 0, 0, 100,
                             None) == -1
    assert b"swap_rows" in lib.s3r_last_error()
    # ... and its strides / offsets must keep the float4 / uint2 accesses aligned
    assert lib.s3r_layernorm(_p(1), 770, _p(2), _p(3), 0, 0, 1e-6, 8, 768, _p(4), 768, None, None, 0, 0, 0, None) == -1
    assert b"layernorm" in lib.s3r_last_error()
    assert lib.s3r_layernorm(_p(1), 768, _p(2), _p(3), 0, 0, 1e-6, 8, 768, None, 0, _p(5), _p(6), 1792, 2, 0, None) == -1
    assert b"col0" in lib.s3r_last_error()
    # s3r_split: strides and column offset
    assert lib.s3r_split(_p(1), 770, _p(2), _p(3), 768, 0, 8, 768, 0, None) == -1
    assert b"split" in lib.s3r_last_error()
    assert lib.s3r_split(_p(1), 768, _p(2), _p(3), 1792, 1026, 8, 768, 0, None) == -1
    assert b"col0" in lib.s3r_last_error()
    # s3r_im2col_3x3s2 copies 8 channels at a time
    assert lib.s3r_im2col_3x3s2(_p(1), _p(2), 1, 7, 9, 12, 4, 5, _p(3), _p(4), None) == -1
    assert b"im2col_3x3s2" in lib.s3r_last_error()


def test_attention_rejects_partial_batches_and_odd_strides(L):
    lib = L.lib()
    assert lib.s3r_attention(_p(1), _p(2), _p(3), 25, 12, 196, 196, 196, None, None, _p(4), 768, None) == -1
    assert b"heads" in lib.s3r_last_error()
    assert lib.s3r_attention(_p(1), _p(2), _p(3), 24, 12, 196, 196, 196, None, None, _p(4), 769, None) == -1
    assert b"ldo" in lib.s3r_last_error()
    good = dict(q=_p(1), k=_p(2), vt=_p(3), bh=24, heads=12, nq=196, nk=196, nk_pad=196, o_hi=_p(5), o_lo=_p(6),
                o_f32=_p(4), ldo=768)

    def attention(**change):
        a = {**good, **change}
        return lib.s3r_attention(*a.values(), None)

    for change, field in [
        (dict(o_lo=None), "o_hi and o_lo"),           # the kernel writes o_lo whenever o_hi is set
        (dict(o_hi=None), "o_hi and o_lo"),
        (dict(ldo=766), "ldo=766"),                   # narrower than heads * 64
        (dict(bh=65536, heads=16, ldo=1024), "bh=65536"),   # grid.y
        (dict(q=_p(1) + 8), "attention: q="),         # TMA bases: 16 bytes
        (dict(k=_p(2) + 4), "attention: k="),
        (dict(vt=_p(3) + 8), "attention: vt="),
        (dict(o_f32=_p(4) + 4), "attention: o_f32="),  # paired fp32 stores: 8 bytes
        (dict(o_hi=_p(5) + 2), "attention: o_hi="),    # paired bf16 stores: 4 bytes
        (dict(o_lo=_p(6) + 2), "attention: o_lo="),
        (dict(nk_pad=198), "nk_pad=198"),             # V^T rows of whole 16-byte groups
        (dict(nk_pad=192), "nk_pad=192"),             # shorter than nk
        (dict(nq=0, o_lo=None), "o_hi and o_lo"),     # empty sizes are checked too
    ]:
        assert attention(**change) == -1, change
        assert field.encode() in lib.s3r_last_error(), (change, lib.s3r_last_error())
    assert attention(nq=0) == 0   # empty: nothing to launch
