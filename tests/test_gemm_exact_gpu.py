"""The tensor-core GEMMs bit for bit: s3r_gemm, s3r_conv_wgrad and the native training Functions on operands whose
products and sums are exact in fp32 (gemm_exact.py), against the one correct answer computed in fp64.

Every comparison is `torch.equal` (through gemm_exact.assert_same, which reports the wrong elements per tile).  Operands,
bias and residuals are followed by NaN, and output memory outside the written window (columns past n inside ldo / ldp,
rows past M, the V^T padding, roles not written) holds a sentinel: no NaN may reach an output, no sentinel may change.
The premise -- at most 2^22 quanta of absolute terms per output -- is asserted on every case's data."""
import pytest
import torch

import gemm_exact as E

pytestmark = pytest.mark.gpu

SENT = -7.0e30       # fp32 sentinel of output memory outside the written window
PSENT = 3.0          # bf16 plane sentinel


@pytest.fixture(scope="module")
def L():
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


def _guarded(t: torch.Tensor) -> torch.Tensor:
    """A device copy of t followed by NaN: any read past its end poisons the result."""
    buf = torch.full((t.numel() + 4096,), float("nan"), dtype=t.dtype, device="cuda")
    v = buf[:t.numel()].view(t.shape)
    v.copy_(t)
    return v


def _strided(t: torch.Tensor, ld: int) -> torch.Tensor:
    """[rows, n] -> a [rows + 2, ld] buffer holding t in its first n columns, NaN everywhere else."""
    buf = torch.full((t.shape[0] + 2, ld), float("nan"), dtype=t.dtype, device="cuda")
    buf[:t.shape[0], :t.shape[1]] = t
    return buf


def _check_window(name, buf, exp, col0=0, tiles=None, sentinel=SENT):
    """buf [rows + extra, ld]: exp at [:rows, col0:col0 + n], the sentinel everywhere else."""
    rows, n = exp.shape
    E.assert_same(name, buf[:rows, col0:col0 + n], exp, tiles)
    rest = buf.clone()
    rest[:rows, col0:col0 + n] = sentinel
    bad = rest != sentinel
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} elements written outside the window, first at " \
                                f"{bad.nonzero()[0].tolist()}"


def _premise(terms: torch.Tensor, q: float):
    worst = float(terms.max())
    assert worst <= E.BUDGET * q, f"premise: {worst / q:.0f} quanta of absolute terms > 2^22"


def _gemm(L, G, NB, H, W, Kc, taps, N, *, precision=0, lo="planes", force_bn=0, bias=True, res1=True, res2=False,
          inplace=False, relu=False, plane_relu=False, ldo_pad=32, ldp_pad=32, col0=0, stats=False, a_swap=False,
          swap_col0=0, seed=0):
    """One EPI_PLAIN launch on exact operands: out_f32, both planes and (optionally) stats_out against fp64."""
    K = taps * Kc
    gen, emax = (E.Gen(1, 0), E.STATS_EPI) if stats else (E.pick_gen(K), E.EPI_MAX)
    q = gen.q
    rows = G * NB * H * W
    a = E.planes((G * NB, H, W, Kc), gen, seed, "cuda")
    b = E.planes((G * N, K), gen, seed + 1, "cuda")
    bias_t = E.ints((G * N,), emax, q, seed + 2, "cuda") if bias else None
    r1 = E.ints((rows, N), emax, q, seed + 3, "cuda") if (res1 or inplace) else None
    r2 = E.ints((rows, N), emax, q, seed + 4, "cuda") if res2 else None

    ah, bh = _guarded(a[0]), _guarded(b[0])
    if precision == 1 and lo == "null":
        al = bl = None
    elif precision == 1:   # lo planes that must never be read
        al, bl = _guarded(torch.full_like(a[1], float("nan"))), _guarded(torch.full_like(b[1], float("nan")))
    else:
        al, bl = _guarded(a[1]), _guarded(b[1])
    d = L.GemmDesc()
    d.a_hi, d.b_hi = ah.data_ptr(), bh.data_ptr()
    d.a_lo, d.b_lo = (al.data_ptr(), bl.data_ptr()) if al is not None else (None, None)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n = G, NB, H, W, Kc, taps, N
    d.epi, d.act, d.plane_relu, d.force_bn, d.precision = L.EPI_PLAIN, L.ACT_RELU if relu else L.ACT_NONE, int(plane_relu), \
        force_bn, precision
    d.a_swap, d.swap_col0 = int(a_swap), swap_col0
    keep = []
    if bias_t is not None:
        keep.append(_guarded(bias_t))
        d.bias = keep[-1].data_ptr()
    ldo = N + ldo_pad
    out = torch.full((rows + 3, ldo), SENT, device="cuda")
    d.out_f32, d.ldo = out.data_ptr(), ldo
    if inplace:
        out[:rows, :N] = r1
        d.res1, d.ldr1 = out.data_ptr(), ldo
    elif r1 is not None:
        keep.append(_strided(r1, N + 8))
        d.res1, d.ldr1 = keep[-1].data_ptr(), N + 8
    if r2 is not None:
        keep.append(_strided(r2, N + 4))
        d.res2, d.ldr2 = keep[-1].data_ptr(), N + 4
    ldp = col0 + N + ldp_pad
    ph = torch.full((rows + 3, ldp), PSENT, dtype=torch.bfloat16, device="cuda")
    pl = torch.full_like(ph, -PSENT)
    d.out_hi, d.out_lo, d.ldp, d.plane_col0 = ph.data_ptr(), pl.data_ptr(), ldp, col0
    st = None
    if stats:
        st = torch.full((rows + 3, N // 16), SENT, device="cuda")
        d.stats_out = st.data_ptr()
    L.gemm(d)
    torch.cuda.synchronize()

    acc = E.gemm_ref(a, b, G, taps, precision, a_swap, swap_col0).reshape(rows, N)
    bias_rows = None if bias_t is None else bias_t.view(G, 1, N).expand(G, rows // G, N).reshape(rows, N)
    terms = E.gemm_ref(a, b, G, taps, precision, a_swap, swap_col0, terms=True).reshape(rows, N)
    for t in (bias_rows, r1, r2):
        if t is not None:
            terms = terms + t.double().abs()
    _premise(terms, q)
    x = E.plain_epilogue(acc, bias_rows, relu, r1, r2)
    tiles = E.tile_ids(G * NB, H, W, N)
    _check_window("out_f32", out, x.float(), tiles=tiles)
    eh, el = E.split_ref(x.clamp_min(0) if plane_relu else x)
    _check_window("out_hi", ph, eh, col0, tiles, PSENT)
    _check_window("out_lo", pl, el, col0, tiles, -PSENT)
    if stats:
        _check_window("stats_out", st, E.stats_ref(x).reshape(rows, N // 16))


# ------------------------------------------------------------------------------------------------ s3r_gemm
PRECISIONS = [(0, "planes"), (1, "nan"), (1, "null")]


@pytest.mark.parametrize("force_bn", [0, 64, 128])
@pytest.mark.parametrize("precision,lo", PRECISIONS, ids=["split", "bf16-nan-lo", "bf16-null-lo"])
@pytest.mark.parametrize("geom", E.GEOMETRY, ids=["x".join(map(str, g)) for g in E.GEOMETRY])
def test_gemm_geometry(L, geom, precision, lo, force_bn):
    """Linear and 3x3 maps 1 x 1, 1 x W, H x 1, 7 x 7, 13 x 19, 130 x 3 with up to 3 images, channel tails
    (8 / 24 / 40 / 200), partial column tiles (32 / 96 / 160), ragged M, two groups; bias + residual."""
    _gemm(L, *geom, precision=precision, lo=lo, force_bn=force_bn, seed=sum(geom))


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("name,G,rows,K,N", E.SWEEP, ids=[s[0] for s in E.SWEEP])
def test_gemm_sweep_shapes(L, name, G, rows, K, N, precision):
    """The 14 launch shapes of tools/gemm_sweep.py at the planner's tile width."""
    _gemm(L, G, 1, 1, rows, K, 1, N, precision=precision, seed=K + N)


@pytest.mark.parametrize("rows,Kc,N,bn", E.RING)
def test_gemm_ring_wrap(L, rows, Kc, N, bn):
    """Persistent CTAs that wrap the operand ring over many tiles (test_gemm_ring_gpu.test_persistent_ring_wrap)."""
    _gemm(L, 1, 1, 1, rows, Kc, 1, N, force_bn=bn, seed=rows + Kc)


@pytest.mark.parametrize("force_bn", [64, 128])
@pytest.mark.parametrize("swap_col0", [0, 256])
@pytest.mark.parametrize("geom", [(2, 1, 1, 300, 96, 1, 512), (2, 2, 13, 19, 40, 9, 512)], ids=["linear", "3x3"])
def test_gemm_groups_a_swap(L, geom, swap_col0, force_bn):
    """groups = 2 with different data per group; a_swap from column swap_col0 on (0: every column)."""
    _gemm(L, *geom, force_bn=force_bn, a_swap=True, swap_col0=swap_col0, seed=7 + swap_col0)


MEMORY_READ = {   # G (slots), rows, Kc, N, lda, ldb, b_group_rows, res1
    # out = P V^T + feat: P rows mem_cap apart, Kc = bank length; V^T [1024, cap] per slot
    "value": (2, 77, 196, 96, 264, 200, 128, True),
    # S = Q K^T: each slot's keys cap rows apart, N = bank length (the chunk tail past N is unspecified)
    "score": (2, 77, 96, 100, 0, 0, 136, False),
}


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("layout", list(MEMORY_READ))
def test_gemm_memory_read_layout(L, layout, precision):
    """lda, ldb and b_group_rows as the engine's memory read sets them, with B staged before the dependency wait
    (b_static = 1).  The operands sit in NaN-padded buffers: a read of the padding would poison the result."""
    G, rows, Kc, N, lda, ldb, bgr, res = MEMORY_READ[layout]
    gen = E.pick_gen(Kc)
    q = gen.q
    a = E.planes((G, 1, rows, Kc), gen, 51, "cuda")
    b = E.planes((G * N, Kc), gen, 52, "cuda")
    bias = E.ints((G * N,), E.EPI_MAX, q, 53, "cuda")
    r1 = E.ints((G * rows, N), E.EPI_MAX, q, 54, "cuda") if res else None

    def b_rows(t):   # [G * b_group_rows, ldb]: group g's N rows from row g * b_group_rows on, NaN elsewhere
        buf = torch.full((G * bgr + 2, ldb or Kc), float("nan"), dtype=t.dtype, device="cuda")
        for g in range(G):
            buf[g * bgr:g * bgr + N, :Kc] = t[g * N:(g + 1) * N]
        return buf

    ap = [_strided(t.reshape(G * rows, Kc), lda or Kc) for t in a[:1 + (precision == 0)]]
    bp = [b_rows(t) for t in b[:1 + (precision == 0)]]
    bg = _guarded(bias)
    d = L.GemmDesc()
    d.a_hi, d.b_hi = ap[0].data_ptr(), bp[0].data_ptr()
    d.a_lo, d.b_lo = (ap[1].data_ptr(), bp[1].data_ptr()) if precision == 0 else (None, None)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n, d.precision = G, 1, 1, rows, Kc, 1, N, precision
    d.lda, d.ldb, d.b_group_rows, d.b_static = lda, ldb, bgr, 1
    d.epi, d.bias = L.EPI_PLAIN, bg.data_ptr()
    ldo = N + 32
    out = torch.full((G * rows + 3, ldo), SENT, device="cuda")
    d.out_f32, d.ldo = out.data_ptr(), ldo
    if r1 is not None:
        rg = _strided(r1, N + 8)
        d.res1, d.ldr1 = rg.data_ptr(), N + 8
    L.gemm(d)
    torch.cuda.synchronize()

    acc = E.gemm_ref(a, b, G, 1, precision).reshape(G * rows, N)
    bias_rows = bias.view(G, 1, N).expand(G, rows, N).reshape(G * rows, N)
    terms = E.gemm_ref(a, b, G, 1, precision, terms=True).reshape(G * rows, N) + bias_rows.double().abs()
    if r1 is not None:
        terms = terms + r1.double().abs()
    _premise(terms, q)
    out[:G * rows, N:(N + 31) // 32 * 32] = SENT   # the last chunk's columns past N hold unspecified values
    _check_window("out_f32", out, E.plain_epilogue(acc, bias_rows, False, r1).float(), tiles=E.tile_ids(G, 1, rows, N))


EPILOGUES = {
    "bare": dict(bias=False, res1=False),
    "bias": dict(res1=False),
    "bias-res1-res2": dict(res2=True),
    "inplace-res1-stats": dict(inplace=True, stats=True),
    "res1-res2-stats": dict(res2=True, stats=True),
    "relu": dict(relu=True),
    "plane-relu-res1-res2": dict(res2=True, plane_relu=True),
    "plane-window": dict(col0=256, ldp_pad=64, ldo_pad=96),
    "dense-ld": dict(ldo_pad=0, ldp_pad=0),
}


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("geom", [(1, 1, 1, 333, E.STATS_KC, 1, 160), (2, 2, 7, 9, 32, 9, 96)], ids=["linear", "3x3"])
@pytest.mark.parametrize("epi", list(EPILOGUES))
def test_gemm_epilogues(L, epi, geom, precision):
    """Bias, res1, res2, in-place res1, ReLU, plane_relu, plane_col0 / ldp windows and stats_out."""
    kw = dict(EPILOGUES[epi])
    G, NB, H, W, Kc, taps, N = geom
    if kw.get("stats"):
        geom = (G, NB, H, W, E.STATS_KC if taps == 1 else 8, taps, N)   # 9 x 8 = 72 terms: small outputs
    _gemm(L, *geom, precision=precision, seed=len(epi), **kw)


@pytest.mark.parametrize("s,cout,G,NB,H,W", [(2, 32, 1, 2, 7, 9), (4, 96, 1, 1, 14, 14), (2, 64, 2, 3, 3, 1),
                                             (4, 32, 2, 1, 1, 5)])
@pytest.mark.parametrize("precision", [0, 1])
def test_gemm_pixshuf(L, s, cout, G, NB, H, W, precision):
    """EPI_PIXSHUF (ConvTranspose2d with kernel == stride): column (i, j, co) of pixel (h, w) goes to pixel
    (h s + i, w s + j), channel co; bias per (group, co); a residual in the output layout; fp32 and planes."""
    Kc, N = 40, s * s * cout
    gen = E.pick_gen(Kc)
    q = gen.q
    a = E.planes((G * NB, H, W, Kc), gen, 11, "cuda")
    b = E.planes((G * N, Kc), gen, 12, "cuda")
    bias = E.ints((G * cout,), E.EPI_MAX, q, 13, "cuda")
    orows = G * NB * H * s * W * s
    res = E.ints((orows, cout), E.EPI_MAX, q, 14, "cuda")
    ah, bh = _guarded(a[0]), _guarded(b[0])
    al, bl = (_guarded(a[1]), _guarded(b[1])) if precision == 0 else (None, None)
    bg, rg = _guarded(bias), _strided(res, cout + 4)
    out = torch.full((orows + 3, cout + 32), SENT, device="cuda")
    ph = torch.full((orows + 3, cout + 64), PSENT, dtype=torch.bfloat16, device="cuda")
    pl = torch.full_like(ph, -PSENT)
    d = L.GemmDesc()
    d.a_hi, d.b_hi = ah.data_ptr(), bh.data_ptr()
    d.a_lo, d.b_lo = (al.data_ptr(), bl.data_ptr()) if al is not None else (None, None)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n, d.precision = G, NB, H, W, Kc, 1, N, precision
    d.epi, d.ps_s, d.ps_cout, d.bias = L.EPI_PIXSHUF, s, cout, bg.data_ptr()
    d.res1, d.ldr1 = rg.data_ptr(), cout + 4
    d.out_f32, d.ldo = out.data_ptr(), cout + 32
    d.out_hi, d.out_lo, d.ldp, d.plane_col0 = ph.data_ptr(), pl.data_ptr(), cout + 64, 32
    L.gemm(d)
    torch.cuda.synchronize()
    acc = E.gemm_ref(a, b, G, 1, precision)                                 # [G*NB, H, W, s*s*cout]
    y = acc.view(G * NB, H, W, s, s, cout).permute(0, 1, 3, 2, 4, 5).reshape(G, orows // G, cout)
    x = (y + bias.double().view(G, 1, cout)).reshape(orows, cout) + res.double()
    terms = E.gemm_ref(a, b, G, 1, precision, terms=True).abs().max() + bias.abs().max() + res.abs().max()
    _premise(terms, q)
    _check_window("out_f32", out, x.float())
    eh, el = E.split_ref(x)
    _check_window("out_hi", ph, eh, 32, sentinel=PSENT)
    _check_window("out_lo", pl, el, 32, sentinel=-PSENT)


def _quarter_turns(maxpos, seed):
    """[maxpos, 16, 2] (cos, sin) in {(1, 0), (0, 1), (-1, 0), (0, -1)}, random per position and pair: RoPE is exact."""
    k = torch.randint(0, 4, (maxpos, 16), generator=torch.Generator().manual_seed(seed))
    cs = torch.tensor([[1.0, 0.0], [0.0, 1.0], [-1.0, 0.0], [0.0, -1.0]])[k]
    return cs.contiguous().cuda()


QKV_CASES = {   # G, q_nb, ntok, ntok_pad, heads, role_base, roles, rope, a_swap (swap_col0 = 3 q_c)
    "merged-5-roles-swap": (2, 2, 37, 40, 4, 0, 5, 1, 1),
    "qkv-3-roles": (1, 3, 50, 52, 2, 0, 3, 1, 0),
    "kv": (2, 1, 64, 64, 4, 1, 2, 1, 0),
    "k2-vt2": (2, 2, 21, 24, 1, 3, 2, 1, 0),
    "q-only": (2, 1, 130, 132, 2, 0, 1, 1, 0),
    "no-rope": (1, 2, 33, 36, 2, 0, 3, 0, 0),
}


@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("case", list(QKV_CASES))
def test_gemm_qkv(L, case, precision):
    """EPI_QKV: head split of q / k / V^T (and the second K / V^T pair, roles 3 and 4), RoPE under random quarter turns
    (pairing, position lookup and the positions of the swapped group exact), q scaled by 0.125, tf32 rounding exact on
    values below 2^11 quanta.  Buffers of roles the launch does not write, and the V^T padding, keep their sentinel."""
    G, q_nb, ntok, npad, heads, base, nroles, rope, swap = QKV_CASES[case]
    qc, Kc = 64 * heads, E.QKV_KC
    n, rows = nroles * qc, q_nb * ntok
    swap_col0 = 3 * qc if swap else 0
    gen = E.Gen(1, 1)
    q = gen.q
    a = E.planes((G, 1, rows, Kc), gen, 21, "cuda")
    b = E.planes((G * n, Kc), gen, 22, "cuda")
    bias = E.ints((G * n,), E.QKV_BIAS, q, 23, "cuda")
    maxpos = 40
    pos = torch.randint(0, maxpos, (G * rows, 2), generator=torch.Generator().manual_seed(24)).to(torch.int32).cuda()
    cs = _quarter_turns(maxpos, 25)
    ah, bh = _guarded(a[0]), _guarded(b[0])
    al, bl = (_guarded(a[1]), _guarded(b[1])) if precision == 0 else (None, None)
    bg, csg = _guarded(bias), _guarded(cs)   # positions index the table: no poison past their end
    shape_qk = (G * q_nb, heads, ntok, 64)
    shape_vt = (G * q_nb, heads, 64, npad)
    outs = {r: torch.full((torch.Size(shape_vt if r in (2, 4) else shape_qk).numel() + 64,), SENT, device="cuda")
            for r in range(5)}
    d = L.GemmDesc()
    d.a_hi, d.b_hi = ah.data_ptr(), bh.data_ptr()
    d.a_lo, d.b_lo = (al.data_ptr(), bl.data_ptr()) if al is not None else (None, None)
    d.groups, d.nb, d.h, d.w, d.kc, d.taps, d.n, d.precision = G, 1, 1, rows, Kc, 1, n, precision
    d.epi, d.bias = L.EPI_QKV, bg.data_ptr()
    d.q_c, d.q_role_base, d.q_ntok, d.q_ntok_pad, d.q_rope, d.q_nb = qc, base, ntok, npad, rope, q_nb
    d.q_pos, d.q_cs, d.q_scale = pos.data_ptr(), csg.data_ptr(), 0.125
    d.q_out, d.k_out, d.vt_out, d.k2_out, d.vt2_out = (outs[r].data_ptr() for r in range(5))
    d.a_swap, d.swap_col0 = swap, swap_col0
    L.gemm(d)
    torch.cuda.synchronize()

    acc = E.gemm_ref(a, b, G, 1, precision, bool(swap), swap_col0).view(G, rows, n)
    y = acc + bias.double().view(G, 1, n)
    _premise(E.gemm_ref(a, b, G, 1, precision, bool(swap), swap_col0, terms=True).view(G, rows, n)
             + bias.double().abs().view(G, 1, n), q)
    assert float(y.abs().max()) < 2 ** 11 * q
    exp = {r: torch.full_like(outs[r], SENT) for r in range(5)}
    yr = y.view(G, q_nb, ntok, nroles, heads, 64)
    p = pos.long().view(G, q_nb, ntok, 2)
    for ri in range(nroles):
        role = base + ri
        v = yr[:, :, :, ri]                                                  # [G, q_nb, ntok, heads, 64]
        if role not in (2, 4) and rope:
            pg = p.flip(0) if (swap and ri * qc >= swap_col0) else p           # positions of the A rows' group
            t = cs.double()[pg]                                              # [G, q_nb, ntok, 2 (y, x), 16, 2]
            c, s_ = t[..., 0].unsqueeze(3), t[..., 1].unsqueeze(3)           # [G, q_nb, ntok, 1, 2, 16]
            v = v.reshape(G, q_nb, ntok, heads, 2, 2, 16)
            u, w = v[..., 0, :], v[..., 1, :]
            v = torch.stack((u * c - w * s_, w * c + u * s_), -2).reshape(G, q_nb, ntok, heads, 64)
        if role == 0:
            v = v * 0.125
        if role in (2, 4):
            vt = torch.full(shape_vt, SENT, dtype=torch.float64, device="cuda")
            vt[..., :ntok] = v.permute(0, 1, 3, 4, 2).reshape(G * q_nb, heads, 64, ntok)
            exp[role][:vt.numel()] = vt.reshape(-1).float()
        else:
            exp[role][:v.numel()] = v.permute(0, 1, 3, 2, 4).reshape(-1).float()
    for r, name in enumerate(("q_out", "k_out", "vt_out", "k2_out", "vt2_out")):
        E.assert_same(name, outs[r].view(-1, 64), exp[r].view(-1, 64))


# ------------------------------------------------------------------------------------------------ s3r_conv_wgrad
WGRAD = E.wgrad_cases()


@pytest.mark.parametrize("shape", WGRAD, ids=["x".join(map(str, s)) for s in WGRAD])
def test_conv_wgrad_exact(L, shape):
    """dW of every DPT / patch-embedding conv at 224 x 224, 288 x 224 and 512 x 384 (B = 1, 4) and the ragged shapes:
    the split contraction over pixels and the fixed-order reduce of the splits give the exact sum."""
    nb, h, w, n, kc, taps = shape
    P = nb * h * w
    gen = E.pick_gen(P, E.BUDGET)
    dy = E.planes((nb, h, w, n), gen, P % 997, "cuda")
    x = E.planes((nb, h, w, kc), gen, P % 991 + 1, "cuda")
    g = [_guarded(t) for t in dy + x]
    lib = L.lib()
    ws_bytes = lib.s3r_conv_wgrad_workspace_bytes(nb, h, w, n, kc, taps)
    assert ws_bytes > 0
    ws = torch.empty(ws_bytes // 4, device="cuda")
    dw = torch.full((n * taps * kc + 64,), SENT, device="cuda")
    L.check(lib.s3r_conv_wgrad(L.ptr(g[0]), L.ptr(g[1]), n, L.ptr(g[2]), L.ptr(g[3]), kc, nb, h, w, n, kc, taps,
                               L.ptr(ws), ws_bytes, L.ptr(dw), L.stream_ptr()), "s3r_conv_wgrad")
    torch.cuda.synchronize()
    _premise(E.wgrad_ref(dy, x, taps, terms=True), gen.q)
    exp = E.wgrad_ref(dy, x, taps).float()
    tiles = (torch.arange(n)[:, None, None] // 128 * 10000 + torch.arange(taps)[None, :, None] * 100 +
             torch.arange(kc)[None, None, :] // 128).view(n, -1)
    E.assert_same("dW", dw[:exp.numel()].view(n, -1), exp.view(n, -1), tiles)
    assert bool((dw[exp.numel():] == SENT).all()), "dW written past its end"


# ------------------------------------------------------------------------------------------------ native Functions
@pytest.mark.parametrize("rows,K,N", [(77, 96, 64), (1000, 768, 256), (3, 64, 32)])
def test_native_linear_exact(rows, K, N):
    """_NativeLinear on bf16-exact fp32 inputs (lo planes 0): y, dx, dW and db are exact; 77 and 3 rows pad the wgrad
    contraction with zeros to a multiple of 8."""
    from spann3r_b200._native_linear import _NativeLinear
    x = E.exact_f32((rows, K), 31, "cuda", e=-1).requires_grad_(True)
    w = E.exact_f32((N, K), 32, "cuda").requires_grad_(True)
    b = E.exact_f32((N,), 33, "cuda", M=100).requires_grad_(True)
    gy = E.exact_f32((rows, N), 34, "cuda", M=5)
    y = _NativeLinear.apply(x, w, b)
    gx, gw, gb = torch.autograd.grad(y, (x, w, b), gy)
    xd, wd, gd = x.detach().double(), w.detach().double(), gy.double()
    E.assert_same("y", y.detach(), (xd @ wd.t() + b.detach().double()).float())
    E.assert_same("dx", gx, (gd @ wd).float())
    E.assert_same("dW", gw, (gd.t() @ xd).float())
    E.assert_same("db", gb, gd.sum(0).float())


NATIVE_CONVS = [   # kind, cin, cout, nb, h, w
    ("1x1", 96, 64, 2, 7, 9), ("3x3", 64, 32, 2, 13, 19), ("3x3", 32, 96, 1, 1, 5), ("3x3s2", 32, 64, 2, 7, 9),
    ("3x3s2", 64, 32, 1, 14, 14), ("convT2", 64, 32, 2, 5, 7), ("convT4", 96, 96, 1, 3, 4), ("patch", 3, 64, 2, 32, 48),
]


@pytest.mark.parametrize("kind,cin,cout,nb,h,w", NATIVE_CONVS, ids=[f"{c[0]}-{c[1]}-{c[2]}-{c[4]}x{c[5]}" for c in NATIVE_CONVS])
def test_native_conv_exact(kind, cin, cout, nb, h, w):
    """_native_conv's Functions (1x1, 3x3, 3x3 stride 2 through im2col / col2im, ConvTranspose, patch) on bf16-exact
    inputs: y, dx, dW and db equal fp64 autograd bit for bit."""
    from test_native_conv_gpu import _native_call, _torch_call
    if kind.startswith("convT"):
        s = int(kind[-1])
        wt = E.exact_f32((cin, cout, s, s), 41, "cuda")
    else:
        k = 16 if kind == "patch" else (1 if kind == "1x1" else 3)
        wt = E.exact_f32((cout, cin, k, k), 41, "cuda")
    x = E.exact_f32((nb, cin, h, w), 42, "cuda", e=-2)
    bias = E.exact_f32((cout,), 43, "cuda", M=50)
    wt.requires_grad_(True)
    bias.requires_grad_(True)
    x.requires_grad_(kind != "patch")
    y = _native_call(kind, x, wt, bias)
    gy = E.exact_f32(tuple(y.shape), 44, "cuda", M=2)
    wrt = [t for t in (x, wt, bias) if t.requires_grad]
    got = torch.autograd.grad(y, wrt, gy)
    ref_in = [t.detach().double().requires_grad_(t.requires_grad) for t in (x, wt, bias)]
    yr = _torch_call(kind, *ref_in)
    ref = torch.autograd.grad(yr, [t for t in ref_in if t.requires_grad], gy.double())
    E.assert_same("y", y.detach().contiguous(), yr.detach().float().contiguous())
    for name, a, r in zip([nm for nm, t in zip(("dx", "dW", "db"), (x, wt, bias)) if t.requires_grad], got, ref):
        E.assert_same(name, a.contiguous(), r.float().contiguous())
