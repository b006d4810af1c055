"""The eval attention core (`s3r_attention`, csrc/attention.cu) against fp64, element by element.

Inputs are rounded to tf32 with the kernel's own round-to-nearest (`tf32`), as its contract requires (the QKV epilogue
does it in the engine); q carries the 64^-0.5 scale.  The reference is softmax(q k^T) v in fp64.

Per-element bound.  Write the kernel's weight of key j in row r as P~_j = c_r p_j (1 + g_j), p the fp64 softmax and c_r
a factor common to the row.  O_r = sum_j P~_j v_j / sum_j P~_j because the row sum l adds the SAME rounded values the
P V product multiplies, so c_r cancels and, with d_j = v_j - ref_r (sum_j p_j d_j = 0),

    O_r - ref_r = sum_j p_j g_j d_j / (1 + sum_j p_j g_j).

g_j = eta_j + xi_j: eta_j is the tf32 rounding of P (round-to-nearest: |eta_j| <= u = 2^-11), xi_j the fp32 error of the
exponent (scores, running max, exp2f).  The row's maximum key gets exp2f(~0) = 1, which tf32 holds exactly: eta = 0 for
it.  Hence, with j* the fp64 argmax,

    |O_rc - ref_rc| <= (u sum_{j != j*} p_j |d_jc| + eps_r sum_j p_j |d_jc|) / (1 - u - eps_r) + kappa sum_j p_j |v_jc|

    eps_r  = 2 ds_r + 2^-24 (1.5 |m_r| + 6 R_r) + 2^-22 (nblk + 1)
    ds_r   = 2^-20 max_j sum_c |q_rc k_jc|            scores: 8 wgmma k-steps, <= 1 ulp of the running |sum| each
    kappa  = 2^-23 ceil(nk / 8) + 2^-24 (35 nblk + 4) P V: 1 ulp per 8-key k-step; the block rescales, 1 / l, l's sums

m_r is the row's top score, R_r = min(m_r - min_j s_rj, 104) its range (weights below e^-104 are under fp32's denormals and
carry nothing), nblk = ceil(nk / 128) the key blocks.  The score and P V terms model the tensor core's fp32 accumulation
as at most one ulp of the running absolute sum per k-step; they are assumptions about the hardware, not a specification,
and the GPU tests report how much of the bound the kernel uses.

Truncating P instead of rounding it keeps the normalisation consistent, so a bias common to every weight cancels; what
the bound sees is that the max key's weight stays exact while every other weight moves by up to 2 u, all downwards.  On
rows with two dominant keys whose second weight has a mantissa just above a power of two and a fractional part in the
upper half of a tf32 ulp (`two_key_rows`), truncation uses 1.8x the bound in the fp64 emulation and rounding 0.47x.  On
random rows the emulated truncation leaves the bound only sometimes (0.8x .. 1.6x over the CPU cases), so only the two-key
rows are relied on to tell the two apart (`test_bound_holds_for_rn_emulation_and_fails_for_truncation`).

Largest |O - ref| / bound measured on H100 80GB HBM3 cards at 400 W and at 700 W power limits (the same on both):
engine shapes 0.63, ragged sizes 0.71, two-key rows 0.47, peaked rows 0.045, uniform rows 1.1e-4.  The bound is rigorous
under the model above, so each test asserts the ratio stays below 1.

The bound cannot see changes of about one ulp to the kernel's arithmetic, such as l summing the unrounded e, an
approximate 1 / l or a stale rescale.  test_attn_core_exact_gpu.py pins those: on exactly representable inputs
(attn_core_exact.py) it holds the kernel to its one correct fp32 answer bit for bit, at the same shapes as this file.
"""
import math

import pytest
import torch

U = 2.0 ** -11
MAX_RANGE = 104.0


# ------------------------------------------------------------------------------------------------
# helpers (pure; checked on the CPU below)
# ------------------------------------------------------------------------------------------------
def tf32(x: torch.Tensor) -> torch.Tensor:
    """fp32 -> tf32 with the kernel's round-to-nearest (add half an ulp of the 10-bit mantissa, clear the low 13 bits)."""
    return ((x.float().contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)


def tf32_trunc(x: torch.Tensor) -> torch.Tensor:
    return (x.float().contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def emulate(q, k, v, rounding=tf32):
    """fp64 emulation of the kernel's softmax arithmetic on [BH, nq, 64] / [BH, nk, 64] inputs: e = fp32(exp(s - max)),
    P = rounding(e), l = sum P (consistent with P), O = P V / l."""
    s = q.double() @ k.double().transpose(-1, -2)
    e = (s - s.amax(-1, keepdim=True)).exp().float()
    p = rounding(e).double()
    return (p @ v.double()) / p.sum(-1, keepdim=True)


def bound(q, k, v, chunk=8):
    """(ref [BH, nq, 64], bound [BH, nq, 64]) in fp64: the per-element bound of the module docstring."""
    BH, nq, _ = q.shape
    nk = k.shape[1]
    nblk = (nk + 127) // 128
    kappa = 2.0 ** -23 * math.ceil(nk / 8) + 2.0 ** -24 * (35 * nblk + 4)
    refs, bounds = [], []
    for b0 in range(0, BH, chunk):
        qd, kd, vd = q[b0:b0 + chunk].double(), k[b0:b0 + chunk].double(), v[b0:b0 + chunk].double()
        s = qd @ kd.transpose(-1, -2)
        p = s.softmax(-1)
        ref = p @ vd
        m = s.amax(-1)
        rng = (m - s.amin(-1)).clamp(max=MAX_RANGE)
        ds = 2.0 ** -20 * (qd.abs() @ kd.abs().transpose(-1, -2)).amax(-1)
        eps = 2 * ds + 2.0 ** -24 * (1.5 * m.abs() + 6 * rng) + 2.0 ** -22 * (nblk + 1)
        jstar = s.argmax(-1)                                                          # [b, nq]
        pv_abs = p @ vd.abs()
        spd = torch.empty_like(ref)
        sxd = torch.empty_like(ref)
        for r0 in range(0, nq, 256):                                                  # sum_j p_j |v_j - ref_r|
            d = (vd[:, None, :, :] - ref[:, r0:r0 + 256, None, :]).abs()             # [b, rows, nk, 64]
            pr = p[:, r0:r0 + 256]
            spd[:, r0:r0 + 256] = torch.einsum("brj,brjc->brc", pr, d)
            js = jstar[:, r0:r0 + 256]
            dstar = torch.gather(d, 2, js[..., None, None].expand(-1, -1, 1, 64)).squeeze(2)
            sxd[:, r0:r0 + 256] = spd[:, r0:r0 + 256] - torch.gather(pr, 2, js[..., None]) * dstar
        e = eps[..., None]
        bnd = (U * sxd.clamp_min(0) + e * spd) / (1 - U - e) + kappa * pv_abs + 2.0 ** -100 * vd.abs().amax()
        refs.append(ref)
        bounds.append(bnd)
    return torch.cat(refs), torch.cat(bounds)


def bound_ratio(o, ref, bnd):
    """Largest |o - ref| / bound (NaN in o counts as a violation)."""
    err = (o.double() - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    return float((err / bnd).max())


def two_key_gaps(n: int) -> torch.Tensor:
    """n score gaps g (tf32-exact) whose weight exp(-g) has a mantissa in [1, 1.1) and a fractional part in [0.75, 0.95)
    of a tf32 ulp: round-to-nearest moves it by <= 0.5 u, truncation by >= 1.36 u."""
    x = torch.linspace(0.05, 6.0, 400000, dtype=torch.float64)
    g = tf32(x.float()).double().unique()
    e = (-g).exp()
    E = torch.floor(torch.log2(e))
    mant = e / 2.0 ** E
    frac = torch.remainder(e / 2.0 ** (E - 10), 1.0)
    g = g[(mant < 1.1) & (frac >= 0.75) & (frac < 0.95)]
    return g[torch.arange(n) % g.numel()]


def two_key_rows(BH: int, nq: int, seed: int):
    """q [BH, nq, 64], k [BH, 2, 64], v [BH, 2, 64]: key 0 scores 0, key 1 scores -g_r (`two_key_gaps`), both exact."""
    gen = torch.Generator().manual_seed(seed)
    g = two_key_gaps(BH * nq).view(BH, nq)
    q = torch.zeros(BH, nq, 64)
    q[..., 0] = g.float()
    k = torch.zeros(BH, 2, 64)
    k[:, 1, 0] = -1.0
    v = tf32(torch.randn(BH, 2, 64, generator=gen))
    return q, k, v


def peaked_rows(BH: int, nq: int, nk: int, seed: int):
    """Each row's top score exceeds its next by 20 .. 60: q_r = beta_r k_{j*} with beta_r set from that row's margin."""
    gen = torch.Generator().manual_seed(seed)
    k = tf32(torch.randn(BH, nk, 64, generator=gen))
    js = torch.randint(0, nk, (BH, nq), generator=gen)
    kstar = torch.gather(k, 1, js[..., None].expand(-1, -1, 64))                     # [BH, nq, 64]
    dots = kstar.double() @ k.double().transpose(-1, -2)                            # [BH, nq, nk]
    top = torch.gather(dots, 2, js[..., None]).squeeze(-1)
    other = dots.scatter(2, js[..., None], -float("inf")).amax(-1) if nk > 1 else top - 64
    gap = 20 + 40 * torch.rand(BH, nq, generator=gen, dtype=torch.float64)
    beta = gap / (top - other)
    return tf32((beta[..., None] * kstar.double()).float()), k, tf32(torch.randn(BH, nk, 64, generator=gen))


def random_rows(BH, nq, nk, seed, qscale=0.3):
    gen = torch.Generator().manual_seed(seed)
    q = tf32(torch.randn(BH, nq, 64, generator=gen) * qscale)
    k = tf32(torch.randn(BH, nk, 64, generator=gen))
    v = tf32(torch.randn(BH, nk, 64, generator=gen))
    return q, k, v


# ------------------------------------------------------------------------------------------------
# CPU: the bound against the emulation, and the helpers
# ------------------------------------------------------------------------------------------------
def test_tf32_rounding_helpers():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -11 + 2 ** -20, 1.0 + 2 ** -10, -(1.0 + 3 * 2 ** -12)])
    assert tf32(x).tolist() == [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -10, 1.0 + 2 ** -10, -(1.0 + 2 ** -10)]
    assert tf32_trunc(x).tolist() == [1.0, 1.0, 1.0, 1.0 + 2 ** -10, -1.0]
    y = torch.randn(10000, dtype=torch.float64).float()
    assert float(((tf32(y).double() - y.double()) / y.double()).abs().max()) <= U
    assert float(((tf32_trunc(y).double() - y.double()) / y.double()).abs().max()) < 2 * U
    g = two_key_gaps(64)
    e = (-g).exp()
    assert float(((tf32_trunc(e.float()).double() - e) / e).abs().min()) > 1.3 * U
    assert float(((tf32(e.float()).double() - e) / e).abs().max()) <= 0.5 * U


def test_peaked_rows_have_the_asked_margin():
    q, k, v = peaked_rows(3, 50, 70, seed=1)
    s = (q.double() @ k.double().transpose(-1, -2)).sort(-1, descending=True).values
    gap = s[..., 0] - s[..., 1]
    assert float(gap.min()) > 19.0 and float(gap.max()) < 61.0


@pytest.mark.parametrize("nq,nk", [(64, 2), (100, 300), (200, 768), (33, 129)])
def test_bound_holds_for_rn_emulation_and_fails_for_truncation(nq, nk):
    """The emulation (tf32 RN of P, consistent l, everything else exact) stays inside the bound on random, peaked and
    uniform rows; with P truncated it leaves the bound on two-dominant-key rows."""
    for q, k, v in (random_rows(2, nq, nk, seed=3), random_rows(2, nq, nk, seed=4, qscale=1.0),
                    peaked_rows(2, nq, nk, seed=5), (torch.zeros(2, nq, 64),) + random_rows(2, nq, nk, seed=6)[1:]):
        ref, bnd = bound(q, k, v)
        assert bound_ratio(emulate(q, k, v), ref, bnd) < 1.0
    q, k, v = two_key_rows(2, nq, seed=7)
    ref, bnd = bound(q, k, v)
    assert bound_ratio(emulate(q, k, v), ref, bnd) < 0.6
    assert bound_ratio(emulate(q, k, v, tf32_trunc), ref, bnd) > 1.5


def test_bound_catches_a_wrong_row():
    """The bound is per element: one row averaged over one key too many leaves it."""
    q, k, v = random_rows(1, 40, 100, seed=8)
    ref, bnd = bound(q, k, v)
    bad = emulate(q, k, v).clone()
    bad[0, 17] = emulate(q[:, 17:18], k[:, :99], v[:, :99])[0, 0]
    assert bound_ratio(bad, ref, bnd) > 10


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from spann3r_b200 import _lib
    _lib.require_device()
    return _lib


SENT = -3.0 * 2.0 ** 100   # sentinel of the output columns / rows the kernel must not write (exact in fp32 and bf16)


def run(L, q, k, v, heads, nk_pad=None, pad_fill=0.0, ldo=None, f32=True, planes=True, guard=0):
    """s3r_attention on [BH, nq, 64] q, [BH, nk, 64] k and v (V^T built with nk_pad columns, the extra ones = pad_fill).
    Returns (o [rows + guard, ldo] fp32 or None, hi, lo or None) with every cell the kernel must not touch = SENT."""
    BH, nq, _ = q.shape
    nk = k.shape[1]
    nk_pad = nk_pad or (nk + 3) // 4 * 4
    ldo = ldo or heads * 64
    vt = torch.full((BH, 64, nk_pad), pad_fill, device="cuda")
    vt[..., :nk] = v.cuda().transpose(1, 2)
    rows = BH // heads * nq
    o = torch.full((rows + guard, ldo), SENT, device="cuda") if f32 else None
    hi = torch.full((rows + guard, ldo), SENT, dtype=torch.bfloat16, device="cuda") if planes else None
    lo = torch.full_like(hi, SENT) if planes else None
    qc, kc = q.cuda().contiguous(), k.cuda().contiguous()
    L.check(L.lib().s3r_attention(L.ptr(qc), L.ptr(kc), L.ptr(vt), BH, heads, nq, nk, nk_pad, L.ptr(hi), L.ptr(lo),
                                  L.ptr(o), ldo, L.stream_ptr()), "s3r_attention")
    torch.cuda.synchronize()
    return o, hi, lo


def heads_view(o, BH, heads, nq):
    """[B nq, >= heads 64] kernel output -> [BH, nq, 64]."""
    return o[: BH // heads * nq, : heads * 64].reshape(BH // heads, nq, heads, 64).transpose(1, 2).reshape(BH, nq, 64)


def check_bound(L, name, q, k, v, heads, **kw):
    BH, nq, _ = q.shape
    o, _, _ = run(L, q, k, v, heads, planes=False, **kw)
    ref, bnd = bound(q.cuda(), k.cuda(), v.cuda())
    r = bound_ratio(heads_view(o, BH, heads, nq), ref, bnd)
    print(f"{name} BH={BH} heads={heads} nq={nq} nk={k.shape[1]}: max |O - ref| / bound = {r:.3e}")
    assert r < 1.0, (name, r)
    return o


# (BH, heads, N) of every geometry of tests/test_stages_gpu.py: the encoder (16 heads, 2 B or 3 images) and the decoder
# (12 heads x 2 B) at N = 196, 768, 672 (21 x 32) and 195 (13 x 15, V^T padded to 196)
ENGINE_SHAPES = [(48, 16, 196), (24, 12, 196), (80, 16, 196), (48, 12, 196), (48, 16, 768), (24, 12, 768),
                 (48, 16, 672), (24, 12, 672), (48, 16, 195), (24, 12, 195)]


@pytest.mark.gpu
@pytest.mark.parametrize("BH,heads,N", ENGINE_SHAPES)
def test_engine_shapes_within_bound(L, BH, heads, N):
    q, k, v = random_rows(BH, N, N, seed=N + BH)
    check_bound(L, "engine_shapes", q, k, v, heads)


SQUARE = [1, 2, 63, 64, 65, 127, 128, 129, 195, 255, 256, 257]
RECT = [(127, 129), (129, 127), (1, 300), (300, 1), (128, 257), (257, 128), (200, 64), (64, 200)]


@pytest.mark.gpu
@pytest.mark.parametrize("nq,nk", [(n, n) for n in SQUARE] + RECT)
def test_ragged_sizes_within_bound(L, nq, nk):
    q, k, v = random_rows(6, nq, nk, seed=nq * 1000 + nk, qscale=0.5)
    check_bound(L, "ragged", q, k, v, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("nk", [1, 2, 129, 195, 300])
def test_peaked_and_uniform_rows(L, nk):
    """Peaked rows (top score 20 .. 60 above the next) return their key's value; uniform rows (q = 0) the mean of V."""
    q, k, v = peaked_rows(4, 130, nk, seed=nk)
    check_bound(L, "peaked", q, k, v, 2)
    zq = torch.zeros(4, 130, 64)
    check_bound(L, "uniform", zq, k, v, 2)       # the fp64 reference of these rows is the mean of V


@pytest.mark.gpu
def test_two_dominant_keys_within_bound(L):
    """Rows where truncating P instead of rounding it would leave the bound (see the module docstring)."""
    q, k, v = two_key_rows(4, 200, seed=9)
    check_bound(L, "two_keys", q, k, v, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("nk", [195, 257, 301])
def test_padded_vt_columns_are_never_read(L, nk):
    """V^T with nk_pad > nk: NaN in the padding columns (one more 16-byte group than needed, too) changes no bit."""
    q, k, v = random_rows(24, 200, nk, seed=nk)
    o0, _, _ = run(L, q, k, v, 12, planes=False)
    o1, _, _ = run(L, q, k, v, 12, pad_fill=float("nan"), planes=False)
    o2, _, _ = run(L, q, k, v, 12, nk_pad=(nk + 3) // 4 * 4 + 8, pad_fill=float("nan"), planes=False)
    assert bool(torch.isfinite(o1).all()) and bool(torch.isfinite(o2).all())
    assert torch.equal(o0, o1) and torch.equal(o0, o2)


@pytest.mark.gpu
@pytest.mark.parametrize("nq,nk", [(195, 195), (129, 64), (257, 300)])
def test_outputs_stay_in_their_columns_and_rows(L, nq, nk):
    """ldo > heads 64 and a guard row: the extra columns and the row after the last are untouched, in the fp32 output
    and in both planes; fp32-only, planes-only and both give the same values, the planes = split(fp32) bit for bit."""
    BH, heads, ldo = 24, 12, 12 * 64 + 6
    rows = BH // heads * nq
    q, k, v = random_rows(BH, nq, nk, seed=nq + nk)
    o, hi, lo = run(L, q, k, v, heads, ldo=ldo, guard=1)
    of, _, _ = run(L, q, k, v, heads, ldo=ldo, guard=1, planes=False)
    _, ph, pl = run(L, q, k, v, heads, ldo=ldo, guard=1, f32=False)
    for t in (o, hi, lo, of, ph, pl):
        assert bool((t[:, heads * 64:].float() == SENT).all()) and bool((t[rows:].float() == SENT).all())
    assert torch.equal(o, of) and torch.equal(hi, ph) and torch.equal(lo, pl)
    sh, sl = L.split(o[:rows, : heads * 64].contiguous())
    assert torch.equal(sh, hi[:rows, : heads * 64]) and torch.equal(sl, lo[:rows, : heads * 64])
    ref, bnd = bound(q.cuda(), k.cuda(), v.cuda())
    assert bound_ratio(heads_view(o, BH, heads, nq), ref, bnd) < 1.0


@pytest.mark.gpu
def test_bitwise_reproducible(L):
    q, k, v = random_rows(48, 195, 195, seed=11)
    a = run(L, q, k, v, 16)
    b = run(L, q, k, v, 16)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
