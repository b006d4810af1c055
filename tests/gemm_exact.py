"""Operands on which the split-bf16 GEMMs have exactly one correct fp32 answer, and that answer.

Every hi-plane entry is m * 2^s and every lo-plane entry m' (|m|, |m'| <= M, small integers), so each of the three
tensor-core products hi*hi, hi*lo, lo*hi is a multiple of the quantum q = 2^s.  When the absolute terms of an output
(products plus bias and residuals) sum to at most BUDGET = 2^22 quanta, every partial sum is a multiple of q below 2^24 q:
exact in fp32, in whatever order and alignment the tensor core and the epilogue add them.  The kernel then has exactly
one correct result, sum_k (a_hi b_hi + a_hi b_lo + a_lo b_hi) (a_hi b_hi alone at precision 1), which fp64 computes
exactly, and its split planes hi = bf16_rn(out), lo = bf16_rn(out - hi) are determined too.  A dropped, added or
misplaced product, k-block, tap, row, group or plane changes some output bits, which `torch.equal` sees.

This module holds the generator, the premise (`Gen.bound`, `premise_terms`), the fp64 references of s3r_gemm and
s3r_conv_wgrad, the case lists the CPU and GPU tests share, and the per-tile mismatch report.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn.functional as F

BUDGET = 1 << 22          # absolute terms of one output, in quanta: 4x headroom under the 24-bit fp32 significand
OPERAND_SHARE = 1 << 21   # of which the GEMM's products may take half; bias, res1 and res2 2^19 each
EPI_MAX = 1 << 19
# stats_out sums squares of a 32-column chunk: outputs of at most 348 quanta keep 32 x^2 within BUDGET
STATS_KC, STATS_EPI = 96, 20
# EPI_QKV rounds to tf32 (11 significant bits): outputs below 2^11 quanta are exact
QKV_KC, QKV_BIAS = 128, 64


@dataclass(frozen=True)
class Gen:
    """hi = m * 2^s, lo = m' with m, m' uniform integers in [-M, M]."""
    M: int
    s: int

    @property
    def q(self) -> float:
        return float(1 << self.s)

    def bound(self, K: int, products: int = 3) -> int:
        """Worst-case sum over K contraction terms of |a_hi b_hi| (+ |a_hi b_lo| + |a_lo b_hi|), in quanta."""
        hh = self.M * self.M * (1 << self.s)
        return K * (hh + (2 * self.M * self.M if products == 3 else 0))


def pick_gen(K: int, budget: int = OPERAND_SHARE) -> Gen:
    """The widest hi / lo separation (largest s), then the largest M, whose worst case fits `budget` over K terms."""
    for s in range(8, -1, -1):
        for M in (4, 2, 1):
            g = Gen(M, s)
            if g.bound(K) <= budget:
                return g
    raise ValueError(f"no exact generator for a {K}-term contraction within {budget} quanta")


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def planes(shape, gen: Gen, seed: int, device="cpu"):
    """(hi, lo) bf16 planes of the given shape drawn from `gen`."""
    g = _gen(device, seed)
    m = torch.randint(-gen.M, gen.M + 1, shape, generator=g, device=device)
    ml = torch.randint(-gen.M, gen.M + 1, shape, generator=g, device=device)
    return (m.float() * gen.q).to(torch.bfloat16), ml.float().to(torch.bfloat16)


def ints(shape, bound: int, q: float, seed: int, device="cpu") -> torch.Tensor:
    """fp32 integers in [-bound, bound], times q."""
    g = _gen(device, seed)
    return torch.randint(-bound, bound + 1, shape, generator=g, device=device).float() * q


def exact_f32(shape, seed: int, device="cpu", M: int = 3, e: int = 0) -> torch.Tensor:
    """fp32 values m * 2^e, |m| <= M: bf16-exact, so their split is (x, 0)."""
    return ints(shape, M, float(2.0 ** e), seed, device)


def split_ref(x: torch.Tensor):
    """hi = bf16_rn(x), lo = bf16_rn(x - hi) of an fp32-representable tensor (the epilogue's split2_bf16)."""
    xf = x.float()
    hi = xf.to(torch.bfloat16)
    return hi, (xf - hi.float()).to(torch.bfloat16)


def split_trunc(x: torch.Tensor):
    """The split with the lo plane truncated instead of rounded (a defect model)."""
    xf = x.float()
    hi = xf.to(torch.bfloat16)
    r = (xf - hi.float()).contiguous()
    return hi, (r.view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ fp64 references
def conv_ref(x: torch.Tensor, w: torch.Tensor, taps: int) -> torch.Tensor:
    """x [nb, H, W, Kc], w [N, taps * Kc] (k = tap * Kc + c, tap = 3 (dy + 1) + dx + 1) -> [nb, H, W, N], in x's dtype."""
    nb, H, W, Kc = x.shape
    N = w.shape[0]
    if taps == 1:
        return (x.reshape(-1, Kc) @ w.t()).view(nb, H, W, N)
    wc = w.reshape(N, 3, 3, Kc).permute(0, 3, 1, 2)
    return F.conv2d(x.permute(0, 3, 1, 2), wc, padding=1).permute(0, 2, 3, 1)


def _products(a, b, taps, precision, f):
    ah, al = (f(t) for t in a)
    bh, bl = (f(t) for t in b)
    if precision == 1:
        return conv_ref(ah, bh, taps)
    return conv_ref(ah, bh + bl, taps) + conv_ref(al, bh, taps)


def gemm_ref(a, b, groups: int, taps: int, precision: int = 0, a_swap: bool = False, swap_col0: int = 0,
             terms: bool = False) -> torch.Tensor:
    """The accumulator of s3r_gemm in fp64: a planes [G*NB, H, W, Kc], b planes [G*N, taps*Kc] -> [G*NB, H, W, N].
    Group g contracts its own A images with its B rows; with a_swap, columns >= swap_col0 read the A images of G-1-g.
    terms: the sum of the products' absolute values instead (the premise)."""
    f = (lambda t: t.double().abs()) if terms else (lambda t: t.double())
    GNB = a[0].shape[0]
    NB, N = GNB // groups, b[0].shape[0] // groups
    out = []
    for g in range(groups):
        ab = lambda gg: tuple(t[gg * NB:(gg + 1) * NB] for t in a)   # noqa: E731
        bb = tuple(t[g * N:(g + 1) * N] for t in b)
        y = _products(ab(g), bb, taps, precision, f)
        if a_swap:
            ys = _products(ab(groups - 1 - g), bb, taps, precision, f)
            y = torch.cat((y[..., :swap_col0], ys[..., swap_col0:]), -1)
        out.append(y)
    return torch.cat(out)


def wgrad_ref(dy, x, taps: int, terms: bool = False) -> torch.Tensor:
    """dW [n, taps, kc] = sum over pixels of dY[p, n] X[p + shift(tap), c] with the three split products, fp64.
    dy planes [nb, h, w, n], x planes [nb, h, w, kc]."""
    f = (lambda t: t.double().abs()) if terms else (lambda t: t.double())
    yh, yl = (f(t) for t in dy)
    xh, xl = (f(t) for t in x)
    nb, h, w, n = yh.shape
    kc = xh.shape[-1]
    ys, ylo = yh.reshape(-1, n), yl.reshape(-1, n)
    out = []
    shifts = [(0, 0)] if taps == 1 else [(dy_, dx_) for dy_ in (-1, 0, 1) for dx_ in (-1, 0, 1)]
    xph, xpl = F.pad(xh, (0, 0, 1, 1, 1, 1)), F.pad(xl, (0, 0, 1, 1, 1, 1))
    for dy_, dx_ in shifts:
        sh = xph[:, 1 + dy_:1 + dy_ + h, 1 + dx_:1 + dx_ + w].reshape(-1, kc)
        sl = xpl[:, 1 + dy_:1 + dy_ + h, 1 + dx_:1 + dx_ + w].reshape(-1, kc)
        out.append(ys.t() @ (sh + sl) + ylo.t() @ sh)
    return torch.stack(out, 1)


def plain_epilogue(acc, bias=None, act_relu=False, res1=None, res2=None):
    """EPI_PLAIN in fp64: (acc + bias), ReLU, + res1 + res2 (all exact on the generator's data)."""
    x = acc + (bias.double() if bias is not None else 0.0)
    if act_relu:
        x = x.clamp_min(0)
    if res1 is not None:
        x = x + res1.double()
    if res2 is not None:
        x = x + res2.double()
    return x


def stats_ref(x: torch.Tensor) -> torch.Tensor:
    """[rows, N] -> [rows, N/32, 2] (sum, sum of squares) per 32-column chunk, fp32 (exact when the premise holds)."""
    c = x.double().reshape(x.shape[0], -1, 32)
    return torch.stack((c.sum(-1), c.square().sum(-1)), -1).float()


# ------------------------------------------------------------------------------------------------ tiles and reports
def next_pow2(x: int) -> int:
    p = 1
    while p < x:
        p <<= 1
    return p


def row_tiles(images: int, H: int, W: int, pix: int = 128) -> torch.Tensor:
    """Output tile of each pixel row [images*H*W] under the engine's bw x bh pixel tiles (bw * bh = pix)."""
    bw = pix if W >= pix else next_pow2(W)
    bh = pix // bw
    th, tw = (H + bh - 1) // bh, (W + bw - 1) // bw
    hh = torch.arange(H)[:, None] // bh
    ww = torch.arange(W)[None, :] // bw
    t = (hh * tw + ww).reshape(-1)
    return (torch.arange(images)[:, None] * (th * tw) + t[None, :]).reshape(-1)


def tile_ids(images: int, H: int, W: int, N: int, bn: int = 64) -> torch.Tensor:
    """[images*H*W, N] tile index of every output element (128-pixel row tiles x bn-column tiles)."""
    r = row_tiles(images, H, W)
    nct = (N + bn - 1) // bn
    return r[:, None] * nct + (torch.arange(N) // bn)[None, :]


def _bad(got, exp):
    ne = got != exp
    if got.is_floating_point():
        ne = ne | (torch.isnan(got) != torch.isnan(exp))
        ne = ne & ~(torch.isnan(got) & torch.isnan(exp))
    return ne


def assert_same(name: str, got: torch.Tensor, exp: torch.Tensor, tiles: torch.Tensor | None = None, shown: int = 6):
    """torch.equal, or an AssertionError with the wrong-element count per tile and the first (row, col, got, expected).
    got / exp: same shape, viewed as [rows, -1]; tiles: optional tile index of every element."""
    assert got.shape == exp.shape and got.dtype == exp.dtype, (name, tuple(got.shape), tuple(exp.shape), got.dtype, exp.dtype)
    if torch.equal(got, exp):
        return
    g2, e2 = got.reshape(got.shape[0], -1), exp.reshape(exp.shape[0], -1)
    bad = _bad(g2, e2)
    if not bool(bad.any()):
        return   # NaN in the same places (guard regions)
    idx = bad.nonzero()[:shown].cpu()
    if tiles is None:
        tiles = (torch.arange(g2.shape[0]) // 128)[:, None].expand(g2.shape)
    tb = tiles.reshape(g2.shape).to(bad.device)[bad]
    ut, cnt = torch.unique(tb, return_counts=True)
    per_tile = ", ".join(f"{int(t)}: {int(c)}" for t, c in list(zip(ut.tolist(), cnt.tolist()))[:12])
    first = "; ".join(f"({int(r)}, {int(c)}) got {float(g2[r, c])!r} expected {float(e2[r, c])!r}" for r, c in idx.tolist())
    raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ in {len(ut)} tiles "
                         f"(wrong per tile: {per_tile}); first: {first}")


# ------------------------------------------------------------------------------------------------ case lists
# s3r_gemm geometry: (groups, NB, H, W, Kc, taps, N); linear layers are the map H = 1, W = rows
GEOMETRY = [
    (1, 1, 1, 300, 8, 1, 32), (1, 1, 1, 300, 24, 1, 96), (1, 1, 1, 300, 40, 1, 160), (1, 1, 1, 333, 200, 1, 160),
    (1, 1, 1, 1, 40, 1, 96), (2, 1, 1, 77, 200, 1, 32),
    (1, 3, 1, 1, 40, 9, 32), (1, 3, 1, 19, 24, 9, 96), (1, 3, 13, 1, 24, 9, 96), (1, 3, 7, 7, 40, 9, 160),
    (1, 2, 13, 19, 8, 9, 96), (1, 3, 13, 19, 200, 9, 32), (2, 2, 13, 19, 40, 9, 160), (1, 1, 130, 3, 24, 9, 32),
]
# tools/gemm_sweep.py: (name, groups, rows, K, N)
SWEEP = [
    ("dec.qkv", 2, 768, 768, 2304), ("dec.proj", 2, 768, 768, 768), ("dec.kv", 2, 768, 768, 1536),
    ("dec.fc1", 2, 768, 768, 3072), ("dec.fc2", 2, 768, 3072, 768), ("key.fc1", 2, 768, 1792, 1792),
    ("val.qkv", 1, 768, 1024, 3072), ("val.proj", 1, 768, 1024, 1024), ("val.fc1", 1, 768, 1024, 4096),
    ("val.fc2", 1, 768, 4096, 1024),
    ("enc.qkv", 1, 7680, 1024, 3072), ("enc.proj", 1, 7680, 1024, 1024), ("enc.fc1", 1, 7680, 1024, 4096),
    ("enc.fc2", 1, 7680, 4096, 1024),
]
# test_gemm_ring_gpu.test_persistent_ring_wrap: (rows, Kc, N, force_bn)
RING = [(7680, 4096, 1024, 0), (7680, 1024, 3072, 64), (7700, 160, 1056, 128)]


def convs(H: int, W: int):
    """(name, kind, Cin, Cout, map h, map w) of one DPT head and the patch embeddings for an H x W frame (the list of
    test_native_conv_gpu._convs)."""
    gh, gw = H // 16, W // 16
    h3, w3 = (gh + 1) // 2, (gw + 1) // 2
    return [
        ("act_postprocess.0.0", "1x1", 1024, 96, gh, gw), ("act_postprocess.1.0", "1x1", 768, 192, gh, gw),
        ("act_postprocess.2.0", "1x1", 768, 384, gh, gw), ("act_postprocess.3.0", "1x1", 768, 768, gh, gw),
        ("act_postprocess.0.1", "convT4", 96, 96, gh, gw), ("act_postprocess.1.1", "convT2", 192, 192, gh, gw),
        ("act_postprocess.3.1", "3x3s2", 768, 768, gh, gw),
        ("layer_rn.0", "3x3nb", 96, 256, 4 * gh, 4 * gw), ("layer_rn.1", "3x3nb", 192, 256, 2 * gh, 2 * gw),
        ("layer_rn.2", "3x3nb", 384, 256, gh, gw), ("layer_rn.3", "3x3nb", 768, 256, h3, w3),
        ("refinenet4.rcu", "3x3", 256, 256, h3, w3), ("refinenet3.rcu", "3x3", 256, 256, gh, gw),
        ("refinenet2.rcu", "3x3", 256, 256, 2 * gh, 2 * gw), ("refinenet1.rcu", "3x3", 256, 256, 4 * gh, 4 * gw),
        ("refinenet4.out_conv", "1x1", 256, 256, gh, gw), ("refinenet3.out_conv", "1x1", 256, 256, 2 * gh, 2 * gw),
        ("refinenet2.out_conv", "1x1", 256, 256, 4 * gh, 4 * gw), ("refinenet1.out_conv", "1x1", 256, 256, 8 * gh, 8 * gw),
        ("head.0", "3x3", 256, 128, H // 2, W // 2), ("head.2", "3x3", 128, 128, H, W),
        ("patch_embed", "patch", 3, 1024, H, W), ("pos_patch_embed", "patch_dx", 3, 1024, H, W),
    ]


def wgrad_shape(kind: str, cin: int, cout: int, h: int, w: int, nb: int):
    """The s3r_conv_wgrad launch (nb, h, w, n, kc, taps) of a conv's weight gradient in _native_conv."""
    if kind in ("3x3", "3x3nb"):
        return nb, h, w, cout, cin, 9
    if kind == "3x3s2":
        return nb, (h + 1) // 2, (w + 1) // 2, cout, 9 * cin, 1
    if kind.startswith("patch"):
        return nb, h // 16, w // 16, cout, 768, 1
    if kind.startswith("convT"):
        s = int(kind[-1])
        return nb, h, w, s * s * cout, cin, 1
    return nb, h, w, cout, cin, 1


def wgrad_cases():
    """Distinct wgrad launches (nb, h, w, n, kc, taps) of every conv at H x W = 224 x 224, 288 x 224 and 512 x 384,
    B = 1 and 4, and the ragged shapes of test_conv_wgrad_is_bitwise_reproducible."""
    seen = []
    for H, W in ((224, 224), (288, 224), (512, 384)):
        for nb in (1, 4):
            for _, kind, cin, cout, h, w in convs(H, W):
                s = wgrad_shape(kind, cin, cout, h, w, nb)
                if s not in seen:
                    seen.append(s)
    for s in ((1, 7, 7, 256, 768, 9), (2, 37, 53, 128, 96, 9), (3, 19, 23, 192, 256, 1), (4, 224, 224, 128, 128, 9)):
        if s not in seen:
            seen.append(s)
    return seen
