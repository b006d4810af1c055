"""Inputs on which the training attention (csrc/attention_train.cu) has one correct fp32 answer, and that answer.

Every product of the four kernels is split-bf16 (hi.hi + hi.lo + lo.hi, fp32 accumulation); the only transcendental
steps are expf and logf.  The inputs here make every step exact:

* Probabilities of exactly 0 or 1.  The scale is 2^-3.  Each query and key of a slice carries SEL = 32 on the two
  selector columns of its group's code (weight 2), or nothing.  A query meets the keys of its own group at s 2 SEL^2 =
  256, keys sharing one code column at 128 and every other key at 0, plus a term eps_ij from the shared columns that is
  the same for every key of one group and differs by at most 12 after scaling across groups.  expf(0) = 1 and
  expf(x) = 0 for x < -103.97, so every kept probability is 1 and every other one 0, in the flash forward (across
  its running max too) and in the backward when it is handed LSE = s max_j S_ij.  A query of no group has Q = 0 on the
  selector and shared columns: its scores are all 0, P = 1 on every key and LSE = log(nk).  The backward is handed
  LSE = 256 there, so P = 0 on that row.
* Every product and partial sum on a grid.  Every value is an integer times a power of two, so each term of an output is
  a multiple of the output's quantum (the smallest lowest set bit among its terms).  When the absolute terms of an
  output sum to at most BUDGET = 2^22 quanta, every partial sum is exact in fp32 whatever the order or alignment of the
  additions.  `premise` measures this on the drawn data, per output element, for every product, for D = rowsum(dO o O)
  and for dS = P o (dP - D).  This assumes that mma.sync's fp32 accumulation loses nothing on such sums, as wgmma's does
  (gemm_exact.py).  It held on an H100 SXM: every case of test_attn_train_exact_gpu.py is bit exact.

So the kernels' results are the fp64 values below, rounded once where the kernel rounds: O = fp32(fp32(sum of the kept
V rows) * fp32(1 / k)); LSE exact for k = 1 and within 1 ulp of fp32(s max + ln k) otherwise (logf's error); dQ, dK and
dV exact.  The backward's in-register split of P and dS into hi / lo planes is `split_ref`, and lo . lo is dropped.

The values are drawn per key group in one of four roles, so that each defect of a split-bf16 kernel moves some output
bit while every output stays within the budget:
* QK: wide Q and K on the shared and one-sided columns, small dS;
* DOV: wide dO and V on disjoint columns;
* WIDE_DS: D large, so that many dS values have more than 17 significant bits and the in-register split rounds their
  lo plane;
* WIDE_IN: Q and K of 18 significant bits on the one-sided columns, so the load's split rounds their lo planes.

One limit: P is 0 or 1, so its lo plane is always zero and a dropped P_lo . V_hi or P_lo . dO_hi product cannot show
here.  The relative-L2 tests of test_native_attn_gpu.py catch that defect: it moves every output by about 2^-9.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from gemm_exact import BUDGET, split_ref, split_trunc

SCALE = 0.125
SEL = 32.0          # selector value: s SEL^2 = 128 per shared code column
TILE = 64           # query / key tile of every kernel
GAP = 110.0         # every kept score is at least this far above every dropped one (expf underflows below -103.97)
QQ, QK, QV, QG = 2.0 ** -5, 2.0 ** -5, 2.0 ** -6, 2.0 ** -6    # quanta of Q, K, V and dO
QK_ROLE, DOV, WIDE_DS, WIDE_IN = range(4)


@dataclass(frozen=True)
class Case:
    B: int
    H: int
    nq: int
    nk: int
    dh: int
    seed: int = 0
    one_to_one: bool = False   # every query matches exactly one key, no uniform rows (the autograd end-to-end case)

    @property
    def id(self) -> str:
        return f"{self.B}x{self.H}x{self.nq}x{self.nk}x{self.dh}" + ("-1to1" if self.one_to_one else "")


# ------------------------------------------------------------------------------------------------ generator
def _ints(g, shape, lo, hi, p0=0.0):
    """Integers of magnitude in [lo, hi] with random signs, zero with probability p0 (fp64)."""
    n = torch.randint(lo, hi + 1, shape, generator=g).double()
    n = n * (torch.randint(0, 2, shape, generator=g).double() * 2 - 1)
    return torch.where(torch.rand(shape, generator=g, dtype=torch.float64) < p0, 0.0, n)


def _mix(g, shape, p0, pw, small=3, wide=(257, 1023)):
    """0 with probability p0, a wide integer (9-10 bits: a non-zero lo plane) with probability pw, else |n| <= small."""
    u = torch.rand(shape, generator=g, dtype=torch.float64)
    return torch.where(u < p0, 0.0, torch.where(u < p0 + pw, _ints(g, shape, *wide), _ints(g, shape, 0, small)))


def _slice(g, nq, nk, dh, one_to_one):
    """One (batch, head) slice: q, k, v, dO and the supplied O as [n, dh] fp64 integers times quanta, and the groups."""
    perm = torch.randperm(dh, generator=g)
    ns, nf = (24, 18) if dh == 64 else (16, 14)
    sel, shared, fq, fk = perm[:ns], perm[ns:ns + 4], perm[ns + 4:ns + 4 + nf], perm[ns + 4 + nf:]
    codes = [(a, b) for a in range(ns) for b in range(a + 1, ns)]
    codes = [codes[i] for i in torch.randperm(len(codes), generator=g).tolist()]

    # key groups of 1..4 keys (1 in the one-to-one case) over a random order of the keys; ~1/5 of the keys in none
    order = torch.randperm(nk, generator=g).tolist()
    kgrp = torch.full((nk,), -1, dtype=torch.long)
    target = nk if (one_to_one or nk < 5) else nk - nk // 5
    pos = ng = 0
    while pos < target and ng < len(codes):
        sz = 1 if one_to_one else int(torch.randint(1, 5, (1,), generator=g))
        for j in order[pos:pos + sz]:
            kgrp[j] = ng
        pos += sz
        ng += 1
    role = torch.randint(0, 4, (ng,), generator=g)
    quni = torch.rand(nq, generator=g) < (0.0 if one_to_one else 0.1)
    qgrp = torch.where(quni, -1, torch.randint(0, ng, (nq,), generator=g))
    seen = [0] * ng                    # at most 6 queries per group (dK and dV sum over them); the rest keep no group
    for i, x in enumerate(qgrp.tolist()):
        if x >= 0 and not one_to_one:
            seen[x] += 1
            if seen[x] > 6:
                qgrp[i] = -1
    quni = qgrp < 0
    qrole = torch.where(qgrp >= 0, role[qgrp.clamp_min(0)], -1)
    krole = torch.where(kgrp >= 0, role[kgrp.clamp_min(0)], -1)

    q = torch.zeros(nq, dh, dtype=torch.float64)
    k = torch.zeros(nk, dh, dtype=torch.float64)
    # selector columns
    code = sel[torch.tensor(codes[:ng])]                  # [ng, 2] columns of each group's code
    for x, grp, quantum in ((q, qgrp, QQ), (k, kgrp, QK)):
        rows = (grp >= 0).nonzero()[:, 0]
        for e in range(2):
            x[rows, code[grp[rows], e]] = SEL / quantum
    # shared columns: kappa per group, the same on every key of it (positive); Q with two + and two - terms, so that
    # |eps| <= 2 (300^2 - 257^2) / 2^10 < 48 on the QK role's rows
    kap = _ints(g, (ng, 4), 257, 300).abs()
    kap = torch.where((role != QK_ROLE)[:, None], _ints(g, (ng, 4), 0, 1), kap)
    kfree = _ints(g, (nk, 4), 257, 300).abs()        # keys of no group
    k[:, shared] = torch.where((kgrp >= 0)[:, None], kap[kgrp.clamp_min(0)], kfree)
    sign = torch.rand(nq, 4, generator=g).argsort(-1) < 2
    qs = _ints(g, (nq, 4), 257, 300).abs() * torch.where(sign, 1.0, -1.0)
    qs = torch.where(((qrole == DOV) | (qrole == WIDE_DS) | (qrole == WIDE_IN))[:, None], _ints(g, (nq, 4), 0, 1), qs)
    q[:, shared] = torch.where(quni[:, None], 0.0, qs)
    # one-sided columns
    q_fq = _mix(g, (nq, nf), 0.3, 0.3)
    q_fq = torch.where(((qrole == DOV) | (qrole == WIDE_DS))[:, None], _ints(g, (nq, nf), 0, 1), q_fq)
    q_fq = torch.where((qrole == WIDE_IN)[:, None], _ints(g, (nq, nf), (1 << 17) + 1, (1 << 18) - 1, 0.3), q_fq)
    q[:, fq] = q_fq
    k_fk = _mix(g, (nk, nf), 0.3, 0.3)
    k_fk = torch.where(((krole == DOV) | (krole == WIDE_DS))[:, None], _ints(g, (nk, nf), 0, 1), k_fk)
    k_fk = torch.where((krole == WIDE_IN)[:, None], _ints(g, (nk, nf), (1 << 17) + 1, (1 << 18) - 1, 0.3), k_fk)
    k[:, fk] = k_fk

    # V, dO and the supplied O
    v = _ints(g, (nk, dh), 0, 3, 0.3)
    go = _ints(g, (nq, dh), 0, 3, 0.3)
    cols = torch.randperm(dh, generator=g)
    wdo, wv = cols[:8], cols[8:16]          # DOV: wide dO and wide V on disjoint columns
    vw = torch.zeros(nk, dh, dtype=torch.float64)
    vw[:, wv] = _ints(g, (nk, 8), 257, 1023, 0.25)
    v = torch.where((krole == DOV)[:, None] & (vw != 0), vw, v)
    v = torch.where((krole == WIDE_IN)[:, None], _ints(g, (nk, dh), 1, 1), v)   # dS = dP = +-1 quantum
    gw = torch.zeros(nq, dh, dtype=torch.float64)
    gw[:, wdo] = _ints(g, (nq, 8), 257, 1023, 0.25)
    go = torch.where((qrole == DOV)[:, None] & (gw != 0), gw, go)
    one = torch.zeros(nq, dh, dtype=torch.float64)
    one[torch.arange(nq), torch.randint(0, dh, (nq,), generator=g)] = _ints(g, (nq,), 1, 1)
    go = torch.where((qrole == WIDE_IN)[:, None], one, go)
    o = torch.zeros(nq, dh, dtype=torch.float64)
    o = torch.where((qrole == DOV)[:, None], _ints(g, (nq, dh), 0, 1, 0.75), o)
    o = torch.where((qrole == WIDE_DS)[:, None], _ints(g, (nq, dh), 160, 320, 0.5), o)
    o = torch.where(quni[:, None], _ints(g, (nq, dh), 0, 2), o)
    go = go * QG
    if one_to_one:
        go = go.float().to(torch.bfloat16).double()   # dO_lo = 0: dP = D exactly on the one kept key
    return dict(q=q * QQ, k=k * QK, v=v * QV, go=go, o=o, qgrp=qgrp, kgrp=kgrp, qrole=qrole, krole=krole)


def make(case: Case):
    """The case's tensors on the CPU: q, k, v [B, H, n, dh], go and o (the supplied O) [B, nq, H * dh], all fp32; lse
    [B * H, nq] (s max_j S_ij, or 256 on rows of no group: P = 0 there), and the groups [B * H, n] (-1: none)."""
    g = torch.Generator().manual_seed(case.seed)
    B, H, nq, nk, dh = case.B, case.H, case.nq, case.nk, case.dh
    sl = [_slice(g, nq, nk, dh, case.one_to_one) for _ in range(B * H)]
    st = lambda key: torch.stack([s[key] for s in sl])   # noqa: E731
    q, k, v = (st(n).float().view(B, H, -1, dh) for n in ("q", "k", "v"))
    tok = lambda x: x.float().view(B, H, nq, dh).transpose(1, 2).reshape(B, nq, H * dh).contiguous()   # noqa: E731
    c = dict(q=q, k=k, v=v, go=tok(st("go")), o=tok(st("o")), qgrp=st("qgrp"), kgrp=st("kgrp"), qrole=st("qrole"),
             krole=st("krole"))
    S = scores(c)
    m = S.max(-1).values
    c["lse"] = torch.where(c["qgrp"] >= 0, m, 256.0).float()
    return c


def slices(x: torch.Tensor, B: int, H: int) -> torch.Tensor:
    """[B, H, n, dh] or token-major [B, n, H * dh] -> [B * H, n, dh]."""
    if x.dim() == 4:
        return x.reshape(B * H, x.shape[2], x.shape[3])
    n = x.shape[1]
    return x.view(B, n, H, -1).transpose(1, 2).reshape(B * H, n, -1)


def tokens(x: torch.Tensor, B: int, H: int) -> torch.Tensor:
    """[B * H, n, dh] -> token-major [B, n, H * dh]."""
    n, dh = x.shape[1], x.shape[2]
    return x.view(B, H, n, dh).transpose(1, 2).reshape(B, n, H * dh)


# ------------------------------------------------------------------------------------------------ fp64 references
def planes(x: torch.Tensor, trunc: bool = False):
    """The split of fp32 values into (hi, lo) as fp64."""
    h, l_ = (split_trunc if trunc else split_ref)(x.float())
    return h.double(), l_.double()


def mm3(a, b, drop: str | None = None):
    """hi.hi + hi.lo + lo.hi of planes a [.., m, t] and b [.., t, n] in fp64 (`drop` leaves one out)."""
    (ah, al), (bh, bl) = a, b
    r = torch.zeros(ah.shape[:-1] + bh.shape[-1:], dtype=torch.float64, device=ah.device)
    if drop != "hh":
        r = r + ah @ bh
    if drop != "hl":
        r = r + ah @ bl
    if drop != "lh":
        r = r + al @ bh
    return r


def _t(p):
    return tuple(x.transpose(-2, -1) for x in p)


def scores(c, device="cpu") -> torch.Tensor:
    """s S = s Q K^T [B * H, nq, nk] (exact on the premise) in fp64."""
    B, H = c["q"].shape[:2]
    Q, K = (planes(slices(c[n], B, H).to(device)) for n in ("q", "k"))
    return mm3(Q, _t(K)) * SCALE


def forward_ref(c, device="cpu"):
    """(O [B, nq, H * dh], LSE [B * H, nq], k [B * H, nq]) of the exact forward; LSE as fp32(s max + ln k)."""
    B, H = c["q"].shape[:2]
    S = scores(c, device)
    m = S.max(-1, keepdim=True).values
    P = (S == m).double()
    k = P.sum(-1)
    V = planes(slices(c["v"], B, H).to(device))
    acc = (P @ (V[0] + V[1])).float()
    o = acc * (1.0 / k.float())[..., None]
    lse = (m[..., 0] + torch.log(k)).float()
    return tokens(o, B, H), lse, k


def backward_ref(c, device="cpu", lse=None, o=None, go=None, parts=False):
    """(dQ, dK, dV) [B, H, n, dh] of the exact backward with the given LSE and O (default: the case's supplied ones).
    parts: also the intermediates (P, dP, D, dS) of the premise and the emulation."""
    B, H = c["q"].shape[:2]
    lse = (c["lse"] if lse is None else lse).to(device).double()
    O = slices((c["o"] if o is None else o).to(device), B, H).double()
    dO = slices((c["go"] if go is None else go).to(device), B, H)
    S = scores(c, device)
    P = (S == lse[..., None]).double()
    Gp = planes(dO)
    V, K, Q = (planes(slices(c[n], B, H).to(device)) for n in ("v", "k", "q"))
    dP = mm3(Gp, _t(V))
    D = (dO.double() * O).sum(-1)
    dS = (P * (dP - D[..., None])).float()
    dq = (mm3(planes(dS), K) * SCALE).float()
    dk = (mm3(_t(planes(dS)), Q) * SCALE).float()
    dv = (P.transpose(-2, -1) @ (Gp[0] + Gp[1])).float()
    shp = lambda x: x.view(B, H, x.shape[1], x.shape[2])   # noqa: E731
    out = (shp(dq), shp(dk), shp(dv))
    return out + ((S, P, dP, D, dS),) if parts else out


# ------------------------------------------------------------------------------------------------ premise
def _lowexp(x: torch.Tensor) -> torch.Tensor:
    """Exponent of the lowest set bit of every non-zero fp64 value (a large value where x = 0)."""
    m, e = torch.frexp(x)
    n = (m.abs() * 2.0 ** 53).long()
    _, e2 = torch.frexp((n & -n).double())
    return torch.where(x == 0, 1 << 12, e.long() - 53 + e2.long() - 1)


def _weight(x: torch.Tensor) -> torch.Tensor:
    """2^(-16 lowexp(x)) where x != 0, else 0: the largest weight of a sum of products marks its finest term."""
    le = _lowexp(x)
    return torch.where(x == 0, 0.0, torch.ldexp(torch.ones_like(x), (-16 * le).clamp(-1000, 1000)))


class Terms:
    """The absolute sum and the quantum of a sum of products, per output element: `quanta` = sum / quantum."""

    def __init__(self, total, weight):
        self.total, self.weight = total, weight

    @staticmethod
    def product(a, b):
        """Of the three split products of planes a [.., m, t] and b [.., t, n]."""
        (ah, al), (bh, bl) = a, b
        A = lambda x: x.abs()   # noqa: E731
        total = A(ah) @ (A(bh) + A(bl)) + A(al) @ A(bh)
        wah, wal, wbh, wbl = (_weight(x) for x in (ah, al, bh, bl))
        return Terms(total, wah @ (wbh + wbl) + wal @ wbh)

    @staticmethod
    def elementwise_sum(x, y):
        """Of sum_d x_d y_d (fp32 products) over the last dimension."""
        return Terms((x * y).abs().sum(-1), (_weight(x) * _weight(y)).sum(-1))

    def __add__(self, other):
        return Terms(self.total + other.total, self.weight + other.weight)

    @property
    def quanta(self) -> torch.Tensor:
        _, e = torch.frexp(self.weight)
        finest = torch.div(e.long() - 1, 16, rounding_mode="floor")   # -(exponent of the finest term's lowest bit)
        return torch.where(self.weight == 0, 0.0, torch.ldexp(self.total, finest))


def premise(c, device="cpu") -> dict:
    """The worst count of quanta of every exact step on the case's data, and the score gap; asserts both.
    Forward: S at the kept pairs, P V.  Backward (supplied LSE and O): S and dP at the kept pairs, D, dS, dS K, dS^T Q,
    P^T dO."""
    B, H = c["q"].shape[:2]
    Q, K, V = (planes(slices(c[n], B, H).to(device)) for n in ("q", "k", "v"))
    dO = slices(c["go"].to(device), B, H)
    O = slices(c["o"].to(device), B, H).double()
    _, _, _, (S, P, dP, D, dS) = backward_ref(c, device, parts=True)
    m = S.max(-1, keepdim=True).values
    Pf = (S == m).double()
    worst = {}

    def note(name, t, mask=None):
        qn = t.quanta if mask is None else torch.where(mask, t.quanta, 0.0)
        worst[name] = float(qn.max()) if qn.numel() else 0.0

    ts = Terms.product(Q, _t(K))
    note("S (forward)", ts, Pf > 0)
    note("S (backward)", ts, P > 0)
    one = (torch.ones_like(Pf), torch.zeros_like(Pf))
    note("P V", Terms.product((Pf, one[1]), V))
    tdp = Terms.product(planes(dO), _t(V))
    note("dP", tdp, P > 0)
    td = Terms.elementwise_sum(dO.double(), O)
    note("D", td, P.sum(-1) > 0)
    tds = tdp + Terms(td.total[..., None].expand_as(tdp.total), td.weight[..., None].expand_as(tdp.weight))
    note("dS", tds, P > 0)
    note("dS K", Terms.product(planes(dS), K))
    note("dS^T Q", Terms.product(_t(planes(dS)), Q))
    note("P^T dO", Terms.product((P.transpose(-2, -1), torch.zeros_like(P).transpose(-2, -1)), planes(dO)))
    for name, w in worst.items():
        assert w <= BUDGET, f"premise: {name} needs {w:.0f} quanta > 2^22"
    # every dropped score lies GAP below the kept ones (forward: below the row's max; backward: below the given LSE)
    lse = c["lse"].to(device).double()[..., None]
    gap_f = torch.where(Pf > 0, math.inf, m - S).min()
    gap_b = torch.where(P > 0, math.inf, lse - S).min()
    worst["gap"] = float(min(gap_f, gap_b))
    assert worst["gap"] >= GAP, f"premise: a dropped score only {worst['gap']} below the kept ones"
    # the backward keeps exactly the forward's pairs on rows of a group
    coded = (c["qgrp"].to(device) >= 0)[..., None]
    assert torch.equal(P * coded, Pf * coded)
    # every split the kernels make is the split the references use: inputs and P are what they are, dS fits fp32
    assert torch.equal(dS.double(), P * (dP - D[..., None]))
    return worst


# ------------------------------------------------------------------------------------------------ tiles and reports
def row_tiles(c, n: int) -> torch.Tensor:
    """Tile index (slice * tiles + row // 64) of every row of a [B * H, n] output."""
    BH = c["q"].shape[0] * c["q"].shape[1]
    nt = (n + TILE - 1) // TILE
    return torch.arange(BH)[:, None] * nt + torch.arange(n)[None, :] // TILE


def tile_report(name, got, exp, tiles, shown=6):
    """torch.equal, or an AssertionError with the wrong elements per (slice, 64-row tile) and the first few.
    got / exp [B * H, n, ...]; tiles [B * H, n]."""
    assert got.shape == exp.shape and got.dtype == exp.dtype, (name, tuple(got.shape), tuple(exp.shape))
    if torch.equal(got, exp):
        return
    g2, e2 = got.reshape(got.shape[0], got.shape[1], -1), exp.reshape(exp.shape[0], exp.shape[1], -1)
    bad = (g2 != e2) & ~(torch.isnan(g2) & torch.isnan(e2))
    if not bool(bad.any()):
        return
    row_bad = bad.any(-1).cpu()
    nt = int(tiles.max()) + 1
    nper = (tiles.shape[1] + TILE - 1) // TILE
    t, cnt = torch.unique(tiles[row_bad], return_counts=True)
    per = ", ".join(f"slice {int(x) // nper} tile {int(x) % nper}: {int(n)} rows" for x, n in zip(t[:10], cnt[:10]))
    idx = bad.nonzero()[:shown].tolist()
    first = "; ".join(f"(slice {s}, row {r}, col {col}) got {float(g2[s, r, col])!r} expected {float(e2[s, r, col])!r}"
                      for s, r, col in idx)
    raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements differ, {len(t)} of {nt} tiles "
                         f"({per}); first: {first}")


# ------------------------------------------------------------------------------------------------ case lists
# every shape of test_native_attn_gpu.SHAPES
SHAPES = [
    (40, 16, 196, 196, 64), (4, 12, 196, 196, 64), (4, 16, 196, 196, 64), (4, 16, 196, 196, 48), (2, 16, 252, 252, 64),
    (2, 12, 252, 252, 64), (3, 16, 252, 252, 48), (2, 16, 768, 768, 64), (1, 12, 768, 768, 64), (2, 12, 196, 252, 64),
    (2, 16, 252, 196, 48), (1, 4, 1, 1, 64), (1, 4, 17, 129, 64), (1, 4, 127, 17, 48), (1, 4, 129, 127, 64),
    (2, 3, 1, 129, 48), (2, 3, 129, 1, 64),
]
_TAILS = (1, 63, 64, 65, 127, 128, 129)
# tails: nq and nk of 1, 63 .. 129, crossed so that nq != nk both ways, at both head dims
TAILS = [(2, 3, nq, nk, dh) for dh in (48, 64) for i, nq in enumerate(_TAILS) for nk in _TAILS[i % 2::2]]


def cases():
    return [Case(*s, seed=17 + i) for i, s in enumerate(SHAPES)] + [Case(*s, seed=101 + i) for i, s in enumerate(TAILS)]


def e2e_cases():
    return [Case(4, 12, 196, 196, 64, seed=5, one_to_one=True), Case(2, 16, 252, 196, 48, seed=6, one_to_one=True),
            Case(2, 3, 129, 65, 64, seed=7, one_to_one=True)]
