"""Inputs on which the eval attention core (csrc/attention.cu) has exactly one correct fp32 answer, and that answer.

The kernel's arithmetic, per 128-query tile, head and 128-key block (the contract stated at the top of attention.cu):
S = Q K^T on tf32 wgmma with fp32 accumulation; keys >= nk set to -inf; running max n = max(m, block max);
al = exp2f((m - n) log2e), 0 on the first block; e = exp2f(fmaf(s, log2e, -n log2e)); P = RN_tf32(e) as
(bits + 0x1000) & ~0x1fff; l = l al + sum P; O = O al + P V on tf32 wgmma with P in registers; out = O * fl(1 / l).

The data here makes every one of those steps exact or deterministic:

* Selector codes.  Each query of a key group carries SEL = 16 on the two selector columns of the group's code and
  -2 SEL^2 on a bias column on which every real key holds 1; each key of the group carries SEL on the same two columns.
  A query then scores its own keys at exactly 0, keys sharing one code column at -256 and every other key at -512.
  Keys of no group hold no code.  A kept score of 0 makes the phantom keys past nk (zero-filled by TMA, so they score
  0 too) tie with the kept keys: one that escaped the mask would add 1 to l.
* Underflow.  Every score that is not kept lies at least GAP = 110 below the row's max, so exp2f's argument is below
  -158 and e underflows to 0 (and any result below 2^-137 would round to a tf32 zero anyway).  Every rise of the
  running max from one key block to a later one is 0 or at least GAP, so al is exactly 1 or exactly 0.
* Grid values.  q, k and v are small integers times powers of two and P is tf32, so every kept score, every sum P and
  every column of sum P v is a sum of terms on one grid; their absolute values stay within gemm_exact.BUDGET = 2^22
  quanta (`premise` measures it per element), so every partial sum is exact in fp32 in any order.
* Fractional weights.  On two-key rows the second key sits at a gap g (`frac_gaps`) whose weight exp(-g) lies in the
  upper part of a tf32 ulp, so that round-to-nearest and truncation differ.  Every such e lies at least 2^-15
  (relative) from any tf32 rounding boundary after allowing for exp2f's documented 2-ulp error, the fmaf's rounding of
  s log2e - fl(n log2e) with |n| <= 2^7, and the rounding of log2e itself to fp32; `premise` measures the margin per
  element on the drawn data.  P is then known bit for bit whatever exp2f's last bits are.

Two further facts are taken as given: exp2f(0) = 1 (kept keys get e = 1; al = 1 when the max does not move) and
exp2f(x) = 0 for x below -150.  The GPU tests confirm both: a one-key row depends on nothing else.

So the kernel's output is fl32(fl32(sum_j P_j v_j) * fl32(1 / sum_j P_j)), with both sums exact and P_j =
RN_tf32(exp(s_j)) known exactly; `expect` computes it in fp64.

Rows take one of six roles, mixed in every 128-query tile and every head (`ROLES`): one kept key (O = v_j); 2, 3, 5
or 7 kept keys (1 / l rounds); uniform rows with q = 0 (every key kept, l = nk, the ragged last block included);
two-key fractional rows; decoy rows whose earlier key block holds a decoy key 110 .. 300 below the final max (al = 0
exactly: a stale or missing rescale keeps the decoy), and the reverse, with the decoys after the kept keys.

Measured on an H100 80GB HBM3 at a 700 W power limit: every case of test_attn_core_exact_gpu.py is bit exact, one-key,
uniform and wider rows alike.  So tf32 wgmma, in the SS form of Q K^T and in the RS form of P V with P in registers,
accumulates grid sums within 2^22 quanta exactly, as bf16 wgmma does (gemm_exact.py); the budget needs no tf32 margin.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from attn_train_exact import Terms
from gemm_exact import BUDGET, split_ref
from test_attention_core_gpu import ENGINE_SHAPES, RECT, SENT, SQUARE, tf32

BQ = BKV = 128          # query tile and key block of the kernel
D = 64
LOG2E = math.log2(math.e)
LOG2E_F32 = float(torch.tensor(LOG2E, dtype=torch.float32))   # the kernel's kLog2e
EXP2F_ULPS = 2          # exp2f's maximum error (CUDA C++ Programming Guide, single-precision functions)
MARGIN = 2.0 ** -15     # least distance of a fractional e from a tf32 rounding boundary, relative, after the errors
N_MAX = 2.0 ** 7        # largest |running max| at which a fractional e is computed
SEL = 16.0
NSEL = 32               # selector columns: 496 codes
BIAS = -2 * SEL * SEL
GAP = 110.0
DECOY = (212, 402)      # decoy rows' q on the decoy column: a decoy key scores -512 + delta in [-300, -110]
FRAC_MAX = 4.0          # fractional gaps g < 4
GQ = 2.0 ** -8          # quantum of the gaps
VQ, VMAX = 2.0 ** -2, 7  # v = VQ * integers in [-VMAX, VMAX]
ONE, MULTI, UNIFORM, FRAC, DECOY_FIRST, DECOY_LAST = range(6)
ROLES = ("one key", "2/3/5/7 keys", "uniform", "two-key fractional", "decoy block first", "decoy block last")
SIZES = (2, 3, 5, 7)


@dataclass(frozen=True)
class Case:
    BH: int
    heads: int
    nq: int
    nk: int
    seed: int = 0

    @property
    def id(self) -> str:
        return f"{self.BH}x{self.heads}x{self.nq}x{self.nk}"


# ------------------------------------------------------------------------------------------------ generator
def frac_gaps() -> torch.Tensor:
    """Gaps g = i 2^-8 in [0.05, 4) whose weight exp(-g) has a fractional part in [0.75, 0.95) of a tf32 ulp: RN rounds
    it up and truncation down (as in test_attention_core_gpu.two_key_gaps, on a grid coarse enough for the budget)."""
    g = torch.arange(13, int(FRAC_MAX / GQ), dtype=torch.float64) * GQ
    e = (-g).exp()
    E = torch.floor(torch.log2(e))
    frac = torch.remainder(e / 2.0 ** (E - 10), 1.0)
    return g[(frac >= 0.75) & (frac < 0.95)]


def _ints(gen, shape, hi, p0=0.0):
    """Integers in [-hi, hi], zero with probability p0 more (fp64)."""
    n = torch.randint(-hi, hi + 1, shape, generator=gen).double()
    return torch.where(torch.rand(shape, generator=gen, dtype=torch.float64) < p0, 0.0, n)


def _pick(gen, xs):
    return xs[int(torch.randint(0, len(xs), (1,), generator=gen))]


def _slice(gen, nq, nk, gaps):
    """One (batch, head) slice: q [nq, 64], k and v [nk, 64] (fp64 on the grid) and each row's role."""
    perm = torch.randperm(D, generator=gen)
    sel, (cb, cg, cd), fq, fk = perm[:NSEL], perm[NSEL:NSEL + 3].tolist(), perm[NSEL + 3:NSEL + 17], perm[NSEL + 17:]
    codes = [(a, b) for a in range(NSEL) for b in range(a + 1, NSEL)]
    codes = torch.tensor(codes)[torch.randperm(len(codes), generator=gen)]

    # key groups over a random order of the keys (sorted within a group); about a fifth of the keys in none
    order = torch.randperm(nk, generator=gen).tolist()
    target = nk if nk < 5 else nk - nk // 5
    groups, kinds, pos = [], [], 0
    while pos < target and len(groups) < len(codes):
        kind = int(torch.randint(0, 3, (1,), generator=gen))
        want = (1, _pick(gen, SIZES), 2)[kind]
        size = max(s for s in (1,) + SIZES if s <= min(want, target - pos))
        groups.append(sorted(order[pos:pos + size]))
        kinds.append(ONE if size == 1 else FRAC if kind == 2 else MULTI)
        pos += size

    k = torch.zeros(nk, D, dtype=torch.float64)
    k[:, cb] = 1.0
    free = torch.ones(nk, dtype=torch.bool)
    for i, keys in enumerate(groups):
        free[keys] = False
        k[keys, sel[codes[i, 0]]] = SEL
        k[keys, sel[codes[i, 1]]] = SEL
        if kinds[i] == FRAC:
            k[keys[1], cg] = -1.0            # the later key of the pair: q_cg = g puts it at -g
    decoy = free & (torch.rand(nk, generator=gen) < 0.5)
    k[decoy, cd] = 1.0
    k[:, fk] = _ints(gen, (nk, len(fk)), 3)   # columns on which q is zero: no score changes, unless misaddressed
    v = _ints(gen, (nk, D), VMAX, 0.25) * VQ

    # candidate groups of each role
    dblk = (decoy.nonzero()[:, 0] // BKV).tolist()
    first = [keys[0] // BKV for keys in groups]
    last = [keys[-1] // BKV for keys in groups]
    plain = [i for i, t in enumerate(kinds) if t != FRAC]
    cand = {ONE: [i for i, t in enumerate(kinds) if t == ONE], MULTI: [i for i, t in enumerate(kinds) if t == MULTI],
            FRAC: [i for i, t in enumerate(kinds) if t == FRAC],
            DECOY_FIRST: [i for i in plain if dblk and first[i] > min(dblk)],
            DECOY_LAST: [i for i in plain if dblk and last[i] < max(dblk)]}
    # every role in every 128-row tile: a shuffled cycle of the roles per tile, falling back where a role has no group
    role = torch.empty(nq, dtype=torch.long)
    for t0 in range(0, nq, BQ):
        n = min(BQ, nq - t0)
        role[t0:t0 + n] = (torch.arange(n) % len(ROLES))[torch.randperm(n, generator=gen)]
    qgrp = torch.full((nq,), -1, dtype=torch.long)
    for r in range(nq):
        want = int(role[r])
        got = next(x for x in (want, ONE, MULTI, FRAC, UNIFORM) if x == UNIFORM or cand.get(x))
        role[r] = got
        if got != UNIFORM:
            qgrp[r] = _pick(gen, cand[got])

    q = torch.zeros(nq, D, dtype=torch.float64)
    rows = (qgrp >= 0).nonzero()[:, 0]
    ci = codes[qgrp[rows]]
    q[rows, sel[ci[:, 0]]] = SEL
    q[rows, sel[ci[:, 1]]] = SEL
    q[rows, cb] = BIAS
    q[rows[:, None], fq[None, :]] = _ints(gen, (len(rows), len(fq)), 3)
    gi = torch.randint(0, len(gaps), (nq,), generator=gen)
    q[:, cg] = torch.where(role == FRAC, gaps[gi], 0.0)
    delta = torch.randint(DECOY[0], DECOY[1] + 1, (nq,), generator=gen).double()
    q[:, cd] = torch.where((role == DECOY_FIRST) | (role == DECOY_LAST), delta, 0.0)
    return q, k, v, role


def make(case: Case) -> dict:
    """q [BH, nq, 64], k and v [BH, nk, 64] fp32 (tf32-exact; q as the kernel takes it, scale included) and the role
    of every row [BH, nq]."""
    gen = torch.Generator().manual_seed(case.seed)
    gaps = frac_gaps()
    sl = [_slice(gen, case.nq, case.nk, gaps) for _ in range(case.BH)]
    q, k, v, role = (torch.stack([s[i] for s in sl]) for i in range(4))
    return dict(q=q.float(), k=k.float(), v=v.float(), role=role)


# ------------------------------------------------------------------------------------------------ the answer
def weights(s: torch.Tensor) -> torch.Tensor:
    """P = RN_tf32(e), e = exp(s - row max) rounded to fp32, in fp64 (exact on the premise)."""
    return tf32((s - s.amax(-1, keepdim=True)).exp().float()).double()


def expect(c: dict, device="cpu", chunk: int = 16) -> torch.Tensor:
    """The kernel's one correct output [BH, nq, 64] fp32: fl32(fl32(P V) * fl32(1 / sum P)), computed in fp64 over
    chunks of slices.  The fp64 quotient and product of fp32 values, rounded to fp32, are the correctly rounded fp32
    results: fp64 carries more than 2 * 24 + 2 bits, so the double rounding is innocuous."""
    out = []
    for b0 in range(0, c["q"].shape[0], chunk):
        q, k, v = (c[n][b0:b0 + chunk].to(device).double() for n in ("q", "k", "v"))
        P = weights(q @ k.transpose(-1, -2))
        acc = (P @ v).float()
        inv = (1.0 / P.sum(-1).float().double()).float()
        out.append((acc.double() * inv.double()[..., None]).float())
    return torch.cat(out).cpu()


def to_rows(x: torch.Tensor, heads: int) -> torch.Tensor:
    """[BH, nq, 64] -> the kernel's output layout [B nq, heads 64]: row b nq + q, columns h 64 + c."""
    BH, nq, _ = x.shape
    return x.view(BH // heads, heads, nq, D).transpose(1, 2).reshape(BH // heads * nq, heads * D)


def buffer(x: torch.Tensor, heads: int, ldo: int, guard: int, dtype=torch.float32) -> torch.Tensor:
    """[B nq + guard, ldo] filled with the sentinel of test_attention_core_gpu.run, with x [B nq, heads 64] in place."""
    buf = torch.full((x.shape[0] + guard, ldo), SENT, dtype=dtype, device=x.device)
    buf[:x.shape[0], :heads * D] = x.to(dtype)
    return buf


def expected_buffers(exp: torch.Tensor, heads: int, ldo: int, guard: int):
    """(fp32, hi, lo) expected output buffers: the planes are split_ref of the expected fp32, bit for bit."""
    rows = to_rows(exp, heads)
    hi, lo = split_ref(rows)
    return (buffer(rows, heads, ldo, guard), buffer(hi, heads, ldo, guard, torch.bfloat16),
            buffer(lo, heads, ldo, guard, torch.bfloat16))


# ------------------------------------------------------------------------------------------------ premise
def _block_max(s: torch.Tensor, nk: int):
    """(block maxima, running maxima) [.., nq, nblk] of scores [.., nq, nk] over 128-key blocks."""
    nblk = (nk + BKV - 1) // BKV
    sp = torch.nn.functional.pad(s, (0, nblk * BKV - nk), value=-math.inf)
    bm = sp.view(*s.shape[:-1], nblk, BKV).amax(-1)
    return bm, bm.cummax(-1).values


def tf32_boundary_distance(e: torch.Tensor) -> torch.Tensor:
    """Relative distance of positive normal fp64 values from the nearest tf32 round-to-nearest boundary."""
    E = torch.floor(torch.log2(e))
    u = torch.ldexp(torch.ones_like(e), (E - 10).long())
    lo = torch.floor(e / u) * u                      # e in [lo, lo + u): boundaries at lo + u / 2 and just below lo
    down = lo - torch.where(lo == torch.ldexp(torch.ones_like(e), E.long()), u / 4, u / 2)
    return torch.minimum((e - lo - u / 2).abs(), e - down) / e


def premise(c: dict, chunk: int = 8) -> dict:
    """Measures, per element, everything the exactness rests on, and asserts it.  Returns the worst values:
    quanta of the kept scores, of sum P and of each column of P V; the least score gap below the max outside the
    fractional range; the least non-zero rise of the running max; the largest |n| at which a fractional e is computed;
    the least margin of a fractional e from a tf32 boundary after exp2f's, the fmaf's and log2e's errors."""
    nk = c["k"].shape[1]
    worst = dict(S=0.0, l=0.0, PV=0.0, gap=math.inf, rise=math.inf, n=0.0, margin=math.inf)
    for b0 in range(0, c["q"].shape[0], chunk):
        q, k, v = (c[n][b0:b0 + chunk].double() for n in ("q", "k", "v"))
        s = q @ k.transpose(-1, -2)
        assert bool((s.amax(-1) == 0).all()), "premise: a row whose max score is not 0"
        P = weights(s)
        kept = P > 0
        z = torch.zeros_like
        ts = Terms.product((q, z(q)), (k.transpose(-1, -2), z(k).transpose(-1, -2)))
        worst["S"] = max(worst["S"], float(torch.where(kept, ts.quanta, 0.0).max()))
        one = torch.ones(nk, 1, dtype=torch.float64)
        worst["l"] = max(worst["l"], float(Terms.product((P, z(P)), (one, z(one))).quanta.max()))
        worst["PV"] = max(worst["PV"], float(Terms.product((P, z(P)), (v, z(v))).quanta.max()))

        bm, rm = _block_max(s, nk)
        rise = rm[..., 1:] - rm[..., :-1]
        worst["rise"] = min(worst["rise"], float(torch.where(rise > 0, rise, math.inf).min()) if rise.numel() else math.inf)
        # the running max n at each key, and the keys whose e survives (computed with the final max)
        n = rm.repeat_interleave(BKV, -1)[..., :nk]
        surv = n == s.amax(-1, keepdim=True)
        x = s - n
        frac = surv & (x < 0) & (x > -FRAC_MAX)
        worst["gap"] = min(worst["gap"], float(torch.where(surv & (x <= -FRAC_MAX), -x, math.inf).min()))
        worst["n"] = max(worst["n"], float(torch.where(frac, n.abs(), 0.0).max()))
        if bool(frac.any()):
            nf, xf = n[frac], x[frac]
            # fmaf(s, L, -fl(n L)) = fl(x L + rho), L = fl32(log2e), rho = n L - fl(n L): its distance from x log2e
            rho = ((nf * LOG2E_F32).float().double() - nf * LOG2E_F32).abs()
            d_arg = xf.abs() * abs(LOG2E_F32 - LOG2E) + rho + 2.0 ** -24 * (xf.abs() * LOG2E_F32 + rho)
            rel = math.log(2) * d_arg * 1.001 + EXP2F_ULPS * 2.0 ** -23
            m = tf32_boundary_distance(xf.exp()) - rel
            worst["margin"] = min(worst["margin"], float(m.min()))
    for name in ("S", "l", "PV"):
        assert worst[name] <= BUDGET, f"premise: {name} needs {worst[name]:.0f} quanta > 2^22"
    assert worst["gap"] >= GAP, f"premise: a dropped score only {worst['gap']} below the row's max"
    assert worst["rise"] >= GAP, f"premise: the running max rises by {worst['rise']} only (al neither 0 nor 1)"
    assert worst["n"] <= N_MAX, f"premise: a fractional e computed at |n| = {worst['n']}"
    assert worst["margin"] >= MARGIN, f"premise: a fractional e {worst['margin']:.3g} from a tf32 boundary"
    return worst


# ------------------------------------------------------------------------------------------------ report
def tiles(case: Case, rows: int, ldo: int) -> torch.Tensor:
    """[rows, ldo] index of the (slice, 128-query tile) of every output element, -1 outside the output."""
    B, ntq = case.BH // case.heads, (case.nq + BQ - 1) // BQ
    r = torch.arange(rows)[:, None]
    col = torch.arange(ldo)[None, :]
    b, q, h = r // case.nq, r % case.nq, col // D
    t = (b * case.heads + h) * ntq + q // BQ
    return torch.where((r < B * case.nq) & (col < case.heads * D), t, -1)


def _where(case: Case, role: torch.Tensor, r: int, col: int) -> str:
    B = case.BH // case.heads
    if r >= B * case.nq or col >= case.heads * D:
        return f"(row {r}, col {col}) outside the output"
    b, q = divmod(r, case.nq)
    h, cc = divmod(col, D)
    return f"(tile {q // BQ}, head {h}, batch {b}, row {q}, col {cc}; {ROLES[int(role[b * case.heads + h, q])]} row)"


def assert_exact(name: str, got: torch.Tensor, exp: torch.Tensor, case: Case, role: torch.Tensor, shown: int = 6):
    """torch.equal on output buffers [rows, ldo], or an AssertionError with the wrong elements per (tile, head) and the
    first few with their tile, head, row, column and the role of the row."""
    assert got.shape == exp.shape and got.dtype == exp.dtype, (name, tuple(got.shape), tuple(exp.shape), got.dtype)
    if torch.equal(got, exp):
        return
    g, e = got.cpu().float(), exp.cpu().float()
    bad = (g != e) & ~(torch.isnan(g) & torch.isnan(e))
    if not bool(bad.any()):
        return
    ntq = (case.nq + BQ - 1) // BQ
    t, cnt = torch.unique(tiles(case, *g.shape)[bad], return_counts=True)
    per = ", ".join("outside" if x < 0 else f"slice {x // ntq} tile {x % ntq}: {n}"
                    for x, n in zip(t[:10].tolist(), cnt[:10].tolist()))
    first = "; ".join(f"{_where(case, role, r, col)} got {float(g[r, col])!r} expected {float(e[r, col])!r}"
                      for r, col in bad.nonzero()[:shown].tolist())
    raise AssertionError(f"{name} {case.id}: {int(bad.sum())} of {bad.numel()} elements differ in {len(t)} (tile, head) "
                         f"pairs ({per}); first: {first}")


# ------------------------------------------------------------------------------------------------ case lists
ENGINE = [Case(BH, heads, N, N, seed=BH + N) for BH, heads, N in ENGINE_SHAPES]
RAGGED = [Case(6, 3, nq, nk, seed=nq * 1000 + nk) for nq, nk in [(n, n) for n in SQUARE] + RECT]
# ldo > heads 64 with a guard row, fp32-only, planes-only and both, nk_pad > nk with NaN padding
CONFIG = [Case(24, 12, 195, 195, seed=3), Case(24, 12, 129, 64, seed=4), Case(24, 12, 257, 300, seed=5),
          Case(24, 12, 200, 1, seed=6)]


def gpu_cases():
    return ENGINE + RAGGED + CONFIG
