"""The premise and the sensitivity of the bit-exact eval attention tests (test_attn_core_exact_gpu.py), on the CPU.

Premise: on every case the GPU file runs, the kept scores, sum P and every column of P V stay within 2^22 quanta per
element, every dropped score lies at least 110 below the row's max, the running max rises by 0 or by at least 110, and
every fractional e keeps its 2^-15 margin from the tf32 rounding boundaries (attn_core_exact.premise).

Emulation: an fp32 model of the kernel's online loop over 128-key blocks, with torch's fp32 exp2, the kernel's RN-tf32
bit trick, the per-block rescale by al and fp32 sums in torch's order.  Without defects it equals the closed-form
expectation bit for bit, also with exp2's results moved by up to 2 ulps, so the expected bits depend neither on the
order of the sums nor on exp2f's last bits.  With one defect switched on, it changes at least one output bit in every
(128-query tile, head) the defect can reach, so `torch.equal` on the GPU cannot pass a kernel with that defect."""
import math

import pytest
import torch

import attn_core_exact as A
from test_attention_core_gpu import bound, bound_ratio, tf32, tf32_trunc


# ------------------------------------------------------------------------------------------------ premise
@pytest.mark.parametrize("case", A.gpu_cases(), ids=lambda c: c.id)
def test_premise(case):
    c = A.make(case)
    A.premise(c)
    for n in ("q", "k", "v"):
        assert torch.equal(c[n], tf32(c[n])), f"{n} is not tf32-exact"
    assert bool(torch.isfinite(A.expect(c)).all())


def test_roles_are_mixed_in_every_tile_and_head():
    """Every (128-query tile, head) of 12 rows or more holds every role, and each role has the structure it is for."""
    case = A.Case(8, 4, 300, 400, seed=7)
    c = A.make(case)
    role = c["role"]
    for t0 in range(0, case.nq, A.BQ):
        for bh in range(case.BH):
            r = role[bh, t0:t0 + A.BQ]
            if r.numel() >= 12:
                assert set(r.tolist()) == set(range(len(A.ROLES))), (bh, t0, r.unique().tolist())
    s = c["q"].double() @ c["k"].double().transpose(-1, -2)
    P = A.weights(s)
    kept = (P > 0).sum(-1)
    frac = ((P > 0) & (P < 1)).sum(-1)
    bm, rm = A._block_max(s, case.nk)
    blk = torch.arange(case.nk) // A.BKV
    kb = torch.where(P > 0, blk, -1)
    first_kept = torch.where(P > 0, blk, 1 << 20).amin(-1)
    last_kept = kb.amax(-1)
    nb = torch.arange(bm.shape[-1])
    decoy = (bm >= -300) & (bm <= -A.GAP)
    for x, want in ((A.ONE, lambda i: kept[i] == 1), (A.UNIFORM, lambda i: kept[i] == case.nk),
                    (A.MULTI, lambda i: (kept[i] >= 2) & (frac[i] == 0)),
                    (A.FRAC, lambda i: (kept[i] == 2) & (frac[i] == 1)),
                    (A.DECOY_FIRST, lambda i: (decoy[i] & (nb < first_kept[i][..., None])).any(-1)),
                    (A.DECOY_LAST, lambda i: (decoy[i] & (nb > last_kept[i][..., None])).any(-1))):
        i = role == x
        assert bool(want(i).all()), A.ROLES[x]
    assert set(kept[role == A.MULTI].unique().tolist()) == set(A.SIZES)


# ------------------------------------------------------------------------------------------------ the emulation
def _pad(x, n):
    return torch.cat((x, x.new_zeros(x.shape[0], n - x.shape[1], x.shape[2])), 1)


def _nudge(ulps):
    """exp2 with every result other than 0 and 1 moved by `ulps` units in the last place."""
    def exp2(x):
        e = torch.exp2(x)
        bits = e.view(torch.int32) + ulps
        return torch.where((e == 0) | (e == 1) | ~torch.isfinite(e), e, bits.view(torch.float32))
    return exp2


def emulate(c, heads, d=frozenset(), exp2=torch.exp2):
    """The kernel's output [B nq, heads 64] (fp32) from its online loop over 128-key blocks, with the defects `d`."""
    q, k, v = c["q"], c["k"], c["v"]
    BH, nq, _ = q.shape
    nk = k.shape[1]
    B = BH // heads
    nqp, nblk = (nq + A.BQ - 1) // A.BQ * A.BQ, (nk + A.BKV - 1) // A.BKV
    kp, vp = _pad(k, nblk * A.BKV), _pad(v, nblk * A.BKV)   # TMA zero-fills rows past nq and nk
    S = (_pad(q, nqp).double() @ kp.double().transpose(-1, -2)).float()
    L2 = torch.tensor(A.LOG2E_F32)
    thr = nk + (1 if "mask_plus_one" in d else -1 if "mask_minus_one" in d else 0)
    m = torch.full((BH, nqp), -math.inf)
    l_ = torch.zeros(BH, nqp)
    o = torch.zeros(BH, nqp, A.D)
    for j in range(nblk):
        s = S[..., j * A.BKV:(j + 1) * A.BKV]
        if (j + 1) * A.BKV > nk and "no_mask" not in d:
            s = torch.where(j * A.BKV + torch.arange(A.BKV) >= thr, -math.inf, s)
        b = s.amax(-1)
        n = b if "max_reset" in d else torch.maximum(m, b)
        al = torch.zeros_like(n) if j == 0 else exp2((m - n) * L2)
        ne = m if ("stale_max" in d and j > 0) else n
        arg = (s.double() * A.LOG2E_F32 + (-ne * L2).double()[..., None]).float()   # fmaf(s, log2e, -n log2e)
        e = exp2(arg)
        P = tf32_trunc(e) if "trunc_p" in d else tf32(e)
        ps = (e if "l_unrounded" in d else P).sum(-1)
        l_ = (l_ if "no_rescale_l" in d else l_ * al) + ps
        pv = (P.double() @ vp[:, j * A.BKV:(j + 1) * A.BKV].double()).float()
        o = (o if "no_rescale_o" in d else o * al[..., None]) + pv
        m = n
    inv = 1.0 / l_
    if "rcp_up" in d or "rcp_down" in d:
        inv = torch.nextafter(inv, torch.full_like(inv, math.inf if "rcp_up" in d else 0.0))
    out = (o * inv[..., None]).view(B, heads, nqp, A.D)
    buf = torch.zeros(B * nq, heads * A.D)
    dst = [(h + 1) % heads for h in range(heads)] if "next_head" in d else list(range(heads))
    b4 = buf.view(B, nq, heads, A.D)
    b4[:, :, dst] = out[:, :, :nq].transpose(1, 2)
    if "write_past_nq" in d:   # rows nq .. of the last query tile land on the next batch's first rows
        for b in range(B):
            r = b * nq + torch.arange(nq, nqp)
            ok = r < B * nq
            buf.view(B * nq, heads, A.D)[r[ok][:, None], torch.tensor(dst)[None, :]] = \
                out[b, :, nq:].transpose(0, 1)[ok]
    return buf


REPRESENTATIVE = [A.Case(6, 3, 150, 300, seed=31), A.Case(4, 2, 200, 257, seed=32), A.Case(6, 3, 140, 200, seed=33)]


@pytest.fixture(scope="module", params=REPRESENTATIVE, ids=lambda c: c.id)
def rep(request):
    case = request.param
    c = A.make(case)
    A.premise(c)
    return case, c, A.to_rows(A.expect(c), case.heads)


@pytest.mark.parametrize("ulps", [0, -2, -1, 1, 2])
def test_emulation_equals_the_closed_form(rep, ulps):
    case, c, exp = rep
    got = emulate(c, case.heads, exp2=_nudge(ulps) if ulps else torch.exp2)
    A.assert_exact("emulation", got, exp, case, c["role"])


def test_emulation_equals_the_closed_form_on_one_key_and_a_full_block():
    for case in (A.Case(6, 3, 130, 1, seed=34), A.Case(4, 2, 128, 256, seed=35)):
        c = A.make(case)
        A.premise(c)
        A.assert_exact("emulation", emulate(c, case.heads), A.to_rows(A.expect(c), case.heads), case, c["role"])


def test_exact_answer_is_inside_the_tf32_bound():
    """The exact expectation stays inside test_attention_core_gpu.bound on the same data: the two oracles agree."""
    for case in (REPRESENTATIVE[0], REPRESENTATIVE[1], A.Case(2, 2, 130, 1, seed=36)):
        c = A.make(case)
        ref, bnd = bound(c["q"], c["k"], c["v"])
        assert bound_ratio(A.expect(c), ref, bnd) < 1.0, case.id


# defect -> what it models:
#   trunc_p: P truncated instead of rounded; l_unrounded: l sums e, not P; no_rescale_l / no_rescale_o: l or O not
#   multiplied by al; stale_max: e computed with the running max before this block's update; max_reset: the running
#   max replaced by the block max; no_mask: keys >= nk kept (TMA reads them as zeros); mask_plus_one / mask_minus_one:
#   the last block's mask off by one either way; rcp_up / rcp_down: 1 / l one ulp off (rcp.approx, __fdividef);
#   next_head: head h written to column block h + 1; write_past_nq: rows >= nq of a ragged query tile written
DEFECTS = ("trunc_p", "l_unrounded", "no_rescale_l", "no_rescale_o", "stale_max", "max_reset", "no_mask",
           "mask_plus_one", "mask_minus_one", "rcp_up", "rcp_down", "next_head", "write_past_nq")


def _reach(case, c, defect):
    """The (slice, 128-query tile) indices whose output the defect can change at all."""
    B, nq, nk, heads = case.BH // case.heads, case.nq, case.nk, case.heads
    ntq = (nq + A.BQ - 1) // A.BQ
    if defect == "next_head":
        rows = torch.full((case.BH, nq), heads > 1)
    elif defect == "write_past_nq":
        tl = A.tiles(case, B * nq, heads * A.D)
        hit = torch.zeros(B * nq, dtype=torch.bool)
        for b in range(B):
            r = b * nq + torch.arange(nq, ntq * A.BQ)
            hit[r[r < B * nq]] = True
        return set(tl[hit].unique().tolist())
    else:
        s = c["q"].double() @ c["k"].double().transpose(-1, -2)
        P = A.weights(s)
        bm, rm = A._block_max(s, nk)
        nonzero = (A.expect(c) != 0).any(-1)
        ragged = nk % A.BKV != 0
        rows = {"trunc_p": ((P > 0) & (P < 1)).any(-1), "l_unrounded": ((P > 0) & (P < 1)).any(-1),
                "no_rescale_l": (rm[..., 1:] > rm[..., :-1]).any(-1),
                "no_rescale_o": (rm[..., 1:] > rm[..., :-1]).any(-1),
                "stale_max": (rm[..., 1:] > rm[..., :-1]).any(-1), "max_reset": (bm[..., 1:] < rm[..., 1:]).any(-1),
                "no_mask": torch.full((case.BH, nq), ragged), "mask_plus_one": torch.full((case.BH, nq), ragged),
                "mask_minus_one": (P[..., -1] > 0) & ragged,
                "rcp_up": torch.ones(case.BH, nq, dtype=torch.bool),
                "rcp_down": torch.ones(case.BH, nq, dtype=torch.bool)}[defect] & nonzero
    t = torch.arange(case.BH)[:, None] * ntq + torch.arange(nq)[None, :] // A.BQ
    return set(t[rows].unique().tolist())


@pytest.mark.parametrize("defect", DEFECTS)
def test_defect_changes_every_tile_it_touches(rep, defect):
    case, c, exp = rep
    got = emulate(c, case.heads, frozenset({defect}))
    tl = A.tiles(case, *exp.shape)
    bad = (got != exp) | (torch.isnan(got) != torch.isnan(exp))
    hit = set(tl[bad].unique().tolist())
    touched = _reach(case, c, defect)
    ntiles = case.BH * ((case.nq + A.BQ - 1) // A.BQ)
    # every tile holds every role, so every defect reaches every tile; write_past_nq reaches the first tile of every
    # head of every batch but the first
    want = case.BH - case.heads if defect == "write_past_nq" else ntiles
    assert len(touched) >= want, (defect, len(touched), want)
    missed = sorted(touched - hit)
    assert not missed, f"{defect}: {len(missed)} of {len(touched)} (slice, tile) pairs unchanged, e.g. {missed[:6]}"
