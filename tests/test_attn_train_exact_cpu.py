"""The premise and the sensitivity of the bit-exact training-attention tests (test_attn_train_exact_gpu.py), on the CPU.

Premise: for every case the GPU file runs, every product, D and dS stays within 2^22 quanta per output element, every
dropped score lies at least 110 below the kept ones (expf underflows to 0 below -103.97), and the data has what the
defect models below need: rounded, not exact, lo planes in the splits of dS and of Q and K.

Emulation: a fp64 model of the four kernels that walks 64-row query and key tiles as they do.  It has the flash
forward's running max and sum, dkdv's loop over query tiles with LSE = +inf past nq, dq's loop over key tiles with the
padded keys masked, and rowdot's lanes.  Without defects it equals the dense references bit for bit.  With one defect
switched on, it changes at least one element of every output tile the defect reaches, so `torch.equal` on the GPU cannot
pass a kernel with that defect.  A tile is reached when it holds a row that keeps a key (dQ, O, LSE) or a key that some
row keeps (dK, dV), narrowed to the rows and keys the defect can affect at all: those keeping a key in the skipped tile,
rows of no group for the padding mask, rows whose running max rises for the rescale, non-zero dropped cross products
of dO V^T, the WIDE_IN role for the inputs' split, rounded dS lo planes, non-zero D, and the slices a swap moves."""
import pytest
import torch

import attn_train_exact as A

S = A.SCALE


# ------------------------------------------------------------------------------------------------ premise
@pytest.mark.parametrize("case", A.cases() + A.e2e_cases(), ids=lambda c: c.id)
def test_premise(case):
    c = A.make(case)
    worst = A.premise(c)
    assert worst["gap"] >= A.GAP
    for n in ("q", "k", "v", "go", "o"):   # the drawn integers times quanta are fp32 values
        x = c[n].double()
        assert torch.equal(x, x.float().double())


@pytest.mark.parametrize("case", [A.Case(2, 3, 150, 190, 64, seed=1), A.Case(2, 16, 768, 768, 64, seed=2),
                                  A.Case(2, 3, 190, 150, 48, seed=3)], ids=lambda c: c.id)
def test_data_has_what_the_defect_models_need(case):
    """Rounded (not exact) lo planes in dS and in Q and K; non-zero lo planes of Q and K on the shared columns and of dO
    and V; rows keeping 1 to 4 keys and rows keeping them all; kept keys in the first, a middle and the ragged last key
    tile, and rows whose kept keys span two tiles."""
    c = A.make(case)
    B, H = case.B, case.H
    *_, (Sc, P, dP, D, dS) = A.backward_ref(c, parts=True)
    kept = dS[P > 0]
    assert int((A.planes(kept)[1] != A.planes(kept, trunc=True)[1]).sum()) > 20
    for n in ("q", "k"):
        x = A.slices(c[n], B, H)
        assert int((A.planes(x)[1] != A.planes(x, trunc=True)[1]).sum()) > 100, n
    for n in ("q", "k", "v", "go"):
        assert int((A.planes(c[n])[1] != 0).sum()) > 100, n
    _, _, k = A.forward_ref(c)
    assert set(k.unique().tolist()) >= {1.0, 2.0, 3.0, 4.0, float(case.nk)}
    tile = torch.arange(case.nk) // A.TILE
    nt = int(tile[-1]) + 1
    seen = set()
    for row in P.reshape(-1, case.nk):
        t = tile[row > 0].unique().tolist()
        if len(t) == 1:
            seen.add("first" if t[0] == 0 else "last" if t[0] == nt - 1 else "middle")
        elif len(t) == 2:
            seen.add("two")
    assert seen >= {"first", "middle", "last", "two"}, seen


# ------------------------------------------------------------------------------------------------ the emulation
def _expf(x):
    return torch.exp(x.float()).double()


def _f32(x):
    return x.float().double()


def _rows(x, r0, n):
    """Rows [r0, r0 + 64) of [BH, n, 64], zero past n."""
    t = x[:, r0:r0 + A.TILE]
    if t.shape[1] < A.TILE:
        t = torch.cat((t, t.new_zeros(t.shape[0], A.TILE - t.shape[1], t.shape[2])), 1)
    return t


def _skipped(d, kernel, tiles):
    for where, i in (("first", 0), ("middle", len(tiles) // 2), ("last", len(tiles) - 1)):
        if f"{kernel}.skip.{where}" in d:
            return tiles[i]
    return None


def _drop(d, kernel, product):
    for p in ("hh", "hl", "lh"):
        if f"{kernel}.{product}.{p}" in d:
            return p
    return None


def _inputs(c, d):
    """q, k, v, dO, O as [BH, n, 64] fp32-valued fp64 (dh = 48 zero-padded, or with the next token's first 16 columns
    under 'pad_read'), read from the swapped slice under 'swap'."""
    B, H, _, dh = c["q"].shape
    out = []
    for n in ("q", "k", "v", "go", "o"):
        x = A.slices(c[n], B, H).double()
        if "swap" in d:
            x = x[torch.tensor([(bh % B) * H + bh // B for bh in range(B * H)])]
        if dh == 48:
            pad = torch.zeros(x.shape[0], x.shape[1], 16, dtype=x.dtype)
            if "pad_read" in d and n in ("q", "k", "v", "go"):
                pad = torch.cat((x[:, 1:, :16], torch.zeros_like(pad[:, :1])), 1)
            x = torch.cat((x, pad), -1)
        out.append(x)
    return out


def emulate(c, d=frozenset()):
    """(O, LSE, dQ, dK, dV) of the four kernels' tile loops with the defects `d`, shaped like the references'."""
    B, H, nq, dh = c["q"].shape
    nk = c["k"].shape[2]
    Q, K, V, G, O = _inputs(c, d)
    ti = "trunc_in" in d
    pl = lambda x: A.planes(x, ti)   # noqa: E731  (the load's split of an input tile)
    ktiles, qtiles = list(range(0, nk, A.TILE)), list(range(0, nq, A.TILE))

    # forward: one pass over the key tiles with the running max m and sum l
    Qp = pl(Q)
    m = torch.full((B * H, nq), -torch.inf, dtype=torch.float64)
    l_ = torch.zeros(B * H, nq, dtype=torch.float64)
    o = torch.zeros(B * H, nq, A.TILE, dtype=torch.float64)
    skip = _skipped(d, "fwd", ktiles)
    for j0 in ktiles:
        if j0 == skip:
            continue
        s = A.mm3(Qp, A._t(pl(_rows(K, j0, nk))), _drop(d, "fwd", "qk")) * S
        if "fwd.no_mask" not in d:
            s = torch.where(j0 + torch.arange(A.TILE) < nk, s, -torch.inf)
        n = torch.maximum(m, s.max(-1).values)
        c0 = _expf(m - n)
        p = _expf(s - n[..., None])
        l_ = (l_ if "fwd.no_rescale_l" in d else l_ * c0) + p.sum(-1)
        o = (o if "fwd.no_rescale_o" in d else o * c0[..., None]) + A.mm3(A.planes(p), pl(_rows(V, j0, nk)))
        m = n
    out_o = (o.float() * (1.0 / l_.float())[..., None])[..., :dh]
    out_lse = (m + torch.log(l_)).float()

    # rowdot: D = rowsum(dO o O), lanes d and d + 32
    cols = 32 if "rowdot.lanes" in d else dh
    D = _f32((G[..., :cols] * O[..., :cols]).sum(-1))
    if "no_D" in d:
        D = torch.zeros_like(D)
    lse = c["lse"].double()
    td = "trunc_ds" in d

    # dkdv: every key tile over the query tiles
    Kp, Vp = pl(K), pl(V)
    dk = torch.zeros(B * H, nk, A.TILE, dtype=torch.float64)
    dv = torch.zeros_like(dk)
    skip = _skipped(d, "dkdv", qtiles)
    for i0 in qtiles:
        if i0 == skip:
            continue
        Qt, Gt = pl(_rows(Q, i0, nq)), pl(_rows(G, i0, nq))
        lt = torch.cat((lse[:, i0:i0 + A.TILE], torch.full((B * H, max(0, i0 + A.TILE - nq)), torch.inf,
                                                            dtype=torch.float64)), 1)
        Dt = torch.cat((D[:, i0:i0 + A.TILE], torch.zeros(B * H, max(0, i0 + A.TILE - nq), dtype=torch.float64)), 1)
        p = _expf(A.mm3(Kp, A._t(Qt), _drop(d, "dkdv", "qk")) * S - lt[:, None, :])
        dv = dv + A.mm3(A.planes(p), Gt)
        dst = _f32(p * (A.mm3(Vp, A._t(Gt), _drop(d, "dkdv", "dov")) - Dt[:, None, :]))
        dk = dk + A.mm3(A.planes(dst, td), Qt, _drop(d, "dkdv", "dsq"))
    out_dk = (dk.float() * (1.0 if "dkdv.no_scale" in d else S))[..., :dh]
    out_dv = (dv.float() * (S if "dkdv.scale_dv" in d else 1.0))[..., :dh]

    # dq: every query tile over the key tiles
    Qp, Gp = pl(Q), pl(G)
    dq = torch.zeros(B * H, nq, A.TILE, dtype=torch.float64)
    skip = _skipped(d, "dq", ktiles)
    for j0 in ktiles:
        if j0 == skip:
            continue
        Kt, Vt = pl(_rows(K, j0, nk)), pl(_rows(V, j0, nk))
        s = A.mm3(Qp, A._t(Kt), _drop(d, "dq", "qk")) * S
        dp = A.mm3(Gp, A._t(Vt), _drop(d, "dq", "dov"))
        p = torch.where(j0 + torch.arange(A.TILE) < nk, _expf(s - lse[..., None]), 0.0)
        ds = _f32(p * (dp - D[..., None]))
        dq = dq + A.mm3(A.planes(ds, td), Kt, _drop(d, "dq", "dsk"))
    out_dq = (dq.float() * (1.0 if "dq.no_scale" in d else S))[..., :dh]
    shp = lambda x: x.reshape(B, H, x.shape[1], dh)   # noqa: E731
    return A.tokens(out_o, B, H), out_lse, shp(out_dq), shp(out_dk), shp(out_dv)


# ragged last tiles of 20 rows or more, B != H so that a batch / head swap moves most slices
REPRESENTATIVE = [A.Case(2, 3, 150, 190, 64, seed=31), A.Case(2, 3, 190, 150, 48, seed=32),
                  A.Case(3, 2, 84, 212, 64, seed=33)]


@pytest.fixture(scope="module", params=REPRESENTATIVE, ids=lambda c: c.id)
def rep(request):
    case = request.param
    c = A.make(case)
    A.premise(c)
    o, lse, _ = A.forward_ref(c)
    return case, c, (o, lse) + A.backward_ref(c)


def test_emulation_equals_the_dense_references(rep):
    case, c, ref = rep
    got = emulate(c)
    for name, g, e in zip(("O", "LSE", "dQ", "dK", "dV"), got, ref):
        assert torch.equal(g, e), name


def test_emulation_of_the_autograd_case_gives_zero_dq_dk():
    case = A.e2e_cases()[-1]
    c = A.make(case)
    o, lse, _ = A.forward_ref(c)
    c = dict(c, lse=lse, o=o)
    got = emulate(c)
    ref = (o, lse) + A.backward_ref(c)
    for name, g, e in zip(("O", "LSE", "dQ", "dK", "dV"), got, ref):
        assert torch.equal(g, e), name
    assert not bool(got[2].any()) and not bool(got[3].any()) and bool(got[4].any())


# defect -> the kernels whose output tiles it must change: "fwd" (O and LSE per query tile), "dq" (dQ per query tile),
# "dkdv" (dK and dV per key tile).  "<kernel>.<product>.<hh | hl | lh>": that product of Q K^T (qk), dO V^T (dov),
# dS^T Q (dsq) or dS K (dsk) left out; "<kernel>.skip.<tile>": a key tile (fwd, dq) or query tile (dkdv) skipped;
# "trunc_in" / "trunc_ds": the lo plane of the inputs' / dS's split truncated; "swap": batch and head swapped;
# "pad_read": at dh = 48 the 16 padding columns read (modelled as the next token's first 16 columns) instead of zeroed.
_PRODUCTS = (("fwd", ("qk",)), ("dkdv", ("qk", "dov", "dsq")), ("dq", ("qk", "dov", "dsk")))
DEFECTS = {f"{k}.{p}.{x}": (k,) for k, ps in _PRODUCTS for p in ps for x in ("hh", "hl", "lh")}
DEFECTS.update({f"{k}.skip.{w}": (k,) for k in ("fwd", "dkdv", "dq") for w in ("first", "middle", "last")})
DEFECTS.update({"fwd.no_mask": ("fwd",), "fwd.no_rescale_o": ("fwd",), "fwd.no_rescale_l": ("fwd",),
                "rowdot.lanes": ("dq", "dkdv"), "no_D": ("dq", "dkdv"), "dq.no_scale": ("dq",),
                "dkdv.no_scale": ("dkdv",), "dkdv.scale_dv": ("dkdv",), "trunc_in": ("dq", "dkdv"),
                "trunc_ds": ("dq", "dkdv"), "swap": ("fwd", "dq", "dkdv"), "pad_read": ("fwd", "dq", "dkdv")})


def _reach(c, kernel, defect):
    """[B * H, n] rows (fwd, dq) or keys (dkdv) whose outputs the defect can change at all: rows that keep a key and
    keys that some row keeps, narrowed for the defects that need a particular tile or datum."""
    B, H, nq, dh = c["q"].shape
    nk = c["k"].shape[2]
    *_, (Sc, P, dP, D, dS) = A.backward_ref(c, parts=True)
    if kernel == "fwd":
        P = (Sc == Sc.max(-1, keepdim=True).values).double()   # the forward keeps every key on rows of no group
    pairs = P > 0
    kt, qt = torch.arange(nk) // A.TILE, torch.arange(nq) // A.TILE
    for where in ("first", "middle", "last"):
        if defect.endswith("skip." + where):
            tiles = qt if kernel == "dkdv" else kt
            nt = int(tiles[-1]) + 1
            t = {"first": 0, "middle": nt // 2, "last": nt - 1}[where]
            pairs = pairs & ((tiles == t)[:, None] if kernel == "dkdv" else (tiles == t)[None, :])
    if defect == "fwd.no_mask":
        pairs = pairs & ((c["qgrp"] < 0)[..., None] if nk % A.TILE else False)
    if defect.startswith("fwd.no_rescale"):   # rows whose running max rises after the first key tile
        first = Sc[..., :A.TILE].max(-1).values < Sc.max(-1).values
        pairs = pairs & first[..., None]
    if defect.endswith(("dov.hl", "dov.lh")):   # pairs where the dropped cross product is not zero (dkdv: V dO^T)
        (gh, gl), (vh, vl) = A.planes(A.slices(c["go"], B, H)), A.planes(A.slices(c["v"], B, H))
        g_hi = defect.endswith("hl") == (kernel == "dq")
        pairs = pairs & ((gh @ vl.transpose(-2, -1) if g_hi else gl @ vh.transpose(-2, -1)) != 0)
    if defect == "trunc_in":
        role = (c["qrole"] if kernel == "dq" else c["krole"]) == A.WIDE_IN
        pairs = pairs & (role[..., None] if kernel == "dq" else role[:, None, :])
    if defect == "trunc_ds":
        pairs = pairs & (A.planes(dS)[1] != A.planes(dS, trunc=True)[1])
    if defect in ("rowdot.lanes", "no_D"):
        G, O = A.slices(c["go"], B, H).double(), A.slices(c["o"], B, H).double()
        part = (G * O)[..., 32:].sum(-1) if defect == "rowdot.lanes" else D
        pairs = pairs & (part != 0)[..., None]
    if defect == "swap":
        moved = torch.tensor([(bh % B) * H + bh // B != bh for bh in range(B * H)])
        pairs = pairs & moved[:, None, None]
    return pairs.any(-2) if kernel == "dkdv" else pairs.any(-1)


def _changed_tiles(c, got, ref, kernel, defect):
    """(touched, changed): the (slice, 64-row tile) indices of the kernel's outputs that the defect can reach, and those
    where some element differs."""
    B, H, nq, _ = c["q"].shape
    nk = c["k"].shape[2]
    sl = lambda x: A.slices(x, B, H) if x.dim() > 2 else x[..., None]   # noqa: E731
    outs, n = {"fwd": ((0, 1), nq), "dq": ((2,), nq), "dkdv": ((3, 4), nk)}[kernel]
    diff = torch.zeros(B * H, n, dtype=torch.bool)
    for i in outs:
        diff |= (sl(got[i]) != sl(ref[i])).any(-1)
    tiles = A.row_tiles(c, n)
    return set(torch.unique(tiles[_reach(c, kernel, defect)]).tolist()), set(torch.unique(tiles[diff]).tolist())


@pytest.mark.parametrize("defect", sorted(DEFECTS))
def test_defect_changes_every_tile_it_touches(rep, defect):
    case, c, ref = rep
    if defect in ("rowdot.lanes", "pad_read") and case.dh != 48:
        pytest.skip("dh = 48 only")
    got = emulate(c, frozenset({defect}))
    for kernel in DEFECTS[defect]:
        touched, hit = _changed_tiles(c, got, ref, kernel, defect)
        assert len(touched) >= len(A.row_tiles(c, 1)) // 2 or defect.startswith(("fwd.skip", "fwd.no_")), \
            (defect, kernel, len(touched))
        missed = sorted(touched - hit)
        assert not missed, f"{defect} on {kernel}: {len(missed)} of {len(touched)} tiles unchanged, e.g. {missed[:6]}"
