"""The spatial memory's kernels against fp64: the read (LN_q, S = Q K_n^T, mem_softmax_kernel, the two-pass column sum into
bank.attn, P V), the append (LN_k rows, LN_v + split_transpose_kernel at column len, bank_bump_kernel), the similarity
gate (cos_rows_kernel + mean_rows_kernel) and the prune's gather, op by op and in lockstep with the oracle.

The reference is oracle.spann3r_oracle run in float64 on the GPU (state dict and inputs in double).  Reads are compared
on the memory term out - feat and on the increment of bank.attn, per batch item.  Banks use three patch grids: 45 tokens
(80 x 144, odd, so an odd frame count gives len % 4 != 0), 196 (224 x 224) and 768 (384 x 512).  Queries are noisy
mixes of three bank keys, one of them among the last three tokens in the first rows, so that the attention has a
realistic peak and the softmax's scalar tail and the last GEMM tiles carry weight.

With the 5e-4 cut, an entry whose fp64 weight lies within 1e-3 relative of the threshold may fall on either side of it
in fp32.  Rows holding such entries are held to the same bar plus the most the cut of those entries can move the
renormalised row (2 m / S in L1: m their weight, S the rest of the kept weight), and must be under 1 % of the rows.

Measured on one H100 80GB HBM3 (SXM, 700 W power limit): see the bars below; each is at most 3x the worst value measured over its cases.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import get_state_dict, rel_l2

C = 1024
GRID = {45: (80, 144), 196: (224, 224), 768: (384, 512)}
THRESH = 5e-4
FLIP_REL = 1e-3
# rel-L2 bars, raw / sharpened checkpoint; worst measured on that H100 over every case that uses them:
TOL_OUT = {False: 1e-4, True: 5e-5}     # out - feat: raw 6.2e-5 (50688 tokens, no cut), sharpened 2.0e-5
TOL_ATTN = {False: 8e-6, True: 5e-5}    # bank.attn increment: raw 2.9e-6, sharpened 1.9e-5
TOL_GATE = 2.5e-7                        # absolute, on mean_p cos: measured 9.4e-8
TOL_PLANES = 7e-6                        # appended split-bf16 planes, rel-L2: measured 2.5e-6


# ------------------------------------------------------------------------------------------------
# helpers (the pure ones are checked on the CPU at the end of the file)
# ------------------------------------------------------------------------------------------------
def flip_slack(w: torch.Tensor, thresh: float, rel: float = FLIP_REL):
    """w [..., M]: fp64 softmax weights before the cut.  Returns (rows holding an entry within `rel` of the threshold,
    per row the largest L1 distance by which cutting or keeping those entries can move the renormalised row: 2 m / S,
    m = their weight, S = the weight kept without them; inf where nothing else is kept)."""
    amb = (w - thresh).abs() <= rel * thresh
    m = (w * amb).sum(-1)
    s = (w * ((w >= thresh) & ~amb)).sum(-1)
    slack = torch.where(amb.any(-1), 2 * m / s, torch.zeros_like(m))
    return amb.any(-1), slack


def check_topk(weights: torch.Tensor, idx: torch.Tensor, k: int, margin: torch.Tensor | float = 0.0, rel: float = 1e-5):
    """weights [B, M] (fp64), idx [B, k'] the kept tokens.  Asserts a valid top-k: k distinct indices, every token whose
    weight is above the k-th largest by more than rel * |k-th| + margin kept, none below it by that much kept.
    Returns how many tokens per batch item the rule decided (0: every token ties with the k-th)."""
    B, M = weights.shape
    assert idx.shape == (B, k), (tuple(idx.shape), k)
    decided = []
    for b in range(B):
        sel = idx[b].long().cpu()
        assert sel.unique().numel() == k and int(sel.min()) >= 0 and int(sel.max()) < M
        w = weights[b].cpu()
        kth = w.sort(descending=True).values[k - 1]
        gap = rel * kth.abs() + margin
        kept = torch.zeros(M, dtype=torch.bool)
        kept[sel] = True
        above, below = w > kth + gap, w < kth - gap
        assert kept[above].all(), f"batch {b}: {int((~kept[above]).sum())} tokens clearly above the k-th weight dropped"
        assert not kept[below].any(), f"batch {b}: {int(kept[below].sum())} tokens clearly below the k-th weight kept"
        decided.append(int(above.sum() + below.sum()))
    return decided


def make_queries(k: torch.Tensor, N: int, sharpen: bool, g: torch.Generator, flat_rows: bool = False):
    """[B, N, C] queries from a bank k [B, M, C]: each row mixes three standardised bank keys (logit of the strongest
    ~ lo..lo + 3, the other two up to 9 below it, so some of them fall under the cut) with unit noise; rows 0-2 take
    their strongest key from the last three tokens.  flat_rows: every odd row is pure noise."""
    B, M, _ = k.shape
    dev = k.device
    w, lo = (8.0, 48.0) if sharpen else (1.0, 14.0)
    kh = (k - k.mean(-1, keepdim=True)) / k.std(-1, keepdim=True, unbiased=False)
    idx = torch.randint(0, M, (B, N, 3), device=dev, generator=g)
    n_tail = min(3, N, M)
    idx[:, :n_tail, 0] = torch.arange(M - 1, M - 1 - n_tail, -1, device=dev)
    t1 = lo + 3 * torch.rand(B, N, 1, device=dev, generator=g)
    t = torch.cat((t1, t1 - 1 - 8 * torch.rand(B, N, 2, device=dev, generator=g)), -1)
    a = t / (32.0 * w)            # logit ~ sqrt(C) * norm weight * correlation / sqrt(C) ... = 32 w a
    if flat_rows:
        a[:, 1::2] = 0.0
    peaks = kh[torch.arange(B, device=dev)[:, None, None], idx]
    noise = torch.randn(B, N, C, device=dev, generator=g)
    q = (a[..., None] * peaks).sum(2) + (1 - (a * a).sum(-1, keepdim=True)).clamp_min(0.05).sqrt() * noise
    return q.contiguous()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _engine(models, sharpen, B, N):
    H, W = GRID[N]
    return models[sharpen]._engine_for(B, H, W)


def _fill(eng, k, v, cap=None):
    """A MemoryBank holding k, v [B, M, C] (M a multiple of the engine's N), appended one frame at a time."""
    from spann3r_b200.engine import MemoryBank
    B, M, _ = k.shape
    N = eng.N
    bank = MemoryBank(B, cap if cap is not None else M + 77, "cuda")
    for t in range(M // N):
        eng.memory_append(bank, k[:, t * N:(t + 1) * N].contiguous(), v[:, t * N:(t + 1) * N].contiguous())
    assert bank.len == M
    return bank


def ref_read(sd64, k, v, q, thresh):
    """fp64 read of oracle.SpatialMemory on a bank k, v: (memory term [B, N, C], attn increment [B, M])."""
    from oracle.spann3r_oracle import SpatialMemory
    sm = SpatialMemory(sd64, attn_thresh=thresh)
    sm.mem_k, sm.mem_v = k.double(), v.double()
    z = torch.zeros(k.shape[0], k.shape[1], 1, dtype=torch.float64, device=k.device)
    sm.mem_attn, sm.mem_count = z, z.clone()
    out = sm.memory_read(q.double(), res=False)
    inc = sm.mem_attn[..., 0]
    assert out.dtype == torch.float64 and inc.dtype == torch.float64
    return out, inc


def ref_weights(sd64, k, q):
    """fp64 softmax weights before the cut [B, N, M] (the first half of oracle.SpatialMemory.memory_read)."""
    from oracle.spann3r_oracle import layernorm
    qn = layernorm(sd64, "norm_q", q.double(), 1e-5)
    kn = layernorm(sd64, "norm_k", k.double(), 1e-5)
    w = torch.softmax(torch.einsum("bpc,bxc->bpx", qn, kn) / math.sqrt(C), dim=-1)
    assert w.dtype == torch.float64
    return w


def ln_v64(sd64, v):
    from oracle.spann3r_oracle import layernorm
    return layernorm(sd64, "norm_v", v.double(), 1e-5)


def check_read(sd64, k, v, q, thresh, out, inc, sharpen, what):
    """out [B, N, C] of the device read with feat = q, inc [B, M] its bank.attn increment, against fp64.
    Returns the worst (out - feat, increment) rel-L2 over the batch items."""
    tol, tol_inc = TOL_OUT[sharpen], TOL_ATTN[sharpen]
    ref_out, ref_inc = ref_read(sd64, k, v, q, thresh)
    assert torch.isfinite(ref_out).all(), f"{what}: the fp64 read has empty rows; the inputs are meant to avoid them"
    mem = out.double() - q.double()
    w = ref_weights(sd64, k, q) if thresh > 0 else None
    vmax = ln_v64(sd64, v).norm(dim=-1).amax(-1)
    if w is not None:
        flips, slacks = flip_slack(w, thresh)
    else:
        flips, slacks = torch.zeros(q.shape[:2], dtype=torch.bool, device=q.device), torch.zeros(q.shape[:2], device=q.device)
    assert float(flips.double().mean()) < 0.01, f"{what}: {int(flips.sum())} of {flips.numel()} rows near the cut"
    worst = [0.0, 0.0]
    for b in range(k.shape[0]):
        flip, slack = flips[b], slacks[b]
        e_out = rel_l2(mem[b][~flip], ref_out[b][~flip])
        if flip.any():
            d = (mem[b][flip] - ref_out[b][flip]).norm(dim=-1)
            bound = tol * ref_out[b][flip].norm(dim=-1) + slack[flip] * vmax[b]
            assert (d <= bound).all(), f"{what} b={b}: a row near the cut is off by more than its entries can move it"
        e_inc = rel_l2(inc[b], ref_inc[b])
        bound_inc = tol_inc + float(slack.sum()) / float(ref_inc[b].norm())
        assert e_out < tol, f"{what} b={b}: out - feat rel-L2 {e_out:.3e} >= {tol:.1e}"
        assert e_inc < bound_inc, f"{what} b={b}: bank.attn increment rel-L2 {e_inc:.3e} >= {bound_inc:.1e}"
        worst = [max(worst[0], e_out), max(worst[1], e_inc)]
    print(f"[measured] {what}: out {worst[0]:.3e} attn {worst[1]:.3e}")
    return worst


# ------------------------------------------------------------------------------------------------
# fixtures
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models():
    from spann3r_b200 import Spann3R, _lib
    _lib.require_device()
    out = {}
    for sharpen in (False, True):
        m = Spann3R(dus3r_name=None)
        m.load_state_dict(get_state_dict(sharpen), strict=True)
        out[sharpen] = m.cuda().eval()
    return out


@pytest.fixture(scope="module")
def sd64():
    return {s: {k: v.cuda().double() for k, v in get_state_dict(s).items() if k.split(".")[0] in ("norm_q", "norm_k", "norm_v")}
            for s in (False, True)}


# ------------------------------------------------------------------------------------------------
# 1. read against fp64
# ------------------------------------------------------------------------------------------------
READ_CASES = [
    # N, frames, B, full bank (cap == len)
    (45, 1, 1, False), (45, 1, 3, False), (45, 2, 2, False), (45, 3, 1, False), (45, 3, 3, False),
    (196, 2, 1, False), (196, 2, 3, False),
    (196, 8, 2, True),       # len 1568 = cap: the ragged last column tile of sequence 0 reads sequence 1's rows
    (768, 5, 2, False), (768, 5, 3, True),
    (768, 16, 2, False),     # 12288 tokens: the softmax row is exactly 48 KB of shared memory
    (768, 17, 2, False),     # past it: the opt-in shared-memory path
    (768, 66, 1, True),      # 50688, the longest bank under the 51200-token row buffer
]


@pytest.mark.gpu
@pytest.mark.parametrize("sharpen", [False, True], ids=["raw", "sharp"])
@pytest.mark.parametrize("N,frames,B,full", READ_CASES)
def test_read_vs_fp64(models, sd64, N, frames, B, full, sharpen):
    """Per batch item, at TOL_OUT / TOL_ATTN.  len 12288 (exactly 48 KB of scores per row) failed to launch before the
    softmax opted in to the large shared-memory buffer for it."""
    eng = _engine(models, sharpen, B, N)
    M = N * frames
    g = _gen(1000 * N + 10 * frames + B)
    k = torch.randn(B, M, C, device="cuda", generator=g)
    v = torch.randn(B, M, C, device="cuda", generator=g)
    bank = _fill(eng, k, v, cap=M if full else None)
    assert (bank.cap == M) == full
    for thresh in (0.0, THRESH):
        q = make_queries(k, N, sharpen, g, flat_rows=thresh == 0.0)
        bank.attn.zero_()
        out = eng.memory_read(bank, q, thresh)
        torch.cuda.synchronize()
        check_read(sd64[sharpen], k, v, q, thresh, out, bank.attn[:, :M], sharpen,
                   f"read N={N} M={M} B={B} full={full} thresh={thresh} sharpen={sharpen}")


# ------------------------------------------------------------------------------------------------
# 2. rows the cut empties
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_read_rows_emptied_by_the_cut(models, sd64):
    """Raw checkpoint, 2304 tokens: a flat (constant) query spreads ~1 / 2304 < 5e-4 over every token, the cut empties
    the row and the renormalisation divides 0 / 0.  NaN exactly where fp64 has it, bank.attn NaN for that sequence;
    the other sequence stays finite and matches fp64."""
    N, B, frames = 768, 2, 3
    M = N * frames
    eng = _engine(models, False, B, N)
    g = _gen(77)
    k = torch.randn(B, M, C, device="cuda", generator=g)
    v = torch.randn(B, M, C, device="cuda", generator=g)
    bank = _fill(eng, k, v)
    q = make_queries(k, N, False, g)
    q[0, ::2] = 0.5                                        # flat rows in sequence 0 only
    out = eng.memory_read(bank, q, THRESH)
    torch.cuda.synchronize()
    sd = sd64[False]
    ref_out, ref_inc = ref_read(sd, k, v, q, THRESH)
    mem = out.double() - q.double()
    nan_dev, nan_ref = torch.isnan(mem).any(-1), torch.isnan(ref_out).any(-1)
    assert int(nan_ref[0].sum()) == N // 2 and not nan_ref[1].any()
    assert torch.equal(nan_dev, nan_ref)
    assert torch.isnan(mem[nan_dev]).all()
    assert torch.isnan(bank.attn[0, :M]).all() and torch.isnan(ref_inc[0]).all()
    assert torch.isfinite(bank.attn[1, :M]).all()
    tol, tol_inc = TOL_OUT[False], TOL_ATTN[False]
    e0 = rel_l2(mem[0][~nan_ref[0]], ref_out[0][~nan_ref[0]])
    e1 = rel_l2(mem[1], ref_out[1])
    ei = rel_l2(bank.attn[1, :M], ref_inc[1])
    print(f"[measured] emptied rows: out {max(e0, e1):.3e} attn {ei:.3e}")
    assert e0 < tol and e1 < tol and ei < tol_inc, (e0, e1, ei)


# ------------------------------------------------------------------------------------------------
# 3. training-mode read: dropout mask across sequences
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("frames", [3, 5])
def test_dropout_read_vs_fp64(models, sd64, frames):
    """B = 2, N = 45, odd len, p = 0.15, no cut: the Philox keep-scale of flat index (b * N + n) * M + i, i.e. the row
    index runs on across sequences.  Bars as the eval read."""
    from spann3r_b200 import _lib
    N, B, p = 45, 2, 0.15
    M = N * frames
    for sharpen in (False, True):
        eng = _engine(models, sharpen, B, N)
        g = _gen(300 + frames)
        k = torch.randn(B, M, C, device="cuda", generator=g)
        v = torch.randn(B, M, C, device="cuda", generator=g)
        bank = _fill(eng, k, v)
        q = make_queries(k, N, sharpen, g, flat_rows=True)
        seed = 12345 + frames
        out = eng.memory_read(bank, q, 0.0, drop_p=p, seed=seed)
        mask = _lib.dropout_mask((B, N, M), seed, p, "cuda").double()
        torch.cuda.synchronize()
        sd = sd64[sharpen]
        w = ref_weights(sd, k, q) * mask
        ref_out = torch.einsum("bpx,bxc->bpc", w, ln_v64(sd, v))
        ref_inc = w.sum(1)
        tol, tol_inc = TOL_OUT[sharpen], TOL_ATTN[sharpen]
        for b in range(B):
            e_out = rel_l2(out[b].double() - q[b].double(), ref_out[b])
            e_inc = rel_l2(bank.attn[b, :M], ref_inc[b])
            print(f"[measured] dropout M={M} sharpen={sharpen} b={b}: out {e_out:.3e} attn {e_inc:.3e}")
            assert e_out < tol and e_inc < tol_inc, (b, e_out, e_inc)


# ------------------------------------------------------------------------------------------------
# 4. append
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N", [45, 196])
def test_append_vs_fp64(models, sd64, N):
    """Three appends at B = 2 with reads in between: raw rows bitwise, count / attn as add_mem, LN_k rows and the
    transposed LN_v columns [len, len + N) of each sequence within 1e-5 of fp64, everything else untouched (the bank is
    pre-filled with a sentinel so that a write to the wrong place shows)."""
    from spann3r_b200.engine import MemoryBank
    B, frames = 2, 3
    eng = _engine(models, True, B, N)
    sd = sd64[True]
    bank = MemoryBank(B, N * frames + 40, "cuda")
    for name in ("kn_hi", "kn_lo", "vnt_hi", "vnt_lo", "k_raw", "v_raw", "attn", "count"):
        getattr(bank, name).fill_(7.0)
    g = _gen(400 + N)
    worst = 0.0
    for t in range(frames):
        M = bank.len
        fk = torch.randn(B, N, C, device="cuda", generator=g) * 2 + 0.3
        fv = torch.randn(B, N, C, device="cuda", generator=g) * 3 - 0.2
        before = {n: getattr(bank, n).clone() for n in ("kn_hi", "kn_lo", "vnt_hi", "vnt_lo", "k_raw", "v_raw", "attn", "count")}
        eng.memory_append(bank, fk, fv)
        torch.cuda.synchronize()
        assert bank.len == M + N
        new = slice(M, M + N)
        assert torch.equal(bank.k_raw[:, new], fk) and torch.equal(bank.v_raw[:, new], fv)
        kn = bank.kn_hi[:, new].double() + bank.kn_lo[:, new].double()
        vn = (bank.vnt_hi[:, :, new].double() + bank.vnt_lo[:, :, new].double()).transpose(1, 2)
        for b in range(B):
            ek = rel_l2(kn[b], F.layer_norm(fk[b].double(), (C,), sd["norm_k.weight"], sd["norm_k.bias"], 1e-5))
            ev = rel_l2(vn[b], ln_v64(sd, fv[b]))
            assert ek < TOL_PLANES and ev < TOL_PLANES, (t, b, ek, ev)
            worst = max(worst, ek, ev)
        assert torch.equal(bank.count[:, :M], before["count"][:, :M] + 1)
        assert torch.equal(bank.attn[:, :M], before["attn"][:, :M])
        assert (bank.count[:, new] == 0).all() and (bank.attn[:, new] == 0).all()
        for name, b4 in before.items():
            cur = getattr(bank, name)
            if name.startswith("vnt"):
                assert torch.equal(cur[:, :, :M], b4[:, :, :M]) and torch.equal(cur[:, :, M + N:], b4[:, :, M + N:]), name
            elif name in ("attn", "count"):
                assert torch.equal(cur[:, M + N:], b4[:, M + N:]), name
            else:
                assert torch.equal(cur[:, :M], b4[:, :M]) and torch.equal(cur[:, M + N:], b4[:, M + N:]), name
        eng.memory_read(bank, fk, 0.0)          # attn of the old tokens becomes non-zero before the next bump
        torch.cuda.synchronize()
    print(f"[measured] append N={N}: planes {worst:.3e}")


# ------------------------------------------------------------------------------------------------
# 5. stale state past len
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,fill,keep", [(768, 12, 5), (45, 13, 5)])
def test_read_after_prune_ignores_stale_state(models, sd64, N, fill, keep):
    """A wide read leaves probabilities out to fill * N in the engine's scratch Pm; the bank is gathered down to a random
    keep * N rows and every bank row / column past len is set to NaN.  The next read is finite, matches fp64 and equals
    bitwise a read from a bank freshly appended with the kept rows."""
    from spann3r_b200.engine import MemoryBank
    B, sharpen = 2, True
    eng = _engine(models, sharpen, B, N)
    M, K = N * fill, N * keep
    g = _gen(500 + N)
    k = torch.randn(B, M, C, device="cuda", generator=g)
    v = torch.randn(B, M, C, device="cuda", generator=g)
    bank = _fill(eng, k, v, cap=M)
    eng.memory_read(bank, make_queries(k, N, sharpen, g, flat_rows=True), 0.0)
    idx = torch.stack([torch.randperm(M, device="cuda", generator=g)[:K] for _ in range(B)])
    bank.gather(idx)
    nan = float("nan")
    for name in ("kn_hi", "kn_lo", "k_raw", "v_raw"):
        getattr(bank, name)[:, K:] = nan
    for name in ("vnt_hi", "vnt_lo"):
        getattr(bank, name)[:, :, K:] = nan
    bank.attn[:, K:] = nan
    bank.count[:, K:] = nan
    kk = torch.gather(k, 1, idx[..., None].expand(-1, -1, C))
    vk = torch.gather(v, 1, idx[..., None].expand(-1, -1, C))
    q = make_queries(kk, N, sharpen, g)
    a0 = bank.attn[:, :K].clone()
    out = eng.memory_read(bank, q, THRESH)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and torch.isfinite(bank.attn[:, :K]).all()
    check_read(sd64[sharpen], kk, vk, q, THRESH, out, bank.attn[:, :K].double() - a0.double(), sharpen,
               f"stale N={N} {M}->{K}")
    fresh = _fill(eng, kk, vk, cap=bank.cap)
    out2 = eng.memory_read(fresh, q, THRESH)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    assert rel_l2(fresh.attn[:, :K], bank.attn[:, :K].double() - a0.double()) < TOL_ATTN[sharpen]


# ------------------------------------------------------------------------------------------------
# 6. scratch growth, 7. determinism
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scratch_growth_between_banks(models, sd64):
    """A fresh engine reads bank A (cap 160), then B (cap 1824: the score / probability scratch is reallocated and the
    plan cache cleared), then A again: all three match fp64, and both reads of A are bitwise equal."""
    from spann3r_b200.engine import Engine
    N, B, sharpen = 45, 2, True
    eng = Engine(models[sharpen]._weights(), B, *GRID[N])
    g = _gen(600)
    data = {}
    for name, frames, cap in (("A", 3, 160), ("B", 40, 1824)):
        k = torch.randn(B, N * frames, C, device="cuda", generator=g)
        v = torch.randn(B, N * frames, C, device="cuda", generator=g)
        data[name] = (k, v, _fill(eng, k, v, cap=cap), make_queries(k, N, sharpen, g))
    assert data["A"][2].cap == 160 and data["B"][2].cap == 1824
    outs, attns = [], []
    for name in ("A", "B", "A"):
        k, v, bank, q = data[name]
        bank.attn.zero_()
        out = eng.memory_read(bank, q, THRESH)
        torch.cuda.synchronize()
        check_read(sd64[sharpen], k, v, q, THRESH, out, bank.attn[:, :bank.len], sharpen, f"growth {name}")
        outs.append(out)
        attns.append(bank.attn.clone())
    assert torch.equal(outs[0], outs[2]) and torch.equal(attns[0], attns[2])


@pytest.mark.gpu
@pytest.mark.parametrize("N,frames,B,sharpen,thresh", [(768, 5, 2, True, THRESH), (45, 3, 3, False, 0.0)])
def test_read_is_deterministic(models, N, frames, B, sharpen, thresh):
    eng = _engine(models, sharpen, B, N)
    g = _gen(700 + N)
    k = torch.randn(B, N * frames, C, device="cuda", generator=g)
    v = torch.randn(B, N * frames, C, device="cuda", generator=g)
    bank = _fill(eng, k, v)
    q = make_queries(k, N, sharpen, g, flat_rows=True)
    a0 = bank.attn.clone()
    o1 = eng.memory_read(bank, q, thresh)
    a1 = bank.attn.clone()
    bank.attn.copy_(a0)
    o2 = eng.memory_read(bank, q, thresh)
    torch.cuda.synchronize()
    assert torch.equal(o1, o2) and torch.equal(a1, bank.attn)


# ------------------------------------------------------------------------------------------------
# 8. similarity gate
# ------------------------------------------------------------------------------------------------
def gate64(k_window, feat_k, N):
    """fp64 mean_p cos(F.normalize(feat_k), F.normalize(window)) of spann3r/model.py:97-118: [B, frames in window]."""
    B = feat_k.shape[0]
    w = k_window.double().reshape(B, -1, N, C)
    return torch.einsum("bpc,btpc->btp", F.normalize(feat_k.double(), p=2, dim=-1), F.normalize(w, p=2, dim=-1)).mean(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [45, 196, 768])
def test_check_sim_vs_fp64(models, N, B):
    """Gate values for wm = 1, 2, 5, 8 against fp64, absolute bar TOL_GATE.  Sequence 0 is a near-duplicate of the last
    frame (~0.99); some tokens are zero vectors (F.normalize's 1e-12 floor) or tiny (norm ~3e-5, far above the floor)."""
    eng = _engine(models, True, B, N)
    g = _gen(800 + N + B)
    frames = 9
    k = torch.randn(B, N * frames, C, device="cuda", generator=g)
    k[:, -N + 1] = 0.0                       # a zero token in the last frame
    k[:, -2 * N + 3] *= 1e-6                 # a tiny one in the frame before
    bank = _fill(eng, k, torch.randn_like(k))
    feat = torch.randn(B, N, C, device="cuda", generator=g)
    feat[0] = k[0, -N:] + 0.14 * torch.randn(N, C, device="cuda", generator=g)
    feat[:, 0] = 0.0
    feat[:, 2] *= 1e-6
    worst = 0.0
    for wm in (1, 2, 5, 8):
        got = eng.check_sim(bank, feat.contiguous(), wm)
        torch.cuda.synchronize()
        ref = gate64(k[:, -wm * N:], feat, N)
        assert ref[0, -1] > 0.9
        err = float((got.double() - ref).abs().max())
        assert err < TOL_GATE, (wm, err)
        worst = max(worst, err)
    print(f"[measured] gate N={N} B={B}: {worst:.3e}")


# ------------------------------------------------------------------------------------------------
# 9. model.SpatialMemory in lockstep with the fp64 oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("N,long_frames,sharpen,frames", [
    (45, 3, True, 24), (196, 3, True, 24), (45, 3, False, 24), (45, 0, True, 10), (196, 0, True, 10)])
def test_lockstep_with_fp64_oracle(models, sd64, monkeypatch, N, long_frames, sharpen, frames):
    """B = 2, work_mem_size 5, long_mem_size = long_frames * N (0: the oldest working frame is dropped).  After every
    frame: len, wm, lm, mem_count and the raw keys equal, the skip decision equal (one frame is a near-duplicate in
    sequence 0 only), the reads and bank.attn within TOL_OUT / TOL_ATTN.  At every prune the device's kept indices are a valid top-k of the fp64
    weights (see check_topk; the margin adds twice the largest gap between the device's and fp64's weights), and the
    fp64 state gathers the same indices.  A prune to 3 N tokens leaves fewer than the 5 working frames, and the gate's
    window is then the whole bank, as in the reference (the device used to refuse the next similarity check)."""
    from oracle import spann3r_oracle as orc
    from spann3r_b200.engine import MemoryBank
    from spann3r_b200.model import SpatialMemory as DevMem
    B, L = 2, long_frames * N
    eng = _engine(models, sharpen, B, N)
    sd = sd64[sharpen]
    gathered = []
    orig_gather = MemoryBank.gather
    monkeypatch.setattr(MemoryBank, "gather", lambda self, idx: (gathered.append(idx.clone()), orig_gather(self, idx))[1])
    dev = DevMem(long_mem_size=L, work_mem_size=5, attn_thresh=THRESH, engine=eng)
    skips = []
    finish = dev.check_sim_finish
    dev.check_sim_finish = lambda pending, thresh=0.7: skips.append(finish(pending, thresh)) or skips[-1]
    ref = orc.SpatialMemory(sd, long_mem_size=L, work_mem_size=5, attn_thresh=THRESH)
    pre = {}
    prunes = []

    def prune64():
        cnt = ref.mem_count[..., 0]
        young = cnt < ref.work_mem_size + 5
        w64 = ref.mem_attn[..., 0] / cnt
        w64[young] = 1e8
        wdev = torch.cat((pre["attn"], torch.zeros(B, N, dtype=torch.float64, device="cuda")), 1) / cnt
        wdev[young] = 1e8
        gap = float((wdev - w64).abs().max())
        idx = gathered[-1]
        prunes.append((check_topk(w64, idx, ref.top_k, margin=2 * gap), gap))
        ie = idx[..., None]
        ref.mem_k = torch.gather(ref.mem_k, 1, ie.expand(-1, -1, C))
        ref.mem_v = torch.gather(ref.mem_v, 1, ie.expand(-1, -1, C))
        ref.mem_attn = torch.gather(ref.mem_attn, 1, ie)
        ref.mem_count = torch.gather(ref.mem_count, 1, ie)

    ref.memory_prune = prune64
    g = _gen(900 + N + long_frames)
    dup_at = frames // 2
    last_k = None
    worst_read, worst_attn = 0.0, 0.0
    for t in range(frames):
        fk = torch.randn(B, N, C, device="cuda", generator=g)
        fv = torch.randn(B, N, C, device="cuda", generator=g)
        if t == dup_at:
            fk[0] = last_k[0] + 0.1 * torch.randn(N, C, device="cuda", generator=g)
        if t > 0:
            q = make_queries(ref.mem_k.float(), N, sharpen, g)
            out = dev.memory_read(q)
            out64 = ref.memory_read(q.double())
            torch.cuda.synchronize()
            e = rel_l2(out.double() - q.double(), out64 - q.double())
            assert e < TOL_OUT[sharpen], (t, e)
            worst_read = max(worst_read, e)
        n_gather = len(gathered)
        skip64 = False
        if ref.mem_k is not None:
            corr = gate64(ref.mem_k[:, -ref.wm * N:], fk, N).max()     # after a prune to 3 N: the whole bank
            assert abs(float(corr) - 0.95) > 1e-5
            skip64 = bool(corr > 0.95)
            pre["attn"] = dev.bank.attn[:, :dev.bank.len].double().clone()
        dev.add_mem_check(fk, fv)
        ref.add_mem_check(fk.double(), fv.double())
        torch.cuda.synchronize()
        assert skips[-1] == skip64 == (t == dup_at), t
        if not skip64:
            last_k = fk
        n = dev.bank.len
        assert n == ref.mem_k.shape[1] and dev.wm == ref.wm and dev.lm == ref.lm, t
        assert torch.equal(dev.bank.count[:, :n].double(), ref.mem_count[..., 0]), t
        assert torch.equal(dev.bank.k_raw[:, :n].double(), ref.mem_k), t
        if long_frames == 0 and len(gathered) > n_gather:
            assert torch.equal(gathered[-1].cpu(), torch.arange(N, n + N)[None].expand(B, -1)), t
        if t > 0:
            e = rel_l2(dev.bank.attn[:, :n], ref.mem_attn[..., 0])
            assert e < TOL_ATTN[sharpen], (t, e)
            worst_attn = max(worst_attn, e)
    if long_frames:
        assert len(prunes) >= 2 and sum(sum(d) for d, _ in prunes) > 0, prunes
    else:
        assert len(gathered) == frames - 5 - 1          # one drop per frame past the working memory, minus the skip
    print(f"[measured] lockstep N={N} long={long_frames} sharpen={sharpen}: read {worst_read:.3e} attn {worst_attn:.3e} "
          f"prunes {[(d, f'{gp:.1e}') for d, gp in prunes]}")


# ------------------------------------------------------------------------------------------------
# 10. the softmax row buffer limit is an argument check
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_read_refuses_banks_past_the_row_buffer(models, sd64):
    """len = 768 * 67 = 51456 > 51200 is refused before anything is launched; a valid read right after matches fp64."""
    from spann3r_b200 import _lib
    from spann3r_b200.engine import MemoryBank
    N, B, sharpen = 768, 1, True
    eng = _engine(models, sharpen, B, N)
    big = MemoryBank(B, N * 67, "cuda")
    big.len = N * 67
    g = _gen(1100)
    q = torch.randn(B, N, C, device="cuda", generator=g)
    with pytest.raises(_lib.S3RError, match="51200"):
        eng.memory_read(big, q, THRESH)
    del big
    k = torch.randn(B, N * 2, C, device="cuda", generator=g)
    v = torch.randn(B, N * 2, C, device="cuda", generator=g)
    bank = _fill(eng, k, v)
    q = make_queries(k, N, sharpen, g)
    out = eng.memory_read(bank, q, THRESH)
    torch.cuda.synchronize()
    check_read(sd64[sharpen], k, v, q, THRESH, out, bank.attn[:, :bank.len], sharpen, "after refusal")


# ------------------------------------------------------------------------------------------------
# CPU checks of the helpers above
# ------------------------------------------------------------------------------------------------
def test_check_topk_accepts_any_split_of_ties_and_rejects_wrong_picks():
    w = torch.tensor([[5.0, 3.0, 3.0, 3.0, 1.0, 1e8, 0.5]], dtype=torch.float64)
    # k = 4: 1e8, 5 and two of the three tied 3s
    for pick in ([5, 0, 1, 2], [5, 0, 2, 3], [0, 3, 5, 1]):
        assert check_topk(w, torch.tensor([pick]), 4) == [4]      # 1e8, 5 above; 1, 0.5 below
    for bad in ([5, 1, 2, 3],            # drops 5, clearly above the k-th
                [5, 0, 1, 4],            # keeps 1, clearly below
                [5, 0, 1, 1],            # not distinct
                [5, 0, 1]):              # wrong count
        with pytest.raises(AssertionError):
            check_topk(w, torch.tensor([bad]), 4)
    # within the margin either side is accepted
    w2 = torch.tensor([[4.0, 2.0, 2.0 + 1e-9, 1.0]], dtype=torch.float64)
    check_topk(w2, torch.tensor([[0, 1]]), 2, margin=1e-8)
    with pytest.raises(AssertionError):
        check_topk(w2, torch.tensor([[0, 1]]), 2, margin=0.0, rel=0.0)
    # every weight tied (the young tokens of a fresh bank): nothing is decided, any k distinct indices pass
    assert check_topk(torch.full((2, 6), 1e8, dtype=torch.float64), torch.tensor([[0, 1, 2], [5, 3, 1]]), 3) == [0, 0]


def test_flip_slack_bounds_every_choice_of_the_ambiguous_entries():
    """Brute force over every keep / cut choice of the entries near the threshold: the renormalised row never moves
    by more than the slack in L1."""
    import itertools
    g = torch.Generator().manual_seed(0)
    t = 0.05
    for _ in range(50):
        w = torch.rand(12, generator=g, dtype=torch.float64) * 0.1
        w[:3] = t * (1 + (torch.rand(3, generator=g, dtype=torch.float64) - 0.5) * 1.8e-3)
        w[3] = 0.15                                   # one entry clearly kept: the fp64 row is not empty
        flip, slack = flip_slack(w[None], t, rel=1e-3)
        assert flip[0] and torch.isfinite(slack[0])
        amb = ((w - t).abs() <= 1e-3 * t).nonzero().flatten().tolist()
        ref = torch.where(w < t, torch.zeros_like(w), w)
        ref = ref / ref.sum()
        for choice in itertools.product((False, True), repeat=len(amb)):
            keep = w >= t
            for i, c in zip(amb, choice):
                keep[i] = c
            row = torch.where(keep, w, torch.zeros_like(w))
            row = row / row.sum()
            assert float((row - ref).abs().sum()) <= float(slack[0]) * (1 + 1e-12)


def test_make_queries_shapes_and_peaks():
    """The query builder on the CPU: shape, rows 0-2 lean on the last, second-last and third-last token, every row has a
    peak of the intended strength, flat rows have none."""
    g = torch.Generator().manual_seed(3)
    k = torch.randn(2, 90, C, generator=g)
    kh = (k - k.mean(-1, keepdim=True)) / k.std(-1, keepdim=True, unbiased=False)
    for sharpen in (False, True):
        q = make_queries(k, 45, sharpen, g)
        assert q.shape == (2, 45, C) and q.is_contiguous()
        corr = torch.einsum("bnc,bmc->bnm", q, kh) / C
        top = corr[:, :3].topk(3, dim=-1).indices
        assert all(89 - r in top[b, r].tolist() for b in range(2) for r in range(3))
        lo = 48.0 / 256 if sharpen else 14.0 / 32          # the strongest key's share: logit lo.. over 32 w
        assert (corr.amax(-1) > 0.8 * lo).all()
    q = make_queries(k, 45, False, g, flat_rows=True)
    corr = torch.einsum("bnc,bmc->bnm", q, kh) / C
    assert corr[:, 1::2].abs().max() < 0.2               # flat rows: pure noise
    assert (corr[:, ::2].amax(-1) > 0.35).all()
