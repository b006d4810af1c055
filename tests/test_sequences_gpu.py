"""Independent sequences in one batch: the per-slot memory stages (s3r_engine_*_slots) against the fp64 oracle run on each
slot alone, and Spann3R.forward_sequences against Spann3R.forward at batch 1, sequence by sequence.

Bars: the op-level ones are those of tests/test_memory_gpu.py (measured on one H100 80GB HBM3, SXM, 700 W power limit);
end to end, 2e-4 rel-L2 is the lockstep bound of tests/test_model_gpu.py (different batch sizes pick different tile
shapes, same arithmetic) and 1e-3 the north star where a prune or the bf16 precision amplifies those differences.  On
that card every end-to-end case measured 0.0: the batched run gave the batch-1 bits.
"""
import functools

import pytest
import torch

from conftest import get_state_dict, rel_l2
from test_memory_gpu import (C, THRESH, TOL_ATTN, TOL_GATE, TOL_OUT, check_read, check_topk, gate64, make_queries)

pytestmark = pytest.mark.gpu

N, HW = 196, (224, 224)


@pytest.fixture(scope="module")
def model():
    from spann3r_b200 import Spann3R, _lib
    _lib.require_device()
    m = Spann3R(dus3r_name=None)
    m.load_state_dict(get_state_dict(True), strict=True)
    return m.cuda().eval()


@pytest.fixture(scope="module")
def sd64():
    return {k: v.cuda().double() for k, v in get_state_dict(True).items() if k.split(".")[0] in ("norm_q", "norm_k", "norm_v")}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------
# op level
# ------------------------------------------------------------------------------------------------
def _slot_bank(eng, frames, g, cap_frames=8):
    """Slots of frames[b] frames each (appended through the slot path, some slots disabled at each step)."""
    from spann3r_b200.engine import MemoryBank
    B = len(frames)
    bank = MemoryBank(B, cap_frames * N, "cuda")
    ks = torch.randn(B, max(frames) * N, C, device="cuda", generator=g)
    vs = torch.randn(B, max(frames) * N, C, device="cuda", generator=g)
    lens = [0] * B
    for t in range(max(frames)):
        on = [t < f for f in frames]
        eng.memory_append_slots(bank, lens, on, ks[:, t * N:(t + 1) * N].contiguous(), vs[:, t * N:(t + 1) * N].contiguous())
        lens = [n + N * o for n, o in zip(lens, on)]
    return bank, lens, ks, vs


def test_slot_read_append_gate_vs_fp64(model, sd64):
    """3 slots of 0, 2 and 5 frames.  Raw rows bitwise, reads / bank.attn per slot at the read bars, the empty slot's read
    is its query bit for bit and leaves its attn alone, gate values per slot at TOL_GATE with -inf past wm[b]; a
    near-duplicate frame fires slot 2's gate only."""
    eng = model._engine_for(3, *HW)
    g = _gen(1)
    frames = [0, 2, 5]
    bank, lens, ks, vs = _slot_bank(eng, frames, g)
    torch.cuda.synchronize()
    for b, f in enumerate(frames):
        assert torch.equal(bank.k_raw[b, :f * N], ks[b, :f * N]) and torch.equal(bank.v_raw[b, :f * N], vs[b, :f * N])
        assert torch.equal(bank.count[b, :f * N].cpu(),
                           torch.cat([torch.full((N,), float(f - 1 - t)) for t in range(f)]) if f else torch.zeros(0))
    q = torch.randn(3, N, C, device="cuda", generator=g)
    for b in (1, 2):
        q[b] = make_queries(ks[b:b + 1, :frames[b] * N], N, True, g)[0]
    a0 = bank.attn.clone()
    out = eng.memory_read_slots(bank, lens, q, THRESH)
    torch.cuda.synchronize()
    assert torch.equal(out[0], q[0]) and torch.equal(bank.attn[0], a0[0])
    for b in (1, 2):
        M = lens[b]
        check_read(sd64, ks[b:b + 1, :M], vs[b:b + 1, :M], q[b:b + 1], THRESH, out[b:b + 1],
                   bank.attn[b:b + 1, :M].double() - a0[b:b + 1, :M].double(), True, f"slot {b} M={M}")
        assert torch.equal(bank.attn[b, M:], a0[b, M:])
    # gate: slot 2 compares with a near-duplicate of its last frame
    fk = torch.randn(3, N, C, device="cuda", generator=g)
    fk[2] = ks[2, 4 * N:5 * N] + 0.1 * torch.randn(N, C, device="cuda", generator=g)
    wm = [0, 2, 3]
    got = eng.check_sim_slots(bank, lens, wm, fk.contiguous())
    torch.cuda.synchronize()
    assert torch.isinf(got[0]).all() and (got[0] < 0).all()
    for b in (1, 2):
        ref = gate64(ks[b:b + 1, lens[b] - wm[b] * N:lens[b]], fk[b:b + 1], N)[0]
        assert float((got[b, :wm[b]].double() - ref).abs().max()) < TOL_GATE, b
        assert torch.isinf(got[b, wm[b]:]).all()
    fired = (got.amax(1) > 0.95).tolist()
    assert fired == [False, False, True], got.amax(1)


def test_slot_tail_garbage_changes_nothing(model):
    """Large finite values planted past every slot's length (K_n / V_n^T / raw rows, attn, count) change no output bit of
    the read, bank.attn below the lengths, or the gate."""
    eng = model._engine_for(3, *HW)
    g = _gen(2)
    bank, lens, ks, _ = _slot_bank(eng, [1, 4, 2], g)
    q = make_queries(ks[:, :N], N, True, g)
    fk = torch.randn(3, N, C, device="cuda", generator=g)
    wm = [1, 3, 2]

    def run():
        a = bank.attn.clone()
        o = eng.memory_read_slots(bank, lens, q, THRESH)
        s = eng.check_sim_slots(bank, lens, wm, fk)
        torch.cuda.synchronize()
        out = (o.clone(), [bank.attn[b, :n].clone() for b, n in enumerate(lens)], s.clone())
        bank.attn.copy_(a)
        return out

    clean = run()
    for b, n in enumerate(lens):
        for name in ("kn_hi", "kn_lo"):
            getattr(bank, name)[b, n:] = 3e37
        for name in ("vnt_hi", "vnt_lo"):
            getattr(bank, name)[b, :, n:] = -3e37
        for name in ("k_raw", "v_raw", "attn", "count"):
            getattr(bank, name)[b, n:] = 1e30
    dirty = run()
    assert torch.equal(clean[0], dirty[0]) and torch.equal(clean[2], dirty[2])
    assert all(torch.equal(a, b) for a, b in zip(clean[1], dirty[1]))


def test_uniform_slots_equal_the_single_length_entry_points(model):
    """Equal lengths through the _slots entry points == the existing entry points, bit for bit: append (every bank
    buffer), read (output and bank.attn) and the gate."""
    from spann3r_b200.engine import MemoryBank
    eng = model._engine_for(3, *HW)
    g = _gen(3)
    k = torch.randn(3, 4 * N, C, device="cuda", generator=g)
    v = torch.randn(3, 4 * N, C, device="cuda", generator=g)
    a, b = MemoryBank(3, 6 * N, "cuda"), MemoryBank(3, 6 * N, "cuda")
    for t in range(4):
        kt, vt = k[:, t * N:(t + 1) * N].contiguous(), v[:, t * N:(t + 1) * N].contiguous()
        eng.memory_append(a, kt, vt)
        eng.memory_append_slots(b, [t * N] * 3, [1] * 3, kt, vt)
        q = make_queries(k[:, :(t + 1) * N], N, True, g)
        o1 = eng.memory_read(a, q, THRESH)
        o2 = eng.memory_read_slots(b, [a.len] * 3, q, THRESH)
        wm = min(t + 1, 3)
        s1 = eng.check_sim(a, q, wm)
        s2 = eng.check_sim_slots(b, [a.len] * 3, [wm] * 3, q)
        torch.cuda.synchronize()
        assert torch.equal(o1, o2) and torch.equal(s1, s2[:, :wm]), t
    for name in ("kn_hi", "kn_lo", "vnt_hi", "vnt_lo", "k_raw", "v_raw", "attn", "count"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


def test_slot_memory_lockstep_with_fp64_oracle(model, sd64, monkeypatch):
    """model.SlotMemory over 3 slots that start at different steps (one stays empty for a while), long_mem_size 3 N so
    that every slot prunes, one near-duplicate frame in slot 1: after every step each slot's length, wm, lm, mem_count and
    raw keys equal its own oracle.SpatialMemory's, reads and bank.attn at the read bars, and every prune keeps a valid
    top-k of that slot's fp64 weights (check_topk, margin twice the largest device / fp64 weight gap)."""
    from oracle import spann3r_oracle as orc
    from spann3r_b200.engine import MemoryBank
    from spann3r_b200.model import SlotMemory
    B, L, steps = 3, 3 * N, 14
    first = [0, 1, 5]                                   # step at which each slot's sequence starts
    eng = model._engine_for(B, *HW)
    mem = SlotMemory(long_mem_size=L, work_mem_size=5, attn_thresh=THRESH, engine=eng)
    refs = [orc.SpatialMemory(sd64, long_mem_size=L, work_mem_size=5, attn_thresh=THRESH) for _ in range(B)]
    gathered = {}
    orig = MemoryBank.gather_slot
    monkeypatch.setattr(MemoryBank, "gather_slot", lambda self, b, idx, n: (gathered.__setitem__(b, idx.clone()),
                                                                            orig(self, b, idx, n))[1])
    pre, prunes = {}, []

    def make_prune(b):
        def prune64():
            r = refs[b]
            cnt = r.mem_count[..., 0]
            young = cnt < r.work_mem_size + 5
            w64 = r.mem_attn[..., 0] / cnt
            w64[young] = 1e8
            wdev = torch.cat((pre[b], torch.zeros(1, N, dtype=torch.float64, device="cuda")), 1) / cnt
            wdev[young] = 1e8
            idx = gathered[b][None]
            prunes.append(check_topk(w64, idx, r.top_k, margin=2 * float((wdev - w64).abs().max())))
            ie = idx[..., None]
            r.mem_k = torch.gather(r.mem_k, 1, ie.expand(-1, -1, C))
            r.mem_v = torch.gather(r.mem_v, 1, ie.expand(-1, -1, C))
            r.mem_attn, r.mem_count = torch.gather(r.mem_attn, 1, ie), torch.gather(r.mem_count, 1, ie)
        return prune64

    gate64_fired = []
    for b in range(B):
        refs[b].memory_prune = make_prune(b)
        refs[b].check_sim = lambda feat_k, thresh, f=refs[b].check_sim: gate64_fired.append(f(feat_k, thresh)) or gate64_fired[-1]
    g = _gen(4)
    last = None
    for t in range(steps):
        active = [t >= f for f in first]
        fk = torch.randn(B, N, C, device="cuda", generator=g)
        fv = torch.randn(B, N, C, device="cuda", generator=g)
        if t == 7:
            fk[1] = last[1] + 0.1 * torch.randn(N, C, device="cuda", generator=g)
        if max(mem.len) > 0:
            q = torch.randn(B, N, C, device="cuda", generator=g)
            for b in range(B):
                if refs[b].mem_k is not None:
                    q[b] = make_queries(refs[b].mem_k.float(), N, True, g)[0]
            out = mem.memory_read(q)
            for b in range(B):
                if refs[b].mem_k is None:
                    assert torch.equal(out[b], q[b])
                    continue
                o64 = refs[b].memory_read(q[b:b + 1].double())
                e = rel_l2(out[b:b + 1].double() - q[b:b + 1].double(), o64 - q[b:b + 1].double())
                assert e < TOL_OUT[True], (t, b, e)
        for b in range(B):
            if refs[b].mem_k is not None:
                pre[b] = mem.bank.attn[b:b + 1, :mem.len[b]].double().clone()
        skip = mem.add_mem_check(fk, fv, active, mem.check_sim_async(fk))
        for b in range(B):
            if active[b]:
                gate64_fired.clear()
                refs[b].add_mem_check(fk[b:b + 1].double(), fv[b:b + 1].double())
                skip64 = bool(gate64_fired and gate64_fired[0])
                assert skip[b] == skip64 == (t == 7 and b == 1), (t, b, skip)
        torch.cuda.synchronize()
        if not skip[1]:
            last = fk
        for b in range(B):
            r = refs[b]
            n = 0 if r.mem_k is None else r.mem_k.shape[1]
            assert (mem.len[b], mem.wm[b], mem.lm[b]) == (n, r.wm, r.lm), (t, b)
            if n:
                assert torch.equal(mem.bank.count[b, :n].double(), r.mem_count[0, :, 0]), (t, b)
                assert torch.equal(mem.bank.k_raw[b, :n].double(), r.mem_k[0]), (t, b)
                assert rel_l2(mem.bank.attn[b, :n], r.mem_attn[0, :, 0]) < TOL_ATTN[True], (t, b)
            assert not mem.bank.k_raw[b, n:].any() and not mem.bank.vnt_hi[b, :, n:].any()
    assert len(prunes) >= 3, prunes
    print(f"[measured] slot lockstep: prunes {prunes}")


# ------------------------------------------------------------------------------------------------
# end to end: forward_sequences vs forward at batch 1
# ------------------------------------------------------------------------------------------------
def _spy(monkeypatch):
    """Records the B = 1 runs' gate decisions / values and each slot's decisions and final state per sequence."""
    from spann3r_b200 import model as M
    rec = {"b1": [], "b1_vals": [], "slots": {}, "final": {}}
    f1 = M.SpatialMemory.check_sim_finish

    def b1(self, pending, thresh=0.7):
        d = f1(self, pending, thresh)
        rec["b1"].append(d)
        rec["b1_vals"].append(float(self._sim_host[0]) if pending is not None else None)
        return d

    fs = M.SlotMemory.check_sim_finish

    def slots(self, pending):
        d = fs(self, pending)
        for b, tag in enumerate(self.tags):
            if tag is not None:
                rec["slots"].setdefault(tag, []).append(d[b])
        return d

    ff = M.SlotMemory.finish

    def finish(self, b):
        if self.tags[b] is not None:
            n = self.len[b]
            rec["final"][self.tags[b]] = dict(len=n, wm=self.wm[b], lm=self.lm[b], count=self.bank.count[b, :n].clone(),
                                              k=self.bank.k_raw[b, :n].clone())
        return ff(self, b)

    monkeypatch.setattr(M.SpatialMemory, "check_sim_finish", b1)
    monkeypatch.setattr(M.SlotMemory, "check_sim_finish", slots)
    monkeypatch.setattr(M.SlotMemory, "finish", finish)
    return rec


def _worst(p_seq, p_single):
    preds, preds_all = p_seq
    rp, rpa = p_single
    assert len(preds) == len(rp) and len(preds_all) == len(rpa)
    worst = 0.0
    for a, b in zip(preds, rp):
        assert list(a) == list(b)
        for k in b:
            assert a[k].shape == b[k].shape, k
            worst = max(worst, rel_l2(a[k], b[k]))
    for (a1, a2), (b1, b2) in zip(preds_all, rpa):
        for k in b2:
            worst = max(worst, rel_l2(a2[k], b2[k]))
    return worst


def _compare(m, seqs, rec, tol, counts_equal=True, max_batch=2, thresh=None):
    """forward_sequences(seqs) against forward(seq) per sequence: outputs within tol, decisions and counters equal."""
    from spann3r_b200 import model as M
    out = m.forward_sequences(seqs, max_batch=max_batch)
    out = [([{k: v.clone() for k, v in p.items()} for p in ps], [tuple({k: v.clone() for k, v in r.items()} for r in pr)
                                                                 for pr in pa]) for ps, pa in out]
    worst = 0.0
    for s, seq in enumerate(seqs):
        rec["b1"].clear()
        preds, preds_all, sp = m.forward(seq, return_memory=True)
        w = _worst(out[s], (preds, preds_all))
        worst = max(worst, w)
        assert w < tol, (s, w)
        assert rec["slots"][s] == rec["b1"], (s, rec["slots"][s], rec["b1"])
        f = rec["final"][s]
        assert (f["len"], f["wm"], f["lm"]) == (sp.bank.len, sp.wm, sp.lm), s
        n = sp.bank.len
        cdiff = int((f["count"] != sp.bank.count[0, :n]).sum())
        kept = rel_l2(f["k"], sp.bank.k_raw[0, :n])
        print(f"[measured] sequence {s} ({len(seq)} frames): worst rel-L2 {w:.2e}, mem_count entries differing {cdiff}, "
              f"kept raw keys rel-L2 {kept:.2e}")
        if counts_equal:
            assert cdiff == 0, s
    rec["slots"].clear()
    rec["final"].clear()
    return worst


def _with_repeat(n, k, seed0):
    from spann3r_b200 import synth
    fr = synth.make_frames(n, *HW, seed0=seed0)
    fr[k + 1] = {"img": fr[k]["img"].clone()}
    return fr


def test_forward_sequences_matches_single_runs(model, monkeypatch):
    """Lengths [2, 5, 3, 7, 4] at 224 x 224 with max_batch 2 and 3 (refills, a ragged tail); sequence 3 repeats a frame.
    The B = 1 run must skip a write at the repeat; if the synthetic checkpoint's gate stays under 0.95 there, both runs use
    one lower sim_thresh between the repeat's value and every other value of that run."""
    from spann3r_b200 import model as M
    from spann3r_b200 import synth
    rec = _spy(monkeypatch)
    lengths = [2, 5, 3, 7, 4]
    seqs = [synth.make_frames(n, *HW, seed0=100 * s + 1) for s, n in enumerate(lengths)]
    seqs[3] = _with_repeat(7, 3, 301)
    model.forward(seqs[3])
    vals = rec["b1_vals"]
    dup = vals[4]                                # step 4 compares frame 4 (= frame 3) with the bank
    others = [v for i, v in enumerate(vals) if v is not None and i != 4]
    print(f"[measured] gate at the repeated frame {dup:.4f}, other steps max {max(others):.4f}")
    assert dup > max(others)
    if not dup > 0.95:
        thresh = (dup + max(others)) / 2
        monkeypatch.setattr(M, "SpatialMemory", functools.partial(M.SpatialMemory, sim_thresh=thresh))
        monkeypatch.setattr(M, "SlotMemory", functools.partial(M.SlotMemory, sim_thresh=thresh))
    rec["b1"].clear()
    model.forward(seqs[3])
    assert rec["b1"][4] and sum(rec["b1"]) == 1, rec["b1"]
    for mb in (2, 3):
        w = _compare(model, seqs, rec, 2e-4, max_batch=mb)
        print(f"[measured] forward_sequences max_batch={mb}: worst rel-L2 {w:.2e}")


def test_long_sequence_prunes_like_batch_one(model, monkeypatch):
    """A 40-frame sequence beside short ones: it prunes at writes 26, 32 and 38 (long_mem_size 4000 at 196 tokens), as at
    B = 1; outputs within 1e-3 and counters equal; the kept-set difference is printed (prune ties may break apart)."""
    from spann3r_b200 import synth
    rec = _spy(monkeypatch)
    seqs = [synth.make_frames(40, *HW, seed0=1001)] + [synth.make_frames(n, *HW, seed0=2000 + 100 * n) for n in (3, 6, 4)]
    _compare(model, seqs, rec, 1e-3, counts_equal=False, max_batch=2)


@pytest.mark.parametrize("variant", ["portrait_mempos", "bf16"])
def test_variants_match_single_runs(monkeypatch, variant):
    """Portrait 288 x 224 frames with mem_pos_enc=True (mixed with a landscape sequence: two groups), and precision
    "bf16": within 1e-3 of forward at B = 1, counters equal."""
    from spann3r_b200 import Spann3R, synth
    m = Spann3R(dus3r_name=None, mem_pos_enc=variant == "portrait_mempos",
                precision="bf16" if variant == "bf16" else "fp32")
    m.load_state_dict(get_state_dict(True), strict=True)
    m = m.cuda().eval()
    rec = _spy(monkeypatch)
    if variant == "portrait_mempos":
        seqs = [synth.make_frames(n, 288, 224, seed0=10 * n) for n in (3, 5, 2)] + [synth.make_frames(3, *HW, seed0=7)]
    else:
        seqs = [synth.make_frames(n, *HW, seed0=10 * n) for n in (3, 5, 2, 4)]
    _compare(m, seqs, rec, 1e-3, max_batch=2)
    if variant == "portrait_mempos":
        assert {k[1:3] for k in m._engines} == {(288, 224), (224, 224)}
