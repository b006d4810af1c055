"""Host logic of the batched independent-sequence mode, without a GPU: the per-slot memory bookkeeping (model.SlotMemory)
against the counters of the reference's add_mem_check, the slot scheduler of Spann3R.forward_sequences on a stub
engine, and the C ABI of the per-slot memory stages."""
import ctypes
import os

import pytest
import torch

from conftest import ROOT

C = 1024


class _SlotEngine:
    """CPU stand-in for engine.Engine's per-slot memory stages: data movement only, as the kernels do it."""

    def __init__(self, B, N):
        self.B, self.N, self.device = B, N, torch.device("cpu")

    def memory_append_slots(self, bank, lens, append, k, v):
        for b in range(self.B):
            if append[b]:
                n = lens[b]
                bank.k_raw[b, n:n + self.N] = k[b]
                bank.v_raw[b, n:n + self.N] = v[b]
                bank.count[b, :n] += 1
                bank.count[b, n:n + self.N] = 0
                bank.attn[b, n:n + self.N] = 0

    def memory_read_slots(self, bank, lens, feat, thresh):
        return feat


@pytest.mark.parametrize("long_frames", [0, 3])
def test_slot_counters_match_the_reference_add_mem_check(monkeypatch, long_frames):
    """Three slots with scripted gate decisions, each against oracle.SpatialMemory (the reference's add_mem_check) run on
    that slot's frames alone with the same decisions: wm, lm, length, mem_count (as a multiset: prune ties may order
    differently) and the kept raw keys, after every step.  long_mem_size 0 drops the oldest working frame; 3 N prunes."""
    from oracle import spann3r_oracle as orc
    from spann3r_b200 import model as M
    B, N, steps = 3, 2, 16
    L = long_frames * N
    eng = _SlotEngine(B, N)
    mem = M.SlotMemory(long_mem_size=L, work_mem_size=5, engine=eng)
    g = torch.Generator().manual_seed(0)
    script = torch.rand(steps, B, generator=g) < 0.25         # True: the gate fires in that slot at that step
    refs = [orc.SpatialMemory(None, long_mem_size=L, work_mem_size=5) for _ in range(B)]
    for b, r in enumerate(refs):
        r.check_sim = lambda feat_k, thresh, b=b: r_script[b]
    r_script = [False] * B
    pruned = []
    orig_prune = mem.memory_prune
    monkeypatch.setattr(mem, "memory_prune", lambda b: (pruned.append(b), orig_prune(b)))
    for t in range(steps):
        fk = torch.randn(B, N, C, generator=g)
        fv = torch.randn(B, N, C, generator=g)
        # an empty bank never skips (the reference checks nothing then)
        decisions = [bool(script[t, b]) and refs[b].mem_k is not None for b in range(B)]
        r_script[:] = decisions
        monkeypatch.setattr(mem, "check_sim_finish", lambda pending: list(decisions))
        skip = mem.add_mem_check(fk, fv, [True] * B, None)
        assert skip == decisions
        for b in range(B):
            refs[b].add_mem_check(fk[b:b + 1], fv[b:b + 1])
            n = refs[b].mem_k.shape[1]
            assert (mem.len[b], mem.wm[b], mem.lm[b]) == (n, refs[b].wm, refs[b].lm), (t, b)
            cnt = mem.bank.count[b, :n]
            assert torch.equal(cnt.sort().values, refs[b].mem_count[0, :, 0].sort().values), (t, b)
            if long_frames == 0 or not pruned:
                assert torch.equal(mem.bank.k_raw[b, :n], refs[b].mem_k[0]), (t, b)
            # the tail a drop or prune leaves behind is zero (the per-slot read's tail contract)
            assert not mem.bank.k_raw[b, n:].any() and not mem.bank.kn_hi[b, n:].any() and not mem.bank.vnt_hi[b, :, n:].any()
    if long_frames:
        assert pruned, "the script is meant to reach a prune"


def test_slot_start_and_finish_reset_only_that_slot():
    from spann3r_b200 import model as M
    B, N = 2, 2
    mem = M.SlotMemory(long_mem_size=8, engine=_SlotEngine(B, N))
    for _ in range(3):
        mem.add_mem_check(torch.ones(B, N, C), torch.ones(B, N, C), [True, True], None)
    assert mem.len == [6, 6] and mem.wm == [3, 3]
    mem.start(1, tag="next")
    assert mem.len == [6, 0] and mem.wm == [3, 0] and mem.lm == [0, 0] and mem.tags == [None, "next"]
    assert not mem.bank.k_raw[1].any() and mem.bank.k_raw[0, :6].all()


# ------------------------------------------------------------------------------------------------
# the scheduler on a stub engine
# ------------------------------------------------------------------------------------------------
class _StubEngine:
    """Engine stand-in whose outputs identify their inputs: a frame's features carry its code (the image's first pixel)
    and head 2's pointmap of a slot carries the code of the frame decoded as view 2 in that slot."""

    def __init__(self, B, H, W, max_images):
        self.B, self.H, self.W, self.N = B, H, W, (H // 16) * (W // 16)
        self.max_images, self.device = max_images, torch.device("cpu")
        self.calls = []

    def encode(self, img):
        self.calls.append(("encode", img.shape[0]))
        return img[:, 0, 0, 0].view(-1, 1, 1).expand(-1, self.N, 1024).contiguous()

    def decode(self, f1, f2):
        self._f2 = f2[:, 0, 0].clone()

    def keyheads(self, f1, f2):
        return f1.clone(), f2.clone()

    def heads(self):
        pts = self._f2.view(1, self.B, 1, 1, 1).expand(2, self.B, self.H, self.W, 3).contiguous()
        return pts, torch.ones(2, self.B, self.H, self.W)

    def value(self, pts3d, feat_k1, transposed=False, rope=False):
        return feat_k1 * 0

    def memory_read_slots(self, bank, lens, feat, thresh):
        self.calls.append(("read", list(lens)))
        return feat

    def memory_append_slots(self, bank, lens, append, k, v):
        self.calls.append(("append", list(append)))


def _stub_model(monkeypatch):
    from spann3r_b200 import Spann3R
    from spann3r_b200 import model as M
    m = Spann3R(dus3r_name=None).eval()
    engines = {}

    def engine_for(B, H, W, n_frames=2, encode_only=False):
        return engines.setdefault((B, H, W), _StubEngine(B, H, W, max(2 * B, min(n_frames * B, 16 * B))))

    monkeypatch.setattr(m, "_engine_for", engine_for)
    monkeypatch.setattr(M.SlotMemory, "check_sim_async", lambda self, feat_k: None)
    starts = []
    orig = M.SlotMemory.start
    monkeypatch.setattr(M.SlotMemory, "start", lambda self, b, tag=None: (starts.append((b, tag)), orig(self, b, tag))[1])
    return m, engines, starts


def _coded_sequences(lengths, H=32, W=48):
    """Frame f of sequence s has every pixel equal to 100 s + f."""
    return [[{"img": torch.full((1, 3, H, W), 100.0 * s + f)} for f in range(n)] for s, n in enumerate(lengths)]


@pytest.mark.parametrize("max_batch,starts_expected", [
    (2, [(0, 0), (1, 1), (0, 2), (0, 3), (1, 4)]),
    (3, [(0, 0), (1, 1), (2, 2), (0, 3), (2, 4)]),
])
def test_scheduler_assigns_and_refills_slots_in_order(monkeypatch, max_batch, starts_expected):
    lengths = [2, 5, 3, 7, 4]
    m, engines, starts = _stub_model(monkeypatch)
    seqs = _coded_sequences(lengths)
    out = m.forward_sequences(seqs, max_batch=max_batch)
    assert starts == starts_expected
    eng = engines[(max_batch, 32, 48)]
    assert len(out) == len(seqs)
    for s, (preds, preds_all) in enumerate(out):
        n = lengths[s]
        assert len(preds) == n and len(preds_all) == n - 1
        assert set(preds[0]) == {"pts3d", "conf"} and all(set(p) == {"pts3d_in_other_view", "conf"} for p in preds[1:])
        assert preds_all[0][0] is preds[0] and preds_all[-1][1] is preds[-1]
        for i in range(1, n):       # head 2 of step i - 1 saw frame i of this very sequence
            v = preds[i]["pts3d_in_other_view"] if i == n - 1 else preds_all[i - 1][1]["pts3d_in_other_view"]
            assert v.shape == (1, 32, 48, 3) and bool((v == 100.0 * s + i).all()), (s, i)
    # idle slots never write; every slot starts its sequence with an empty bank
    steps = sum(n - 1 for n in lengths)
    appends = [c[1] for c in eng.calls if c[0] == "append"]
    assert sum(sum(a) for a in appends) == steps
    # frames are encoded in batched calls within max_images
    enc = [c[1] for c in eng.calls if c[0] == "encode"]
    assert sum(enc) == sum(lengths) and max(enc) <= eng.max_images and len(enc) < len(seqs) + 1


def test_scheduler_groups_resolutions_and_rejects_bad_input(monkeypatch):
    m, engines, starts = _stub_model(monkeypatch)
    a = _coded_sequences([3, 2])
    b = _coded_sequences([4], H=48, W=32)
    out = m.forward_sequences([a[0], b[0], a[1]], max_batch=4)
    assert set(engines) == {(2, 32, 48), (1, 48, 32)}
    assert [len(p) for p, _ in out] == [3, 4, 2]
    assert out[1][0][0]["pts3d"].shape == (1, 32, 48, 3)          # portrait outputs are landscape views
    with pytest.raises(ValueError):
        m.forward_sequences([a[0], a[0][:1]])
    with pytest.raises(ValueError):
        m.forward_sequences([a[0]], max_batch=0)
    m.train()
    with pytest.raises(NotImplementedError):
        m.forward_sequences([a[0]])


def test_run_sharded_independent_passes_the_ranks_sequences():
    from spann3r_b200 import shard
    seqs = [[{"img": torch.zeros(1, 3, 16, 16)}] * n for n in (2, 3, 4, 5, 6)]
    calls = []

    def fwd(my, max_batch):
        calls.append(([len(q) for q in my], max_batch))
        return [([len(q)], None) for q in my]

    out = shard.run_sharded(fwd, seqs, per_gpu_batch=3, rank=1, world_size=2, independent=True)
    assert calls == [([3, 5], 3)] and out == {1: [3], 3: [5]}


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
SLOT_SYMBOLS = {"s3r_engine_memory_read_slots": 7, "s3r_engine_memory_append_slots": 7, "s3r_engine_check_sim_slots": 7}


def test_slot_symbols_are_exported_and_bound_with_their_declared_arity():
    from spann3r_b200 import _lib, engine
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    L = ctypes.CDLL(_lib.LIB_PATH)
    header = open(os.path.join(ROOT, "include", "spann3r_b200.h")).read()
    assert "#define S3R_MAX_SLOTS 64" in header and engine.MAX_SLOTS == 64
    for name, arity in SLOT_SYMBOLS.items():
        assert hasattr(L, name), name
        assert name + "(" in header, name
        assert len(_lib._PROTOS[name][1]) == arity, name
