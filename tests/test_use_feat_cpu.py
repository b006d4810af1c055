"""CPU tests of `Spann3R(use_feat=True)`: the 768-wide value encoder fed with decoder tokens (16 heads of 48).

* the derived key inventory equals the real reference's (tests/golden/state_dict_spec_usefeat.json);
* the module tree round-trips a strict load_state_dict;
* the use_feat oracle (oracle/usefeat_oracle.py) matches the real reference's outputs (tools/make_golden.py --only usefeat);
* the zero-padded 64-wide head slots the library runs (engine.head_slots / pad_qkv_rows / pad_proj_cols and the 16-pair
  RoPE table) restate the oracle's 48-wide attention exactly, in fp64, before any GPU run;
* the training recompute of the use_feat value stage equals the oracle, and the stage partition covers every key once.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_l2
from oracle import spann3r_oracle as orc
from oracle import usefeat_oracle as ufo
from spann3r_b200 import _recompute as R
from spann3r_b200 import engine as E
from spann3r_b200 import synth, train

TOL = 2e-5          # test_oracle_vs_golden.py: fp32 reassociation noise between two eager PyTorch programs

_SD = {}


def usefeat_state_dict():
    if "sd" not in _SD:
        _SD["sd"] = synth.make_state_dict(synth.usefeat_spec(), seed=0, sharpen=True)
    return _SD["sd"]


def _sub_tokens(t):
    return t[:, ::7, ::8]


def test_derived_spec_equals_the_reference_inventory():
    with open(os.path.join(GOLDEN, "state_dict_spec_usefeat.json")) as f:
        ref = json.load(f)
    got = synth.usefeat_spec()["spann3r"]
    assert list(got.items()) == list(ref.items())
    assert len(got) == 1099
    assert not any(k.startswith("pos_patch_embed.") for k in got)
    assert got["value_encoder.0.attn.qkv.weight"] == [2304, 768] and got["value_out.weight"] == [1024, 768]


def test_module_tree_round_trips_a_strict_load():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, use_feat=True)
    sd = usefeat_state_dict()
    assert list(m.state_dict().keys()) == list(sd.keys())
    m.load_state_dict(sd, strict=True)
    back = m.state_dict()
    assert all(torch.equal(back[k], v) for k, v in sd.items())
    with pytest.raises(RuntimeError):          # the default model's keys do not load strictly into a use_feat model
        m.load_state_dict(synth.make_state_dict(seed=0), strict=True)
    m._init_like_reference()                   # the reference constructors' init of the non-DUSt3R keys
    assert torch.equal(m.value_norm.weight.data, torch.ones(768))
    assert float(dict(m.named_parameters())["value_encoder.0.attn.qkv.weight"].detach().abs().max()) <= 768 ** -0.5 + 1e-7


@pytest.mark.parametrize("fname,nf,H,W,mem_pos_enc", [
    ("seq_224_3f_sharp_usefeat.npz", 3, 224, 224, False),
    ("seq_288x224_3f_sharp_usefeat_mempos.npz", 3, 288, 224, True),
])
def test_oracle_matches_reference_golden(fname, nf, H, W, mem_pos_enc):
    g = np.load(os.path.join(GOLDEN, fname))
    sd = usefeat_state_dict()
    trace = []
    preds, preds_all, mem = ufo.forward(sd, synth.make_frames(nf, H, W), return_memory=True, trace=trace,
                                        mem_pos_enc=mem_pos_enc)
    s = int(g["meta/px_stride"])
    for i, p in enumerate(preds):
        assert set(p.keys()) == {k.split("/")[-1] for k in g.files if k.startswith(f"preds/{i}/")}
        for k, v in p.items():
            assert v.shape[1:3] == (min(H, W), max(H, W))
            assert rel_l2(v[:, ::s, ::s], g[f"preds/{i}/{k}"]) < TOL, (i, k)
    for i, (_, r2) in enumerate(preds_all):
        for k, v in r2.items():
            assert rel_l2(v[:, ::s, ::s], g[f"preds_all/{i}/res2/{k}"]) < TOL, (i, k)
    assert rel_l2(_sub_tokens(mem.mem_k), g["mem/mem_k_sub"]) < TOL
    assert rel_l2(_sub_tokens(mem.mem_v), g["mem/mem_v_sub"]) < TOL
    assert rel_l2(mem.mem_attn, g["mem/mem_attn"]) < 1e-4
    assert np.array_equal(mem.mem_count.numpy(), g["mem/mem_count"])
    if "act/value_out#0" in g.files:
        assert rel_l2(_sub_tokens(trace[0]["cur_v"]), g["act/value_out#0"]) < TOL


def test_offline_oracle_matches_reference_golden():
    from test_oracle_vs_golden import _pair_graph
    g = np.load(os.path.join(GOLDEN, "offline_224_4f_sharp_usefeat.npz"))
    sd = usefeat_state_dict()
    frames = synth.make_frames(4, 224, 224)
    graph = _pair_graph(lambda a, b: orc.dust3r_forward(sd, a, b), frames)
    preds, _, idx_used = ufo.offline_reconstruction(sd, frames, graph)
    assert list(idx_used) == list(g["idx_used"])
    s = int(g["meta/px_stride"])
    for i, p in enumerate(preds):
        for k, v in p.items():
            assert rel_l2(v[:, ::s, ::s], g[f"preds/{i}/{k}"]) < TOL, (i, k)


def _padded_attention(x, wq, bq, wp, bp, pos, cs, rope):
    """The library's arithmetic on the packed operands, in fp64: qkv into 64-wide slots, the epilogue's RoPE (pairs
    (j, j + 16) of each 32-wide half over the [maxpos, 16, 2] table), q * 48^-0.5, softmax(q k^T) v, proj over the slots."""
    B, N, _ = x.shape
    qkv = (x @ wq.t() + bq).view(B, N, 3, 16, 64).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    pad = torch.ones(64, dtype=torch.bool)
    pad[torch.cat([torch.arange(12), 16 + torch.arange(12), 32 + torch.arange(12), 48 + torch.arange(12)])] = False
    for t in (q, k, v):
        assert torch.count_nonzero(t[..., pad]) == 0          # padding columns are exactly zero

    def rot(t):
        out = t.clone()
        for s in range(2):
            c = cs[pos[..., s], :, 0][:, None]
            sn = cs[pos[..., s], :, 1][:, None]
            u, w = t[..., 32 * s: 32 * s + 16], t[..., 32 * s + 16: 32 * s + 32]
            out[..., 32 * s: 32 * s + 16] = u * c - w * sn
            out[..., 32 * s + 16: 32 * s + 32] = w * c + u * sn
        return out
    if rope:
        q, k = rot(q), rot(k)
        assert torch.count_nonzero(q[..., pad]) == 0 and torch.count_nonzero(k[..., pad]) == 0
    q = q * 48 ** -0.5
    o = torch.softmax(q @ k.transpose(-2, -1), dim=-1) @ v
    assert torch.count_nonzero(o[..., pad]) == 0
    return o.transpose(1, 2).reshape(B, N, 1024) @ wp.t() + bp


@pytest.mark.parametrize("gh,gw", [(14, 14), (6, 11)])
def test_padded_head_slots_restate_48_wide_attention(gh, gw):
    g = torch.Generator().manual_seed(7)
    C, B, N = 768, 2, gh * gw
    d = torch.float64
    sd = {"a.qkv.weight": torch.randn(3 * C, C, generator=g, dtype=d) * C ** -0.5,
          "a.qkv.bias": torch.randn(3 * C, generator=g, dtype=d) * 0.1,
          "a.proj.weight": torch.randn(C, C, generator=g, dtype=d) * C ** -0.5,
          "a.proj.bias": torch.randn(C, generator=g, dtype=d) * 0.1}
    x = torch.randn(B, N, C, generator=g, dtype=d)
    pos = torch.cartesian_prod(torch.arange(gh), torch.arange(gw)).view(1, N, 2).expand(B, -1, -1).clone()
    slots = E.head_slots(16, 48)
    assert slots.unique().numel() == C and int(slots.max()) < 1024
    wq, bq = E.pad_qkv_rows(sd["a.qkv.weight"], slots), E.pad_qkv_rows(sd["a.qkv.bias"], slots)
    wp = E.pad_proj_cols(sd["a.proj.weight"], slots)
    assert wq.shape == (3072, C) and bq.shape == (3072,) and wp.shape == (C, 1024)
    cs = E.rope_cs_table(head_dim=48).double()
    assert cs.shape == (E.ROPE_MAXPOS, 16, 2)
    assert torch.equal(cs[:, 12:, 0], torch.ones(E.ROPE_MAXPOS, 4, dtype=d)) and torch.count_nonzero(cs[:, 12:, 1]) == 0
    assert torch.equal(E.rope_cs_table(), E.rope_cs_table(head_dim=64))
    for rope in (False, True):
        ref = orc.attention(sd, "a", x, pos, 16, use_rope=rope)
        got = _padded_attention(x, wq, bq, wp, sd["a.proj.bias"], pos, cs, rope)
        assert rel_l2(got, ref) < 1e-12, (rope, rel_l2(got, ref))


def test_padded_rows_stay_zero_through_the_layernorm_fold():
    """norm1 is folded into the padded qkv: the padding rows keep zero weight, bias and column sum (cs), so the epilogue's
    rstd * (acc - mean * cs) + bias is exactly 0 there."""
    g = torch.Generator().manual_seed(2)
    w, b = torch.randn(2304, 768, generator=g), torch.randn(2304, generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(768, generator=g), 0.1 * torch.randn(768, generator=g)
    slots = E.head_slots(16, 48)
    wf, bf = E.fold_layernorm(w, b, gamma, beta)
    wpad, bpad = E.pad_qkv_rows(wf, slots), E.pad_qkv_rows(bf, slots)
    cs = E.split_bf16_host_rowsum(wpad)
    live = torch.zeros(3072, dtype=torch.bool)
    live[torch.cat([r * 1024 + slots for r in range(3)])] = True
    assert torch.count_nonzero(wpad[~live]) == 0 and torch.count_nonzero(bpad[~live]) == 0
    assert torch.count_nonzero(cs[~live]) == 0
    assert torch.equal(wpad[live], wf) and torch.equal(cs[live], E.split_bf16_host_rowsum(wf))


@pytest.mark.parametrize("H,W", [(224, 224), (64, 96)])
def test_recompute_value_stage_equals_the_oracle(H, W):
    sd = usefeat_state_dict()
    g = torch.Generator().manual_seed(4)
    N = (H // 16) * (W // 16)
    dec = torch.randn(1, N, 768, generator=g)
    k1 = torch.randn(1, N, 1024, generator=g)
    pos = torch.cartesian_prod(torch.arange(H // 16), torch.arange(W // 16)).view(1, N, 2)
    with torch.no_grad():
        for rope in (False, True):
            got = R.value_tokens(sd, dec, k1, rope, H, W)
            ref = ufo.encode_cur_value(sd, dec, pos, mem_pos_enc=rope) + k1
            assert rel_l2(got, ref) < 1e-5, (rope, rel_l2(got, ref))


def test_recompute_step_returns_the_decoder_tokens():
    sd = usefeat_state_dict()
    H, W = 64, 96
    fr = synth.make_frames(2, H, W)
    with torch.no_grad():
        ref, pos = orc.encode_image(sd, torch.cat([f["img"] for f in fr]))
        f1, f2 = ref[:1], ref[1:]
        outs = R.step(sd, f1, f1, f2, H, W, dec_tokens=True)
        d1, _ = orc.decoder(sd, f1, pos[:1], f2, pos[1:])
    assert len(outs) == 5 and rel_l2(outs[4], d1[-1]) < 1e-5


def test_stage_partition_covers_every_usefeat_key_once():
    from spann3r_b200 import Spann3R
    m = Spann3R(dus3r_name=None, use_feat=True)
    seen = {}
    for stage in ("encode", "memread", "step", "value"):
        names, params = train.stage_params(m, stage)
        assert len(names) == len(set(names)) and len(names) == len(params)
        for n in names:
            assert n not in seen, (n, stage, seen.get(n))
            seen[n] = stage
    every = [n for n, _ in m.named_parameters(remove_duplicate=False)]
    assert sorted(set(every) - set(seen)) == ["dust3r.mask_token"]
    assert sum(1 for n in seen if seen[n] == "value") == 6 * 12 + 4
