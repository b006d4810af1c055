"""The fp64 training-mode reference of tests/test_train_fp64_gpu.py, pinned on the CPU.

That module holds a training step to `oracle.spann3r_oracle` run in float64, with the memory read replaced by
`MaskedMemory`: the reference's training-mode read (spann3r/model.py:145-183 with attn_thresh = 0 and no similarity gate)
whose nn.Dropout mask is the Philox keep-scale the product draws for that read's seed.  The helpers live here so that the
tests below can pin them without a GPU:

* the masked read equals the read the training backward differentiates (`_recompute.memory_read`) in fp64;
* a mask of the wrong seed, or the right mask shifted by one key, moves that read by far more than the GPU module's
  forward bars, so those bars can tell a wrong mask from rounding;
* `keep_scale` lays the flat Philox stream out as the [B, P, M] attention tensor the reference's dropout acts on.
"""
import functools
import math

import numpy as np
import torch

from conftest import get_state_dict, rel_l2
from oracle import spann3r_oracle as orc
from spann3r_b200 import _recompute as R
from test_train_cpu import philox_keep_scale_numpy


def keep_scale(seed: int, B: int, N: int, M: int, p: float, device="cpu") -> torch.Tensor:
    """Keep-scale (0 or fp32(1 / (1 - p)), what the kernel multiplies by) of the [B, N, M] attention weights of one
    training-mode read with `seed`, in float64: element (b, n, i) is flat index (b * N + n) * M + i of the Philox stream."""
    ks = philox_keep_scale_numpy(seed, B * N * M, p).reshape(B, N, M)
    return torch.from_numpy(ks).to(device, torch.float64)


def masked_read(sd, feat, mem_k, mem_v, ks):
    """spann3r/model.py:145-183 in training mode: softmax(LN_q(feat) LN_k(K)^T / sqrt(C)), times the dropout keep-scale
    `ks` [B, P, M] (no threshold, no renormalisation), then . LN_v(V) + feat."""
    q = orc.layernorm(sd, "norm_q", feat, 1e-5)
    k = orc.layernorm(sd, "norm_k", mem_k, 1e-5)
    attn = torch.softmax(torch.einsum("bpc,bxc->bpx", q, k) / math.sqrt(feat.shape[-1]), dim=-1)
    attn = attn * ks.to(attn.dtype)
    return torch.einsum("bpx,bxc->bpc", attn, orc.layernorm(sd, "norm_v", mem_v, 1e-5)) + feat


class MaskedMemory(orc.SpatialMemory):
    """`orc.SpatialMemory` in training mode: every `memory_read` takes the next keep-scale of `masks` (consumed in order)."""

    def __init__(self, sd, masks, **kw):
        super().__init__(sd, **kw)
        assert self.attn_thresh == 0 and self.sim_thresh == 1.0, "the masked read is the training-mode read (no cut, no gate)"
        self.masks = masks

    def memory_read(self, feat, res=True):
        assert res
        ks = self.masks.pop(0)
        assert tuple(ks.shape) == (feat.shape[0], feat.shape[1], self.mem_k.shape[1]), (ks.shape, feat.shape, self.mem_k.shape)
        return masked_read(self.sd, feat, self.mem_k, self.mem_v, ks)


def masked_memory(masks: list):
    """A stand-in for `orc.SpatialMemory` (monkeypatched in; `orc.forward` and `usefeat_oracle.forward` look it up at call
    time) whose reads pop `masks`."""
    return functools.partial(MaskedMemory, masks=masks)


# The wrong masks the GPU module's sensitivity test builds the reference with
def wrong_seed(seed, B, N, M, p, device="cpu"):
    return keep_scale(seed + 1, B, N, M, p, device)


def rolled_mask(seed, B, N, M, p, device="cpu"):
    return torch.roll(keep_scale(seed, B, N, M, p, device), 1, dims=-1)


B_, N_, P_ = 2, 196, 0.15


def _read_case():
    """fp64 norm_q / norm_k / norm_v of the sharpened checkpoint, a two-frame bank and a query, at B = 2, 224 x 224 tokens."""
    sd = {k: v.double() for k, v in get_state_dict(True).items() if k.startswith("norm_")}
    g = torch.Generator().manual_seed(17)
    ks = [torch.randn(B_, N_, 1024, generator=g, dtype=torch.float64) for _ in range(2)]
    vs = [torch.randn(B_, N_, 1024, generator=g, dtype=torch.float64) for _ in range(2)]
    q = torch.randn(B_, N_, 1024, generator=g, dtype=torch.float64)
    return sd, ks, vs, q


def _oracle_read(sd, ks, vs, q, mask):
    mem = masked_memory([mask])(sd, attn_thresh=0, sim_thresh=1.0)
    for k, v in zip(ks, vs):
        mem.add_mem(k, v)
    out = mem.memory_read(q)
    assert not mem.masks
    return out


def test_masked_oracle_read_equals_the_recompute_read():
    sd, ks, vs, q = _read_case()
    seed = 987654321987
    mask = keep_scale(seed, B_, N_, 2 * N_, P_)
    got = _oracle_read(sd, ks, vs, q, mask)
    ref = R.memory_read(sd, q, torch.cat(ks, 1), torch.cat(vs, 1), mask)
    assert rel_l2(got, ref) < 1e-12
    # with every element kept unscaled it is the oracle's own training-mode read
    plain = orc.SpatialMemory(sd, attn_thresh=0, sim_thresh=1.0)
    for k, v in zip(ks, vs):
        plain.add_mem(k, v)
    assert rel_l2(_oracle_read(sd, ks, vs, q, torch.ones_like(mask)), plain.memory_read(q)) < 1e-12


def test_wrong_masks_move_the_read_far_past_the_forward_bars():
    from test_train_fp64_gpu import FWD
    sd, ks, vs, q = _read_case()
    seed = 987654321987
    args = (seed, B_, N_, 2 * N_, P_)
    right = _oracle_read(sd, ks, vs, q, keep_scale(*args))
    bar = max(g for g, _ in FWD.values())
    for name, mask in (("seed + 1", wrong_seed(*args)), ("rolled", rolled_mask(*args))):
        moved = rel_l2(_oracle_read(sd, ks, vs, q, mask), right)
        print(f"masked read, {name} mask: moved by {moved:.2e} (largest forward bar {bar:.1e})")
        assert moved > 100 * bar, (name, moved, bar)


def test_keep_scale_layout_is_the_flat_philox_stream():
    seed, M = 4242424242, 3 * N_
    ks = keep_scale(seed, B_, N_, M, P_)
    flat = philox_keep_scale_numpy(seed, B_ * N_ * M, P_)
    rng = np.random.default_rng(0)
    for b, n, i in [(0, 0, 0), (1, 0, 0), (1, N_ - 1, M - 1), (0, 5, 3)] + \
            [tuple(int(x) for x in t) for t in zip(rng.integers(0, B_, 64), rng.integers(0, N_, 64), rng.integers(0, M, 64))]:
        assert float(ks[b, n, i]) == float(flat[(b * N_ + n) * M + i]), (b, n, i)
    assert not torch.equal(ks[0], ks[1])                        # batch item 1 continues the stream, it does not repeat it
    assert set(np.unique(flat).tolist()) == {0.0, float(np.float32(1 / (1 - P_)))}
    assert torch.equal(rolled_mask(seed, B_, N_, M, P_)[..., 1:], ks[..., :-1])
