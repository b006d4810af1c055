"""Training mode of `Spann3R.forward` (spann3r/model.py:473-539 with `self.training`): SURVEY.md §8f rank 1 / §8e-train,
staged.

What is native and what is not (said once, here):

* FORWARD: every stage runs the sm_90a kernels of libspann3r_b200.so, exactly as in eval mode, with the reference's
  training-mode branches -- `attn_thresh=0` (no cut / renormalisation in the memory read, :474), `mem_dropout` on the
  attention weights (:167-168; Philox mask, reproducible: `s3r_engine_memory_read_train`), ungated `add_mem` (:518-519).
  The packed weights are refreshed in place from the (optimizer-updated) parameters at the start of every forward.
* BACKWARD: **PyTorch recompute** -- each stage is an `autograd.Function` that saves its inputs and, in `backward`,
  re-evaluates the stage with the differentiable restatement in `_recompute.py` and calls `torch.autograd.grad`.  The
  native dgrad / wgrad kernels are the next step of this row; until they exist, backward time is eager PyTorch.
  Gradients reach the `nn.Parameter`s through the Function's parameter inputs, so `DistributedDataParallel`
  (`spann3r/training.py:322-325`) all-reduces them over NCCL like the reference's.

Stages (= Functions): encoder (per chunk of frames), memory read, frame step (twin decoder + key heads + DPT heads), value
encoder.  Square / landscape frames only (the reference trains at 224 x 224).
"""
from __future__ import annotations

import torch

from . import _lib, _recompute as R

_STAGE_PREFIXES = {
    "encode": ("dust3r.patch_embed.", "dust3r.enc_blocks.", "dust3r.enc_norm."),
    "memread": ("norm_q.", "norm_k.", "norm_v."),
    "step": ("dust3r.decoder_embed.", "dust3r.dec_blocks.", "dust3r.dec_blocks2.", "dust3r.dec_norm.", "attn_head_1.",
             "attn_head_2.", "dust3r.downstream_head1.", "dust3r.downstream_head2."),
    "value": ("pos_patch_embed.", "value_encoder.", "value_norm.", "value_out."),
}


def stage_params(model, stage: str):
    """(names, parameters) of one stage, in state-dict order.  Aliased keys (scratch.layerK_rn == scratch.layer_rn.K-1) appear
    under both names with the same Parameter; the restatement reads only `layer_rn.K-1`, the other input gets no gradient."""
    names, params = [], []
    for n, p in model.named_parameters(remove_duplicate=False):
        if n.startswith(_STAGE_PREFIXES[stage]):
            names.append(n)
            params.append(p)
    return names, params


class _Stage(torch.autograd.Function):
    """forward: `native(*acts)` (CUDA library, no autograd graph) -> tuple of tensors;
    backward: recompute `torch_fn(P, *acts)` under autograd and differentiate it (PyTorch recompute backward)."""

    @staticmethod
    def forward(ctx, native, torch_fn, names, n_act, *tensors):
        acts = tensors[:n_act]
        with torch.no_grad():
            outs = native(*acts)
        outs = outs if isinstance(outs, tuple) else (outs,)
        ctx.save_for_backward(*tensors)
        ctx.torch_fn, ctx.names, ctx.n_act = torch_fn, names, n_act
        return outs if len(outs) > 1 else outs[0]

    @staticmethod
    def backward(ctx, *gouts):
        tensors = ctx.saved_tensors
        n_act = ctx.n_act
        acts = [t.detach().requires_grad_(t.is_floating_point()) for t in tensors[:n_act]]
        params = [t.detach().requires_grad_(True) for t in tensors[n_act:]]
        with torch.enable_grad():
            outs = ctx.torch_fn(dict(zip(ctx.names, params)), *acts)
        outs = outs if isinstance(outs, tuple) else (outs,)
        pairs = [(o, g) for o, g in zip(outs, gouts) if g is not None and o.requires_grad]
        wrt = [t for t in acts if t.requires_grad] + params
        grads = torch.autograd.grad([o for o, _ in pairs], wrt, [g for _, g in pairs], allow_unused=True)
        it = iter(grads)
        g_acts = [next(it) if t.requires_grad else None for t in acts]
        g_params = [g if g is None else g.contiguous() for g in it]   # DDP's buckets expect the parameters' own (dense) strides
        return (None, None, None, None, *g_acts, *g_params)


def set_native_linear(on: bool = True):
    """Run the Linear layers of the backward (recompute forward, dgrad, wgrad) on the wgmma GEMM engine (`_native_linear.py`)
    instead of `F.linear` + PyTorch autograd."""
    from . import _native_linear
    _native_linear.ENABLED = bool(on)


def _apply(native, torch_fn, names, params, *acts):
    return _Stage.apply(native, torch_fn, names, len(acts), *acts, *params)


class TrainMemory:
    """SpatialMemory in training mode: ungated `add_mem` (spann3r/model.py:80-95, 518-519) into the engine's bank for the
    native read, plus the autograd-tracked raw keys / values the read's backward differentiates through."""

    def __init__(self, engine, drop_p: float, names, params):
        from .engine import MemoryBank
        self.engine, self.drop_p = engine, float(drop_p)
        self.names, self.params = names, params            # norm_q / norm_k / norm_v
        self.bank = None
        self.keys, self.vals = [], []
        self.MemoryBank = MemoryBank

    def add_mem(self, feat_k, feat_v):
        if self.bank is None:
            self.bank = self.MemoryBank(self.engine.B, 4000 + 8 * self.engine.N, self.engine.device)
        if self.bank.len + self.engine.N > self.bank.cap:
            raise RuntimeError("training-mode memory holds at most %d frames" % (self.bank.cap // self.engine.N))
        self.engine.memory_append(self.bank, feat_k.detach().contiguous(), feat_v.detach().contiguous())
        self.keys.append(feat_k)
        self.vals.append(feat_v)

    def memory_read(self, feat):
        mem_k, mem_v = torch.cat(self.keys, dim=1), torch.cat(self.vals, dim=1)
        names, params = self.names, self.params
        p = self.drop_p
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if p > 0 else 0   # drawn from torch's CPU generator
        eng, bank = self.engine, self.bank

        def native(feat_, mem_k_, mem_v_):
            return eng.memory_read(bank, feat_.contiguous(), 0.0, drop_p=p, seed=seed)

        def torch_fn(P, feat_, mem_k_, mem_v_):
            ks = _lib.dropout_mask((feat_.shape[0], feat_.shape[1], mem_k_.shape[1]), seed, p, feat_.device) if p > 0 else None
            return R.memory_read(P, feat_, mem_k_, mem_v_, ks)
        return _apply(native, torch_fn, names, params, feat, mem_k, mem_v)


def forward_train(model, frames, return_memory=False):
    """`Spann3R.forward` with `self.training` (spann3r/model.py:473-539).  Same outputs / keys as eval mode; every tensor
    in `preds` / `preds_all` carries an autograd graph back to the parameters."""
    F_ = len(frames)
    B, _, H, W = frames[0]["img"].shape
    if H > W:
        raise NotImplementedError("training mode supports square / landscape frames (the reference trains at 224 x 224)")
    model._check_true_shape(frames, H, W)
    eng = model._engine_for(B, H, W, n_frames=F_, training=True)
    N = eng.N
    mem = TrainMemory(eng, model.memory_dropout, *stage_params(model, "memread"))
    imgs = [model._dev(f["img"]) for f in frames]

    enc_names, enc_params = stage_params(model, "encode")
    feats = []
    chunk = max(1, eng.max_images // B)
    for s in range(0, F_, chunk):
        part = imgs[s: s + chunk]
        x = torch.cat(part, dim=0) if len(part) > 1 else part[0]
        out = _apply(lambda im: eng.encode(im.contiguous()), R.encode, enc_names, enc_params, x)
        feats += list(out.view(len(part), B, N, 1024).unbind(0))

    step_names, step_params = stage_params(model, "step")
    val_names, val_params = stage_params(model, "value")
    rope_v = bool(model.mem_pos_enc)

    def native_step(feat_fuse, feat1, feat2):
        eng.decode(feat_fuse.contiguous(), feat2.contiguous())
        k1, k2 = eng.keyheads(feat1.contiguous(), feat2.contiguous())
        pts, conf = eng.heads()
        return k1, k2, pts, conf

    feat_k2 = None
    preds, preds_all = None, []
    for i in range(F_ - 1):
        feat1, feat2 = feats[i], feats[i + 1]
        feat_fuse = mem.memory_read(feat_k2) if feat_k2 is not None else feat1
        feat_k1, feat_k2, pts, conf = _apply(native_step, lambda P, a, b, c: R.step(P, a, b, c, H, W), step_names,
                                             step_params, feat_fuse, feat1, feat2)
        res1 = {"pts3d": pts[0], "conf": conf[0]}
        res2 = {"pts3d_in_other_view": pts[1], "conf": conf[1]}
        mem_v = _apply(lambda p3, k1: eng.value(p3.contiguous(), k1.contiguous(), transposed=False, rope=rope_v),
                       lambda P, p3, k1: R.value(P, p3, k1, rope_v), val_names, val_params, pts[0], feat_k1)
        mem.add_mem(feat_k1, mem_v)                         # training: no similarity gate (spann3r/model.py:518-519)
        if preds is None:
            preds = [res1]
            preds_all = [(res1, res2)]
        else:
            res1["pts3d_in_other_view"] = res1.pop("pts3d")
            preds.append(res1)
            preds_all.append((res1, res2))
    preds.append(res2)
    if return_memory:
        return preds, preds_all, mem
    return preds, preds_all
