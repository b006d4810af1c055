"""Drop-in `Spann3R` / `SpatialMemory` / DUSt3R module for the reference's callers.

Mirrors the reference's public surface (spann3r/model.py:11-226,473-539; dust3r/model.py:84-225) --
same class names, constructor signature, `state_dict` keys (1101, or 1099 with `use_feat=True`; strict-loadable both ways), the
`.dust3r` attribute, `forward(frames, return_memory=False) -> (preds, preds_all[, sp_mem])` with the
same dict keys / shapes -- so `demo.py` / `eval.py` run by changing one import (INTEGRATION.md).

The modules below hold parameters only.  All arithmetic runs in libspann3r_b200.so through
`engine.Engine`; there is no eager-PyTorch, CPU or Triton path -- on a machine without an sm_90
GPU `forward` raises.  Training mode (`train.py`): the same CUDA forward with the reference's
training branches (attn_thresh=0, memory dropout, ungated add_mem) and a PyTorch-recompute backward (SURVEY.md §8f rank 1, staged).
`offline_reconstruction` (SURVEY.md §8f rank 2) is built on the same engine stages.  Portrait frames follow the
reference's landscape wrapper (`_to_landscape`).  Every constructor option is supported: `mem_pos_enc=True` puts RoPE into the
value encoder; `use_feat=True` builds the reference's 768-wide value encoder (16 heads of 48, no `pos_patch_embed`), fed
with head 1's last decoder tokens instead of the pointmap.  The library runs its 48-wide heads zero-padded to 64-wide slots
(include/spann3r_b200.h, s3r_model_w.value_dim), an exact repacking of the same arithmetic.

Precision: `Spann3R(precision="fp32")` (default) holds the forward within 1e-3 of the fp32 reference: every GEMM multiplies
split-bf16 operands with three tensor-core products.  `precision="bf16"` (or `set_precision("bf16")`) is an opt-in for speed
over parity, inference only: the GEMMs of the encoder, decoder, key heads and value encoder multiply bf16 operands once,
with fp32 accumulation; the DPT heads, the spatial memory and the attention cores are unchanged (the reference's own
`use_amp` inference likewise keeps its heads in fp32).
"""
from __future__ import annotations

import argparse
import os

import torch
import torch.nn as nn

from . import offline, synth
from ._lib import conf_score as _conf_score
from .engine import MAX_SLOTS, PRECISIONS, Engine, MemoryBank, PackedWeights


# ------------------------------------------------------------------------------------------------
# parameter tree with the reference's exact key layout
# ------------------------------------------------------------------------------------------------
class ParamModule(nn.Module):
    """A container of parameters / sub-containers (no forward: compute lives in the CUDA library)."""

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("spann3r_b200 leaf modules hold parameters only; call Spann3R.forward / the .dust3r "
                           "stage methods (the fused CUDA path) instead")


def build_param_tree(root: nn.Module, keys_shapes: dict, prefix: str = ""):
    """Create nested ParamModules under `root` so that root.state_dict() has exactly the given keys, in order.
    Aliased keys (dpt scratch.layerK_rn == scratch.layer_rn.K-1) share one Parameter, as in the reference."""
    shared = {}
    for key, shape in keys_shapes.items():
        if not key.startswith(prefix):
            continue
        parts = key[len(prefix):].split(".")
        mod = root
        for p in parts[:-1]:
            if p not in mod._modules:
                mod.add_module(p, ParamModule())
            mod = mod._modules[p]
        canon = synth.canonical_key(key)
        if canon not in shared:
            # zero-filled, never uninitialised memory; `Spann3R._init_like_reference` gives the keys a DUSt3R
            # checkpoint does not cover the reference constructors' default init
            shared[canon] = nn.Parameter(torch.zeros(tuple(shape), dtype=torch.float32))   # trainable, like the reference's
        mod.register_parameter(parts[-1], shared[canon])
    return root


def _to_landscape(t: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """transpose_to_landscape / wrapper_yes (dust3r/utils/misc.py:66-94) as Spann3R configures it (landscape_only=True,
    spann3r/model.py:222) over PatchEmbedDust3R tokens: the head runs at the frame's own (H, W); for a portrait
    frame every output then has axes 1 and 2 swapped -- a VIEW, like the reference's `swapaxes`."""
    return t.swapaxes(1, 2) if H > W else t


class AsymmetricCroCo3DStereo(ParamModule):
    """Parameter holder + stage methods of dust3r/model.py:53-225 (ViT-L encoder, twin ViT-B decoder, DPT heads)."""

    enc_embed_dim, dec_embed_dim, enc_depth, dec_depth = 1024, 768, 24, 12

    def __init__(self, spec=None):
        super().__init__()
        spec = spec or synth.load_spec()
        build_param_tree(self, spec["spann3r"], prefix="dust3r.")
        self._owner = None  # set by Spann3R

    def load_state_dict(self, ckpt, strict=True, **kw):
        # dust3r/model.py:94-101: a checkpoint without dec_blocks2 duplicates dec_blocks into it
        new = dict(ckpt)
        if not any(k.startswith("dec_blocks2") for k in ckpt):
            for k, v in ckpt.items():
                if k.startswith("dec_blocks"):
                    new[k.replace("dec_blocks", "dec_blocks2")] = v
        if self._owner is not None:
            self._owner._packed_dirty = True
        return super().load_state_dict(new, strict=strict, **kw)

    # -- stage methods, same names / argument meaning as the reference -------------------------------
    def _encode_image(self, image, true_shape=None):
        """dust3r/model.py:131-154 -> (x [B,N,1024], pos [B,N,2] int64, None)."""
        eng = self._owner._engine_for(image.shape[0], image.shape[-2], image.shape[-1], encode_only=True)
        x = eng.encode(self._owner._dev(image))
        return x, self._owner._positions(image.shape[0], image.shape[-2], image.shape[-1]), None

    def _decoder(self, f1, pos1, f2, pos2):
        """dust3r/model.py:186-205 -> (dec1, dec2), 13 tensors each ([f_enc, d1..d12], d12 normed)."""
        o = self._owner
        # the patch grid comes from the POSITIONS, as in the reference (its RoPE is position-driven): 768 tokens can be
        # 24 x 32 or 32 x 24, and only pos tells which
        grids = []
        for pos in (pos1, pos2):
            if pos is None:
                raise RuntimeError("_decoder needs the token positions (pos1, pos2) returned by _encode_image")
            gh, gw = int(pos[..., 0].max()) + 1, int(pos[..., 1].max()) + 1
            grids.append((gh, gw))
        if grids[0] != grids[1] or grids[0][0] * grids[0][1] != f1.shape[1] or f2.shape[1] != f1.shape[1]:
            raise RuntimeError(f"_decoder: positions describe patch grids {grids} but the features have "
                               f"{f1.shape[1]} / {f2.shape[1]} tokens (both views must share one grid)")
        eng = o._engine_for(f1.shape[0], 16 * grids[0][0], 16 * grids[0][1])
        dec_all = eng.decode(f1.contiguous(), f2.contiguous(), want_all=True)
        dec1 = [f1] + [dec_all[l, 0] for l in range(12)]
        dec2 = [f2] + [dec_all[l, 1] for l in range(12)]
        o._last_dec = (id(dec1[-1]), id(dec2[-1]))
        return dec1, dec2

    def forward(self, view1, view2):
        """Pairwise DUSt3R forward (dust3r/model.py:213-225) for `dust3r.inference.inference`."""
        o = self._owner
        img1, img2 = o._dev(view1["img"]), o._dev(view2["img"])
        B, _, H, W = img1.shape
        eng = o._engine_for(B, H, W)
        feats = eng.encode(torch.cat((img1, img2), dim=0).contiguous())
        eng.decode(feats[:B].contiguous(), feats[B:].contiguous())
        pts, conf = eng.heads()
        return ({"pts3d": _to_landscape(pts[0], H, W), "conf": _to_landscape(conf[0], H, W)},
                {"pts3d_in_other_view": _to_landscape(pts[1], H, W), "conf": _to_landscape(conf[1], H, W)})


# ------------------------------------------------------------------------------------------------
# spatial memory
# ------------------------------------------------------------------------------------------------
class SpatialMemory:
    """spann3r/model.py:11-210 with the bank resident in pre-allocated device buffers (engine.MemoryBank).

    Same attributes (`mem_k`, `mem_v`, `mem_attn`, `mem_count`, `wm`, `lm`, `num_patches`) and methods
    (`add_mem`, `add_mem_check`, `check_sim`, `memory_read`, `memory_prune`) as the reference class;
    `norm_q/k/v` are applied inside the CUDA library (LN_k / LN_v once at write time)."""

    def __init__(self, norm_q=None, norm_k=None, norm_v=None, mem_dropout=None, long_mem_size=4000, work_mem_size=5,
                 attn_thresh=5e-4, sim_thresh=0.95, save_attn=False, num_patches=None, *, engine: Engine = None):
        if engine is None:
            raise RuntimeError("SpatialMemory needs the CUDA engine (no CPU path)")
        if mem_dropout is not None and getattr(mem_dropout, "training", False):
            raise NotImplementedError("training-mode memory dropout is not implemented (inference path only)")
        self.engine = engine
        self.attn_thresh = attn_thresh
        self.long_mem_size = long_mem_size
        self.work_mem_size = work_mem_size
        self.top_k = long_mem_size
        self.sim_thresh = sim_thresh
        self.num_patches = num_patches
        self.bank = None
        self._sim_host = None
        self.init_mem()

    def init_mem(self):
        self.lm = 0
        self.wm = 0
        if self.bank is not None:
            self.bank.len = 0

    def _ensure_bank(self, P):
        if self.bank is None:
            cap = self.long_mem_size + (self.work_mem_size + 3) * P
            self.bank = MemoryBank(self.engine.B, cap, self.engine.device)

    # reference-compatible views
    @property
    def mem_k(self):
        return None if self.bank is None or self.bank.len == 0 else self.bank.k_raw[:, : self.bank.len]

    @property
    def mem_v(self):
        return None if self.bank is None or self.bank.len == 0 else self.bank.v_raw[:, : self.bank.len]

    @property
    def mem_attn(self):
        return None if self.bank is None or self.bank.len == 0 else self.bank.attn[:, : self.bank.len, None]

    @property
    def mem_count(self):
        return None if self.bank is None or self.bank.len == 0 else self.bank.count[:, : self.bank.len, None]

    def add_mem(self, feat_k, feat_v, pts_cur=None, img_cur=None):  # :80-95
        if self.num_patches is None:
            self.num_patches = feat_k.shape[1]
        self._ensure_bank(self.num_patches)
        self.engine.memory_append(self.bank, feat_k, feat_v)

    def check_sim(self, feat_k, thresh=0.7):  # :97-118
        return self.check_sim_finish(self.check_sim_async(feat_k, thresh), thresh)

    def check_sim_async(self, feat_k, thresh=0.7):
        """First half of check_sim: enqueue the similarity kernels and an async copy of max(mean_corr) to pinned host
        memory.  The reference reads the value with a blocking `.item()` right away (:114); the forward loop instead
        enqueues this as soon as feat_k exists and reads it (check_sim_finish) after the DPT heads and the value encoder
        have been enqueued, so the GPU never drains while the host decides whether to append.  Same inputs (the bank does
        not change in between), same value, same decision."""
        if self.bank is None or self.bank.len == 0 or thresh == 1.0:
            return None
        # the window is the last wm * P tokens, or the whole bank when a prune to long_mem_size < wm * P tokens left
        # fewer (mem_k[:, -wm * P:] of the reference)
        mean_corr = self.engine.check_sim(self.bank, feat_k, min(self.wm, self.bank.len // self.num_patches))
        if self._sim_host is None:
            self._sim_host = torch.empty(1, dtype=torch.float32, pin_memory=True)
        self._sim_host.copy_(mean_corr.max().reshape(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(mean_corr.device))
        return ev

    def check_sim_finish(self, pending, thresh=0.7):
        if pending is None:
            return False
        pending.synchronize()
        mx = float(self._sim_host[0])
        if mx > thresh:
            print("Similarity detected:", mx)
            return True
        return False

    def add_mem_check(self, feat_k, feat_v, pts_cur=None, img_cur=None, sim_pending="now"):  # :120-143
        if self.num_patches is None:
            self.num_patches = feat_k.shape[1]
        if sim_pending == "now":
            sim_pending = self.check_sim_async(feat_k, thresh=self.sim_thresh)
        if self.check_sim_finish(sim_pending, thresh=self.sim_thresh):
            return
        self.add_mem(feat_k, feat_v, pts_cur, img_cur)
        self.wm += 1
        if self.wm > self.work_mem_size:
            self.wm -= 1
            if self.long_mem_size == 0:
                P = self.num_patches
                idx = torch.arange(P, self.bank.len, device=self.engine.device)[None].expand(self.bank.batch, -1)
                self.bank.gather(idx.contiguous())
            else:
                self.lm += self.num_patches
        if self.lm > self.long_mem_size:
            self.memory_prune()
            self.lm = self.top_k - self.wm * self.num_patches

    def memory_read(self, feat, res=True):  # :145-183
        if not res:
            raise NotImplementedError("memory_read(res=False) is never used by the reference")
        return self.engine.memory_read(self.bank, feat, self.attn_thresh)

    def memory_prune(self):  # :185-210 -- selection stays torch.topk on identical inputs (SURVEY.md §7.3-#3)
        n = self.bank.len
        weights = self.bank.attn[:, :n] / self.bank.count[:, :n]
        weights[self.bank.count[:, :n] < self.work_mem_size + 5] = 1e8
        _, idx = torch.topk(weights, self.top_k, dim=1)
        self.bank.gather(idx)
        print("Memory pruned:", n, "->", self.bank.len)


class SlotMemory:
    """One SpatialMemory per batch item ("slot") of an engine, for independent sequences run as one batch
    (`Spann3R.forward_sequences`).  Each slot applies the reference's add_mem_check / memory_prune
    (spann3r/model.py:120-143,185-210) exactly as a batch-1 run would: its own length, similarity gate, `wm`, `lm` and
    prune.  The slots share one MemoryBank (slot b = batch item b) and the per-slot engine stages, so a step costs one
    launch sequence and one host synchronisation for all gates, as SpatialMemory's lockstep batch does."""

    def __init__(self, long_mem_size=4000, work_mem_size=5, attn_thresh=5e-4, sim_thresh=0.95, *, engine: Engine):
        if engine.B > MAX_SLOTS:
            raise ValueError(f"at most {MAX_SLOTS} slots, the engine has a batch of {engine.B}")
        self.engine = engine
        self.attn_thresh = attn_thresh
        self.long_mem_size = long_mem_size
        self.work_mem_size = work_mem_size
        self.top_k = long_mem_size
        self.sim_thresh = sim_thresh
        self.num_patches = P = engine.N
        B = engine.B
        self.bank = MemoryBank(B, long_mem_size + (work_mem_size + 3) * P, engine.device)
        self.len, self.wm, self.lm = [0] * B, [0] * B, [0] * B
        self.tags = [None] * B            # what the caller runs in each slot (forward_sequences: the sequence index)
        self._sim_host = None

    def start(self, b, tag=None):
        """Empty slot b for a new sequence (init_mem of spann3r/model.py:66-78)."""
        self.finish(b)
        self.tags[b] = tag

    def finish(self, b):
        """Slot b's sequence has ended: zero its bank region (the tail contract) and its counters."""
        self.bank.zero_slot_tail(b, 0, self.len[b])
        self.len[b] = self.wm[b] = self.lm[b] = 0
        self.tags[b] = None

    def memory_read(self, feat):
        """Slot b reads its own bank; an empty slot returns feat[b] itself."""
        return self.engine.memory_read_slots(self.bank, self.len, feat, self.attn_thresh)

    def check_sim_async(self, feat_k):
        """Every slot's gate value (max over its window of mean_p cos) copied to pinned host memory; None when no slot has
        a window.  The window is the last wm frames, or the whole bank after a prune left fewer (spann3r/model.py:102-105)."""
        P = self.num_patches
        wm = [min(w, n // P) for w, n in zip(self.wm, self.len)]
        if max(wm) == 0 or self.sim_thresh == 1.0:
            return None
        vals = self.engine.check_sim_slots(self.bank, self.len, wm, feat_k)
        if self._sim_host is None:
            self._sim_host = torch.empty(self.engine.B, dtype=torch.float32, pin_memory=True)
        self._sim_host.copy_(vals.amax(1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(vals.device))
        return ev

    def check_sim_finish(self, pending):
        """Per slot: True where the gate fired (the write is skipped)."""
        if pending is None:
            return [False] * self.engine.B
        pending.synchronize()
        out = []
        for b, mx in enumerate(self._sim_host.tolist()):
            out.append(mx > self.sim_thresh)
            if out[-1]:
                print(f"Similarity detected (slot {b}):", mx)
        return out

    def add_mem_check(self, feat_k, feat_v, active, sim_pending):
        """add_mem_check of spann3r/model.py:120-143 for every slot with active[b]; returns the per-slot skip decisions."""
        skip = self.check_sim_finish(sim_pending)
        append = [bool(a) and not s for a, s in zip(active, skip)]
        if any(append):
            self.engine.memory_append_slots(self.bank, self.len, append, feat_k, feat_v)
        P = self.num_patches
        for b, a in enumerate(append):
            if not a:
                continue
            self.len[b] += P
            self.wm[b] += 1
            if self.wm[b] > self.work_mem_size:
                self.wm[b] -= 1
                if self.long_mem_size == 0:
                    n = self.len[b]
                    self.bank.gather_slot(b, torch.arange(P, n, device=self.engine.device), n)
                    self.len[b] = n - P
                else:
                    self.lm[b] += P
            if self.lm[b] > self.long_mem_size:
                self.memory_prune(b)
                self.lm[b] = self.top_k - self.wm[b] * P
        return skip

    def memory_prune(self, b):  # :185-210 on slot b alone, selection by torch.topk on its [1, n] weights
        n = self.len[b]
        weights = self.bank.attn[b:b + 1, :n] / self.bank.count[b:b + 1, :n]
        weights[self.bank.count[b:b + 1, :n] < self.work_mem_size + 5] = 1e8
        _, idx = torch.topk(weights, self.top_k, dim=1)
        self.bank.gather_slot(b, idx[0], n)
        self.len[b] = self.top_k
        print(f"Memory pruned (slot {b}):", n, "->", self.top_k)


# ------------------------------------------------------------------------------------------------
# Spann3R
# ------------------------------------------------------------------------------------------------
class Spann3R(ParamModule):
    def __init__(self, dus3r_name="./checkpoints/DUSt3R_ViTLarge_BaseDecoder_512_dpt.pth", use_feat=False,
                 mem_pos_enc=False, memory_dropout=0.15, max_encode_batch: int = 16, precision: str = "fp32"):
        super().__init__()
        self.set_precision(precision)
        self.use_feat, self.mem_pos_enc = bool(use_feat), mem_pos_enc
        # use_feat (spann3r/model.py:225-242): a 768-wide value encoder and no pos_patch_embed
        spec = synth.usefeat_spec() if self.use_feat else synth.load_spec()
        self.dust3r = AsymmetricCroCo3DStereo(spec)
        object.__setattr__(self.dust3r, "_owner", self)
        rest = {k: v for k, v in spec["spann3r"].items() if not k.startswith("dust3r.")}
        build_param_tree(self, rest)
        self.memory_dropout = memory_dropout
        self.max_encode_batch = max_encode_batch
        self._packed = None
        self._packed_dirty = True
        self._packed_moved = False
        self._engines = {}
        self._pos_cache = {}
        if dus3r_name is not None:
            self._init_like_reference()
            self._load_dust3r(dus3r_name)

    def set_precision(self, precision: str):
        """"fp32" (default): fp32-grade GEMMs everywhere.  "bf16": one bf16 tensor-core product per GEMM in the encoder,
        decoder, key heads and value encoder (inference only).  Engines of both precisions share the packed weights."""
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
        self.precision = precision

    # -- checkpoint plumbing -----------------------------------------------------------------------
    def _load_dust3r(self, path):
        """dust3r/model.py:27-51 load_model: {'args': Namespace(model=...), 'model': state_dict}, strict=False."""
        if not os.path.isfile(path):
            raise FileNotFoundError(path)
        torch.serialization.add_safe_globals([argparse.Namespace])
        ckpt = torch.load(path, map_location="cpu")
        args = ckpt["args"].model if "args" in ckpt else synth.DUST3R_ARGS
        flat = args.replace(" ", "")
        for need in ("enc_embed_dim=1024", "enc_depth=24", "dec_embed_dim=768", "dec_depth=12", "head_type='dpt'"):
            if need not in flat:
                raise ValueError(f"unsupported DUSt3R architecture (need {need}): {args}")
        print("... loading model from", path)
        print(self.dust3r.load_state_dict(ckpt["model"], strict=False))
        if not self.use_feat:
            # spann3r/model.py:240-242: pos_patch_embed (default value encoder only) starts as a copy of dust3r.patch_embed
            self.pos_patch_embed.proj.weight.data.copy_(self.dust3r.patch_embed.proj.weight.data)
            self.pos_patch_embed.proj.bias.data.copy_(self.dust3r.patch_embed.proj.bias.data)

    @torch.no_grad()
    def _init_like_reference(self):
        """The parameters a DUSt3R checkpoint does NOT cover get what the reference's constructors give them
        (spann3r/model.py:228-261: stock nn.Linear / nn.LayerNorm / Block init), so that a `strict=False` or partial
        Spann3R checkpoint load never runs on zeros: LayerNorm weight 1 / bias 0, Linear and conv weights
        kaiming_uniform(a=sqrt(5)), biases U(+-1/sqrt(fan_in))."""
        import math
        for name, p in self.named_parameters():
            if name.startswith("dust3r."):
                continue
            leaf = name.split(".")[-1]
            mod = name.split(".")[-2]
            is_norm = mod.startswith("norm") or mod.endswith("_norm") or mod.endswith("norm")
            if is_norm:
                p.fill_(1.0 if leaf == "weight" else 0.0)
            elif leaf == "weight":
                nn.init.kaiming_uniform_(p, a=math.sqrt(5))
            else:
                w = dict(self.named_parameters())[name[: -len("bias")] + "weight"]
                fan_in = w[0].numel()
                p.uniform_(-1.0 / math.sqrt(fan_in), 1.0 / math.sqrt(fan_in))

    # The packed device copy of the weights is rebuilt when the parameters may have changed: load_state_dict, any
    # _apply (.to / .cuda / .float) and an explicit invalidate_packed() after in-place edits of `.data`.
    def invalidate_packed(self):
        self._packed_dirty = True

    def load_state_dict(self, *a, **k):
        self._packed_dirty = True
        return super().load_state_dict(*a, **k)

    def _apply(self, fn, *a, **k):
        self._packed_dirty = True
        self._packed_moved = True
        return super()._apply(fn, *a, **k)

    def _weights(self) -> PackedWeights:
        if self._packed is None or self._packed_dirty:
            dev = next(self.parameters()).device
            if dev.type != "cuda":
                raise RuntimeError("spann3r_b200.Spann3R runs on an H100 only: call .to('cuda') first (no CPU path)")
            self._engines.clear()
            self._packed = None
            self._packed = PackedWeights(self.state_dict(), device=dev)
            self._packed_dirty = False
        return self._packed

    def _weights_train(self) -> PackedWeights:
        """Training: the parameters change every optimizer step, so every forward re-packs them -- with device arithmetic
        and IN PLACE (`PackedWeights.refresh`), which keeps the engines and their cached tile plans valid."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("spann3r_b200.Spann3R runs on an H100 only: call .to('cuda') first (no CPU path)")
        sd = self.state_dict()
        if self._packed is None or self._packed.host_math or self._packed.device != dev or self._packed_moved:
            self._engines.clear()
            self._packed = None
            self._packed = PackedWeights(sd, device=dev, host_math=False)
            self._packed_moved = False
        else:
            self._packed.refresh(sd)
        self._packed_dirty = True      # a later eval-mode call must re-pack: the optimizer steps after this forward
        return self._packed

    def _engine_for(self, B, H, W, n_frames=2, encode_only=False, training=False) -> Engine:
        if training and self.precision != "fp32":
            raise NotImplementedError(f"precision {self.precision!r} is inference only: the training backward recomputes the "
                                      "fp32-grade forward, not this one (set_precision('fp32') to train)")
        w = self._weights_train() if training else self._weights()
        max_images = max(2 * B, min(n_frames * B, self.max_encode_batch * B))
        key = (B, H, W, self.precision)
        eng = self._engines.get(key)
        if eng is None or eng.max_images < max_images:
            self._engines.pop(key, None)
            eng = Engine(w, B, H, W, max_images=max_images, precision=self.precision)
            self._engines[key] = eng
        return eng

    def _dev(self, t):
        dev = next(self.parameters()).device
        return t.to(dev, torch.float32, non_blocking=True).contiguous()

    @staticmethod
    def _check_true_shape(frames, H, W):
        """The reference takes (H, W) from view['true_shape'] when present (spann3r/model.py:263-287); with the
        PatchEmbedDust3R it runs, that is the tensor's own shape for every frame a dataset produces."""
        for f in frames:
            if tuple(f["img"].shape[-2:]) != (H, W):
                raise ValueError("all frames of a sequence must have the same height and width")
            ts = f.get("true_shape")
            if ts is not None and any((int(h), int(w)) != (H, W) for h, w in torch.as_tensor(ts).reshape(-1, 2).tolist()):
                raise NotImplementedError(f"true_shape {ts} differs from the image tensor shape {(H, W)}")

    def _positions(self, B, H, W):
        key = (H, W)
        if key not in self._pos_cache:
            dev = next(self.parameters()).device
            y, x = torch.arange(H // 16, device=dev), torch.arange(W // 16, device=dev)
            self._pos_cache[key] = torch.cartesian_prod(y, x)
        return self._pos_cache[key].view(1, -1, 2).expand(B, -1, 2).clone()

    # -- forward -----------------------------------------------------------------------------------
    def forward(self, frames, return_memory=False):
        """spann3r/model.py:473-539.  Eval mode: the inference path below.  Training mode (`self.training`): the same CUDA
        forward with the reference's training branches and a PyTorch-recompute backward (`train.py`)."""
        if self.training:      # also under torch.no_grad(): the training BRANCHES are what .train() selects, as in the reference
            if self.precision != "fp32":
                raise NotImplementedError(f"precision {self.precision!r} is inference only (set_precision('fp32') to train)")
            from .train import forward_train
            return forward_train(self, frames, return_memory)
        return self._forward_eval(frames, return_memory)

    @torch.no_grad()
    def _forward_eval(self, frames, return_memory=False):
        F_ = len(frames)
        img0 = frames[0]["img"]
        B, _, H, W = img0.shape
        self._check_true_shape(frames, H, W)
        eng = self._engine_for(B, H, W, n_frames=F_)
        sp_mem = SpatialMemory(engine=eng)

        # The encoder has no dependence on the memory loop: encode every frame up front in large batches
        # (SURVEY.md §3.1); per-image results are identical to the reference's pair / single-frame calls.
        feats = self._encode_frames(eng, [self._dev(f["img"]) for f in frames])
        return self._frame_loop(F_, H, W, eng, sp_mem, lambda i: feats[i], return_memory)

    @staticmethod
    def _encode_frames(eng, imgs):
        """Encode the frames imgs ([B, 3, H, W] each) in calls of up to eng.max_images images -> one [B, N, 1024] each."""
        B = imgs[0].shape[0]
        feats = []
        chunk = max(1, eng.max_images // B)
        for s in range(0, len(imgs), chunk):
            part = imgs[s: s + chunk]
            out = eng.encode(torch.cat(part, dim=0) if len(part) > 1 else part[0])
            feats += list(out.view(len(part), B, eng.N, 1024).unbind(0))
        return feats

    def _frame_loop(self, F_, H, W, eng, sp_mem, feat_of, return_memory):
        """The frame loop of spann3r/model.py:484-533 over the already encoded frames."""
        portrait = H > W        # heads run at (H, W); outputs and the pointmap value encoder's input are the landscape views
        feat_k2 = None
        preds, preds_all = None, []
        for i in range(F_ - 1):
            feat1, feat2 = feat_of(i), feat_of(i + 1)
            feat_fuse = sp_mem.memory_read(feat_k2, res=True) if feat_k2 is not None else feat1
            eng.decode(feat_fuse, feat2)
            feat_k1, feat_k2 = eng.keyheads(feat1, feat2)
            sim = sp_mem.check_sim_async(feat_k1, thresh=sp_mem.sim_thresh)   # read back in add_mem_check below
            pts, conf = eng.heads()
            res1 = {"pts3d": _to_landscape(pts[0], H, W), "conf": _to_landscape(conf[0], H, W)}
            res2 = {"pts3d": _to_landscape(pts[1], H, W), "conf": _to_landscape(conf[1], H, W)}
            mem_v = self._value(eng, pts[0], feat_k1, portrait)
            sp_mem.add_mem_check(feat_k1, mem_v, sim_pending=sim)
            res2["pts3d_in_other_view"] = res2.pop("pts3d")
            if preds is None:
                preds = [res1]
                preds_all = [(res1, res2)]
            else:
                res1["pts3d_in_other_view"] = res1.pop("pts3d")
                preds.append(res1)
                preds_all.append((res1, res2))
        preds.append(res2)
        if return_memory:
            return preds, preds_all, sp_mem
        return preds, preds_all

    def _value(self, eng, pts1, feat_k1, portrait):
        """encode_cur_value(res1, dec1, pos1, shape1) + feat_k1 (spann3r/model.py:312-320, 519-521) after the engine's last
        decode / heads.  Default: the pointmap of head 1, which the engine reads through the landscape view's strides.
        use_feat: dec1[-1], the engine's resident dec_norm tokens of stream 1, on the frame's own grid."""
        if self.use_feat:
            return eng.value(None, feat_k1, rope=self.mem_pos_enc, tokens=True)
        return eng.value(pts1, feat_k1, transposed=portrait, rope=self.mem_pos_enc)

    # -- independent sequences in one batch ------------------------------------------------------------------
    def forward_sequences(self, sequences, max_batch: int = 8):
        """Reconstruct many sequences, batched, each exactly as `forward(sequence)` would at batch 1: its own similarity
        gate, working / long-term counters, prune and bank length (`SlotMemory`).  `forward` with B > 1 instead couples
        the batch (one gate, shared counters: the reference's semantics); this does not.

        sequences: list of sequences, each a list of >= 2 view dicts {'img': [1, 3, H, W]}; they may differ in length and
        resolution.  Sequences of one resolution run on one engine with up to `max_batch` slots; a slot whose sequence
        ends takes the next waiting one, and slots left without a sequence run on zero features with no memory writes.
        Returns one (preds, preds_all) per sequence, in input order, with the keys and shapes of `forward`.  Eval only."""
        if self.training:
            raise NotImplementedError("forward_sequences is an inference path; call .eval() first")
        if not 1 <= max_batch <= MAX_SLOTS:
            raise ValueError(f"max_batch must be in [1, {MAX_SLOTS}], got {max_batch}")
        groups = {}
        for s, seq in enumerate(sequences):
            if len(seq) < 2:
                raise ValueError(f"sequence {s} has {len(seq)} frame(s); the frame loop needs at least 2")
            img0 = seq[0]["img"]
            if img0.dim() != 4 or img0.shape[0] != 1:
                raise ValueError(f"sequence {s}: frames must be single views [1, 3, H, W], got {tuple(img0.shape)}")
            H, W = img0.shape[-2:]
            self._check_true_shape(seq, H, W)
            groups.setdefault((int(H), int(W)), []).append(s)
        results = [None] * len(sequences)
        with torch.no_grad():
            for (H, W), ids in groups.items():
                self._run_slots([sequences[s] for s in ids], ids, H, W, min(max_batch, len(ids)), results)
        return results

    def _run_slots(self, seqs, ids, H, W, B, results):
        """The frame loop of `_frame_loop` over B slots, each advancing its own sequence; refills in input order."""
        portrait = H > W
        eng = self._engine_for(B, H, W, n_frames=max(len(q) for q in seqs))
        N = eng.N
        mem = SlotMemory(engine=eng)
        waiting = list(range(len(seqs)))          # positions in seqs, taken in order
        slot = [None] * B                          # per slot: dict of the running sequence, or None when idle
        zeros = torch.zeros(1, N, 1024, dtype=torch.float32, device=eng.device)

        def fill(free):
            """Start the next waiting sequences in the free slots; their frames are encoded in batched calls."""
            new = []
            for b in free:
                if not waiting:
                    break
                j = waiting.pop(0)
                mem.start(b, ids[j])
                slot[b] = {"j": j, "i": 0, "feats": [], "preds": None, "preds_all": []}
                new.append(b)
            imgs = [(b, self._dev(f["img"])) for b in new for f in seqs[slot[b]["j"]]]
            for s in range(0, len(imgs), eng.max_images):
                part = imgs[s: s + eng.max_images]
                out = eng.encode(torch.cat([im for _, im in part], dim=0))
                for (b, _), f in zip(part, out.view(len(part), 1, N, 1024).unbind(0)):
                    slot[b]["feats"].append(f)

        fill(range(B))
        feat_k2 = None
        while any(st is not None for st in slot):
            active = [st is not None for st in slot]
            f1 = torch.cat([st["feats"][st["i"]] if st else zeros for st in slot]).contiguous()
            f2 = torch.cat([st["feats"][st["i"] + 1] if st else zeros for st in slot]).contiguous()
            # a slot's first step reads nothing (feat_fuse = feat1, spann3r/model.py:495-500): its bank is empty, and the
            # read of an empty slot returns its query, here feat1
            q = f1 if feat_k2 is None else torch.stack(
                [f1[b] if (st is None or st["i"] == 0) else feat_k2[b] for b, st in enumerate(slot)]).contiguous()
            feat_fuse = mem.memory_read(q) if max(mem.len) > 0 else q
            eng.decode(feat_fuse, f2)
            feat_k1, feat_k2 = eng.keyheads(f1, f2)
            sim = mem.check_sim_async(feat_k1)
            pts, conf = eng.heads()
            mem_v = self._value(eng, pts[0], feat_k1, portrait)
            mem.add_mem_check(feat_k1, mem_v, active, sim)
            done = []
            for b, st in enumerate(slot):
                if st is None:
                    continue
                res1 = {"pts3d": _to_landscape(pts[0, b:b + 1], H, W), "conf": _to_landscape(conf[0, b:b + 1], H, W)}
                res2 = {"pts3d": _to_landscape(pts[1, b:b + 1], H, W), "conf": _to_landscape(conf[1, b:b + 1], H, W)}
                res2["pts3d_in_other_view"] = res2.pop("pts3d")
                if st["preds"] is None:
                    st["preds"] = [res1]
                    st["preds_all"] = [(res1, res2)]
                else:
                    res1["pts3d_in_other_view"] = res1.pop("pts3d")
                    st["preds"].append(res1)
                    st["preds_all"].append((res1, res2))
                st["i"] += 1
                if st["i"] == len(seqs[st["j"]]) - 1:
                    st["preds"].append(res2)
                    results[ids[st["j"]]] = (st["preds"], st["preds_all"])
                    mem.finish(b)
                    slot[b] = None
                    done.append(b)
            if done:
                fill(done)

    # -- offline mode (SURVEY.md §8f rank 2) ------------------------------------------------------------
    def find_initial_pair(self, graph, n_frames):
        """spann3r/model.py:333-357: the pair with the highest summed confidence score in the pairwise graph
        (`graph` = output of the reference's dust3r.inference.inference run on `model.dust3r`)."""
        view1, view2, pred1, pred2 = graph["view1"], graph["view2"], graph["pred1"], graph["pred2"]
        conf_matrix = torch.zeros(n_frames, n_frames)
        for i in range(len(view1["idx"])):
            c1, c2 = pred1["conf"][i].float(), pred2["conf"][i].float()
            if c1.is_cuda:
                sc = float(_conf_score(c1.contiguous())) + float(_conf_score(c2.contiguous()))
            else:   # the reference moves the graph to the CPU (dust3r/inference.py:73): tiny host-side reductions
                sc = float(((c1 - 1) / c1).mean() + ((c2 - 1) / c2).mean())
            conf_matrix[int(view1["idx"][i]), int(view2["idx"][i])] = sc
        flat = int(conf_matrix.argmax())
        pair_idx = (flat // n_frames, flat % n_frames)
        print(f"init pair:{pair_idx}, conf: {conf_matrix.max()}")
        return pair_idx

    @torch.no_grad()
    def offline_reconstruction(self, frames, graph=None, *, scene_graph="complete", prefilter=None, max_batch=None):
        """spann3r/model.py:394-471 + find_next_best_view :359-392 (eval mode).  Every frame is encoded once up front
        (the reference re-encodes each candidate on every iteration; the features are identical).

        graph: the output of the reference's `inference(make_pairs(...), model.dust3r)` (or `offline.inference`).  With
        graph=None the initial pair comes from `offline.pair_scores` over `scene_graph` / `prefilter` (single views only),
        and no pairwise maps are materialised.
        max_batch: next-best-view candidates decoded per engine call (default 8 without a graph, 1 with one).  Above 1,
        each step scores its candidates in batches with one host read; the winner is then decoded again at batch 1, so
        the outputs for a chosen frame do not depend on max_batch -- only a near-tie between candidates can.  Frames of
        batch B > 1 (the reference's lockstep batch, scored by a mean over the batch) always take the serial loop."""
        if self.training:
            raise NotImplementedError("spann3r_b200 implements the inference path; call .eval() first")
        if max_batch is None:
            max_batch = 8 if graph is None else 1
        if max_batch < 1:
            raise ValueError(f"max_batch must be >= 1, got {max_batch}")
        n_frames = len(frames)
        idx_todo = list(range(n_frames))
        B, _, H, W = frames[0]["img"].shape
        self._check_true_shape(frames, H, W)
        if graph is None and B != 1:
            raise ValueError(f"offline_reconstruction without a graph needs single views [1, 3, H, W], got batch {B}")
        portrait = H > W
        eng = self._engine_for(B, H, W, n_frames=n_frames)
        sp_mem = SpatialMemory(engine=eng)
        if graph is not None:
            p0, p1 = self.find_initial_pair(graph, n_frames)
        feats = self._encode_frames(eng, [self._dev(f["img"]) for f in frames])
        if graph is None:
            p0, p1 = offline.initial_pair(self, feats, H, W, scene_graph, prefilter, max_batch)
        idx_used = [p0, p1]
        idx_todo.remove(p0)
        idx_todo.remove(p1)
        # the candidate engine: batch K, its own workspace, so the main engine's state is only touched by the winner
        cand_eng = self._engine_for(min(max_batch, n_frames - 2), H, W) if max_batch > 1 and B == 1 and idx_todo else None

        def decode_heads(f_fuse, f2):
            eng.decode(f_fuse, f2)
            pts, conf = eng.heads()
            return ({"pts3d": _to_landscape(pts[0], H, W), "conf": _to_landscape(conf[0], H, W), "_raw": pts[0]},
                    {"pts3d": _to_landscape(pts[1], H, W), "conf": _to_landscape(conf[1], H, W)})

        feat1, feat2 = feats[p0], feats[p1]
        feat_fuse = feat1
        res1, res2 = decode_heads(feat_fuse, feat2)
        feat_k2, preds, preds_all = None, None, []
        while True:
            if feat_k2 is not None:
                feat1 = feat2
                feat_fuse = sp_mem.memory_read(feat_k2, res=True)
                if cand_eng is not None:
                    best_id, best_conf = offline.next_best_view(cand_eng, feat_fuse, feats, idx_todo)
                else:
                    best_conf, best_id = 0.0, None
                    for i in idx_todo:                               # find_next_best_view
                        r1, r2 = decode_heads(feat_fuse, feats[i])
                        total = float(_conf_score(r1["conf"].contiguous())) + float(_conf_score(r2["conf"].contiguous()))
                        if total > best_conf:
                            best_conf, best_id = total, i
                idx_todo.remove(best_id)
                idx_used.append(best_id)
                print(f"next best view: {best_id}, conf: {best_conf}")
                feat2 = feats[best_id]
                res1, res2 = decode_heads(feat_fuse, feat2)          # restores the engine's hooks for the winner
            feat_k1, feat_k2 = eng.keyheads(feat1, feat2)
            mem_v = self._value(eng, res1.pop("_raw"), feat_k1, portrait)
            sp_mem.add_mem_check(feat_k1, mem_v)
            res2["pts3d_in_other_view"] = res2.pop("pts3d")
            if preds is None:
                preds = [res1]
                preds_all = [(res1, res2)]
            else:
                res1["pts3d_in_other_view"] = res1.pop("pts3d")
                preds.append(res1)
                preds_all.append((res1, res2))
            if len(idx_todo) == 0:
                break
        preds.append(res2)
        return preds, preds_all, idx_used
