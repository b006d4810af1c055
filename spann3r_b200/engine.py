"""Host side of the model-level C ABI: weight packing and the `Engine` wrapper.

`PackedWeights` converts a reference-layout state dict (1101 keys, SURVEY.md §8b; 1099 for use_feat) ONCE into the
split-bf16 planes / fp32 tables of `s3r_model_w` (include/spann3r_b200.h); `Engine` owns one
`s3r_engine` handle per (batch, height, width) and exposes its stages on torch tensors.
Everything here is plumbing (pointers, shapes, one-time layout permutes); all arithmetic of the
forward path runs in libspann3r_b200.so.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib
from ._lib import _f, _i, _i64, _vp  # noqa: F401
from ._lib import Bank, BlockW, DecBlockW, DptW, FusionW, Lin, LN, ModelW, Planes, RcuW  # noqa: F401


ROPE_MAXPOS = 64
MAX_SLOTS = 64      # include/spann3r_b200.h: S3R_MAX_SLOTS, the batch limit of the per-slot memory stages
VALUE_PTS_TRANSPOSED, VALUE_ROPE, VALUE_DEC_TOKENS = 1, 2, 4   # include/spann3r_b200.h: flags of s3r_engine_value


def rope_cs_table(maxpos: int = ROPE_MAXPOS, base: float = 100.0, head_dim: int = 64) -> torch.Tensor:
    """(cos, sin) of pos * base^(-j/P), j < P = head_dim / 4: exactly the fp32 table the reference's PyTorch RoPE2D
    builds (croco/models/pos_embed.py:120-129 with D = head_dim / 2), as [maxpos, 16, 2].  The QKV epilogue rotates the
    pairs (j, j + 16) of each 32-wide half of a 64-wide head slot; for 48-wide heads (P = 12, the use_feat value encoder)
    entries 12..15 are (1, 0) and leave the zero padding pairs at zero."""
    D = head_dim // 2
    inv_freq = 1.0 / (base ** (torch.arange(0, D, 2).float() / D))
    t = torch.arange(maxpos, dtype=inv_freq.dtype)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    cs = torch.stack((freqs.cos(), freqs.sin()), dim=-1)
    if cs.shape[1] < 16:
        pad = torch.zeros(maxpos, 16 - cs.shape[1], 2)
        pad[..., 0] = 1.0
        cs = torch.cat((cs, pad), dim=1)
    return cs.contiguous()


def head_slots(heads: int = 16, head_dim: int = 48) -> torch.Tensor:
    """Column of every model feature c = h * head_dim + d in the 64-wide head slots the attention kernel runs on:
    head h, half s (y / x), in-half index i -> 64 h + 32 s + (i < P ? i : 16 + (i - P)), P = head_dim / 4.  Each half's
    RoPE pairs (i, i + P) land on the epilogue's pairs (j, j + 16); everything else in the slot is zero padding."""
    half, P = head_dim // 2, head_dim // 4
    c = torch.arange(heads * head_dim)
    h, d = c // head_dim, c % head_dim
    s, i = d // half, d % half
    return 64 * h + 32 * s + torch.where(i < P, i, 16 + (i - P))


def pad_qkv_rows(t: torch.Tensor, slots: torch.Tensor) -> torch.Tensor:
    """qkv weight [3 C, K] / bias [3 C] -> [3 * 64 heads, K] / [3 * 64 heads] with each role's rows at their slots, zeros
    elsewhere (any dtype / device)."""
    C, width = slots.numel(), 64 * ((int(slots.max()) + 64) // 64)
    out = t.new_zeros((3 * width,) + tuple(t.shape[1:]))
    idx = torch.cat([r * width + slots for r in range(3)]).to(t.device)
    return out.index_copy_(0, idx, t.reshape((3 * C,) + tuple(t.shape[1:])))


def pad_proj_cols(w: torch.Tensor, slots: torch.Tensor) -> torch.Tensor:
    """proj weight [N, C] -> [N, 64 * heads] reading the attention output's slot columns, zeros elsewhere."""
    width = 64 * ((int(slots.max()) + 64) // 64)
    return w.new_zeros(w.shape[0], width).index_copy_(1, slots.to(w.device), w)


def fold_layernorm(w: torch.Tensor, b: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor):
    """Fold the affine part of a LayerNorm into the Linear that consumes it (exact algebra, done in fp64):

        LN(x) W^T + b = rstd (x W'^T - mean rowsum(W')) + b',   W' = W diag(gamma),  b' = b + W beta

    so the GEMM can run on the raw residual stream x and its epilogue applies the per-row (mean, rstd)
    (include/spann3r_b200.h: s3r_gemm_desc.ln_stats / ln_cs).  Returns (W', b') as fp32."""
    w64, b64 = w.double(), b.double()
    return (w64 * gamma.double()[None, :]).float(), (b64 + w64 @ beta.double()).float()


def split_bf16_host_rowsum(w: torch.Tensor) -> torch.Tensor:
    """Row sums of hi + lo where hi = bf16(w), lo = bf16(w - hi): the same round-to-nearest-even split the device kernel
    (`s3r_split`) makes, evaluated on the host in fp64 -- the column-sum vector `cs` of a LayerNorm-folded Linear must be the
    sum of what the tensor core actually multiplies (tests/test_ops_gpu.py checks host == device planes)."""
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return (hi.double() + lo.double()).sum(dim=1).float()


def bf16_hi_rowsum(w: torch.Tensor) -> torch.Tensor:
    """Row sums of the hi plane bf16(w) alone, in fp64: the `cs_hi` of a LayerNorm-folded Linear, which a bf16-precision
    GEMM (one product, hi x hi) subtracts instead of `cs`."""
    return w.to(torch.bfloat16).double().sum(dim=1).float()


class PackedWeights:
    """Device-resident packed weights + the `s3r_model_w` pointer table."""

    def __init__(self, state_dict: dict, device="cuda", host_math: bool = True):
        """host_math=True (inference): the one-time layout arithmetic runs on the CPU copy of the checkpoint.
        host_math=False (training, where the weights change every optimizer step): the same arithmetic as torch ops on
        the device tensors, and `refresh()` re-packs IN PLACE (same buffers, so engines and cached tile plans stay valid)."""
        _lib.require_device()
        self.device = torch.device(device)
        self.host_math = host_math
        self._keep = []          # tensors the pointer table refers to, in creation order
        self._slot = None        # refresh(): index of the next tensor to overwrite (None = allocating)
        self.sd = state_dict
        self.struct = ModelW()
        self.param_bytes = 0
        self._build()
        del self.sd
        torch.cuda.synchronize(self.device)

    @torch.no_grad()
    def refresh(self, state_dict: dict):
        """Re-pack a changed state dict into the existing device buffers (same shapes, same order)."""
        self.sd = state_dict
        self._slot = 0
        self._build()
        assert self._slot == len(self._keep), "refresh walked a different number of tensors than the first pack"
        self._slot = None
        del self.sd

    # -- helpers ---------------------------------------------------------------------------------
    # Inference: all one-time layout work (stacking groups, permutes, LayerNorm folding, column sums) is host arithmetic
    # on the CPU copy of the checkpoint; the device sees one upload per tensor and the library's own split kernel.
    # (Round 1 did this with fp64 torch ops on the GPU: ~900 library launches before the first tensor-core kernel.)
    def _t(self, key):
        return self.sd[key].detach().to("cpu" if self.host_math else self.device, torch.float32)

    def _store(self, t: torch.Tensor) -> torch.Tensor:
        """Keep `t` alive on the device (first pack) or copy it into the buffer made then (refresh)."""
        if self._slot is None:
            t = t.contiguous().to(self.device)
            self._keep.append(t)
            return t
        dst = self._keep[self._slot]
        self._slot += 1
        dst.copy_(t.reshape(dst.shape))
        return dst

    def _f32(self, t: torch.Tensor):
        t = self._store(t)
        if self._slot is None:
            self.param_bytes += t.numel() * 4
        return t.data_ptr()

    def _planes(self, w2d: torch.Tensor) -> Planes:
        p = Planes()
        if self._slot is None:
            hi, lo = _lib.split(w2d.contiguous().to(self.device))
            self._keep += [hi, lo]
            self.param_bytes += hi.numel() * 4
        else:
            hi, lo = self._keep[self._slot], self._keep[self._slot + 1]
            self._slot += 2
            _lib.split(w2d.contiguous().to(self.device), out=(hi, lo))
        p.hi, p.lo = hi.data_ptr(), lo.data_ptr()
        return p

    def _lin(self, weights, biases=None) -> Lin:
        """weights: list of 2-D [N, K] tensors (one per group), stacked along N."""
        l = Lin()
        l.w = self._planes(torch.cat([w.reshape(w.shape[0], -1) for w in weights], dim=0))
        if biases is not None:
            l.b = self._f32(torch.cat([b.reshape(-1) for b in biases], dim=0))
        return l

    def _ln(self, names) -> LN:
        n = LN()
        n.w = self._f32(torch.stack([self._t(k + ".weight") for k in names]))
        n.b = self._f32(torch.stack([self._t(k + ".bias") for k in names]))
        return n

    def _linear(self, names, slots=None) -> Lin:
        """slots: read the input through the 64-wide head slots (`pad_proj_cols`) -- proj of the use_feat value blocks."""
        ws = [self._t(k + ".weight") for k in names]
        if slots is not None:
            ws = [pad_proj_cols(w, slots) for w in ws]
        return self._lin(ws, [self._t(k + ".bias") for k in names])

    def _linear_ln(self, names, ln_names, slots=None) -> Lin:
        """Linear that follows a LayerNorm, with the LayerNorm folded in (include/spann3r_b200.h, s3r_lin.cs):
        LN(x) W^T + b = rstd (x W'^T - mean cs) + b'  with  W' = W diag(gamma), b' = b + W beta, cs = rowsum(W').
        Exact algebra; cs is summed over the split-bf16 planes the tensor core will actually multiply, cs_hi over the hi
        plane alone (bf16 precision)."""
        ws, bs = [], []
        for k, ln in zip(names, ln_names):
            wf, bf = fold_layernorm(self._t(k + ".weight"), self._t(k + ".bias"), self._t(ln + ".weight"), self._t(ln + ".bias"))
            if slots is not None:   # qkv of the use_feat value blocks: rows into 64-wide head slots, zero weight / bias / cs
                wf, bf = pad_qkv_rows(wf, slots), pad_qkv_rows(bf, slots)
            ws.append(wf)
            bs.append(bf)
        l = self._lin(ws, bs)
        l.cs = self._f32(torch.cat([split_bf16_host_rowsum(w.reshape(w.shape[0], -1)) for w in ws], dim=0))
        l.cs_hi = self._f32(torch.cat([bf16_hi_rowsum(w.reshape(w.shape[0], -1)) for w in ws], dim=0))
        return l

    def _conv3(self, names, bias=True) -> Lin:   # [Cout, Cin, 3, 3] -> [Cout, tap, Cin]
        ws = [self._t(k + ".weight").permute(0, 2, 3, 1) for k in names]
        return self._lin(ws, [self._t(k + ".bias") for k in names] if bias else None)

    def _convT(self, names) -> Lin:              # [Cin, Cout, s, s] -> rows (i, j, co), cols ci
        ws = [self._t(k + ".weight").permute(2, 3, 1, 0) for k in names]
        return self._lin([w.reshape(-1, w.shape[-1]) for w in ws], [self._t(k + ".bias") for k in names])

    def _block(self, prefix, slots=None) -> BlockW:
        b = BlockW()
        b.norm1 = self._ln([prefix + ".norm1"])
        b.qkv = self._linear_ln([prefix + ".attn.qkv"], [prefix + ".norm1"], slots)
        b.proj = self._linear([prefix + ".attn.proj"], slots)
        b.norm2 = self._ln([prefix + ".norm2"])
        b.fc1 = self._linear_ln([prefix + ".mlp.fc1"], [prefix + ".norm2"])
        b.fc2 = self._linear([prefix + ".mlp.fc2"])
        return b

    def _decblock(self, l) -> DecBlockW:
        ps = [f"dust3r.dec_blocks.{l}", f"dust3r.dec_blocks2.{l}"]
        d = DecBlockW()
        d.norm1 = self._ln([p + ".norm1" for p in ps])
        # one launch per layer for the self-attention qkv AND the cross-attention k, v projections (the latter read the
        # other stream's layer input, norm_y folded): per group [attn.qkv; cross_attn.projk; cross_attn.projv]
        d.qkv = self._linear_ln([p + s for p in ps for s in (".attn.qkv", ".cross_attn.projk", ".cross_attn.projv")],
                                [p + s for p in ps for s in (".norm1", ".norm_y", ".norm_y")])
        d.proj = self._linear([p + ".attn.proj" for p in ps])
        d.norm_y = self._ln([p + ".norm_y" for p in ps])
        d.norm2 = self._ln([p + ".norm2" for p in ps])
        d.q = self._linear_ln([p + ".cross_attn.projq" for p in ps], [p + ".norm2" for p in ps])
        d.cproj = self._linear([p + ".cross_attn.proj" for p in ps])
        d.norm3 = self._ln([p + ".norm3" for p in ps])
        d.fc1 = self._linear_ln([p + ".mlp.fc1" for p in ps], [p + ".norm3" for p in ps])
        d.fc2 = self._linear([p + ".mlp.fc2" for p in ps])
        return d

    def _build(self):
        s = self.struct
        s.patch_embed = self._linear(["dust3r.patch_embed.proj"])
        for i in range(24):
            s.enc[i] = self._block(f"dust3r.enc_blocks.{i}")
        s.enc_norm = self._ln(["dust3r.enc_norm"])
        s.decoder_embed = self._linear(["dust3r.decoder_embed"])
        for i in range(12):
            s.dec[i] = self._decblock(i)
        s.dec_norm = self._ln(["dust3r.dec_norm"])
        s.key_fc1 = self._linear(["attn_head_1.0", "attn_head_2.0"])
        s.key_fc2 = self._linear(["attn_head_1.2", "attn_head_2.2"])
        hp = ["dust3r.downstream_head1.dpt", "dust3r.downstream_head2.dpt"]
        d = s.dpt
        d.act1_conv = self._linear([p + ".act_postprocess.0.0" for p in hp])
        d.act1_up = self._convT([p + ".act_postprocess.0.1" for p in hp])
        d.act2_conv = self._linear([p + ".act_postprocess.1.0" for p in hp])
        d.act2_up = self._convT([p + ".act_postprocess.1.1" for p in hp])
        d.act3_conv = self._linear([p + ".act_postprocess.2.0" for p in hp])
        d.act4_conv = self._linear([p + ".act_postprocess.3.0" for p in hp])
        d.act4_down = self._conv3([p + ".act_postprocess.3.1" for p in hp])
        for i in range(4):
            d.layer_rn[i] = self._conv3([p + f".scratch.layer_rn.{i}" for p in hp], bias=False)
            rn = [p + f".scratch.refinenet{i + 1}" for p in hp]
            f = d.refine[i]
            if i < 3:   # refinenet4.resConfUnit1 exists in the checkpoint but is never used (dpt_block.py:196)
                f.rcu1.conv1 = self._conv3([p + ".resConfUnit1.conv1" for p in rn])
                f.rcu1.conv2 = self._conv3([p + ".resConfUnit1.conv2" for p in rn])
            f.rcu2.conv1 = self._conv3([p + ".resConfUnit2.conv1" for p in rn])
            f.rcu2.conv2 = self._conv3([p + ".resConfUnit2.conv2" for p in rn])
            f.out_conv = self._linear([p + ".out_conv" for p in rn])
        d.head0 = self._conv3([p + ".head.0" for p in hp])
        d.head2 = self._conv3([p + ".head.2" for p in hp])
        d.head4_w = self._f32(torch.stack([self._t(p + ".head.4.weight").reshape(4, 128) for p in hp]))
        d.head4_b = self._f32(torch.stack([self._t(p + ".head.4.bias") for p in hp]))
        # value encoder: 1024 wide (default), or 768 wide with 48-wide heads (use_feat; no pos_patch_embed), packed into
        # 64-wide head slots (include/spann3r_b200.h, s3r_model_w.value_dim)
        s.value_dim = self.value_dim = int(self.sd["value_norm.weight"].shape[0])
        slots = head_slots(16, self.value_dim // 16) if self.value_dim == 768 else None
        if slots is None:
            s.pos_patch_embed = self._linear(["pos_patch_embed.proj"])
        for i in range(6):
            s.val[i] = self._block(f"value_encoder.{i}", slots)
        s.value_norm = self._ln(["value_norm"])
        s.value_out = self._linear(["value_out"])
        s.norm_q, s.norm_k, s.norm_v = self._ln(["norm_q"]), self._ln(["norm_k"]), self._ln(["norm_v"])
        s.rope_cs = self._f32(rope_cs_table())
        s.rope_maxpos = ROPE_MAXPOS
        if slots is not None:
            s.rope_cs_v = self._f32(rope_cs_table(head_dim=self.value_dim // 16))


class MemoryBank:
    """Device buffers of one batch of sequences' spatial memory (s3r_bank)."""

    def __init__(self, batch: int, cap: int, device):
        cap = (cap + 31) // 32 * 32
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=device)  # noqa: E731
        self.kn_hi, self.kn_lo = z(batch, cap, 1024, dt=torch.bfloat16), z(batch, cap, 1024, dt=torch.bfloat16)
        self.vnt_hi, self.vnt_lo = z(batch, 1024, cap, dt=torch.bfloat16), z(batch, 1024, cap, dt=torch.bfloat16)
        self.k_raw, self.v_raw = z(batch, cap, 1024), z(batch, cap, 1024)
        self.attn, self.count = z(batch, cap), z(batch, cap)
        self.cap, self.len, self.batch = cap, 0, batch

    def struct(self) -> Bank:
        b = Bank()
        b.kn_hi, b.kn_lo = self.kn_hi.data_ptr(), self.kn_lo.data_ptr()
        b.vnt_hi, b.vnt_lo = self.vnt_hi.data_ptr(), self.vnt_lo.data_ptr()
        b.k_raw, b.v_raw = self.k_raw.data_ptr(), self.v_raw.data_ptr()
        b.attn, b.count = self.attn.data_ptr(), self.count.data_ptr()
        b.cap, b.len = self.cap, self.len
        return b

    def gather(self, idx: torch.Tensor):
        """Keep rows idx [B, k] (the prune of spann3r/model.py:193-200), in that order.  Pure data movement."""
        k = idx.shape[1]
        ie = idx.unsqueeze(-1).expand(-1, -1, 1024)
        for name in ("kn_hi", "kn_lo", "k_raw", "v_raw"):
            t = getattr(self, name)
            t[:, :k] = torch.gather(t[:, : self.len], 1, ie)
        it = idx.unsqueeze(1).expand(-1, 1024, -1)
        for name in ("vnt_hi", "vnt_lo"):
            t = getattr(self, name)
            t[:, :, :k] = torch.gather(t[:, :, : self.len], 2, it)
        for name in ("attn", "count"):
            t = getattr(self, name)
            t[:, :k] = torch.gather(t[:, : self.len], 1, idx)
        self.len = k

    # -- per-slot use (model.SlotMemory): slot b is batch item b with its own length -------------------------------
    def zero_slot_tail(self, b: int, start: int, end: int):
        """Zero rows / columns [start, end) of slot b, so that the region past the slot's length stays finite (the
        tail contract of the per-slot read, include/spann3r_b200.h)."""
        if end > start:
            for name in ("kn_hi", "kn_lo", "k_raw", "v_raw", "attn", "count"):
                getattr(self, name)[b, start:end] = 0
            for name in ("vnt_hi", "vnt_lo"):
                getattr(self, name)[b, :, start:end] = 0

    def gather_slot(self, b: int, idx: torch.Tensor, n: int):
        """Keep rows idx [k] of slot b (length n), in that order, and zero the tail [k, n) they leave behind."""
        k = idx.shape[0]
        ie = idx[:, None].expand(-1, 1024)
        for name in ("kn_hi", "kn_lo", "k_raw", "v_raw"):
            t = getattr(self, name)
            t[b, :k] = torch.gather(t[b, :n], 0, ie)
        for name in ("vnt_hi", "vnt_lo"):
            t = getattr(self, name)
            t[b, :, :k] = torch.gather(t[b, :, :n], 1, idx[None].expand(1024, -1))
        for name in ("attn", "count"):
            t = getattr(self, name)
            t[b, :k] = torch.gather(t[b, :n], 0, idx)
        self.zero_slot_tail(b, k, n)


PRECISIONS = {"fp32": 0, "bf16": 1}   # Spann3R(precision=...) -> s3r_engine_create_ex's GEMM precision


class Engine:
    def __init__(self, weights: PackedWeights, batch: int, height: int, width: int, max_images: int = 0,
                 precision: str = "fp32"):
        """precision "bf16": the GEMMs of encode / decode / keyheads / value multiply the hi planes only (one tensor-core
        product); everything else runs as in "fp32" (include/spann3r_b200.h, s3r_engine_create_ex)."""
        if precision not in PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, got {precision!r}")
        self.weights = weights   # keeps the packed tensors alive
        self.precision = precision
        self.B, self.H, self.W = batch, height, width
        self.N = (height // 16) * (width // 16)
        self.max_images = max(max_images, 2 * batch)
        self.device = weights.device
        L = _lib.lib()
        with torch.cuda.device(self.device):     # the engine allocates its workspace on the CURRENT device
            self._h = L.s3r_engine_create_ex(C.byref(weights.struct), batch, height, width, self.max_images,
                                             PRECISIONS[precision])
        if not self._h:
            raise _lib.S3RError("s3r_engine_create failed: " + L.s3r_last_error().decode())

    def _call(self, name, *args):
        """One engine stage on the engine's own device and that device's current stream (the library launches on the
        current device; the C side refuses a call made while another device is current)."""
        _lib.call(name, self.device, self._h, *args)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                _lib.lib().s3r_engine_destroy(h)
            except Exception:
                pass

    def _new(self, *shape):
        return torch.empty(*shape, dtype=torch.float32, device=self.device)

    @staticmethod
    def _chk(x, shape=None):
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous(), "fp32 contiguous CUDA tensor expected"
        if shape is not None:
            assert tuple(x.shape) == tuple(shape), (tuple(x.shape), tuple(shape))
        return x

    def encode(self, img: torch.Tensor) -> torch.Tensor:
        nimg = img.shape[0]
        self._chk(img, (nimg, 3, self.H, self.W))
        feat = self._new(nimg, self.N, 1024)
        self._call("s3r_engine_encode", _lib.ptr(img), nimg, _lib.ptr(feat))
        return feat

    def decode(self, f1, f2, want_all=False):
        self._chk(f1, (self.B, self.N, 1024)); self._chk(f2, (self.B, self.N, 1024))
        dec_all = self._new(12, 2, self.B, self.N, 768) if want_all else None
        self._call("s3r_engine_decode", _lib.ptr(f1), _lib.ptr(f2), _lib.ptr(dec_all))
        return dec_all

    def keyheads(self, feat1, feat2):
        self._chk(feat1, (self.B, self.N, 1024)); self._chk(feat2, (self.B, self.N, 1024))
        k1, k2 = self._new(self.B, self.N, 1024), self._new(self.B, self.N, 1024)
        self._call("s3r_engine_keyheads", _lib.ptr(feat1), _lib.ptr(feat2), _lib.ptr(k1), _lib.ptr(k2))
        return k1, k2

    def heads(self):
        pts = self._new(2, self.B, self.H, self.W, 3)
        conf = self._new(2, self.B, self.H, self.W)
        self._call("s3r_engine_heads", _lib.ptr(pts), _lib.ptr(conf))
        return pts, conf

    def value(self, pts3d, feat_k1, transposed: bool = False, rope: bool = False, tokens: bool = False):
        """pts3d: head 1's map in the head's own [B, H, W, 3] layout; transposed=True reads it as the [B, W, H, 3]
        landscape view the reference's head wrapper returns for portrait frames (S3R_VALUE_PTS_TRANSPOSED).
        tokens=True (use_feat weights, S3R_VALUE_DEC_TOKENS): the input is dec1[-1] [B, N, 768] instead, or None for the
        engine's own copy from the last `decode`."""
        if tokens:
            if pts3d is not None:
                self._chk(pts3d, (self.B, self.N, 768))
        else:
            self._chk(pts3d, (self.B, self.H, self.W, 3))
        self._chk(feat_k1, (self.B, self.N, 1024))
        out = self._new(self.B, self.N, 1024)
        flags = (VALUE_PTS_TRANSPOSED if transposed else 0) | (VALUE_ROPE if rope else 0) | (VALUE_DEC_TOKENS if tokens else 0)
        self._call("s3r_engine_value", _lib.ptr(pts3d), _lib.ptr(feat_k1), flags, _lib.ptr(out))
        return out

    def memory_read(self, bank: MemoryBank, feat, thresh: float, drop_p: float = 0.0, seed: int = 0):
        """drop_p > 0: the training-mode read (nn.Dropout(drop_p) on the attention weights, Philox mask of `seed`)."""
        self._chk(feat, (self.B, self.N, 1024))
        out = self._new(self.B, self.N, 1024)
        bs = bank.struct()
        if drop_p > 0.0:
            self._call("s3r_engine_memory_read_train", C.byref(bs), _lib.ptr(feat), float(thresh), float(drop_p),
                       int(seed) & 0xFFFFFFFFFFFFFFFF, _lib.ptr(out))
        else:
            self._call("s3r_engine_memory_read", C.byref(bs), _lib.ptr(feat), float(thresh), _lib.ptr(out))
        return out

    def memory_append(self, bank: MemoryBank, feat_k, feat_v):
        self._chk(feat_k, (self.B, self.N, 1024)); self._chk(feat_v, (self.B, self.N, 1024))
        bs = bank.struct()
        self._call("s3r_engine_memory_append", C.byref(bs), _lib.ptr(feat_k), _lib.ptr(feat_v))
        bank.len += self.N

    def check_sim(self, bank: MemoryBank, feat_k, wm: int) -> torch.Tensor:
        out = self._new(self.B, wm)
        bs = bank.struct()
        self._call("s3r_engine_check_sim", C.byref(bs), _lib.ptr(feat_k), wm, _lib.ptr(out))
        return out

    # -- per-slot memory stages (independent sequences, one per batch item) ------------------------------------
    def _slot_ints(self, vals):
        vals = [int(v) for v in vals]
        if len(vals) != self.B:
            raise ValueError(f"expected {self.B} per-slot values, got {len(vals)}")
        return (_i * self.B)(*vals)

    def memory_read_slots(self, bank: MemoryBank, lens, feat, thresh: float):
        """memory_read with slot b reading its first lens[b] tokens; a slot of length 0 returns its feat row unchanged."""
        self._chk(feat, (self.B, self.N, 1024))
        out = self._new(self.B, self.N, 1024)
        self._call("s3r_engine_memory_read_slots", C.byref(bank.struct()), self._slot_ints(lens),
                   _lib.ptr(feat), float(thresh), _lib.ptr(out))
        return out

    def memory_append_slots(self, bank: MemoryBank, lens, append, feat_k, feat_v):
        """Slot b with append[b] takes its N tokens at offset lens[b]; the caller tracks the lengths."""
        self._chk(feat_k, (self.B, self.N, 1024)); self._chk(feat_v, (self.B, self.N, 1024))
        self._call("s3r_engine_memory_append_slots", C.byref(bank.struct()), self._slot_ints(lens),
                   self._slot_ints(append), _lib.ptr(feat_k), _lib.ptr(feat_v))

    def check_sim_slots(self, bank: MemoryBank, lens, wm, feat_k) -> torch.Tensor:
        """[B, 8]: slot b's gate values against its last wm[b] frames ending at lens[b]; -inf past wm[b]."""
        self._chk(feat_k, (self.B, self.N, 1024))
        out = self._new(self.B, 8)
        self._call("s3r_engine_check_sim_slots", C.byref(bank.struct()), self._slot_ints(lens),
                   self._slot_ints(wm), _lib.ptr(feat_k), _lib.ptr(out))
        return out

    def take_flops(self) -> float:
        return float(_lib.lib().s3r_engine_take_flops(self._h))

    def _on(self):
        return torch.cuda.device(self.device)

    def profile(self, on: bool):
        _lib.lib().s3r_engine_profile(self._h, int(on))

    def profile_read(self) -> dict:
        out = (C.c_double * 6)()
        with self._on():
            _lib.check(_lib.lib().s3r_engine_profile_read(self._h, out), "profile_read")
        return dict(gemm_ms=out[0], gemm_flops=out[1], gemm_launches=int(out[2]), attn_ms=out[3], attn_flops=out[4],
                    attn_launches=int(out[5]))

    def profile_list(self, cap: int = 4096):
        """[(ms, flops, kind)] of the launches recorded since profile(True), in launch order (kind 0 split GEMM,
        1 attention, 2 one-product bf16 GEMM)."""
        ms, fl, kd = (C.c_double * cap)(), (C.c_double * cap)(), (C.c_int * cap)()
        with self._on():
            n = _lib.lib().s3r_engine_profile_list(self._h, ms, fl, kd, cap)
        if n < 0:
            _lib.check(n, "profile_list")
        return [(ms[i], fl[i], kd[i]) for i in range(min(n, cap))]

    def take_launches(self) -> int:
        return int(_lib.lib().s3r_engine_take_launches(self._h))
