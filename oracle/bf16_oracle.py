"""ORACLE -- TEST INFRASTRUCTURE ONLY.  Emulation of `Spann3R(precision="bf16")` in fp64.

The bf16 precision changes one thing (include/spann3r_b200.h, s3r_engine_create_ex): every GEMM of encode, decode,
keyheads and value multiplies the bf16 hi planes of its operands once and accumulates in fp32.  This module restates those
four stages in fp64 and rounds to bf16 exactly where the engine does, so that the GPU result can be held to the format's own
error rather than to the fp32-grade bars:
  - the A operand of each GEMM is bf16 of the fp32 tensor its planes are written from: the raw residual stream for a folded
    LayerNorm, GELU(fc1) for fc2, the attention output for proj, the im2col'd pixels (points) for the patch embeddings,
    cat(feat, dec_norm) for the key heads' fc1, value_norm's output for value_out;
  - the weights are bf16 of the packed fp32 weights; a LayerNorm-folded Linear uses W' = W diag(gamma) and b' = b + W beta
    from `spann3r_b200.engine.fold_layernorm` and applies  rstd (acc - mean rowsum(bf16(W'))) + b'  (the cs_hi vector);
  - everything else -- LayerNorm statistics, RoPE, the attention cores, GELU, residual adds, dec_norm, the DPT heads and the
    spatial memory -- is `oracle.spann3r_oracle`'s fp64 arithmetic, unchanged.

`Emu(sd, rounding=False)` drops every rounding (and folds the LayerNorms in fp64): it is then the same function as
`spann3r_oracle` up to fp64 reassociation, which pins the restatement itself (tests/test_bf16_cpu.py).  With rounding on, its
distance to the fp64 truth is what the bf16 format costs.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import spann3r_oracle as orc


def bf16(x: torch.Tensor) -> torch.Tensor:
    """bf16 (round to nearest even) of the fp32 value of x, returned in x's dtype: the hi plane the engine's producers
    write from an fp32 tensor."""
    return x.float().to(torch.bfloat16).to(x.dtype)


class Emu:
    def __init__(self, sd, rounding: bool = True):
        self.sd, self.rounding = sd, rounding
        self._fold = {}

    def r(self, x):
        return bf16(x) if self.rounding else x

    # -- GEMMs ---------------------------------------------------------------------------------------
    def linear(self, name, x):
        """Plain Linear: A = x (fp32 tensor the planes are written from), B = the packed weight."""
        sd = self.sd
        return F.linear(self.r(x), self.r(sd[name + ".weight"]), sd.get(name + ".bias"))

    def _folded(self, name, ln):
        key = (name, ln)
        if key not in self._fold:
            sd = self.sd
            w, b, g, be = sd[name + ".weight"], sd[name + ".bias"], sd[ln + ".weight"], sd[ln + ".bias"]
            if self.rounding:     # what PackedWeights packs: the fold in fp64, stored as fp32
                from spann3r_b200.engine import fold_layernorm
                wf, bf = fold_layernorm(w, b, g, be)
                wf, bf = bf16(wf.to(w.dtype)), bf.to(w.dtype)
            else:
                wf, bf = w.double() * g.double()[None, :], b.double() + w.double() @ be.double()
                wf, bf = wf.to(w.dtype), bf.to(w.dtype)
            self._fold[key] = (wf, bf, wf.sum(dim=1))
        return self._fold[key]

    def linear_ln(self, name, ln, x, eps=1e-6):
        """LN(x) W^T + b with the LayerNorm folded: A = the raw x, rstd (x W'^T - mean cs) + b'."""
        wf, bf, cs = self._folded(name, ln)
        mean = x.mean(dim=-1, keepdim=True)
        rstd = torch.rsqrt(x.var(dim=-1, unbiased=False, keepdim=True) + eps)
        return rstd * (F.linear(self.r(x), wf) - mean * cs) + bf

    def patch_embed(self, name, img):
        """Conv2d(k = s = 16) = GEMM over the im2col'd patches; rounding each pixel is rounding each im2col element."""
        sd = self.sd
        x = F.conv2d(self.r(img), self.r(sd[name + ".proj.weight"]), sd[name + ".proj.bias"], stride=16)
        B, _, gh, gw = x.shape
        pos = torch.cartesian_prod(torch.arange(gh, device=img.device), torch.arange(gw, device=img.device))
        return x.flatten(2).transpose(1, 2), pos.view(1, gh * gw, 2).expand(B, -1, 2).clone()

    # -- blocks (croco/models/blocks.py:94-130, 149-191) ----------------------------------------------
    @staticmethod
    def _core(q, k, v, scale):
        return ((q @ k.transpose(-2, -1)) * scale).softmax(dim=-1) @ v

    def attention(self, name, ln, x, xpos, heads, use_rope=True):
        B, N, C = x.shape
        qkv = self.linear_ln(name + ".qkv", ln, x).reshape(B, N, 3, heads, C // heads).transpose(1, 3)
        q, k, v = [qkv[:, :, i] for i in range(3)]
        if use_rope:
            q, k = orc.rope2d(q, xpos), orc.rope2d(k, xpos)
        o = self._core(q, k, v, (C // heads) ** -0.5).transpose(1, 2).reshape(B, N, C)
        return self.linear(name + ".proj", o)

    def mlp(self, name, ln, x):
        return self.linear(name + ".fc2", F.gelu(self.linear_ln(name + ".fc1", ln, x)))

    def block(self, name, x, xpos, heads, use_rope=True):
        x = x + self.attention(name + ".attn", name + ".norm1", x, xpos, heads, use_rope)
        return x + self.mlp(name + ".mlp", name + ".norm2", x)

    def decoder_block(self, name, x, y, xpos, ypos, heads=orc.DEC_HEADS):
        x = x + self.attention(name + ".attn", name + ".norm1", x, xpos, heads)
        B, Nq, C = x.shape
        Nk, dh, ca = y.shape[1], C // heads, name + ".cross_attn"
        q = self.linear_ln(ca + ".projq", name + ".norm2", x).reshape(B, Nq, heads, dh).permute(0, 2, 1, 3)
        k = self.linear_ln(ca + ".projk", name + ".norm_y", y).reshape(B, Nk, heads, dh).permute(0, 2, 1, 3)
        v = self.linear_ln(ca + ".projv", name + ".norm_y", y).reshape(B, Nk, heads, dh).permute(0, 2, 1, 3)
        o = self._core(orc.rope2d(q, xpos), orc.rope2d(k, ypos), v, dh ** -0.5).transpose(1, 2).reshape(B, Nq, C)
        x = x + self.linear(ca + ".proj", o)
        return x + self.mlp(name + ".mlp", name + ".norm3", x)

    # -- the four stages ---------------------------------------------------------------------------
    def encode_image(self, img):
        """dust3r/model.py:131-154 -> (feat, pos)."""
        x, pos = self.patch_embed("dust3r.patch_embed", img)
        for i in range(orc.ENC_DEPTH):
            x = self.block(f"dust3r.enc_blocks.{i}", x, pos, orc.ENC_HEADS)
        return orc.layernorm(self.sd, "dust3r.enc_norm", x, 1e-6), pos

    def decoder(self, f1, pos1, f2, pos2):
        """dust3r/model.py:186-205 -> (dec1, dec2), 13 tensors each."""
        out = [(f1, f2)]
        a, b = self.linear("dust3r.decoder_embed", f1), self.linear("dust3r.decoder_embed", f2)
        for i in range(orc.DEC_DEPTH):
            a, b = (self.decoder_block(f"dust3r.dec_blocks.{i}", a, b, pos1, pos2),
                    self.decoder_block(f"dust3r.dec_blocks2.{i}", b, a, pos2, pos1))
            out.append((a, b))
        out[-1] = tuple(orc.layernorm(self.sd, "dust3r.dec_norm", t, 1e-6) for t in out[-1])
        return list(zip(*out))

    def key_head(self, num, feat, dec_last):
        """spann3r/model.py:299-303."""
        x = F.gelu(self.linear(f"attn_head_{num}.0", torch.cat((feat, dec_last), dim=-1)))
        return self.linear(f"attn_head_{num}.2", x)

    def encode_cur_value(self, pts3d, mem_pos_enc=False):
        """spann3r/model.py:305-320, default value encoder: pts3d [B, h, w, 3] (the landscape view)."""
        x, pos = self.patch_embed("pos_patch_embed", pts3d.permute(0, 3, 1, 2))
        return self._value_tail(x, pos, 16, mem_pos_enc)

    def encode_cur_value_usefeat(self, dec_last, pos, mem_pos_enc=False):
        """use_feat value encoder on dec1[-1] (16 heads of 48; the engine's zero-padded 64-wide slots round to the same)."""
        return self._value_tail(dec_last, pos, 16, mem_pos_enc)

    def _value_tail(self, x, pos, heads, mem_pos_enc):
        for i in range(6):
            x = self.block(f"value_encoder.{i}", x, pos, heads, use_rope=mem_pos_enc)
        return self.linear("value_out", orc.layernorm(self.sd, "value_norm", x, 1e-6))


@torch.no_grad()
def forward(sd, frames, rounding=True, use_feat=False, mem_pos_enc=False, **mem_kw):
    """Spann3R.forward in eval mode (spann3r/model.py:473-539) with the emulated stages: `spann3r_oracle.forward` with
    encode, decode, the key heads and the value encoder replaced, the DPT heads and the memory unchanged."""
    e = Emu(sd, rounding)
    sp_mem = orc.SpatialMemory(sd, **mem_kw)
    feat1 = feat2 = pos1 = pos2 = feat_k2 = None
    preds, preds_all = None, []
    H, W = frames[0]["img"].shape[-2:]
    for i in range(len(frames) - 1):
        if feat1 is None:
            out, pos = e.encode_image(torch.cat((frames[i]["img"], frames[i + 1]["img"]), dim=0))
            feat1, feat2 = out.chunk(2, dim=0)
            pos1, pos2 = pos.chunk(2, dim=0)
        else:
            feat1, pos1 = feat2, pos2
            feat2, pos2 = e.encode_image(frames[i + 1]["img"])
        feat_fuse = sp_mem.memory_read(feat_k2, res=True) if feat_k2 is not None else feat1
        dec1, dec2 = e.decoder(feat_fuse, pos1, feat2, pos2)
        feat_k1, feat_k2 = e.key_head(1, feat1, dec1[-1]), e.key_head(2, feat2, dec2[-1])
        res1 = orc.downstream_head(sd, "dust3r.downstream_head1", dec1, H, W)
        res2 = orc.downstream_head(sd, "dust3r.downstream_head2", dec2, H, W)
        if use_feat:
            cur_v = e.encode_cur_value_usefeat(dec1[-1], pos1, mem_pos_enc)
        else:
            cur_v = e.encode_cur_value(res1["pts3d"], mem_pos_enc)
        sp_mem.add_mem_check(feat_k1, cur_v + feat_k1)
        res2["pts3d_in_other_view"] = res2.pop("pts3d")
        if preds is None:
            preds, preds_all = [res1], [(res1, res2)]
        else:
            res1["pts3d_in_other_view"] = res1.pop("pts3d")
            preds.append(res1)
            preds_all.append((res1, res2))
    preds.append(res2)
    return preds, preds_all
