"""PyTorch RECOMPUTE of the four engine stages -- used ONLY by the backward pass of training mode (`train.py`).

This is NOT a forward path: `Spann3R.forward` always runs the sm_90a kernels (training mode included), and nothing here
is reachable from eval-mode code.  The native dgrad / wgrad kernels of SURVEY.md §8f rank 1 are not written yet; until
they are, `torch.autograd.Function.backward` of every stage re-evaluates that stage with these differentiable
restatements (activation checkpointing at stage granularity) and lets PyTorch autograd produce the gradients -- labelled
"PyTorch recompute backward" wherever a number from it is reported.  Each function cites the reference lines it restates
(paths relative to the reference root); `tests/test_train_cpu.py` pins them to the oracle on the CPU.

P: dict parameter name (the reference's state-dict keys) -> tensor.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import _native_linear

ENC_HEADS, DEC_HEADS, VAL_HEADS = 16, 12, 16


def _lin(P, n, x):
    # F.linear + PyTorch autograd by default; with the switch on, forward / dgrad / wgrad on the wgmma GEMM engine
    return _native_linear.linear(x, P[n + ".weight"], P[n + ".bias"])


def _ln(P, n, x, eps):
    return F.layer_norm(x, x.shape[-1:], P[n + ".weight"], P[n + ".bias"], eps)


def _rope_cs(gh: int, gw: int, device, base: float = 100.0):
    """cos / sin of pos * base^(-j/16), j < 16 (croco/models/pos_embed.py:120-129, D = 32), for the row-major patch grid:
    returns (cos_y, sin_y, cos_x, sin_x), each [gh*gw, 16]."""
    inv = 1.0 / (base ** (torch.arange(0, 32, 2, device=device).float() / 32))
    ys = torch.arange(gh, device=device).float().repeat_interleave(gw)
    xs = torch.arange(gw, device=device).float().repeat(gh)
    fy, fx = ys[:, None] * inv[None], xs[:, None] * inv[None]
    return fy.cos(), fy.sin(), fx.cos(), fx.sin()


def _rope(t, cs):
    """2-D RoPE on [B, heads, N, 64] (pos_embed.py:131-159): the head dim is [y half | x half], each half 16 (u, v) pairs
    (j, j + 16) rotated by its position's angle."""
    cy, sy, cx, sx = cs
    y, x = t[..., :32], t[..., 32:]

    def rot(h, c, s):
        u, v = h[..., :16], h[..., 16:]
        return torch.cat((u * c - v * s, v * c + u * s), dim=-1)
    return torch.cat((rot(y, cy, sy), rot(x, cx, sx)), dim=-1)


def _sdpa(q, k, v):
    """softmax(q k^T / sqrt(dh)) v in plain fp32 ops (not F.scaled_dot_product_attention: which fused backend it picks, and that
    backend's internal precision, is PyTorch's choice; the backward of a path held to 1e-3 should not depend on it)."""
    a = torch.softmax((q @ k.transpose(-2, -1)) * (q.shape[-1] ** -0.5), dim=-1)
    return a @ v


def _self_attn(P, n, x, heads, cs):
    """croco/models/blocks.py:94-112."""
    B, N, C = x.shape
    qkv = _lin(P, n + ".qkv", x).view(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if cs is not None:
        q, k = _rope(q, cs), _rope(k, cs)
    o = _sdpa(q, k, v)
    return _lin(P, n + ".proj", o.transpose(1, 2).reshape(B, N, C))


def _cross_attn(P, n, xq, y, heads, cs):
    """croco/models/blocks.py:149-169."""
    B, N, C = xq.shape
    dh = C // heads
    q = _lin(P, n + ".projq", xq).view(B, N, heads, dh).transpose(1, 2)
    k = _lin(P, n + ".projk", y).view(B, -1, heads, dh).transpose(1, 2)
    v = _lin(P, n + ".projv", y).view(B, -1, heads, dh).transpose(1, 2)
    o = _sdpa(_rope(q, cs), _rope(k, cs), v)
    return _lin(P, n + ".proj", o.transpose(1, 2).reshape(B, N, C))


def _mlp(P, n, x):
    return _lin(P, n + ".fc2", F.gelu(_lin(P, n + ".fc1", x)))


def _block(P, n, x, heads, cs):
    """croco/models/blocks.py:127-130 (LayerNorm eps 1e-6)."""
    x = x + _self_attn(P, n + ".attn", _ln(P, n + ".norm1", x, 1e-6), heads, cs)
    return x + _mlp(P, n + ".mlp", _ln(P, n + ".norm2", x, 1e-6))


def _dec_block(P, n, x, y, cs):
    """croco/models/blocks.py:186-191."""
    x = x + _self_attn(P, n + ".attn", _ln(P, n + ".norm1", x, 1e-6), DEC_HEADS, cs)
    y_ = _ln(P, n + ".norm_y", y, 1e-6)
    x = x + _cross_attn(P, n + ".cross_attn", _ln(P, n + ".norm2", x, 1e-6), y_, DEC_HEADS, cs)
    return x + _mlp(P, n + ".mlp", _ln(P, n + ".norm3", x, 1e-6))


# ------------------------------------------------------------------------------------------------ stages
def encode(P, img):
    """dust3r/model.py:131-154 + dust3r/patch_embed.py:19-29: img [n, 3, H, W] -> [n, N, 1024]."""
    x = F.conv2d(img, P["dust3r.patch_embed.proj.weight"], P["dust3r.patch_embed.proj.bias"], stride=16)
    gh, gw = x.shape[-2:]
    cs = _rope_cs(gh, gw, img.device)
    x = x.flatten(2).transpose(1, 2)
    for i in range(24):
        x = _block(P, f"dust3r.enc_blocks.{i}", x, ENC_HEADS, cs)
    return _ln(P, "dust3r.enc_norm", x, 1e-6)


def memory_read(P, feat, mem_k, mem_v, keep_scale=None):
    """spann3r/model.py:145-183 in TRAINING mode (attn_thresh = 0: no cut, no renormalisation; `keep_scale` = the
    dropout mask times 1 / (1 - p), or None): out = dropout(softmax(LN_q(feat) LN_k(K)^T / 32)) LN_v(V) + feat."""
    q = _ln(P, "norm_q", feat, 1e-5)
    k = _ln(P, "norm_k", mem_k, 1e-5)
    attn = torch.softmax(torch.einsum("bpc,bxc->bpx", q, k) / 32.0, dim=-1)
    if keep_scale is not None:
        attn = attn * keep_scale
    return torch.einsum("bpx,bxc->bpc", attn, _ln(P, "norm_v", mem_v, 1e-5)) + feat


def _rcu(P, n, x):
    """ResidualConvUnit_custom, croco/models/dpt_block.py:121-142."""
    o = F.conv2d(F.relu(x), P[n + ".conv1.weight"], P[n + ".conv1.bias"], padding=1)
    o = F.conv2d(F.relu(o), P[n + ".conv2.weight"], P[n + ".conv2.bias"], padding=1)
    return o + x


def _fusion(P, n, path, skip=None):
    """FeatureFusionBlock_custom, dpt_block.py:189-218 (bilinear x2, align_corners=True, then out_conv)."""
    o = path if skip is None else path + _rcu(P, n + ".resConfUnit1", skip)
    o = _rcu(P, n + ".resConfUnit2", o)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    return F.conv2d(o, P[n + ".out_conv.weight"], P[n + ".out_conv.bias"])


def _dpt(P, p, hooks, gh, gw):
    """DPTOutputAdapter_fix.forward, dust3r/heads/dpt_head.py:34-65 + postprocess.py:10-58 -> (pts3d [B,H,W,3], conf)."""
    L = [t.view(t.shape[0], gh, gw, t.shape[-1]).permute(0, 3, 1, 2) for t in hooks]
    ap = p + ".act_postprocess"
    l0 = F.conv_transpose2d(F.conv2d(L[0], P[ap + ".0.0.weight"], P[ap + ".0.0.bias"]), P[ap + ".0.1.weight"],
                            P[ap + ".0.1.bias"], stride=4)
    l1 = F.conv_transpose2d(F.conv2d(L[1], P[ap + ".1.0.weight"], P[ap + ".1.0.bias"]), P[ap + ".1.1.weight"],
                            P[ap + ".1.1.bias"], stride=2)
    l2 = F.conv2d(L[2], P[ap + ".2.0.weight"], P[ap + ".2.0.bias"])
    l3 = F.conv2d(F.conv2d(L[3], P[ap + ".3.0.weight"], P[ap + ".3.0.bias"]), P[ap + ".3.1.weight"], P[ap + ".3.1.bias"],
                  stride=2, padding=1)
    ls = [F.conv2d(t, P[p + f".scratch.layer_rn.{i}.weight"], None, padding=1) for i, t in enumerate((l0, l1, l2, l3))]
    path = _fusion(P, p + ".scratch.refinenet4", ls[3])[:, :, : ls[2].shape[2], : ls[2].shape[3]]
    path = _fusion(P, p + ".scratch.refinenet3", path, ls[2])
    path = _fusion(P, p + ".scratch.refinenet2", path, ls[1])
    path = _fusion(P, p + ".scratch.refinenet1", path, ls[0])
    o = F.conv2d(path, P[p + ".head.0.weight"], P[p + ".head.0.bias"], padding=1)
    o = F.interpolate(o, scale_factor=2, mode="bilinear", align_corners=True)
    o = F.relu(F.conv2d(o, P[p + ".head.2.weight"], P[p + ".head.2.bias"], padding=1))
    o = F.conv2d(o, P[p + ".head.4.weight"], P[p + ".head.4.bias"]).permute(0, 2, 3, 1)
    xyz = o[..., :3]
    d = xyz.norm(dim=-1, keepdim=True)
    return xyz / d.clip(min=1e-8) * torch.expm1(d), 1 + o[..., 3].exp()


def step(P, feat_fuse, feat1, feat2, H, W):
    """One frame step between the memory read and the memory write: the twin decoder (dust3r/model.py:186-205), the two
    key heads (spann3r/model.py:299-303) and the two DPT heads.  Returns (feat_k1, feat_k2, pts [2,B,H,W,3], conf)."""
    gh, gw = H // 16, W // 16
    cs = _rope_cs(gh, gw, feat1.device)
    a, b = _lin(P, "dust3r.decoder_embed", feat_fuse), _lin(P, "dust3r.decoder_embed", feat2)
    h1, h2 = [feat_fuse], [feat2]
    for i in range(12):
        a, b = (_dec_block(P, f"dust3r.dec_blocks.{i}", a, b, cs), _dec_block(P, f"dust3r.dec_blocks2.{i}", b, a, cs))
        if i in (5, 8):
            h1.append(a)
            h2.append(b)
    a, b = _ln(P, "dust3r.dec_norm", a, 1e-6), _ln(P, "dust3r.dec_norm", b, 1e-6)
    h1.append(a)
    h2.append(b)

    def key_head(n, feat, d):
        return _lin(P, n + ".2", F.gelu(_lin(P, n + ".0", torch.cat((feat, d), dim=-1))))
    k1, k2 = key_head("attn_head_1", feat1, a), key_head("attn_head_2", feat2, b)
    p1, c1 = _dpt(P, "dust3r.downstream_head1.dpt", h1, gh, gw)
    p2, c2 = _dpt(P, "dust3r.downstream_head2.dpt", h2, gh, gw)
    return k1, k2, torch.stack((p1, p2)), torch.stack((c1, c2))


def value(P, pts3d, feat_k1, rope: bool):
    """spann3r/model.py:305-320 encode_cur_value (+ `cur_v + feat_k1`, :519-521): pts3d [B, H, W, 3] -> [B, N, 1024]."""
    x = F.conv2d(pts3d.permute(0, 3, 1, 2), P["pos_patch_embed.proj.weight"], P["pos_patch_embed.proj.bias"], stride=16)
    gh, gw = x.shape[-2:]
    cs = _rope_cs(gh, gw, x.device) if rope else None
    x = x.flatten(2).transpose(1, 2)
    for i in range(6):
        x = _block(P, f"value_encoder.{i}", x, VAL_HEADS, cs)
    return _lin(P, "value_out", _ln(P, "value_norm", x, 1e-6)) + feat_k1
