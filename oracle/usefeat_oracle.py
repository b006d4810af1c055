"""ORACLE -- TEST INFRASTRUCTURE ONLY.  `Spann3R(use_feat=True)` on top of the primitives of `spann3r_oracle`.

With use_feat the reference's value encoder is six `Block(768, 16 heads)` -- heads 48 wide, attention scale 48^-0.5,
RoPE2D over 24-wide halves with mem_pos_enc -- plus `value_norm` (768) and `value_out` (768 -> 1024), and it is fed
dec1[-1] (dec_norm of head 1's last decoder layer) with the positions pos1 of the frame's own patch grid instead of the
pointmap (spann3r/model.py:225-242, 305-320).  Everything else is the default model's frame loop and offline mode, restated
here with that one call changed; `tests/test_use_feat_cpu.py` pins both to outputs of the real reference
(`tools/make_golden.py --only usefeat`).
"""
from __future__ import annotations

import torch

from . import spann3r_oracle as orc


def encode_cur_value(sd, dec_last, pos, mem_pos_enc=False):
    """spann3r/model.py:305-314 (use_feat=True): dec_last [B, N, 768], pos [B, N, 2] (y, x) -> cur_v [B, N, 1024]."""
    x = dec_last
    for i in range(6):
        x = orc.block(sd, f"value_encoder.{i}", x, pos, 16, use_rope=mem_pos_enc)
    x = orc.layernorm(sd, "value_norm", x, 1e-6)
    return orc.linear(sd, "value_out", x)


@torch.no_grad()
def forward(sd, frames, return_memory=False, trace=None, mem_pos_enc=False, **mem_kw):
    """Spann3R.forward (spann3r/model.py:473-539) of a use_feat model; the eval-mode branches unless mem_kw selects the
    training ones (attn_thresh=0, sim_thresh=1.0), as `spann3r_oracle.forward`."""
    sp_mem = orc.SpatialMemory(sd, **mem_kw)
    feat1 = feat2 = pos1 = pos2 = None
    feat_k2 = None
    preds, preds_all = None, []
    H, W = frames[0]["img"].shape[-2:]
    for i in range(len(frames) - 1):
        if feat1 is None:
            out, pos = orc.encode_image(sd, torch.cat((frames[i]["img"], frames[i + 1]["img"]), dim=0))
            feat1, feat2 = out.chunk(2, dim=0)
            pos1, pos2 = pos.chunk(2, dim=0)
        else:
            feat1, pos1 = feat2, pos2
            feat2, pos2 = orc.encode_image(sd, frames[i + 1]["img"])
        feat_fuse = sp_mem.memory_read(feat_k2, res=True) if feat_k2 is not None else feat1
        dec1, dec2 = orc.decoder(sd, feat_fuse, pos1, feat2, pos2)
        feat_k1 = orc.key_head(sd, 1, feat1, dec1[-1])
        feat_k2 = orc.key_head(sd, 2, feat2, dec2[-1])
        res1 = orc.downstream_head(sd, "dust3r.downstream_head1", dec1, H, W)
        res2 = orc.downstream_head(sd, "dust3r.downstream_head2", dec2, H, W)
        cur_v = encode_cur_value(sd, dec1[-1], pos1, mem_pos_enc)
        sp_mem.add_mem_check(feat_k1, cur_v + feat_k1)
        if trace is not None:
            trace.append(dict(feat1=feat1, feat_fuse=feat_fuse, dec1=dec1, pos1=pos1, feat_k1=feat_k1, feat_k2=feat_k2,
                              cur_v=cur_v))
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


@torch.no_grad()
def offline_reconstruction(sd, frames, graph, mem_pos_enc=False, **mem_kw):
    """Spann3R.offline_reconstruction (spann3r/model.py:394-471, find_next_best_view :359-392) of a use_feat model."""
    n_frames = len(frames)
    idx_todo = list(range(n_frames))
    H, W = frames[0]["img"].shape[-2:]
    sp_mem = orc.SpatialMemory(sd, **mem_kw)
    p0, p1 = orc.find_initial_pair(graph, n_frames)
    idx_used = [p0, p1]
    idx_todo.remove(p0)
    idx_todo.remove(p1)
    out, pos = orc.encode_image(sd, torch.cat((frames[p0]["img"], frames[p1]["img"]), dim=0))
    feat1, feat2 = out.chunk(2, dim=0)
    pos1, pos2 = pos.chunk(2, dim=0)
    dec1, dec2 = orc.decoder(sd, feat1, pos1, feat2, pos2)
    res1 = orc.downstream_head(sd, "dust3r.downstream_head1", dec1, H, W)
    res2 = orc.downstream_head(sd, "dust3r.downstream_head2", dec2, H, W)
    feat_k2, preds, preds_all = None, None, []
    while True:
        if feat_k2 is not None:
            feat1, pos1 = feat2, pos2
            feat_fuse = sp_mem.memory_read(feat_k2, res=True)
            best_conf, best = 0.0, None
            for i in idx_todo:
                f2, ps2 = orc.encode_image(sd, frames[i]["img"])
                d1, d2 = orc.decoder(sd, feat_fuse, pos1, f2, ps2)
                r1 = orc.downstream_head(sd, "dust3r.downstream_head1", d1, H, W)
                r2 = orc.downstream_head(sd, "dust3r.downstream_head2", d2, H, W)
                total = orc.conf_score(r1["conf"]) + orc.conf_score(r2["conf"])
                if total > best_conf:
                    best_conf, best = total, (i, d1, d2, r1, r2, f2, ps2)
            id_n, dec1, dec2, res1, res2, feat2, pos2 = best
            idx_todo.remove(id_n)
            idx_used.append(id_n)
        feat_k1 = orc.key_head(sd, 1, feat1, dec1[-1])
        feat_k2 = orc.key_head(sd, 2, feat2, dec2[-1])
        cur_v = encode_cur_value(sd, dec1[-1], pos1, mem_pos_enc)
        sp_mem.add_mem_check(feat_k1, cur_v + feat_k1)
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
