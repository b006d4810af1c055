"""Spann3R's training and test criteria on the GPU (spann3r/loss.py:129-369 of the reference, with dust3r's L21).

    from spann3r_b200.loss import *
    criterion = eval("ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)")   # training.py:36-38
    loss, details, factor_loss = criterion.compute_frame_loss(views, preds_all)
    (loss + factor_loss).backward()

The reference's names, constructor arguments and return structures, computed by the kernels of csrc/loss.cu: one
forward call (no host synchronisation) and, for `compute_frame_loss`, one device-to-host copy of the logged details.
`loss` and `factor_loss` come from one autograd Function whose backward is one native call; it differentiates the norm
factor of the prediction (as the reference does) and treats the medians of the shift / scale variants as constants
(they are `no_grad` in the reference).

Inputs: `gts` = the views, each with CUDA `pts3d [B,H,W,3]` fp32, `valid_mask [B,H,W]` bool and `camera_pose [B,4,4]`
fp32; `preds` = `preds_all` as `Spann3R.forward` returns it (eval or training mode).

Differences from the reference (INTEGRATION.md, "Training and test criteria"):
  * with norm_mode=False the shift / scale variants return new tensors instead of modifying the caller's predictions
    in place;
  * get_all_pts3d_t returns tensors without autograd history; compute_frame_loss's `conf_mean` is a detached 0-d tensor;
  * the MultiLoss `+` / `*` algebra and reductions other than 'mean' (standalone) and 'none' (under ConfLoss_t) raise
    NotImplementedError;
  * a term without a valid pixel under ConfLoss_t raises ValueError (the reference fails in torch.stack).
"""
from __future__ import annotations

import ctypes as C
from copy import copy, deepcopy

import torch
from torch import nn

from . import _lib

__all__ = ["L21", "L21Loss", "Regr3D_t", "Regr3D_t_ShiftInv", "Regr3D_t_ScaleInv", "Regr3D_t_ScaleShiftInv",
           "ConfLoss_t"]

_NORM_MODES = {"avg_dis": 1, "avg_log1p": 2}
_H, _PB = _lib.LOSS_RES_HEADER, _lib.LOSS_RES_PER_B


class L21Loss(nn.Module):
    """Euclidean distance between 3-D points (dust3r/losses.py:52-59): the pixel criterion of the Spann3R criteria.
    It selects the native kernel's distance; it is not evaluated on its own."""

    def __init__(self, reduction="mean"):
        super().__init__()
        self.reduction = reduction


L21 = L21Loss()


# ---------------------------------------------------------------------------------------------------------------------
# input parsing
# ---------------------------------------------------------------------------------------------------------------------
def _pred_slots(preds, F):
    """Pred slots in the native order: L[0..F-2] then R[0..F-2] (dust3r/inference.py:87-109 get_pred_pts3d)."""
    if len(preds) != F - 1:
        raise ValueError(f"preds has {len(preds)} pairs, the {F} views need {F - 1}")
    pts, conf = [], []
    for side in (0, 1):
        for k in range(F - 1):
            p = preds[k][side]
            use_pose = side == 1 or k != 0
            if "pts3d" in p:
                if use_pose:
                    raise ValueError(f"preds[{k}][{side}] holds 'pts3d', which needs a camera pose (not produced by Spann3R)")
                pts.append(p["pts3d"])
            elif "pts3d_in_other_view" in p:
                if not use_pose:
                    raise ValueError("preds[0][0] must hold 'pts3d'")
                pts.append(p["pts3d_in_other_view"])
            else:
                raise ValueError(f"preds[{k}][{side}] has no 'pts3d' / 'pts3d_in_other_view'")
            conf.append(p.get("conf"))
    return pts, conf


def _check(t, name, shape, dtype, dev):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
    if t.device != dev:
        raise ValueError(f"{name} is on {t.device}, expected {dev}")
    return t.contiguous()


class _Call:
    """One native evaluation: validated inputs, the descriptor (with the host pointer arrays it references) and the
    workspace, kept alive together until the backward has run."""

    def __init__(self, crit, gts, preds, dist_clip, conf_loss, alpha, need_conf):
        F = len(gts)
        if F < 2:
            raise ValueError("the criteria need at least 2 views")
        pts, conf = _pred_slots(preds, F)
        p0 = gts[0]["pts3d"]
        if not isinstance(p0, torch.Tensor) or not p0.is_cuda:
            raise ValueError("gts[0]['pts3d'] must be a CUDA tensor")
        if p0.dim() != 4 or p0.shape[-1] != 3:
            raise ValueError(f"pts3d must be [B,H,W,3], got {tuple(p0.shape)}")
        B, H, W, _ = p0.shape
        dev = p0.device
        self.B, self.H, self.W, self.F, self.dev = B, H, W, F, dev
        self.gt = [_check(g["pts3d"], f"gts[{i}]['pts3d']", (B, H, W, 3), torch.float32, dev) for i, g in enumerate(gts)]
        self.valid = [_check(g["valid_mask"], f"gts[{i}]['valid_mask']", (B, H, W), torch.bool, dev)
                      for i, g in enumerate(gts)]
        self.pose0 = _check(gts[0]["camera_pose"], "gts[0]['camera_pose']", (B, 4, 4), torch.float32, dev)
        self.pred = [_check(p, f"pred slot {k}", (B, H, W, 3), torch.float32, dev) for k, p in enumerate(pts)]
        if need_conf or all(c is not None for c in conf):
            if any(c is None for c in conf):
                raise ValueError("every prediction needs a 'conf' map")
            self.conf = [_check(c, f"conf slot {k}", (B, H, W), torch.float32, dev) for k, c in enumerate(conf)]
        else:
            self.conf = None
        nm = crit.norm_mode
        if nm and nm not in _NORM_MODES:
            raise ValueError(f"norm_mode {nm!r} is not one of {list(_NORM_MODES)} or False")
        S = 2 * (F - 1)
        V = C.c_void_p
        self._arr = [(V * F)(*[t.data_ptr() for t in self.gt]), (V * F)(*[t.data_ptr() for t in self.valid]),
                     (V * S)(*[t.data_ptr() for t in self.pred])]
        if self.conf is not None:
            self._arr.append((V * S)(*[t.data_ptr() for t in self.conf]))
        d = _lib.LossDesc()
        d.frames, d.batch, d.height, d.width = F, B, H, W
        d.norm_mode = _NORM_MODES.get(nm, 0) if nm else 0
        d.gt_scale, d.fix_first = int(bool(crit.gt_scale)), int(bool(crit.fix_first))
        d.shift_inv, d.scale_inv = int(crit._shift), int(crit._scale)
        d.conf_loss, d.alpha = int(conf_loss), float(alpha)
        d.has_dist_clip, d.dist_clip = int(dist_clip is not None), float(dist_clip if dist_clip is not None else 0.0)
        d.pose0 = self.pose0.data_ptr()
        d.gt_pts, d.valid, d.pred = self._arr[0], self._arr[1], self._arr[2]
        d.conf = self._arr[3] if self.conf is not None else None
        self.desc = d
        L = _lib.lib()
        self.ws_bytes = L.s3r_loss_workspace_bytes(C.byref(d))
        if self.ws_bytes == 0:
            raise ValueError("s3r_loss_workspace_bytes: " + L.s3r_last_error().decode(errors="replace"))
        self.ws = torch.empty(self.ws_bytes, dtype=torch.uint8, device=dev)
        self.results = torch.empty(_H + _PB * B, dtype=torch.float64, device=dev)

    def forward(self, maps=False):
        B, H, W, F = self.B, self.H, self.W, self.F
        gt_out = pred_out = valid_out = None
        if maps:
            gt_out = torch.empty((F, B, H, W, 3), dtype=torch.float32, device=self.dev)
            pred_out = torch.empty((2 * (F - 1), B, H, W, 3), dtype=torch.float32, device=self.dev)
            valid_out = torch.empty((F, B, H, W), dtype=torch.uint8, device=self.dev)
        _lib.call("s3r_loss_forward", self.dev, C.byref(self.desc), _lib.ptr(self.ws), self.ws_bytes, _lib.ptr(gt_out),
                  _lib.ptr(pred_out), _lib.ptr(valid_out), _lib.ptr(self.results))
        return gt_out, pred_out, valid_out

    def backward(self, upstream):
        B, H, W, S = self.B, self.H, self.W, 2 * (self.F - 1)
        gp = torch.empty((S, B, H, W, 3), dtype=torch.float32, device=self.dev)
        gc = torch.empty((S, B, H, W), dtype=torch.float32, device=self.dev) if self.desc.conf_loss else None
        _lib.call("s3r_loss_backward", self.dev, C.byref(self.desc), _lib.ptr(self.ws), self.ws_bytes, _lib.ptr(upstream),
                  _lib.ptr(gp), _lib.ptr(gc))
        return gp, gc

    def per_b(self, i):
        """Per-batch-element result i (0 gt_factor, 1 pr_factor, 2 gt_shift_z, 3 pred_shift_z, 4 gt_scale,
        5 pred_scale) as fp32 [B] on the device."""
        return self.results[_H + i::_PB].float()


class _Criterion(torch.autograd.Function):
    """(loss, factor_loss) of one native forward; inputs: the pred slots, then the conf slots."""

    @staticmethod
    def forward(ctx, call, *tensors):
        call.forward()
        ctx.call = call
        # saved so that autograd's version check rejects an in-place change of an input before the backward, which
        # reads the inputs again through the workspace's pointer table
        ctx.save_for_backward(*tensors)
        r = call.results
        return r[0].float(), r[1].float()

    @staticmethod
    def backward(ctx, g_loss, g_factor):
        _ = ctx.saved_tensors                 # raises if an input was modified in place since the forward
        call = ctx.call
        z = torch.zeros((), dtype=torch.float32, device=call.dev)
        up = torch.stack([z if g_loss is None else g_loss.float().reshape(()),
                          z if g_factor is None else g_factor.float().reshape(())]).contiguous()
        gp, gc = call.backward(up)
        S = gp.shape[0]
        grads = [gp[k] for k in range(S)]
        if call.conf is not None:
            grads += [gc[k] if gc is not None else None for k in range(S)]
        return (None, *grads)


# ---------------------------------------------------------------------------------------------------------------------
# the reference's classes
# ---------------------------------------------------------------------------------------------------------------------
class Regr3D_t(nn.Module):
    """spann3r/loss.py:129-247: regression of the normalised pointmaps of every view in the first camera's frame."""
    _shift = False
    _scale = False

    def __init__(self, criterion, norm_mode="avg_dis", gt_scale=False, fix_first=True):
        super().__init__()
        if not isinstance(criterion, L21Loss):
            raise NotImplementedError(f"{criterion} is not L21Loss: only the L21 pixel criterion is implemented")
        if norm_mode and norm_mode not in _NORM_MODES:
            raise NotImplementedError(f"norm_mode {norm_mode!r}: only {list(_NORM_MODES)} or False")
        self.criterion = copy(criterion)
        self.norm_mode = norm_mode
        self.gt_scale = gt_scale
        self.fix_first = fix_first

    def get_name(self):
        return f"{type(self).__name__}({self.criterion})"

    def with_reduction(self, mode):
        res = deepcopy(self)
        res.criterion.reduction = "none"      # as the reference: the per-pixel losses, whatever `mode` says
        return res

    def __add__(self, other):
        raise NotImplementedError("the MultiLoss algebra is not implemented")

    __mul__ = __rmul__ = __radd__ = __add__

    def _call(self, gts, preds, dist_clip=None, conf_loss=False, alpha=1.0, need_conf=False):
        return _Call(self, gts, preds, dist_clip, conf_loss, alpha, need_conf)

    def _pts3d(self, gts, preds, dist_clip):
        call = self._call(gts, preds, dist_clip)
        gt, pr, valid = call.forward(maps=True)
        F, B = call.F, call.B
        gt_pts = [gt[i] for i in range(F)]
        pr_pts = ([pr[k] for k in range(F - 1)], [pr[F - 1 + k] for k in range(F - 1)])
        factors = bool(self.norm_mode)
        pr_factor = call.per_b(1).view(B, 1, 1, 1) if factors else None
        gt_factor = call.per_b(0).view(B, 1, 1, 1) if factors and not self.gt_scale else None
        masks = [valid[i].view(torch.bool) for i in range(F)]
        monitoring = {}
        if self._shift:
            monitoring.update(gt_shift_z=call.results[11].float(), pred_shift_z=call.results[12].float())
        if self._scale:
            monitoring.update(gt_scale=call.results[13].float(), pred_scale=call.results[14].float())
        return gt_pts, pr_pts, gt_factor, pr_factor, masks, monitoring

    def get_all_pts3d_t(self, gts, preds, dist_clip=None):
        """(gt_pts [F], (pr_l [F-1], pr_r [F-1]), gt_factor, pr_factor, masks [F], monitoring) as the reference."""
        return self._pts3d(gts, preds, dist_clip)

    def _details(self, call, host):
        name = type(self).__name__
        d = {name + "_pts3d_1": host[2], name + "_pts3d_2": host[3], name + "loss_left": host[4],
             name + "loss_right": host[5], name + "conf_left": host[6], name + "conf_right": host[7]}
        if self._shift:
            d.update(gt_shift_z=host[11], pred_shift_z=host[12])
        if self._scale:
            d.update(gt_scale=host[13], pred_scale=host[14])
        return d

    def _frame_loss(self, gts, preds, conf_loss, alpha, dist_clip=None):
        call = self._call(gts, preds, dist_clip, conf_loss, alpha, need_conf=True)
        tensors = call.pred + call.conf
        loss, factor = _Criterion.apply(call, *tensors)
        host = call.results[:_H].cpu().tolist()           # the one device-to-host copy: logged values
        if conf_loss and host[16] > 0:
            raise ValueError(f"{int(host[16])} loss term(s) without a valid pixel: ConfLoss_t is undefined there")
        factor_loss = factor if host[15] > 0 else 0.0
        return call, loss, factor_loss, host

    def compute_frame_loss(self, gts, preds, **kw):
        """(loss, details, factor_loss): loss = sum of the per-term mean L21 distances (reduction 'mean')."""
        if self.criterion.reduction != "mean":
            raise NotImplementedError(f"reduction {self.criterion.reduction!r} of a standalone {type(self).__name__}: "
                                      "only 'mean' (and 'none' under ConfLoss_t)")
        call, loss, factor_loss, host = self._frame_loss(gts, preds, False, 1.0, **kw)
        return loss, self._details(call, host), factor_loss


class Regr3D_t_ShiftInv(Regr3D_t):
    """Invariant to depth shift: the lower median z of each point set is subtracted (spann3r/loss.py:294-322)."""
    _shift = True

    def get_all_pts3d_t(self, gts, preds):
        return self._pts3d(gts, preds, None)


class Regr3D_t_ScaleInv(Regr3D_t):
    """Invariant to scale: median distance to the median centre (spann3r/loss.py:325-364); gt_scale=True brings the
    prediction to the ground truth's scale."""
    _scale = True

    def get_all_pts3d_t(self, gts, preds):
        return self._pts3d(gts, preds, None)


class Regr3D_t_ScaleShiftInv(Regr3D_t_ScaleInv, Regr3D_t_ShiftInv):
    """Shift first, then scale (the reference's MRO)."""


class ConfLoss_t(nn.Module):
    """spann3r/loss.py:250-291: the per-pixel loss weighted by the learned confidence, d c - alpha log c."""

    def __init__(self, pixel_loss, alpha=1):
        super().__init__()
        assert alpha > 0
        if not isinstance(pixel_loss, Regr3D_t):
            raise NotImplementedError("ConfLoss_t is implemented over the Regr3D_t family only")
        self.alpha = alpha
        self.pixel_loss = pixel_loss.with_reduction("none")

    def get_name(self):
        return f"ConfLoss({self.pixel_loss})"

    def __add__(self, other):
        raise NotImplementedError("the MultiLoss algebra is not implemented")

    __mul__ = __rmul__ = __radd__ = __add__

    def compute_frame_loss(self, gts, preds, **kw):
        """(loss, details, factor_loss) as the reference."""
        pl = self.pixel_loss
        if pl.criterion.reduction != "none":
            raise NotImplementedError("ConfLoss_t needs a pixel loss with reduction 'none'")
        call, loss, factor_loss, host = pl._frame_loss(gts, preds, True, self.alpha, **kw)
        conf_mean = call.results[10].float()
        details = dict(conf_loss_1=host[8], conf_loss2=host[9], conf_mean=conf_mean, **pl._details(call, host))
        return loss, details, factor_loss
