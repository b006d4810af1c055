"""PyTorch restatement of Spann3R's criteria (spann3r/loss.py:129-369 with dust3r's L21), for tests: any device, any
float dtype, autograd through the prediction's norm factor; medians and scales are constants (no_grad), as there.

    out = criterion(gts, preds, norm_mode='avg_dis', fix_first=False, conf_alpha=0.4, dtype=torch.float64)

returns a dict with loss, factor_loss (tensor, or 0.0), details (floats, the reference's keys and order), gt_pts, pr_l,
pr_r, gt_factor, pr_factor, masks and monitoring (the pre-alignment points too, for the median checks).
"""
import torch


def pred_slots(preds, F):
    L = [preds[0][0]["pts3d"]] + [preds[k][0]["pts3d_in_other_view"] for k in range(1, F - 1)]
    R = [preds[k][1]["pts3d_in_other_view"] for k in range(F - 1)]
    cl = [preds[k][0]["conf"] for k in range(F - 1)]
    cr = [preds[k][1]["conf"] for k in range(F - 1)]
    return L, R, cl, cr


def _nanmed(vals, masks):
    """lower median over the valid entries of all maps, per batch element: vals [B, ...] list."""
    cat = torch.cat([torch.where(m, v, torch.full_like(v, float("nan"))).reshape(len(v), -1) for v, m in zip(vals, masks)], 1)
    return torch.nanmedian(cat, dim=1).values


def criterion(gts, preds, norm_mode="avg_dis", gt_scale=False, fix_first=True, shift=False, scale=False,
              conf_alpha=None, dist_clip=None, name=None, dtype=torch.float64, check_empty=True):
    """check_empty: under ConfLoss_t (conf_alpha set) a loss term without a valid pixel raises ValueError, as
    spann3r_b200.loss does (the reference fails in torch.stack there); False returns NaN for it."""
    F = len(gts)
    L, R, cl, cr = pred_slots(preds, F)
    L = [p.to(dtype) for p in L]
    R = [p.to(dtype) for p in R]
    cl = [c.to(dtype) for c in cl]
    cr = [c.to(dtype) for c in cr]
    T = torch.linalg.inv(gts[0]["camera_pose"].double()).to(dtype)
    gt, masks = [], []
    for g in gts:
        p = g["pts3d"].to(dtype)
        gt.append(torch.einsum("bij,bhwj->bhwi", T[:, :3, :3], p) + T[:, None, None, :3, 3])
        m = g["valid_mask"].clone()
        if dist_clip is not None:
            m = m & (g["pts3d"].to(dtype).norm(dim=-1) <= dist_clip)
        masks.append(m)
    prim = L + [R[-1]]
    nf = 1 if fix_first else F
    n_tot = sum(masks[f].sum() for f in range(nf)).to(dtype)

    def factor(pts):
        s = 0
        for f in range(nf):
            d = pts[f].norm(dim=-1)
            if norm_mode == "avg_log1p":
                d = torch.log1p(d)
            s = s + torch.where(masks[f], d, torch.zeros_like(d)).flatten(1).sum(1)
        return (s / (n_tot + 1e-8)).clip(min=1e-8).view(-1, 1, 1, 1)

    pr_factor = gt_factor = None
    if norm_mode:
        pr_factor = factor(prim)
        L = [p / pr_factor for p in L]
        R = [p / pr_factor for p in R]
        if not gt_scale:
            gt_factor = factor(gt)
            gt = [p / gt_factor for p in gt]
    mon = {"pre_gt": [g.detach() for g in gt], "pre_pr": [p.detach() for p in L + [R[-1]]]}
    monitoring = {}
    if shift:
        with torch.no_grad():
            gs = _nanmed([g[..., 2] for g in gt], masks)
            ps = _nanmed([p[..., 2] for p in L + [R[-1]]], masks)
        sub = lambda p, s: p - torch.stack([torch.zeros_like(s), torch.zeros_like(s), s], -1).view(-1, 1, 1, 3)  # noqa: E731
        gt = [sub(g, gs) for g in gt]
        L = [sub(p, ps) for p in L]
        R = [sub(p, ps) for p in R]
        monitoring.update(gt_shift_z=gs.mean(), pred_shift_z=ps.mean())
        mon.update(gt_shift=gs, pred_shift=ps)
    if scale:
        with torch.no_grad():
            def cs(pts):
                c = torch.stack([_nanmed([p[..., i] for p in pts], masks) for i in range(3)], -1)
                mon.setdefault("centres", []).append(c)
                return _nanmed([(p - c.view(-1, 1, 1, 3)).norm(dim=-1) for p in pts], masks)
            gsc = cs(gt)
            psc = cs(L + [R[-1]]).clip(min=1e-3, max=1e3)
        if gt_scale:
            r = (gsc / psc).view(-1, 1, 1, 1)
            L = [p * r for p in L]
            R = [p * r for p in R]
        else:
            r = (psc / gsc).view(-1, 1, 1, 1)
            L = [p * r for p in L]
            R = [p * r for p in R]
            gt = [g * (gsc / psc).view(-1, 1, 1, 1) for g in gt]
        monitoring.update(gt_scale=gsc.mean(), pred_scale=psc.mean())
    # terms in the reference's order: left / right interleaved per frame
    terms = []
    for i in range(F):
        if i != F - 1:
            terms.append(("L", i, L[i], cl[i]))
        if i != 0:
            terms.append(("R", i - 1, R[i - 1], cr[i - 1]))
    dists, confs = [], []
    for side, k, p, c in terms:
        f = k if side == "L" else k + 1
        m = masks[f]
        dists.append((p[m] - gt[f][m]).norm(dim=-1))
        confs.append(c[m])
    means = [d.mean() if d.numel() else d.new_zeros(()) for d in dists]
    left = sum(float(means[t]) for t, (s, k, _, _) in enumerate(terms) if s == "L" and k != 0)
    right = sum(float(means[t]) for t, (s, k, _, _) in enumerate(terms) if s == "R" and k != F - 2)
    conf_l = sum(float(cl[k].mean()) for k in range(1, F - 1))
    conf_r = sum(float(cr[k].mean()) for k in range(0, F - 2))
    name = name or "Regr3D_t"
    details = {name + "_pts3d_1": float(means[0]), name + "_pts3d_2": float(means[1]), name + "loss_left": left,
               name + "loss_right": right, name + "conf_left": conf_l, name + "conf_right": conf_r}
    details.update({k: float(v) for k, v in monitoring.items()})
    if conf_alpha is not None and check_empty and any(d.numel() == 0 for d in dists):
        raise ValueError("a loss term without a valid pixel: ConfLoss_t is undefined there")
    if conf_alpha is None:
        loss = sum(means)
    else:
        cls = torch.stack([(d * c - conf_alpha * torch.log(c)).mean() for d, c in zip(dists, confs)]) * 2.0
        loss = cls.mean()
        conf_mean = sum(c.mean() for c in confs) / len(confs)
        details = dict(conf_loss_1=float(cls[0]), conf_loss2=float(cls[1]), conf_mean=float(conf_mean), **details)
    factor_loss = 0.0
    if pr_factor is not None and gt_factor is not None:
        sel = pr_factor[pr_factor > gt_factor]
        if len(sel) > 0:
            factor_loss = (sel - gt_factor).abs().mean()
    return {"loss": loss, "factor_loss": factor_loss, "details": details, "gt_pts": gt, "pr_l": L, "pr_r": R,
            "gt_factor": gt_factor, "pr_factor": pr_factor, "masks": masks, "monitoring": monitoring, "pre": mon}
