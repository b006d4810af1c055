"""Spann3R's criteria on the H100 at the inputs where they go wrong (csrc/loss.cu through spann3r_b200.loss): batch
elements with 0 / 1 / 2 / odd / even valid pixels, valid pixels only at the 2048-pixel block edges, P = 1, P < 256 and
P = k 2048 +- 1, two frames, a 64-frame eval sequence, planar scenes with tied medians, +-inf and NaN, norm factors
either side of the 1e-8 clip, points at dist_clip, d == 0 pixels, conf 1 and 1e30, and the two upstream gradients
alone and together.  Per case:
  * medians bit for bit against the host radix select over the same header (tests/native/loss_host_check.cpp) and
    equal to torch.nanmedian of the kernel's own fp32 stage values; aligned maps bit for bit against the float32
    restatement given the kernel's factor and medians; the factor within 1 ulp of the fp64 sum of the same fp32 terms;
  * loss, factor_loss, details, monitoring and every gradient against fp64 autograd of oracle/loss_oracle.py, within
    bounds derived from the fp32 roundings on each value's path (see K and check_against_fp64);
  * the NaN pattern of the oracle and of the reference's goldens; gradients exactly 0 at invalid pixels; two runs
    bitwise equal."""
import math

import numpy as np
import pytest
import torch

import loss_host as lh
from oracle import loss_oracle as lo
from spann3r_b200 import _lib, synth
from test_loss_adversarial_cpu import close, load_adv_golden, np_align, np_stage_value, same_bits
from test_loss_cpu import oracle_kwargs, slot_tensors

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24
# Roundings between an input and the distance d of a pixel: the division by the fp32 factor, the shift subtraction,
# the scale multiplication (each side), the difference, three squares, two additions and the square root, plus the
# fp32 rounding of the factor, the medians and the scale ratio themselves: 14 of them, each <= u relative to the
# magnitude it acts on.  K = 16 covers them with the fp64 sums' own error (< 1e-12 relative) to spare.
K = 16
_H, _PB = _lib.LOSS_RES_HEADER, _lib.LOSS_RES_PER_B

TRAIN = "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)"
TEST = "Regr3D_t_ScaleShiftInv(L21, gt_scale=True)"
EVAL = "Regr3D_t_ScaleShiftInv(L21, norm_mode=False, gt_scale=True)"
CRITERIA = [TRAIN, TEST, EVAL,
            "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_log1p', fix_first=True), alpha=0.2)",
            "Regr3D_t(L21, norm_mode='avg_dis')",
            "Regr3D_t(L21, norm_mode=False)",
            "Regr3D_t_ShiftInv(L21, norm_mode='avg_log1p', fix_first=False)",
            "Regr3D_t_ScaleInv(L21, gt_scale=False, fix_first=False)",
            "Regr3D_t_ScaleShiftInv(L21, gt_scale=False)"]


def native(crit_str):
    ns = {}
    exec("from spann3r_b200.loss import *", ns)
    return eval(crit_str, ns)


def to_dev(gts, preds):
    return ([{k: t.to(DEV) for k, t in d.items()} for d in gts],
            [tuple({k: t.to(DEV) for k, t in d.items()} for d in p) for p in preds])


# ---------------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------------
def data(B=2, F=3, H=16, W=24, invalid=0.3, seed=0):
    return synth.make_loss_case(B, F, H, W, invalid=invalid, seed=seed)


def with_counts(counts, F=3, H=8, W=12, seed=1):
    """B = len(counts) elements, element b with counts[b] valid pixels over all frames (None: all of them)."""
    gts, preds = data(len(counts), F, H, W, invalid=0.0, seed=seed)
    g = torch.Generator().manual_seed(seed)
    for b, n in enumerate(counts):
        if n is None:
            continue
        flat = torch.zeros(F * H * W, dtype=torch.bool)
        flat[torch.randperm(F * H * W, generator=g)[:n]] = True
        for f in range(F):
            gts[f]["valid_mask"][b] = flat[f * H * W:(f + 1) * H * W].view(H, W)
    return gts, preds


def block_edges():
    """P = 4097: valid pixels only at p = 2047, 2048 and in the last, one-pixel block (p = 4096) of every frame."""
    gts, preds = data(2, 3, 17, 241, invalid=0.0, seed=2)
    for g in gts:
        m = torch.zeros(2, 17 * 241, dtype=torch.bool)
        m[:, [2047, 2048, 4096]] = True
        m[1, 2047] = False
        g["valid_mask"] = m.view(2, 17, 241)
    return gts, preds


def planar():
    gts, preds = synth.make_loss_adv_case("planar")
    return gts, preds


def inf_nan_valid():
    """+-inf and NaN at valid pixels and NaN at invalid ones of the ground truth and the predictions' z."""
    gts, preds = data(2, 3, 16, 24, invalid=0.3, seed=3)
    for f, g in enumerate(gts):
        g["pts3d"][~g["valid_mask"]] = float("nan")
        g["valid_mask"][:, 0, :4] = True
        g["pts3d"][:, 0, 0, 2] = float("inf")
        g["pts3d"][:, 0, 1, 2] = -float("inf")
        g["pts3d"][:, 0, 2, 0] = float("nan")
    for k in range(len(preds)):
        synth.loss_slot(preds, k, 0)[:, 0, 3, 2] = float("inf")
        synth.loss_slot(preds, k, 1)[:, 0, 2, 2] = float("nan")
    return gts, preds


def shift_to_zero():
    """Integer depths: after the median shift many z are exactly +0.0, and some inputs are -0.0."""
    gts, preds = data(2, 3, 16, 24, invalid=0.2, seed=4)
    for g in gts:
        g["camera_pose"] = torch.eye(4).repeat(2, 1, 1)
        g["pts3d"][..., 2] = torch.round(g["pts3d"][..., 2] * 2) / 2
        g["pts3d"][:, ::3, ::5, 0] = -0.0
    for k in range(len(preds)):
        for side in (0, 1):
            p = synth.loss_slot(preds, k, side)
            p[..., 2] = torch.round(p[..., 2] * 4) / 4
    return gts, preds


def factor_at(t, mode):
    """Element 0's predictions scaled so that its raw prediction norm factor is t * 1e-8 (t != 1: the fp32 rounding of
    the scaled inputs, ~1e-7 relative, keeps it on its side of the clip)."""
    gts, preds = data(2, 3, 16, 24, invalid=0.3, seed=5)
    F = len(gts)
    prim = [synth.loss_slot(preds, k, 0) for k in range(F - 1)] + [synth.loss_slot(preds, F - 2, 1)]
    n = sum(int(g["valid_mask"].sum()) for g in gts)
    s = sum(float(p[0].double().norm(dim=-1)[g["valid_mask"][0]].sum()) for p, g in zip(prim, gts))
    c = t * 1e-8 * (n + 1e-8) / s
    for k in range(F - 1):
        for side in (0, 1):
            p = synth.loss_slot(preds, k, side)
            p[0] = (p[0].double() * c).float()
    return gts, preds


def conf_extremes():
    gts, preds = synth.make_loss_adv_case("d_zero")
    return gts, preds


CASES = {}
for i, c in enumerate(CRITERIA):
    CASES[f"counts_{i}"] = (c, lambda: with_counts([0, 1, 2, 3, 4, 7, 8, None]), {})
    CASES[f"edges_{i}"] = (c, block_edges, {})
    CASES[f"f2_{i}"] = (c, lambda: data(2, 2, 16, 24, seed=6), {})
for i, c in enumerate([TRAIN, TEST, CRITERIA[8]]):
    for H, W in [(1, 1), (8, 12), (23, 89), (3, 683), (45, 91), (17, 241)]:
        CASES[f"size{H}x{W}_{i}"] = (c, (lambda H=H, W=W: data(2, 3, H, W, invalid=0.0 if H * W == 1 else 0.3, seed=7)), {})
for i, c in enumerate([TEST, EVAL, CRITERIA[6], CRITERIA[7], CRITERIA[8]]):
    CASES[f"planar_{i}"] = (c, planar, {})
    CASES[f"infnan_{i}"] = (c, inf_nan_valid, {})
    CASES[f"zero_{i}"] = (c, shift_to_zero, {})
for t in (0.5, 0.999, 1.001, 2.0):
    for mode in ("avg_dis", "avg_log1p"):
        CASES[f"clip{t}_{mode}"] = (f"ConfLoss_t(Regr3D_t(L21, norm_mode='{mode}', fix_first=False), alpha=0.4)",
                                    (lambda t=t, mode=mode: factor_at(t, mode)), {})
        CASES[f"clip{t}_{mode}_regr"] = (f"Regr3D_t(L21, norm_mode='{mode}', fix_first=False)",
                                         (lambda t=t, mode=mode: factor_at(t, mode)), {})
for tag, c in (("train", TRAIN), ("log1p", CRITERIA[3])):
    CASES[f"distclip_{tag}"] = (c, lambda: synth.make_loss_adv_case("dist_clip_eq"), {"dist_clip": 3.0})
CASES["dzero_conf"] = ("ConfLoss_t(Regr3D_t(L21, norm_mode=False), alpha=0.4)", conf_extremes, {})
CASES["dzero_regr"] = ("Regr3D_t(L21, norm_mode='avg_dis', fix_first=False)", conf_extremes, {})
CASES["train_5f"] = (TRAIN, lambda: data(2, 5, 64, 64, seed=8), {})


# ---------------------------------------------------------------------------------------------------------------------
# the checks
# ---------------------------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy()


def kernel_state(crit, gts, preds, dist_clip):
    """The native forward's maps and per-element results, and the kernel's transformed, unaligned ground truth."""
    pl = getattr(crit, "pixel_loss", crit)
    call = pl._call(gts, preds, dist_clip)
    gt_out, pr_out, valid = call.forward(maps=True)
    plain = native("Regr3D_t(L21, norm_mode=False)")._call(gts, preds, dist_clip)
    gtT = plain.forward(maps=True)[0]
    return (pl, _np(gt_out), _np(pr_out), _np(valid).astype(bool), call.results.cpu().numpy(), _np(gtT),
            np.stack([_np(p) for p in call.pred]))


def check_medians_and_maps(crit_str, gts, preds, dist_clip):
    crit = native(crit_str)
    pl, gt_out, pr_out, valid, res, gtT, pred = kernel_state(crit, gts, preds, dist_clip)
    F, B = gtT.shape[0], gtT.shape[1]
    S = 2 * (F - 1)
    prim = list(range(F - 1)) + [S - 1]
    nm = pl.norm_mode
    nf = 1 if pl.fix_first else F
    n_tot = float(valid[:nf].sum())
    for b in range(B):
        r = lambda i: np.float32(res[_H + b * _PB + i])                        # noqa: E731
        m = valid[:, b].reshape(-1)
        sets = {"gt": (gtT[:, b].reshape(-1, 3), r(0), 2, 4), "pr": (pred[prim, b].reshape(-1, 3), r(1), 3, 5)}
        aln = {}
        for name, (pts, fac, si, ci) in sets.items():
            # the factor: 1 ulp of the fp64 sum of the same fp32 norms (log1p: 2 ulp, CUDA's log1pf and numpy's may
            # each be an ulp from the exact value)
            use = nm and not (name == "gt" and pl.gt_scale)
            if use:
                nrm = lh.norm3(np.concatenate([sets[name][0].reshape(F, -1, 3)[f] for f in range(nf)]))
                vals = nrm if nm == "avg_dis" else np.log1p(nrm.astype(np.float64))
                vals = vals[valid[:nf, b].reshape(-1)].astype(np.float64)
                want = max(math.fsum(vals.tolist()) / (n_tot + 1e-8), 1e-8)
                ulps = 1 if nm == "avg_dis" else 2
                if math.isfinite(want):
                    assert abs(float(fac) - want) <= ulps * float(np.spacing(np.float32(want))), (name, b, fac, want)
                else:
                    assert float(fac) == want or (fac != fac and want != want), (name, b, fac, want)
            else:
                assert fac == 1.0
            shift, centre = np.float32(0), np.zeros(3, np.float32)
            with np.errstate(all="ignore"):
                if pl._shift:
                    shift = lh.median(pts, m, fac, 0.0, centre, 0)
                    assert same_bits(shift, r(si)), (name, b, shift, r(si))
                    _torch_median_equals(np_stage_value(pts, fac, 0.0, centre, 0)[m], shift)
                scale = np.float32(1)
                if pl._scale:
                    for kind in (1, 2, 3):
                        centre[kind - 1] = lh.median(pts, m, fac, shift, centre, kind)
                        _torch_median_equals(np_stage_value(pts, fac, shift, centre, kind)[m], centre[kind - 1])
                    scale = lh.median(pts, m, fac, shift, centre, 4)
                    _torch_median_equals(np_stage_value(pts, fac, shift, centre, 4)[m], scale)
                    if name == "pr" and scale == scale:
                        scale = np.float32(min(max(scale, np.float32(1e-3)), np.float32(1e3)))
                    assert same_bits(scale, r(ci)), (name, b, scale, r(ci))
            aln[name] = (fac, shift, scale)
        mg = mp = np.float32(1)
        if pl._scale:
            gs, ps = aln["gt"][2], aln["pr"][2]
            with np.errstate(all="ignore"):
                if pl.gt_scale:
                    mp = gs / ps
                else:
                    mp, mg = ps / gs, gs / ps
        with np.errstate(all="ignore"):
            for f in range(F):
                want = np_align(gtT[f, b].reshape(-1, 3), aln["gt"][0], aln["gt"][1], mg)
                assert same_bits(gt_out[f, b].reshape(-1, 3), want), ("gt map", f, b)
            for k in range(S):
                want = np_align(pred[k, b].reshape(-1, 3), aln["pr"][0], aln["pr"][1], mp)
                assert same_bits(pr_out[k, b].reshape(-1, 3), want), ("pred map", k, b)
    return valid, res


def _torch_median_equals(vals, m):
    t = torch.from_numpy(np.ascontiguousarray(vals)).to(DEV)
    want = t.nanmedian() if t.numel() else torch.tensor(float("nan"))
    w = float(want)
    assert (math.isnan(w) and m != m) or w == float(m), (w, m)


def run_native(crit_str, gts, preds, kw, upstream):
    crit = native(crit_str)
    slots = slot_tensors(preds)
    for p, c in slots.values():
        p.grad = c.grad = None
    loss, details, fl = crit.compute_frame_loss(gts, preds, **kw)
    backward(loss, fl, upstream)
    grads = {key: (_np(p.grad) if p.grad is not None else np.zeros(p.shape, np.float32),
                   _np(c.grad) if c.grad is not None else np.zeros(c.shape, np.float32)) for key, (p, c) in slots.items()}
    return float(loss), float(fl), {k: float(v) for k, v in details.items()}, grads


def backward(loss, fl, upstream):
    fl_t = isinstance(fl, torch.Tensor)
    if upstream == "loss" or (upstream == "both" and not fl_t):
        loss.backward()
    elif upstream == "factor":
        fl.backward()
    else:
        (loss + fl).backward()


def check_against_fp64(crit_str, gts, preds, kw, upstream, valid, res):
    okw = oracle_kwargs(crit_str)
    alpha = okw["conf_alpha"] or 0.0
    conf = okw["conf_alpha"] is not None
    a = run_native(crit_str, gts, preds, kw, upstream)
    b = run_native(crit_str, gts, preds, kw, upstream)
    assert a[:3] == b[:3] or _nan_equal(a[:3], b[:3])
    for key in a[3]:                                                             # bitwise reproducible
        assert same_bits(a[3][key][0], b[3][key][0]) and same_bits(a[3][key][1], b[3][key][1])
    loss, fl, details, grads = a
    slots = slot_tensors(preds)
    for p, c in slots.values():
        p.grad = c.grad = None
    out = lo.criterion(gts, preds, dtype=torch.float64, dist_clip=kw.get("dist_clip"), **okw)
    backward(out["loss"], out["factor_loss"], upstream)
    F = len(gts)
    S, B = 2 * (F - 1), gts[0]["pts3d"].shape[0]
    for f in range(F):
        assert np.array_equal(_np(out["masks"][f]).astype(bool), valid[f]), f
    # per-pixel error of d: K u (|pr| + |gt| + |shift_p mul_p| + |shift_g mul_g|), the aligned magnitudes before the
    # shift, with the kernel's medians and ratios
    r = res[_H:].reshape(B, _PB)
    mul = np.ones((B, 2))
    if okw["scale"]:
        mul[:, 1] = r[:, 4] / r[:, 5] if okw["gt_scale"] else r[:, 5] / r[:, 4]
        if not okw["gt_scale"]:
            mul[:, 0] = r[:, 4] / r[:, 5]
    # a median of fp32 values moves by at most the largest fp32 error among them, <= 2 u max|pre| for the shift
    # (pre: the normalised points before the shift) and <= 8 u max|pre| for the scale (|v - c|, v and c shifted);
    # the shift error enters d scaled by mul, the scale error relative to the scale through the ratio mul
    pre = [_np(t) for t in out["pre"]["pre_gt"]] + [_np(t) for t in out["pre"]["pre_pr"]]
    maxpre = np.zeros((B, 2))
    for i, p in enumerate(pre):
        for b in range(B):
            v = np.abs(p[b][valid[i % F][b]])
            maxpre[b, i // F] = max(maxpre[b, i // F], v[np.isfinite(v)].max(initial=0.0))
    shifts = maxpre * np.abs(mul) if okw["shift"] else np.zeros((B, 2))
    rel_mul = np.zeros(B)
    if okw["scale"]:
        with np.errstate(all="ignore"):
            rel_mul = np.nan_to_num(maxpre[:, 0] / np.abs(r[:, 4]) + maxpre[:, 1] / np.abs(r[:, 5]), posinf=0.0) / 2
    pr_al = out["pr_l"] + out["pr_r"]
    fr = [k if k < F - 1 else k - (F - 1) + 1 for k in range(S)]
    conf_maps = [preds[k][0]["conf"] for k in range(F - 1)] + [preds[k][1]["conf"] for k in range(F - 1)]
    e_term, eK = [], np.zeros(S)
    coef_mag = np.zeros(B)
    with np.errstate(all="ignore"):
        for k in range(S):
            m = valid[fr[k]]
            n = m.sum()
            pk, gk = _np(pr_al[k]), _np(out["gt_pts"][fr[k]])
            mag = np.linalg.norm(pk, axis=-1) + np.linalg.norm(gk, axis=-1)
            A = mag * (1 + rel_mul[:, None, None]) + (shifts[:, 0] + shifts[:, 1])[:, None, None]
            d = np.linalg.norm(pk - gk, axis=-1)
            c = _np(conf_maps[k]).astype(np.float64) if conf else np.ones_like(d)
            eD = K * U * A
            eT = c * eD + K * U * (d * c + alpha * np.abs(np.log(c))) if conf else eD
            w = (2.0 / (S * n) if conf else 1.0 / n) if n else 0.0
            e_term.append((eD, A, d, c, w))
            eK[k] = eT[m].sum() / n if n else 0.0
            x = _np(slots[(0, k) if k < F - 1 else (1, k - F + 1)][0]).astype(np.float64)
            xn = np.linalg.norm(x, axis=-1)
            fpv = r[:, 1] if okw["norm_mode"] else np.ones(B)
            # d == 0 pixels add nothing to the factor's gradient (the kernel skips them, torch's norm backward is 0)
            contrib = np.where(m & (d > 0), w * c * xn * (A / np.where(d > 0, d, 1.0) + 1.0), 0.0).reshape(B, -1).sum(1)
            coef_mag += np.abs(mul[:, 1]) / fpv ** 2 * contrib
    lref = float(out["loss"])
    fref = float(out["factor_loss"])
    loss_bound = (eK.sum() * (2.0 / S) if conf else eK.sum()) + 1e-12 * abs(lref)
    assert _scalar_ok(loss, lref, loss_bound), (loss, lref, loss_bound)
    fl_bound = K * U * (np.abs(r[:, 0]).max() + np.abs(r[:, 1]).max()) + 1e-12
    assert _scalar_ok(fl, fref, fl_bound), (fl, fref, fl_bound)
    keys = list(out["details"])
    assert list(details) == keys
    name = keys[3 if conf else 0].rsplit("_pts3d_1", 1)[0]
    mon_b = K * U * np.mean([max([np.nan_to_num(np.abs(p[b][valid[i % F][b]]), posinf=0).max(initial=0.0)
                                  for i, p in enumerate(pre)]) for b in range(B)])
    dbound = {"conf_loss_1": 2 * eK[0], "conf_loss2": 2 * eK[1], name + "_pts3d_1": eK[0], name + "_pts3d_2": eK[1],
              name + "loss_left": eK[1:F - 1].sum(), name + "loss_right": eK[F - 1:2 * F - 3].sum(),
              "conf_mean": 2 * U * abs(float(out["details"].get("conf_mean", 0.0)))}   # returned as an fp32 tensor
    for key in keys:
        ref = float(out["details"][key])
        # monitoring: the median bound, and the fp32 rounding of the reported value (the 1e-3 clip of pred_scale is
        # applied in fp32, as the reference applies it)
        bd = dbound.get(key, mon_b * (1 + abs(ref)) + 2 * U * abs(ref) if "shift" in key or "scale" in key else 0.0)
        assert _scalar_ok(details[key], ref, bd + 1e-10 * abs(ref) + 1e-300), (key, details[key], ref, bd)
    # gradients, per pixel
    gl = 0.0 if upstream == "factor" else 1.0
    n_tot = valid[:1 if okw["fix_first"] else F].sum()
    coef_err = 2 * K * U * gl * coef_mag / (n_tot + 1e-8) if okw["norm_mode"] else np.zeros(B)
    for k in range(S):
        key = (0, k) if k < F - 1 else (1, k - F + 1)
        p, c = slots[key]
        gp_ref = _np(p.grad) if p.grad is not None else np.zeros(p.shape)
        gc_ref = _np(c.grad) if c.grad is not None else np.zeros(c.shape)
        gp, gc = grads[key]
        m = valid[fr[k]]
        assert np.all(gp[~m] == 0) and not np.signbit(gp[~m]).any(), ("grad at invalid pixel", key)
        assert np.all(gc[~m] == 0), ("conf grad at invalid pixel", key)
        eD, A, d, cc, w = e_term[k]
        fpv = r[:, 1] if okw["norm_mode"] else np.ones(B)
        scale = (np.abs(mul[:, 1]) / fpv)[:, None, None]
        with np.errstate(all="ignore"):
            t1 = gl * w * cc * scale * K * U * A / d
            bound = t1[..., None] + coef_err[:, None, None, None] + K * U * np.abs(gp_ref) + 1e-37
            cbound = gl * w * eD + K * U * np.abs(gc_ref) + 1e-37
        for b in range(B):
            sel = m[b]
            if not np.isfinite(gp_ref[b][sel]).all():     # the criterion is undefined for this element: see INTEGRATION
                continue
            err = np.abs(gp[b][sel].astype(np.float64) - gp_ref[b][sel])
            assert np.isfinite(gp[b][sel]).all() and np.all(err <= bound[b][sel]), ("grad", key, b, err.max())
            if conf:
                errc = np.abs(gc[b][sel].astype(np.float64) - gc_ref[b][sel])
                assert np.all(errc <= cbound[b][sel]), ("conf grad", key, b, errc.max())
    return out


def _nan_equal(a, b):
    fa, fb = np.array(a[:2], np.float64), np.array(b[:2], np.float64)
    return np.array_equal(fa, fb, equal_nan=True) and all(
        (x == y) or (x != x and y != y) for x, y in zip(a[2].values(), b[2].values()))


def _scalar_ok(v, ref, bound):
    if v == ref:
        return True
    if ref != ref or abs(ref) == math.inf:
        return (v != v and ref != ref) or v == ref
    return v == v and abs(v - ref) <= bound


def _prepare(make):
    gts, preds = to_dev(*make())
    for p, c in slot_tensors(preds).values():
        p.requires_grad_(True)
        c.requires_grad_(True)
    return gts, preds


def _conf_loss_refuses(crit_str, gts, valid):
    F = len(gts)
    return crit_str.startswith("ConfLoss_t") and any(valid[f].sum() == 0 for f in range(F))


@pytest.mark.parametrize("name", sorted(CASES))
def test_case(name):
    crit_str, make, kw = CASES[name]
    gts, preds = _prepare(make)
    with torch.no_grad():
        valid, res = check_medians_and_maps(crit_str, gts, preds, kw.get("dist_clip"))
    if _conf_loss_refuses(crit_str, gts, valid):
        with pytest.raises(ValueError, match="without a valid pixel"):
            native(crit_str).compute_frame_loss(gts, preds, **kw)
        return
    check_against_fp64(crit_str, gts, preds, kw, "both", valid, res)


@pytest.mark.parametrize("upstream", ["loss", "factor", "both"])
@pytest.mark.parametrize("crit_str", [TRAIN, "Regr3D_t_ScaleInv(L21, gt_scale=False, fix_first=False)"])
def test_upstream_gradients(crit_str, upstream):
    gts, preds = _prepare(lambda: data(2, 3, 16, 24, seed=9))
    with torch.no_grad():
        valid, res = check_medians_and_maps(crit_str, gts, preds, None)
    _, _, fl = native(crit_str).compute_frame_loss(gts, preds)
    assert isinstance(fl, torch.Tensor)                  # predictions are smaller than the gt: factor_loss is live
    check_against_fp64(crit_str, gts, preds, {}, upstream, valid, res)


def test_long_eval_sequence():
    """eval.py's criterion on a 64-frame 224 x 224 sequence: medians over 3.2 M pooled pixels, maps bit for bit."""
    gts, preds = to_dev(*data(1, 64, 224, 224, invalid=0.2, seed=10))
    with torch.no_grad():
        check_medians_and_maps(EVAL, gts, preds, None)
        crit = native(EVAL)
        gt, (pl, pr), gf, pf, masks, mon = crit.get_all_pts3d_t(gts, preds)
        out = lo.criterion(gts, preds, dtype=torch.float64, **oracle_kwargs(EVAL))
        for k, v in out["monitoring"].items():
            assert abs(float(mon[k]) - float(v)) <= K * U * 10 * (1 + abs(float(v))), k


def test_d_zero_pixels_have_zero_gradient():
    """Pixels whose prediction equals the ground truth exactly: d == 0, and the gradient there is 0 (torch's norm
    backward), with conf 1 and 1e30 around them."""
    crit_str = "ConfLoss_t(Regr3D_t(L21, norm_mode=False), alpha=0.4)"
    gts, preds = _prepare(conf_extremes)
    loss, _, fl = native(crit_str).compute_frame_loss(gts, preds)
    loss.backward()
    for (side, k), (p, c) in slot_tensors(preds).items():
        g = p.grad[:, :, 0::2]
        assert torch.isfinite(p.grad).all() and (g == 0).all(), (side, k)


def test_alpha_zero_against_fp64():
    """alpha = 0 (ConfLoss_t itself asserts alpha > 0, as the reference; the native layer takes it): loss = mean d c."""
    crit_str = TRAIN
    gts, preds = _prepare(lambda: data(2, 3, 16, 24, seed=11))
    pl = native(crit_str).pixel_loss
    _, loss, _, host = pl._frame_loss(gts, preds, True, 0.0)
    okw = dict(oracle_kwargs(crit_str), conf_alpha=0.0)
    out = lo.criterion(gts, preds, dtype=torch.float64, **okw)
    assert abs(float(loss) - float(out["loss"])) <= 1e-6 * abs(float(out["loss"]))


@pytest.mark.parametrize("name", sorted(synth.LOSS_ADV_CASES))
def test_native_matches_adversarial_goldens(name):
    """The reference's own values on the adversarial cases: NaN for NaN, ValueError where it raises, values within the
    fp32-vs-fp32 tolerance of the oracle's test (1e-5 maps and scalars, 1e-4 gradients, of |ref| + rms(ref))."""
    case = synth.LOSS_ADV_CASES[name]
    g = load_adv_golden(name)
    kw = case.get("kw", {})
    crit = native(case["criterion"])
    gts, preds = to_dev(*synth.make_loss_adv_case(name))
    pl = getattr(crit, "pixel_loss", crit)
    with torch.no_grad():
        gt, (pls, prs), gf, pf, masks, mon = (pl.get_all_pts3d_t(gts, preds, **kw) if kw
                                             else pl.get_all_pts3d_t(gts, preds))
    F = len(gts)
    for i in range(F):
        assert close(_np(gt[i]), g[f"gt_{i}"], 1e-5), i
        assert np.array_equal(_np(masks[i]), g[f"mask_{i}"])
    for k in range(F - 1):
        assert close(_np(pls[k]), g[f"pr_l_{k}"], 1e-5) and close(_np(prs[k]), g[f"pr_r_{k}"], 1e-5), k
    assert list(mon) == list(g["mon_keys"])
    assert close([float(v) for v in mon.values()], g["mon_vals"], 1e-5)
    if case["call"] != "loss":
        return
    gts, preds = _prepare(lambda: synth.make_loss_adv_case(name))
    if str(g["raises"]):
        with pytest.raises(ValueError, match="without a valid pixel"):
            crit.compute_frame_loss(gts, preds, **kw)
        return
    loss, details, fl = crit.compute_frame_loss(gts, preds, **kw)
    (loss + fl).backward()
    assert close(float(loss), g["loss"], 1e-5) and close(float(fl), g["factor_loss"], 1e-5)
    assert list(details) == list(g["detail_keys"])
    assert close([float(v) for v in details.values()], g["detail_vals"], 1e-5)
    for (side, k), (p, c) in slot_tensors(preds).items():
        ref = g[f"grad_pts_{side}_{k}"]
        fin = np.isfinite(ref).all(axis=-1)
        assert close(_np(p.grad)[fin], ref[fin], 1e-4), (side, k)
        assert (_np(p.grad)[~fin] == 0).all()
        gc = _np(c.grad) if c.grad is not None else np.zeros(c.shape, np.float32)
        assert close(gc, g[f"grad_conf_{side}_{k}"], 1e-4), (side, k)
