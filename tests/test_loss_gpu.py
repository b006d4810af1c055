"""Spann3R's criteria on the H100 (spann3r_b200.loss over csrc/loss.cu): values and gradients against the reference's
goldens, gradients against fp64 autograd of the PyTorch restatement, exact medians, bitwise reproducibility, one
synchronising copy per compute_frame_loss and none in the backward, input checks, a training step of the model driven by
the native criterion, and the eval.py recipe of INTEGRATION.md."""
import warnings

import pytest
import torch

from oracle import loss_oracle as lo
from spann3r_b200 import synth
from test_loss_cpu import CASES, check_against_golden, grads_of, oracle_kwargs, rel, slot_tensors

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True)
def _restore_tf32():
    """Tests below turn TF32 off for their comparisons: give the tests after them the settings they started with."""
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def native(crit_str):
    ns = {}
    exec("from spann3r_b200.loss import *", ns)
    return eval(crit_str, ns)


def case_on_gpu(name, grad=True):
    case = synth.LOSS_CASES[name]
    gts, preds = synth.make_loss_case(**case["data"], device=DEV)
    if grad:
        for p, c in slot_tensors(preds).values():
            p.requires_grad_(True)
            c.requires_grad_(True)
    return case, gts, preds


def run_native(name):
    case, gts, preds = case_on_gpu(name, grad=case_is_loss(name))
    crit = native(case["criterion"])
    kw = case.get("kw", {})
    if case["call"] == "loss":
        loss, details, fl = crit.compute_frame_loss(gts, preds, **kw)
        (loss + fl).backward()
        return {"loss": loss, "factor_loss": fl, "details": details}, grads_of(preds)
    gt, (pl, pr), gf, pf, masks, mon = crit.get_all_pts3d_t(gts, preds, **kw)
    return {"gt_pts": gt, "pr_l": pl, "pr_r": pr, "gt_factor": gf, "pr_factor": pf, "masks": masks,
            "monitoring": mon}, None


def case_is_loss(name):
    return synth.LOSS_CASES[name]["call"] == "loss"


@pytest.mark.parametrize("name", CASES)
def test_native_matches_reference_goldens(name):
    out, grads = run_native(name)
    check_against_golden(name, out, grads, 1e-5, 1e-5, 1e-4)


@pytest.mark.parametrize("name", [n for n in CASES if case_is_loss(n)])
def test_gradients_match_fp64_autograd(name):
    case, gts, preds = case_on_gpu(name)
    loss, _, fl = native(case["criterion"]).compute_frame_loss(gts, preds, **case.get("kw", {}))
    (loss + fl).backward()
    ours = grads_of(preds)
    for p, c in slot_tensors(preds).values():
        p.grad = c.grad = None
    out = lo.criterion(gts, preds, dtype=torch.float64, dist_clip=case.get("kw", {}).get("dist_clip"),
                       **oracle_kwargs(case["criterion"]))
    (out["loss"] + out["factor_loss"]).backward()
    ref = grads_of(preds)
    for key in ours:
        assert rel(ours[key][0], ref[key][0]) < 1e-5, (key, rel(ours[key][0], ref[key][0]))
        if abs(ref[key][1]).sum() > 0:
            assert rel(ours[key][1], ref[key][1]) < 1e-5, key
    assert abs(float(loss) - float(out["loss"])) <= 1e-5 * abs(float(out["loss"]))


def _lower_median(vals, masks):
    cat = torch.cat([torch.where(m, v, torch.full_like(v, float("nan"))).reshape(len(v), -1) for v, m in zip(vals, masks)], 1)
    return torch.nanmedian(cat, dim=1).values


@pytest.mark.parametrize("name", ["eval", "even_pts"])
def test_medians_are_torch_nanmedian_of_the_native_points(name):
    case, gts, preds = case_on_gpu(name, grad=False)
    crit = native(case["criterion"])
    F = len(gts)
    plain = native("Regr3D_t(L21, norm_mode=False)")
    gtT, _, _, _, masks, _ = plain.get_all_pts3d_t(gts, preds)          # the transformed ground truth, unaligned
    call = crit._call(gts, preds)
    call.forward(maps=True)
    per_b = lambda i: call.per_b(i)                                          # noqa: E731
    gfac, pfac = per_b(0).view(-1, 1, 1, 1), per_b(1).view(-1, 1, 1, 1)
    pr = [p / pfac for p in call.pred[:F - 1] + [call.pred[-1]]]
    gt = [g / gfac for g in gtT]
    for pts, shift_i, scale_i in ((gt, 2, 4), (pr, 3, 5)):
        shift = _lower_median([p[..., 2] for p in pts], masks)
        assert torch.equal(shift, per_b(shift_i)), (shift, per_b(shift_i))
        s = shift.view(-1, 1, 1)
        sh = [torch.stack((p[..., 0], p[..., 1], p[..., 2] - s), -1) for p in pts]
        centre = torch.stack([_lower_median([p[..., i] for p in sh], masks) for i in range(3)], -1).view(-1, 1, 1, 3)
        nrm = []
        for p in sh:
            d = p - centre
            nrm.append((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]).sqrt())
        scale = _lower_median(nrm, masks)
        if scale_i == 5:
            scale = scale.clip(1e-3, 1e3)
        assert torch.equal(scale, per_b(scale_i)), (scale, per_b(scale_i))
    if name == "even_pts":   # all pixels valid: an even count per batch element, so the lower median is a real choice
        assert (F * gts[0]["pts3d"].shape[1] * gts[0]["pts3d"].shape[2]) % 2 == 0


def test_bitwise_reproducible():
    results = []
    for _ in range(2):
        case, gts, preds = case_on_gpu("train")
        loss, details, fl = native(case["criterion"]).compute_frame_loss(gts, preds)
        (loss + fl).backward()
        results.append((loss.item(), fl.item(), {k: float(v) for k, v in details.items()}, grads_of(preds)))
    a, b = results
    assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2]
    for key in a[3]:
        assert (a[3][key][0] == b[3][key][0]).all() and (a[3][key][1] == b[3][key][1]).all()


def test_one_synchronising_copy():
    case, gts, preds = case_on_gpu("train")
    crit = native(case["criterion"])
    crit.compute_frame_loss(gts, preds)       # warm-up: library load, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("warn")
    try:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            loss, details, fl = crit.compute_frame_loss(gts, preds)
        fwd = [x for x in w if "synchroniz" in str(x.message)]
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            (loss + fl).backward()
        bwd = [x for x in w if "synchroniz" in str(x.message)]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert len(fwd) == 1, [str(x.message) for x in fwd]
    assert len(bwd) == 0, [str(x.message) for x in bwd]


def test_invalid_inputs_raise_value_error():
    case, gts, preds = case_on_gpu("regr_mean", grad=False)
    crit = native(case["criterion"])
    bad = [dict(g) for g in gts]
    bad[1]["pts3d"] = bad[1]["pts3d"].double()
    with pytest.raises(ValueError, match="float32"):
        crit.compute_frame_loss(bad, preds)
    bad = [dict(g) for g in gts]
    bad[2]["valid_mask"] = bad[2]["valid_mask"][:, :-1]
    with pytest.raises(ValueError, match="shape"):
        crit.compute_frame_loss(bad, preds)
    bad = [dict(g) for g in gts]
    bad[0]["camera_pose"] = bad[0]["camera_pose"].cpu()
    with pytest.raises(ValueError, match="CUDA"):
        crit.compute_frame_loss(bad, preds)


def test_empty_term_under_confloss_raises():
    case, gts, preds = case_on_gpu("train", grad=False)
    gts[2]["valid_mask"] = torch.zeros_like(gts[2]["valid_mask"])
    with pytest.raises(ValueError, match="without a valid pixel"):
        native(case["criterion"]).compute_frame_loss(gts, preds)


def test_in_place_change_of_an_input_before_backward_is_rejected():
    case, gts, preds = case_on_gpu("regr_mean")
    loss, _, fl = native(case["criterion"]).compute_frame_loss(gts, preds)
    (loss + fl).backward(retain_graph=True)
    first = {k: (v[0].copy(), v[1].copy()) for k, v in grads_of(preds).items()}
    for p, c in slot_tensors(preds).values():
        p.grad = c.grad = None
    (loss + fl).backward(retain_graph=True)                   # a second backward through the same graph
    for key, (gp, _) in grads_of(preds).items():
        assert (gp == first[key][0]).all()
    with torch.no_grad():
        preds[1][0]["pts3d_in_other_view"].mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (loss + fl).backward()


def test_training_step_parameter_gradients_match_the_oracle_criterion():
    """One training-mode step of Spann3R (CUDA forward, recompute backward) driven by the native training criterion,
    against the same step driven by the PyTorch restatement of the criterion (fp64 autograd): parameter gradients on a
    sample of every stage, as tests/test_train_gpu.py samples them."""
    from conftest import get_state_dict, rel_l2
    from spann3r_b200 import Spann3R
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    model = Spann3R(dus3r_name=None, memory_dropout=0.0)
    model.load_state_dict(get_state_dict(True), strict=True)
    model = model.cuda()
    gts, _ = synth.make_loss_case(1, 3, 224, 224, invalid=0.3, seed=21, device=DEV)
    for g, f in zip(gts, synth.make_frames(3, 224, 224)):
        g["img"] = f["img"].to(DEV)
    crit_str = "ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)"
    watch = ["dust3r.enc_blocks.3.attn.qkv.weight", "dust3r.enc_norm.weight", "dust3r.dec_blocks.7.cross_attn.projk.weight",
             "dust3r.dec_blocks2.2.mlp.fc1.bias", "attn_head_2.0.weight", "norm_k.weight", "value_encoder.4.mlp.fc2.weight",
             "value_out.bias", "dust3r.downstream_head1.dpt.scratch.refinenet2.resConfUnit1.conv1.weight",
             "dust3r.downstream_head2.dpt.head.4.weight", "pos_patch_embed.proj.weight"]
    named = dict(model.named_parameters())
    grads, losses = {}, {}
    try:
        model.train()
        for arm in ("native", "oracle"):
            model.zero_grad(set_to_none=True)
            _, preds_all = model(gts)
            if arm == "native":
                loss, _, fl = native(crit_str).compute_frame_loss(gts, preds_all)
            else:
                out = lo.criterion(gts, preds_all, dtype=torch.float64, **oracle_kwargs(crit_str))
                loss, fl = out["loss"], out["factor_loss"]
            total = loss + fl
            total.backward()
            losses[arm] = float(total)
            grads[arm] = {k: named[k].grad.detach().clone() for k in watch}
    finally:
        model.zero_grad(set_to_none=True)
        model.eval()
    assert abs(losses["native"] - losses["oracle"]) <= 1e-5 * abs(losses["oracle"])
    errs = {k: rel_l2(grads["native"][k].cpu(), grads["oracle"][k].cpu()) for k in watch}
    print({k: "%.1e" % v for k, v in errs.items()})
    assert max(errs.values()) < 1e-4, errs


def _integration_eval_recipe():
    """The eval.py block of INTEGRATION.md ("Training and test criteria on the GPU"), as it stands there."""
    import os
    from conftest import ROOT
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    sec = text[text.index("## Training and test criteria on the GPU"):]
    sec = sec[sec.index("eval.py:128-218 on the device"):]
    start = sec.index("```python\n") + len("```python\n")
    return sec[start: sec.index("```", start)]


def _numpy_eval_py(gts, preds):
    """eval.py:128-189 in numpy: the criterion's points (the PyTorch restatement, fp32 on the CPU, standing in for the
    reference's criterion), gt_shift_z added back to z, geotrf by view 0's camera_pose, the valid masks."""
    import numpy as np
    cpu = lambda d: {k: v.cpu() for k, v in d.items()}                  # noqa: E731
    out = lo.criterion([cpu(g) for g in gts], [tuple(cpu(d) for d in p) for p in preds], norm_mode=False, gt_scale=True,
                       shift=True, scale=True, dtype=torch.float32)
    gt_shift_z = float(out["monitoring"]["gt_shift_z"])
    in_camera1 = gts[0]["camera_pose"][0].cpu().numpy()
    pred_pts = (out["pr_l"], out["pr_r"])
    pts_all, pts_gt_all, masks_all = [], [], []
    for j, view in enumerate(gts):
        pts = (pred_pts[0][j] if j < len(pred_pts[0]) else pred_pts[1][-1]).detach().numpy()[0].copy()
        pts_gt = out["gt_pts"][j].detach().numpy()[0].copy()
        pts[..., -1] += gt_shift_z
        pts = pts @ in_camera1[:3, :3].T + in_camera1[:3, 3]
        pts_gt[..., -1] += gt_shift_z
        pts_gt = pts_gt @ in_camera1[:3, :3].T + in_camera1[:3, 3]
        pts_all.append(pts[None])
        pts_gt_all.append(pts_gt[None])
        masks_all.append(view["valid_mask"].cpu().numpy()[0][None])
    return (np.concatenate(pts_all).astype(np.float32), np.concatenate(pts_gt_all).astype(np.float32),
            np.concatenate(masks_all))


def test_integration_eval_recipe_matches_numpy_eval_py():
    from spann3r_b200 import recon_eval
    torch.backends.cuda.matmul.allow_tf32 = False
    gts, preds = synth.make_loss_case(1, 4, 224, 224, invalid=0.2, seed=31, device=DEV)
    ns = {"torch": torch, "batch": gts, "preds": preds, "name_data": "synthetic"}
    exec(_integration_eval_recipe(), ns)
    ours = ns["metrics"]
    pts_all, pts_gt_all, masks_all = _numpy_eval_py(gts, preds)
    assert abs(ns["pts_all"].cpu().numpy() - pts_all).max() <= 1e-5 * abs(pts_all).max()
    ref = recon_eval.evaluate_reconstruction(torch.from_numpy(pts_all).to(DEV), torch.from_numpy(pts_gt_all).to(DEV),
                                             torch.from_numpy(masks_all).to(DEV), 0.1)
    for k, a, b in zip(ours._fields, ours, ref):
        assert abs(a - b) <= 1e-4 * abs(b) + 1e-7, (k, a, b)
