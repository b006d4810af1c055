"""Spann3R's criteria (spann3r_b200.loss) without a GPU: the PyTorch restatement (oracle/loss_oracle.py) against the
reference's own criteria (tests/golden/loss_*.npz, tools/make_golden_loss.py), the Python layer's argument checks and
the reference's criterion strings, and the sm_90a build of csrc/loss.cu (no spills)."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT
from oracle import loss_oracle as lo
from spann3r_b200 import synth

CASES = sorted(synth.LOSS_CASES)


def load_golden(name):
    return dict(np.load(os.path.join(GOLDEN, f"loss_{name}.npz")))


def oracle_kwargs(crit: str):
    """criterion string -> loss_oracle.criterion keyword arguments"""
    inner = crit
    conf_alpha = None
    m = re.match(r"ConfLoss_t\((.*), alpha=([0-9.]+)\)$", crit)
    if m:
        inner, conf_alpha = m.group(1), float(m.group(2))
    name = inner.split("(")[0]
    kw = {"conf_alpha": conf_alpha, "name": name, "shift": "Shift" in name, "scale": "Scale" in name}
    args = dict(norm_mode="avg_dis", gt_scale=False, fix_first=True)
    for k, v in re.findall(r"(\w+)=('[^']*'|\w+)", inner):
        args[k] = eval(v)
    kw.update(args)
    return kw


def _np(x):
    return x.detach().cpu().double().numpy() if isinstance(x, torch.Tensor) else np.asarray(x, np.float64)


def rel(a, b):
    a, b = _np(a), _np(b)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def check_against_golden(name, out, grads, tol_scalar, tol_map, tol_grad):
    """out: loss_oracle-shaped dict (tensors); grads: {(side, k): (dpts, dconf)} or None"""
    g = load_golden(name)
    sub = int(g["sub"])
    case = synth.LOSS_CASES[name]
    if case["call"] == "loss":
        assert abs(float(out["loss"]) - float(g["loss"])) <= tol_scalar * max(abs(float(g["loss"])), 1e-3)
        assert abs(float(out["factor_loss"]) - float(g["factor_loss"])) <= tol_scalar * max(abs(float(g["factor_loss"])), 1e-3)
        assert list(out["details"].keys()) == list(g["detail_keys"])
        for k, ref in zip(g["detail_keys"], g["detail_vals"]):
            v = float(out["details"][k])
            assert abs(v - ref) <= tol_scalar * max(abs(ref), 1e-3), (k, v, ref)
        for (s, k), (gp, gc) in grads.items():
            assert rel(gp[:, ::sub, ::sub], g[f"grad_pts_{s}_{k}"]) < tol_grad, (s, k)
            if np.abs(g[f"grad_conf_{s}_{k}"]).sum() > 0:
                assert rel(gc[:, ::sub, ::sub], g[f"grad_conf_{s}_{k}"]) < tol_grad, (s, k)
    else:
        for i, gt in enumerate(out["gt_pts"]):
            assert rel(gt[:, ::sub, ::sub], g[f"gt_{i}"]) < tol_map
            assert np.array_equal(_np(out["masks"][i][:, ::sub, ::sub]).astype(bool), g[f"mask_{i}"])
        for k in range(len(out["pr_l"])):
            assert rel(out["pr_l"][k][:, ::sub, ::sub], g[f"pr_l_{k}"]) < tol_map
            assert rel(out["pr_r"][k][:, ::sub, ::sub], g[f"pr_r_{k}"]) < tol_map
        for key in ("gt_factor", "pr_factor"):
            if g[key].size == 0:
                assert out[key] is None
            else:
                assert rel(out[key].flatten(), g[key]) < tol_scalar
        assert list(out["monitoring"].keys()) == list(g["mon_keys"])
        for k, ref in zip(g["mon_keys"], g["mon_vals"]):
            assert abs(float(out["monitoring"][k]) - ref) <= tol_scalar * max(abs(ref), 1e-3), k


def slot_tensors(preds):
    F = len(preds) + 1
    out = {}
    for k in range(F - 1):
        out[(0, k)] = (preds[k][0]["pts3d" if k == 0 else "pts3d_in_other_view"], preds[k][0]["conf"])
        out[(1, k)] = (preds[k][1]["pts3d_in_other_view"], preds[k][1]["conf"])
    return out


def grads_of(preds):
    return {key: (p.grad.detach().cpu().numpy(), c.grad.detach().cpu().numpy() if c.grad is not None else np.zeros(c.shape))
            for key, (p, c) in slot_tensors(preds).items()}


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_goldens(name):
    case = synth.LOSS_CASES[name]
    gts, preds = synth.make_loss_case(**case["data"])
    for p, c in slot_tensors(preds).values():
        p.requires_grad_(True)
        c.requires_grad_(True)
    out = lo.criterion(gts, preds, dtype=torch.float32, dist_clip=case.get("kw", {}).get("dist_clip"),
                       **oracle_kwargs(case["criterion"]))
    grads = None
    if case["call"] == "loss":
        (out["loss"] + out["factor_loss"]).backward()
        grads = grads_of(preds)
    out = {k: ([t.detach() for t in v] if isinstance(v, list) else v) for k, v in out.items()}
    check_against_golden(name, out, grads, 1e-5, 1e-6, 1e-4)


def test_golden_files_are_small():
    for name in CASES:
        assert os.path.getsize(os.path.join(GOLDEN, f"loss_{name}.npz")) < 1 << 20


def test_reference_criterion_strings_evaluate():
    ns = {}
    exec("from spann3r_b200.loss import *", ns)
    train = eval("ConfLoss_t(Regr3D_t(L21, norm_mode='avg_dis', fix_first=False), alpha=0.4)", ns)
    test = eval("Regr3D_t_ScaleShiftInv(L21, gt_scale=True)", ns)
    assert train.get_name().startswith("ConfLoss(Regr3D_t(") and train.alpha == 0.4
    assert train.pixel_loss.criterion.reduction == "none" and not train.pixel_loss.fix_first
    assert test.get_name() == "Regr3D_t_ScaleShiftInv(L21Loss())" and test._shift and test._scale and test.gt_scale
    assert isinstance(train, torch.nn.Module) and isinstance(test, torch.nn.Module)


def test_python_layer_validates_arguments():
    from spann3r_b200.loss import L21, ConfLoss_t, Regr3D_t, Regr3D_t_ScaleShiftInv
    with pytest.raises(NotImplementedError):
        Regr3D_t(L21, norm_mode="median_dis")
    with pytest.raises(NotImplementedError):
        Regr3D_t(L21) + Regr3D_t(L21)
    crit = ConfLoss_t(Regr3D_t(L21, norm_mode="avg_dis", fix_first=False), alpha=0.4)
    gts, preds = synth.make_loss_case(1, 3, 16, 16, seed=0)
    with pytest.raises(ValueError, match="CUDA"):            # CPU tensors
        crit.compute_frame_loss(gts, preds)
    with pytest.raises(ValueError, match="CUDA"):
        Regr3D_t_ScaleShiftInv(L21, gt_scale=True).get_all_pts3d_t(gts, preds)
    with pytest.raises(ValueError, match="pairs"):
        crit.compute_frame_loss(gts, preds[:1])
    bad = [tuple(dict(d) for d in p) for p in preds]
    bad[1][0]["pts3d"] = bad[1][0].pop("pts3d_in_other_view")
    with pytest.raises(ValueError, match="camera pose"):
        crit.compute_frame_loss(gts, bad)
    with pytest.raises(NotImplementedError):                 # a standalone criterion with reduction 'none'
        Regr3D_t(L21).with_reduction("none").compute_frame_loss(gts, preds)


def test_loss_cu_builds_without_spills(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not installed")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-Xptxas", "-v", "-c", os.path.join(ROOT, "spann3r_b200", "csrc", "loss.cu"), "-o",
                        str(tmp_path / "loss.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) >= 7 and all(s == ("0", "0") for s in spills), spills


def test_c_abi_rejects_bad_descriptors_without_a_device():
    import ctypes as C
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_abi_sizeof(3) == C.sizeof(_lib.LossDesc)
    d = _lib.LossDesc()
    d.frames, d.batch, d.height, d.width = 1, 1, 8, 8
    assert L.s3r_loss_workspace_bytes(C.byref(d)) == 0
    assert b"frames >= 2" in L.s3r_last_error()
    d.frames = 2
    assert L.s3r_loss_workspace_bytes(C.byref(d)) == 0                    # null pointers
    assert L.s3r_loss_forward(C.byref(d), None, 0, None, None, None, None, None) == -1
    assert L.s3r_loss_backward(C.byref(d), None, 0, None, None, None, None) == -1
    assert L.s3r_loss_forward(None, None, 0, None, None, None, None, None) == -1
    assert b"null descriptor" in L.s3r_last_error()
