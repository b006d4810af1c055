"""ORACLE -- TEST INFRASTRUCTURE ONLY (imported by tests/ only; nothing under spann3r_b200/ touches it).

CPU restatement (numpy + scipy) of the post-forward stages of the reference's eval.py:189-218, the checker of
spann3r_b200.recon_eval:
  * k-NN normals (`pcd.estimate_normals()`, Open3D's default KDTreeSearchParamKNN(30)): the k nearest points of each
    point, itself included; the unit eigenvector of the smallest eigenvalue of their mean-centred covariance; (0, 0, 1)
    with fewer than 3 points or a zero covariance; sign as the solver returns it.
  * point-to-point ICP (`registration_icp(..., TransformationEstimationPointToPoint())`, default ICPConvergenceCriteria:
    max_iteration 30, relative_fitness 1e-6, relative_rmse 1e-6): pass j pairs each source point under T with its
    nearest target point within the correspondence distance (inclusive); fitness = pairs / source points, inlier_rmse =
    sqrt(sum d^2 / pairs) (0 without pairs); stop after pass j if j >= 1 and both changes against pass j-1 are below
    their thresholds, or j == max_iteration; else T <- Umeyama(pairs) T (no scaling, reflection fixed by det; identity
    without pairs).  The T of the last pass is returned with that pass's fitness and rmse.
  * accuracy / completion with normal consistency exactly as spann3r/tools/eval_recon.py computes them.

open3d is not installable here, so Open3D itself was never run against this restatement: the ICP and normal semantics
above are a restatement of Open3D's documented behaviour.  Known divergences from Open3D: Open3D transforms the source
cloud in place after every update (rounding accumulates differently from applying the composed T to the original
points, as here); its covariance is formed from raw moments in one pass (here mean-centred); it returns early with the
initial transform when the correspondence distance is <= 0; its eigen solver (and so the sign of a normal) differs.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


def box_centre(points: np.ndarray) -> np.ndarray:
    p = np.asarray(points, np.float64)
    return 0.5 * (p.min(0) + p.max(0))


def knn_normals(points: np.ndarray, k: int = 30, return_diagnostics: bool = False):
    """[N, 3] fp64 normals.  With return_diagnostics also (d_k, d_k+1, eigenvalues ascending) per point, which tell
    whether a point's normal is well-posed (unambiguous k-NN set, separated smallest eigenvalues)."""
    p = np.asarray(points, np.float64)
    n = len(p)
    ke = min(k, n)
    out = np.zeros((n, 3))
    out[:, 2] = 1.0
    diag = None
    if ke < 3:
        return (out, diag) if return_diagnostics else out
    tree = cKDTree(p)
    kq = min(ke + 1, n)
    d, idx = tree.query(p, k=kq, workers=-1)
    nb = p[idx[:, :ke]]                                  # [N, k, 3]
    mu = nb.mean(1, keepdims=True)
    dd = nb - mu
    C = np.einsum("nki,nkj->nij", dd, dd) / ke
    w, V = np.linalg.eigh(C)
    out = V[:, :, 0].copy()
    zero = np.abs(C).reshape(n, 9).max(1) == 0
    out[zero] = (0.0, 0.0, 1.0)
    if return_diagnostics:
        dk1 = d[:, ke] if kq > ke else np.full(n, np.inf)
        diag = (d[:, ke - 1], dk1, w)
    return (out, diag) if return_diagnostics else out


def _umeyama(ps: np.ndarray, qs: np.ndarray, c: np.ndarray) -> np.ndarray:
    """3x4 [R | t] with q ~ R p + t from paired points given relative to the shift c."""
    T = np.zeros((3, 4))
    T[:, :3] = np.eye(3)
    n = len(ps)
    if n == 0:
        return T
    ms, md = ps.sum(0) / n, qs.sum(0) / n
    S = (qs.T @ ps) / n - np.outer(md, ms)              # cov(dst, src)
    U, _, Vt = np.linalg.svd(S)
    D = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        D[2, 2] = -1
    R = U @ D @ Vt
    T[:, :3] = R
    T[:, 3] = (md - R @ ms) + (c - R @ c)
    return T


def _apply(T: np.ndarray, p: np.ndarray) -> np.ndarray:
    return p @ T[:3, :3].T + T[:3, 3]


def registration_icp(source, target, max_correspondence_distance: float, init=None, max_iteration: int = 30,
                     relative_fitness: float = 1e-6, relative_rmse: float = 1e-6, target_tree=None):
    """-> dict(transformation 4x4, fitness, inlier_rmse, passes, pass_correspondences, pass_rmse)."""
    src = np.asarray(source, np.float64)
    tgt = np.asarray(target, np.float64)
    tree = target_tree if target_tree is not None else cKDTree(tgt)
    c = box_centre(tgt)
    T = np.eye(4) if init is None else np.asarray(init, np.float64).copy()
    counts, rmses = [], []
    prev = None
    j = 0
    while True:
        x = _apply(T, src)
        d, idx = tree.query(x, workers=-1)
        ok = d <= max_correspondence_distance
        cnt = int(ok.sum())
        fitness = cnt / len(src)
        rmse = float(np.sqrt(np.sum(d[ok] ** 2) / cnt)) if cnt else 0.0
        counts.append(cnt)
        rmses.append(rmse)
        if (j >= 1 and abs(prev[0] - fitness) < relative_fitness and abs(prev[1] - rmse) < relative_rmse) or j == max_iteration:
            break
        U = np.eye(4)
        U[:3] = _umeyama(x[ok] - c, tgt[idx[ok]] - c, c)
        T = U @ T
        prev = (fitness, rmse)
        j += 1
    return {"transformation": T, "fitness": fitness, "inlier_rmse": rmse, "passes": j + 1,
            "pass_correspondences": counts, "pass_rmse": rmses}


def accuracy(gt_points, rec_points, gt_normals=None, rec_normals=None, tree=None):
    tree = tree if tree is not None else cKDTree(gt_points)
    distances, idx = tree.query(rec_points, workers=-1)
    res = [np.mean(distances), np.median(distances)]
    if gt_normals is not None and rec_normals is not None:
        nd = np.abs(np.sum(gt_normals[idx] * rec_normals, axis=-1))
        res += [np.mean(nd), np.median(nd)]
    return tuple(float(v) for v in res)


def completion(gt_points, rec_points, gt_normals=None, rec_normals=None, tree=None):
    tree = tree if tree is not None else cKDTree(rec_points)
    distances, idx = tree.query(gt_points, workers=-1)
    res = [np.mean(distances), np.median(distances)]
    if gt_normals is not None and rec_normals is not None:
        nd = np.abs(np.sum(gt_normals * rec_normals[idx], axis=-1))
        res += [np.mean(nd), np.median(nd)]
    return tuple(float(v) for v in res)


def evaluate_reconstruction(pts, pts_gt, masks, threshold: float, knn: int = 30) -> dict:
    """eval.py:189-218 in numpy: mask, ICP, normals of the transformed prediction and of the ground truth, accuracy and
    completion -> the eight numbers eval.py logs (plus the ICP result)."""
    keep = np.asarray(masks) > 0
    pred = np.asarray(pts, np.float64)[keep].reshape(-1, 3)
    gt = np.asarray(pts_gt, np.float64)[keep].reshape(-1, 3)
    gt_tree = cKDTree(gt)
    reg = registration_icp(pred, gt, threshold, target_tree=gt_tree)
    pred_t = _apply(reg["transformation"], pred)
    n_pred = knn_normals(pred_t, knn)
    n_gt = knn_normals(gt, knn)
    acc, acc_med, nc1, nc1_med = accuracy(gt, pred_t, n_gt, n_pred, tree=gt_tree)
    comp, comp_med, nc2, nc2_med = completion(gt, pred_t, n_gt, n_pred)
    return {"acc": acc, "comp": comp, "nc1": nc1, "nc2": nc2, "acc_med": acc_med, "comp_med": comp_med,
            "nc1_med": nc1_med, "nc2_med": nc2_med, "icp": reg}
