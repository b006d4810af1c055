"""Reconstruction metrics on the GPU: the post-forward stages of the reference's eval.py:189-218 without host copies.

eval.py masks each reconstruction, registers it onto the ground truth with Open3D's point-to-point ICP, estimates 30-NN
normals on both clouds and calls `accuracy` / `completion` of spann3r/tools/eval_recon.py (scipy cKDTree queries in each
direction, mean and median distance, mean and median |n_gt . n_pred|).  The same calls are here, computed on the device by
libspann3r_b200.so (csrc/pointcloud.cu) over an exact spatial index; there is no CPU fallback.

Semantics that differ from the reference's libraries (INTEGRATION.md, "Reconstruction metrics on the GPU"):
  * nearest-neighbour ties break to the smallest point index (scipy's tie order depends on its tree);
  * the ICP and normal semantics restate Open3D's documented behaviour (registration_icp with
    TransformationEstimationPointToPoint and the default ICPConvergenceCriteria; estimate_normals with
    KDTreeSearchParamKNN(30)); Open3D itself was not run against this module.  Normals use a mean-centred covariance
    and keep the solver's sign; eval.py only reads |n . n|;
  * the `-mask.ply` / `-gt.ply` files are not written here: `spann3r_b200.vis.write_point_cloud` writes them.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import numpy as np
import torch

from . import _lib


def _points(x, name: str) -> torch.Tensor:
    if not isinstance(x, torch.Tensor):
        raise ValueError(f"{name}: expected a CUDA tensor [N, 3], got {type(x).__name__}")
    if not x.is_cuda:
        raise ValueError(f"{name}: expected a CUDA tensor, got one on {x.device}")
    if x.dtype not in (torch.float32, torch.float64) or x.dim() != 2 or x.shape[1] != 3:
        raise ValueError(f"{name}: expected [N, 3] float32 / float64, got {tuple(x.shape)} {x.dtype}")
    if not 1 <= x.shape[0] < 2 ** 31:
        raise ValueError(f"{name}: need 1 <= N < 2^31 points, got {x.shape[0]}")
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f"{name}: contains non-finite coordinates")
    return x.contiguous()


def _rigid(T, device, name: str):
    """4x4 (or 3x4) rigid transform -> contiguous fp64 [3, 4] on `device`, or None."""
    if T is None:
        return None
    T = torch.as_tensor(T, dtype=torch.float64)
    if tuple(T.shape) not in ((4, 4), (3, 4)):
        raise ValueError(f"{name}: expected a 4x4 or 3x4 transform, got {tuple(T.shape)}")
    if not bool(torch.isfinite(T).all()):
        raise ValueError(f"{name}: contains non-finite values")
    return T[:3].to(device).contiguous()


def _is_f64(x: torch.Tensor) -> int:
    return int(x.dtype == torch.float64)


class PointIndex:
    """Exact spatial index over one cloud [N, 3] (optionally under a rigid transform), built on the device.  It holds the
    cloud's points in fp64, so queries, normals and ICP against it need nothing else."""

    def __init__(self, points: torch.Tensor, transform=None, _device_rt: torch.Tensor | None = None):
        points = _points(points, "points")
        _lib.require_device()
        self.device = points.device
        self.n = points.shape[0]
        # _device_rt: a [3, 4] fp64 transform this module computed on the device (the ICP result), used as is
        T = _device_rt if _device_rt is not None else _rigid(transform, self.device, "transform")
        self.ws = torch.empty(int(_lib.lib().s3r_pcl_index_bytes(self.n)), dtype=torch.uint8, device=self.device)
        _lib.call("s3r_pcl_index_build", points, _lib.ptr(points), _is_f64(points), self.n, _lib.ptr(T), _lib.ptr(self.ws))

    def query(self, queries: torch.Tensor, max_dist: float = math.inf, transform=None):
        """1-NN of every query (each first mapped by `transform` if given) -> (dist [Q] fp64, idx [Q] int64).  Nothing within
        max_dist (inclusive) -> idx -1, dist inf.  Ties -> the smallest index."""
        queries = _points(queries, "queries")
        if queries.device != self.device:
            raise ValueError("queries and the indexed cloud must be on the same device")
        if not max_dist >= 0:
            raise ValueError(f"max_dist must be >= 0, got {max_dist}")
        T = _rigid(transform, self.device, "transform")
        nq = queries.shape[0]
        dist = torch.empty(nq, dtype=torch.float64, device=self.device)
        idx = torch.empty(nq, dtype=torch.int64, device=self.device)
        _lib.call("s3r_pcl_nearest", self.device, _lib.ptr(self.ws), self.n, _lib.ptr(queries), _is_f64(queries), nq,
                  _lib.ptr(T), float(max_dist), _lib.ptr(dist), _lib.ptr(idx))
        return dist, idx

    def normals(self, knn: int = 30) -> torch.Tensor:
        """[N, 3] fp64 unit normals of the indexed points from their `knn` nearest neighbours (themselves included)."""
        if not 1 <= int(knn) <= 32:
            raise ValueError(f"knn must be in 1..32, got {knn}")
        out = torch.empty(self.n, 3, dtype=torch.float64, device=self.device)
        _lib.call("s3r_pcl_normals", self.device, _lib.ptr(self.ws), self.n, int(knn), _lib.ptr(out))
        return out


def nearest_neighbors(queries: torch.Tensor, points: torch.Tensor, max_dist: float = math.inf, transform=None):
    """Exact 1-NN of every query among `points` (scipy's `cKDTree(points).query(queries)`), optionally after mapping the
    queries by a rigid `transform` (4x4 / 3x4) and bounded by `max_dist` -> (dist [Q] fp64, idx [Q] int64; -1 = none)."""
    return PointIndex(points).query(queries, max_dist, transform)


def estimate_normals(points: torch.Tensor, knn: int = 30) -> torch.Tensor:
    """`pcd.estimate_normals()` of eval.py:211-212 (Open3D's default KDTreeSearchParamKNN(30)) -> [N, 3] fp64."""
    return PointIndex(points).normals(knn)


class RegistrationResult:
    """What eval.py reads of Open3D's result: `.transformation` (4x4 fp64, on the device), `.fitness`, `.inlier_rmse`;
    plus `.passes` and the per-pass correspondence counts / inlier rmse."""

    def __init__(self, out: torch.Tensor, host: np.ndarray, max_iteration: int):
        self.transformation = out[:16].view(4, 4)
        self.fitness = float(host[16])
        self.inlier_rmse = float(host[17])
        self.passes = int(host[18])
        m = max_iteration + 1
        self.pass_correspondences = [int(v) for v in host[19: 19 + self.passes]]
        self.pass_rmse = [float(v) for v in host[19 + m: 19 + m + self.passes]]


def _icp(source: torch.Tensor, target: PointIndex, max_correspondence_distance, init, max_iteration, relative_fitness,
         relative_rmse) -> torch.Tensor:
    if not max_correspondence_distance >= 0:
        raise ValueError(f"max_correspondence_distance must be >= 0, got {max_correspondence_distance}")
    if not 0 <= int(max_iteration) <= 10000:
        raise ValueError(f"max_iteration must be in 0..10000, got {max_iteration}")
    T0 = _rigid(init, target.device, "init")
    ws = torch.empty(int(_lib.lib().s3r_pcl_icp_workspace_bytes()), dtype=torch.uint8, device=target.device)
    out = torch.empty(19 + 2 * (int(max_iteration) + 1), dtype=torch.float64, device=target.device)
    _lib.call("s3r_pcl_icp", target.device, _lib.ptr(source), _is_f64(source), source.shape[0], _lib.ptr(target.ws),
              target.n, float(max_correspondence_distance), _lib.ptr(T0), int(max_iteration), float(relative_fitness),
              float(relative_rmse), _lib.ptr(ws), _lib.ptr(out))
    return out


def registration_icp(source: torch.Tensor, target: torch.Tensor, max_correspondence_distance: float, init=None,
                     max_iteration: int = 30, relative_fitness: float = 1e-6, relative_rmse: float = 1e-6):
    """Point-to-point ICP of `source` onto `target` as eval.py:204-206 calls Open3D's
    `registration_icp(pcd, pcd_gt, threshold, trans_init, TransformationEstimationPointToPoint())` with the default
    ICPConvergenceCriteria (max_iteration 30, relative_fitness / relative_rmse 1e-6).  The iteration runs on the device
    without host synchronisation; one device->host copy reads fitness and rmse."""
    source = _points(source, "source")
    tgt = PointIndex(target)
    if source.device != tgt.device:
        raise ValueError("source and target must be on the same device")
    out = _icp(source, tgt, max_correspondence_distance, init, max_iteration, relative_fitness, relative_rmse)
    return RegistrationResult(out, out.cpu().numpy(), int(max_iteration))


def _stats_into(x: torch.Tensor, out: torch.Tensor, threshold: float = 0.0):
    """out[0:3] = mean, median, count(x < threshold) of the fp64 vector x (device, no synchronisation)."""
    ws = torch.empty(int(_lib.lib().s3r_pcl_stats_workspace_bytes()), dtype=torch.uint8, device=x.device)
    _lib.call("s3r_pcl_stats", x, _lib.ptr(x), x.numel(), float(threshold), _lib.ptr(ws), _lib.ptr(out))


def _abs_dot(a: torch.Tensor, b: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    out = torch.empty(a.shape[0], dtype=torch.float64, device=a.device)
    _lib.call("s3r_pcl_abs_dot", a, _lib.ptr(a), _lib.ptr(b), _lib.ptr(idx), a.shape[0], _lib.ptr(out))
    return out


def _normals(x, name: str, n: int) -> torch.Tensor:
    x = _points(x, name)
    if x.shape[0] != n:
        raise ValueError(f"{name}: {x.shape[0]} normals for {n} points")
    return x.to(torch.float64).contiguous()


def _one_direction(index: PointIndex, queries, idx_normals, q_normals, query_rt=None):
    """Distances from every query (mapped by the device [3, 4] transform query_rt if given) to the indexed cloud, and
    |n_index[nn] . n_query| -> (mean, median[, mean, median]) on the device."""
    if query_rt is None:
        dist, idx = index.query(queries)
    else:
        nq = queries.shape[0]
        dist = torch.empty(nq, dtype=torch.float64, device=index.device)
        idx = torch.empty(nq, dtype=torch.int64, device=index.device)
        _lib.call("s3r_pcl_nearest", index.device, _lib.ptr(index.ws), index.n, _lib.ptr(queries), _is_f64(queries), nq,
                  _lib.ptr(query_rt), math.inf, _lib.ptr(dist), _lib.ptr(idx))
    res = torch.empty(6, dtype=torch.float64, device=index.device)
    _stats_into(dist, res[0:3])
    if idx_normals is None:
        return res[0:2]
    _stats_into(_abs_dot(q_normals, idx_normals, idx), res[3:6])
    return torch.stack((res[0], res[1], res[3], res[4]))


def accuracy(gt_points, rec_points, gt_normals=None, rec_normals=None):
    """spann3r/tools/eval_recon.py `accuracy`: distances from every reconstructed point to the ground truth ->
    (mean, median) or, with both normal sets, (mean, median, mean |n . n|, median |n . n|) as Python floats."""
    gt = PointIndex(gt_points)
    rec = _points(rec_points, "rec_points")
    with_n = gt_normals is not None and rec_normals is not None
    gn = _normals(gt_normals, "gt_normals", gt.n) if with_n else None
    rn = _normals(rec_normals, "rec_normals", rec.shape[0]) if with_n else None
    return tuple(float(v) for v in _one_direction(gt, rec, gn, rn).cpu().tolist())


def completion(gt_points, rec_points, gt_normals=None, rec_normals=None):
    """spann3r/tools/eval_recon.py `completion`: distances from every ground-truth point to the reconstruction ->
    (mean, median) or, with both normal sets, (mean, median, mean |n . n|, median |n . n|) as Python floats."""
    rec = PointIndex(rec_points)
    gt = _points(gt_points, "gt_points")
    with_n = gt_normals is not None and rec_normals is not None
    gn = _normals(gt_normals, "gt_normals", gt.shape[0]) if with_n else None
    rn = _normals(rec_normals, "rec_normals", rec.n) if with_n else None
    return tuple(float(v) for v in _one_direction(rec, gt, rn, gn).cpu().tolist())


def completion_ratio(gt_points, rec_points, dist_th: float = 0.05) -> float:
    """spann3r/tools/eval_recon.py `completion_ratio`: the share of ground-truth points closer than dist_th to the
    reconstruction, rounded to float32 as np.mean of the float32 indicator returns it."""
    rec = PointIndex(rec_points)
    gt = _points(gt_points, "gt_points")
    dist, _ = rec.query(gt)
    res = torch.empty(3, dtype=torch.float64, device=rec.device)
    _stats_into(dist, res, dist_th)
    below = float(res[2].cpu())
    return float(np.float32(below / gt.shape[0]))


class ReconMetrics(NamedTuple):
    """The eight numbers eval.py:221 logs per scene, in its order."""
    acc: float
    comp: float
    nc1: float
    nc2: float
    acc_med: float
    comp_med: float
    nc1_med: float
    nc2_med: float


def evaluate_reconstruction(pts, pts_gt, masks, threshold: float, knn: int = 30) -> ReconMetrics:
    """eval.py:189-218 on the device: keep the points where masks > 0, register the prediction onto the ground truth by
    point-to-point ICP (max correspondence distance `threshold`: eval.py uses 100 on DTU, 0.1 elsewhere; identity
    start), estimate `knn`-NN normals of the transformed prediction and of the ground truth, then accuracy and completion
    with normal consistency.  pts, pts_gt [..., 3] and masks [...] on one CUDA device.  Each cloud's spatial index is built
    once and reused for ICP, normals and the queries; one device->host copy reads the eight numbers."""
    for name, x in (("pts", pts), ("pts_gt", pts_gt), ("masks", masks)):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise ValueError(f"{name}: expected a CUDA tensor")
    if pts.shape != pts_gt.shape or pts.shape[-1] != 3 or tuple(masks.shape) != tuple(pts.shape[:-1]):
        raise ValueError(f"expected pts, pts_gt [..., 3] and masks [...] of matching shapes, got {tuple(pts.shape)}, "
                         f"{tuple(pts_gt.shape)}, {tuple(masks.shape)}")
    keep = masks > 0
    pred = _points(pts[keep].reshape(-1, 3), "pts[masks > 0]")
    gt = _points(pts_gt[keep].reshape(-1, 3), "pts_gt[masks > 0]")
    gt_index = PointIndex(gt)
    out = _icp(pred, gt_index, threshold, None, 30, 1e-6, 1e-6)
    T = out[:12].view(3, 4)
    pred_index = PointIndex(pred, _device_rt=T)           # the transformed prediction, pcd.transform(transformation)
    n_gt = gt_index.normals(knn)
    n_pred = pred_index.normals(knn)
    acc = _one_direction(gt_index, pred, n_gt, n_pred, query_rt=T)
    comp = _one_direction(pred_index, gt, n_pred, n_gt)
    a, c = (v for v in torch.stack((acc, comp)).cpu().tolist())
    return ReconMetrics(acc=a[0], comp=c[0], nc1=a[2], nc2=c[2], acc_med=a[1], comp_med=c[1], nc1_med=a[3], nc2_med=c[3])
