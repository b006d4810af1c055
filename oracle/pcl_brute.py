"""ORACLE -- TEST INFRASTRUCTURE ONLY (imported by tests/ only; nothing under spann3r_b200/ touches it).

Tie-exact brute-force nearest neighbours in fp64, the checker of the spatial index in csrc/pointcloud.cu.  Every squared
distance is formed exactly as pointcloud_math.cuh's dist2 forms it, ((dx*dx + dy*dy) + dz*dz) with every step rounded,
by separate torch elementwise ops (no cdist, no matmul expansion, no pow, nothing a compiler could fuse into an FMA), so
the distances are bitwise the kernel's.  Queries under a rigid transform follow apply_rt: ((T0 x + T1 y) + T2 z) + t.

  * 1-NN: the minimum over all points, then the smallest original index among the exact minima.
  * k-NN: the first k points in the lexicographic order (d2, original index); `reverse_ties` takes the LARGEST indices
    among the points tied at the k-th distance instead (a wrong rule, which tests use to show that they tell the two
    apart).

Work runs in chunks of queries on the device of the points (CUDA or CPU).
"""
from __future__ import annotations

import math

import numpy as np
import torch

_CHUNK = 1 << 24          # pair distances per chunk


def _t64(x, device) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=torch.float64)
    return torch.as_tensor(np.asarray(x, np.float64), device=device)


def apply_rt(T, x: torch.Tensor) -> torch.Tensor:
    """x' = R x + t for a [3, 4] (or 4x4) rigid transform, each row summed as ((r0 x + r1 y) + r2 z) + t."""
    T = _t64(T, x.device)[:3]
    rows = []
    for r in range(3):
        a = T[r, 0] * x[:, 0]
        b = T[r, 1] * x[:, 1]
        c = T[r, 2] * x[:, 2]
        rows.append(((a + b) + c) + T[r, 3])
    return torch.stack(rows, 1)


def dist2(q: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """[m, n] squared distances between queries q [m, 3] and points p [n, 3], rounded like pointcloud_math.cuh."""
    dx = q[:, 0, None] - p[None, :, 0]
    dy = q[:, 1, None] - p[None, :, 1]
    dz = q[:, 2, None] - p[None, :, 2]
    xx = dx * dx
    yy = dy * dy
    zz = dz * dz
    return (xx + yy) + zz


class BruteIndex:
    """Brute-force stand-in for the spatial index over `points` [n, 3] (any float dtype; promoted to fp64 exactly)."""

    def __init__(self, points, device=None):
        if device is None:
            device = points.device if isinstance(points, torch.Tensor) else ("cuda" if torch.cuda.is_available() else "cpu")
        self.device = torch.device(device)
        self.pts = _t64(points, self.device).reshape(-1, 3).contiguous()
        self.n = self.pts.shape[0]
        self._ar = torch.arange(self.n, device=self.device)

    def _chunks(self, m: int):
        step = max(1, _CHUNK // self.n)
        for i in range(0, m, step):
            yield i, min(m, i + step)

    def nearest_d2(self, queries, transform=None):
        """-> (d2 [m] fp64, idx [m] int64) as torch tensors on the index's device."""
        q = _t64(queries, self.device).reshape(-1, 3)
        if transform is not None:
            q = apply_rt(transform, q)
        d2s, idxs = [], []
        for i0, i1 in self._chunks(q.shape[0]):
            d2 = dist2(q[i0:i1], self.pts)
            m = d2.min(1).values
            idx = torch.where(d2 == m[:, None], self._ar, self.n).min(1).values
            d2s.append(m)
            idxs.append(idx)
        return torch.cat(d2s), torch.cat(idxs)

    def nearest(self, queries, transform=None, max_dist: float = math.inf):
        """Like s3r_pcl_nearest: (dist, idx) with dist = sqrt(d2); nothing with dist <= max_dist -> (inf, -1)."""
        d2, idx = self.nearest_d2(queries, transform)
        d = torch.sqrt(d2)
        miss = d > max_dist
        return torch.where(miss, math.inf, d), torch.where(miss, -1, idx)

    def query(self, x, workers=-1):
        """cKDTree.query(x) for k = 1, as numpy arrays: lets oracle.recon_eval_oracle.registration_icp use this index."""
        d, idx = self.nearest(x)
        return d.cpu().numpy(), idx.cpu().numpy()

    def knn(self, queries, k: int, reverse_ties: bool = False) -> torch.Tensor:
        """[m, min(k, n)] original indices of the k nearest points of each query in the order (d2, index)."""
        q = _t64(queries, self.device).reshape(-1, 3)
        k = min(k, self.n)
        out = []
        for i0, i1 in self._chunks(q.shape[0]):
            d2 = dist2(q[i0:i1], self.pts)
            kth = torch.topk(d2, k, dim=1, largest=False).values[:, k - 1:k]
            below = d2 < kth
            tied = d2 == kth
            room = k - below.sum(1, keepdim=True)             # how many of the tied points fit
            if reverse_ties:
                rank = tied.flip(1).cumsum(1).flip(1)          # 1 for the largest tied index
            else:
                rank = tied.cumsum(1)                          # 1 for the smallest tied index
            take = below | (tied & (rank <= room))
            cols = take.nonzero()[:, 1].reshape(i1 - i0, k)    # ascending index within each row
            order = torch.sort(torch.gather(d2, 1, cols), dim=1, stable=True).indices
            out.append(torch.gather(cols, 1, order))
        return torch.cat(out)
