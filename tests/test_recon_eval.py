"""Reconstruction metrics on the GPU (spann3r_b200.recon_eval): eval.py:189-218 -- ICP, 30-NN normals, accuracy /
completion with normal consistency -- without host copies.

Checkers:
  * tests/golden/recon_eval.json: the reference's own spann3r/tools/eval_recon.py (scipy cKDTree) on the seeded clouds of
    synth.RECON_CASES (tools/make_golden_recon.py);
  * scipy itself, run here, for every nearest-neighbour query;
  * oracle/recon_eval_oracle.py (numpy + scipy) for the normals, the ICP loop and evaluate_reconstruction -- a restatement
    of Open3D's documented semantics; Open3D itself is not run;
  * the device math header compiled for the host (tests/native/recon_host_check.cpp) against numpy.
"""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from conftest import GOLDEN
from spann3r_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(GOLDEN, "recon_eval.json")))


def _case(i):
    return synth.make_recon_case(*synth.RECON_CASES[i])


def _ulp_close(a, b, ulps=1):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b) <= ulps * np.spacing(np.maximum(np.abs(a), np.abs(b)))


# ------------------------------------------------------------------------------------------------------------------
# CPU: the device math on the host, the oracle
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("recon") / "recon_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "recon_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.rc_umeyama.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.rc_smallest_eigvec.argtypes = [C.c_void_p, C.c_void_p]
    L.rc_knn_normal.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.rc_dist2.argtypes = [C.c_void_p] * 2
    L.rc_dist2.restype = C.c_double
    L.rc_box_lb2.argtypes = [C.c_void_p] * 3
    L.rc_box_lb2.restype = C.c_double
    return L


def _p(a):
    return a.ctypes.data


def _umeyama(L, src, dst, c=None):
    src, dst = np.ascontiguousarray(src, np.float64), np.ascontiguousarray(dst, np.float64)
    c = np.ascontiguousarray(np.zeros(3) if c is None else c, np.float64)
    T = np.zeros(12)
    L.rc_umeyama(_p(src), _p(dst), len(src), _p(c), _p(T))
    return T.reshape(3, 4)


def _np_umeyama(src, dst):
    ms, md = src.mean(0), dst.mean(0)
    S = (dst - md).T @ (src - ms) / len(src)
    U, _, Vt = np.linalg.svd(S)
    D = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        D[2, 2] = -1
    R = U @ D @ Vt
    return R, md - R @ ms


def test_umeyama_random_reflected_planar_collinear(host_lib):
    rng = np.random.default_rng(0)
    for trial in range(50):
        R = synth._rotation(rng.normal(0, 1, 3))
        t = rng.normal(0, 3, 3)
        src = rng.normal(0, 1, (40, 3)) + rng.normal(0, 5, 3)
        # random: exact recovery, with and without a shift of the sums
        for c in (None, rng.normal(0, 10, 3)):
            T = _umeyama(host_lib, src, src @ R.T + t, c)
            assert np.abs(T[:, :3] - R).max() < 1e-10 and np.abs(T[:, 3] - t).max() < 1e-9
        # planar (rank 2 covariance): still unique
        pl = src.copy()
        pl[:, 2] = 0.3
        T = _umeyama(host_lib, pl, pl @ R.T + t)
        assert np.abs(T[:, :3] - R).max() < 1e-10 and np.abs(T[:, 3] - t).max() < 1e-9
        # reflected target: the best PROPER rotation, as numpy's SVD with the det fix gives it
        M = R @ np.diag([1.0, 1.0, -1.0])
        dst = src @ M.T + t + rng.normal(0, 0.01, src.shape)
        T = _umeyama(host_lib, src, dst)
        Rn, tn = _np_umeyama(src, dst)
        assert abs(np.linalg.det(T[:, :3]) - 1) < 1e-12
        assert np.abs(T[:, :3] - Rn).max() < 1e-9 and np.abs(T[:, 3] - tn).max() < 1e-8
        # collinear (rank 1): not unique; any proper rotation that maps the line onto the line is optimal
        d = rng.normal(0, 1, 3)
        line = np.outer(rng.normal(0, 1, 30), d) + rng.normal(0, 1, 3)
        T = _umeyama(host_lib, line, line @ R.T + t)
        Rg = T[:, :3]
        assert np.abs(Rg @ Rg.T - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(Rg) - 1) < 1e-12
        assert np.abs(line @ Rg.T + T[:, 3] - (line @ R.T + t)).max() < 1e-9
    # no pairs -> identity
    T = np.zeros(12)
    host_lib.rc_umeyama(None, None, 0, _p(np.zeros(3)), _p(T))
    assert np.array_equal(T.reshape(3, 4), np.eye(3, 4))


def test_smallest_eigenvector_distinct_repeated_zero(host_lib):
    rng = np.random.default_rng(1)
    for _ in range(200):
        Q = synth._rotation(rng.normal(0, 2, 3))
        for w in (np.sort(rng.uniform(0.1, 10, 3)), np.array([0.0, 1.0, 4.0]), np.array([1e-9, 2.0, 3.0])):
            Cm = np.ascontiguousarray(Q @ np.diag(w) @ Q.T)
            n = np.zeros(3)
            host_lib.rc_smallest_eigvec(_p(Cm), _p(n))
            assert abs(np.linalg.norm(n) - 1) < 1e-14
            assert abs(abs(n @ Q[:, 0]) - 1) < 1e-9
        # repeated smallest eigenvalue: any unit vector of that eigenspace
        Cm = np.ascontiguousarray(Q @ np.diag([1.0, 1.0, 5.0]) @ Q.T)
        host_lib.rc_smallest_eigvec(_p(Cm), _p(n))
        assert abs(n @ Q[:, 2]) < 1e-9 and abs(np.linalg.norm(n) - 1) < 1e-14
        # triple: anything unit
        Cm = np.ascontiguousarray(np.eye(3) * 2.5)
        host_lib.rc_smallest_eigvec(_p(Cm), _p(n))
        assert abs(np.linalg.norm(n) - 1) < 1e-14
    host_lib.rc_smallest_eigvec(_p(np.zeros(9)), _p(n))
    assert n.tolist() == [0.0, 0.0, 1.0]
    # k-NN normal of a noisy plane, and the degenerate counts
    pts = np.ascontiguousarray(np.c_[rng.uniform(-1, 1, (30, 2)), 1e-3 * rng.normal(size=30)] @ Q.T + 7.0)
    host_lib.rc_knn_normal(_p(pts), 30, _p(n))
    ref = np.linalg.eigh(np.cov(pts.T, bias=True))[1][:, 0]
    assert abs(abs(n @ ref) - 1) < 1e-9
    for k in (1, 2):
        host_lib.rc_knn_normal(_p(pts), k, _p(n))
        assert n.tolist() == [0.0, 0.0, 1.0]
    host_lib.rc_knn_normal(_p(np.ascontiguousarray(np.ones((5, 3)))), 5, _p(n))
    assert n.tolist() == [0.0, 0.0, 1.0]


def test_box_lower_bound_never_exceeds_the_distance(host_lib):
    rng = np.random.default_rng(2)
    for scale in (1e-3, 1.0, 1e3):
        for _ in range(200):
            P = np.ascontiguousarray(rng.normal(0, 1, (32, 3)) * scale * rng.uniform(0.01, 1) + rng.normal(0, 5 * scale, 3))
            lo, hi = np.ascontiguousarray(P.min(0)), np.ascontiguousarray(P.max(0))
            for q in rng.normal(0, 5 * scale, (8, 3)).tolist() + P[:4].tolist():
                q = np.ascontiguousarray(q, np.float64)
                lb = host_lib.rc_box_lb2(_p(q), _p(lo), _p(hi))
                for p in P:
                    p = np.ascontiguousarray(p)
                    assert lb <= host_lib.rc_dist2(_p(q), _p(p))
    empty_lo, empty_hi = np.full(3, np.inf), np.full(3, -np.inf)
    assert host_lib.rc_box_lb2(_p(np.zeros(3)), _p(empty_lo), _p(empty_hi)) == math.inf


@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_oracle_matches_golden(i):
    from oracle import recon_eval_oracle as ro
    gt, pred, _ = _case(i)
    g = GOLD["cases"][i]
    gt64, pred64 = gt.astype(np.float64), pred.astype(np.float64)
    acc = ro.accuracy(gt64, pred64)
    comp = ro.completion(gt64, pred64)
    assert np.allclose(acc, g["accuracy"], rtol=1e-12, atol=0) and np.allclose(comp, g["completion"], rtol=1e-12, atol=0)


def test_oracle_icp_recovers_a_known_transform():
    from oracle import recon_eval_oracle as ro
    gt, pred, T = _case(4)
    reg = ro.registration_icp(pred, gt, 0.1)
    assert np.abs(reg["transformation"] - T).max() < 1e-6, reg["transformation"] - T
    assert reg["fitness"] == 1.0 and reg["inlier_rmse"] < 1e-6


def test_c_abi_rejects_bad_point_cloud_arguments():
    """Validation of the s3r_pcl_* entries happens before any CUDA call: status -1 and a message, no device needed."""
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_pcl_index_bytes(0) == 0 and L.s3r_pcl_index_bytes(2 ** 31) == 0 and L.s3r_pcl_index_bytes(1000) > 0
    assert L.s3r_pcl_index_build(None, 0, 10, None, None, None) == -1 and b"pcl_index_build" in L.s3r_last_error()
    fake = C.c_void_p(16)
    assert L.s3r_pcl_index_build(fake, 0, 0, None, fake, None) == -1
    assert L.s3r_pcl_index_build(fake, 0, 2 ** 31, None, fake, None) == -1
    assert L.s3r_pcl_nearest(fake, 10, fake, 0, 5, None, -1.0, fake, fake, None) == -1
    assert L.s3r_pcl_nearest(fake, 10, fake, 0, 5, None, float("nan"), fake, fake, None) == -1
    assert L.s3r_pcl_normals(fake, 10, 0, fake, None) == -1 and L.s3r_pcl_normals(fake, 10, 33, fake, None) == -1
    assert b"k=33" in L.s3r_last_error()
    assert L.s3r_pcl_icp(fake, 0, 10, fake, 10, -0.5, None, 30, 1e-6, 1e-6, fake, fake, None) == -1
    assert L.s3r_pcl_icp(fake, 0, 0, fake, 10, 0.5, None, 30, 1e-6, 1e-6, fake, fake, None) == -1
    assert L.s3r_pcl_stats(fake, 0, 0.0, fake, fake, None) == -1
    assert L.s3r_pcl_abs_dot(fake, fake, fake, 0, fake, None) == -1
    assert L.s3r_pcl_icp_workspace_bytes() > 0 and L.s3r_pcl_stats_workspace_bytes() > 0


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


def _check_nn(points, queries, d, idx):
    """d / idx from the GPU against scipy: <= 1 ulp; equal index where the nearest point is unique, else the smallest."""
    tree = cKDTree(points)
    k = min(8, len(points))
    ds, iss = tree.query(queries, k=k, workers=-1)
    ds, iss = ds.reshape(len(queries), k), iss.reshape(len(queries), k)
    assert _ulp_close(d, ds[:, 0]).all(), np.abs(d - ds[:, 0]).max()
    unique = ds[:, 1] > ds[:, 0] if k > 1 else np.ones(len(queries), bool)
    assert np.array_equal(idx[unique], iss[unique, 0])
    for r in np.nonzero(~unique)[0]:
        tied = iss[r][ds[r] == ds[r, 0]]
        assert len(tied) < k, "more ties than the check queried"
        assert idx[r] == tied.min(), (r, idx[r], tied)
    return float((d == ds[:, 0]).mean()), int((~unique).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_gpu_nearest_matches_scipy(i):
    from spann3r_b200 import recon_eval as re_
    gt, pred, _ = _case(i)
    gt64, pred64 = gt.astype(np.float64), pred.astype(np.float64)
    scale = synth.RECON_CASES[i][3]
    for pts, qs, pts_np, qs_np in ((gt, pred, gt64, pred64), (pred, gt, pred64, gt64)):
        d, idx = re_.nearest_neighbors(_cuda(qs), _cuda(pts))
        d, idx = d.cpu().numpy(), idx.cpu().numpy()
        bitwise, ties = _check_nn(pts_np, qs_np, d, idx)
        print(f"case {i}: N={len(pts)} Q={len(qs)} bitwise-equal to scipy {bitwise:.6f}, tied queries {ties}")
        # fp64 input gives the same answer as the exactly promoted fp32 input
        d64, idx64 = re_.nearest_neighbors(_cuda(qs, torch.float64), _cuda(pts, torch.float64))
        assert np.array_equal(d64.cpu().numpy(), d) and np.array_equal(idx64.cpu().numpy(), idx)
        # distance bound: -1 exactly where scipy's distance exceeds it
        md = float(np.median(d))
        dm, im = re_.nearest_neighbors(_cuda(qs), _cuda(pts), max_dist=md)
        dm, im = dm.cpu().numpy(), im.cpu().numpy()
        far = d > md
        assert np.array_equal(im == -1, far) and np.array_equal(im[~far], idx[~far]) and np.all(np.isinf(dm[far]))
    # a transformed query == the query of the pre-transformed points
    T = np.eye(4)
    T[:3, :3] = synth._rotation((0.1, -0.2, 0.3))
    T[:3, 3] = np.array([0.3, -0.1, 0.2]) * scale
    moved = pred64 @ T[:3, :3].T + T[:3, 3]
    dt, it = re_.nearest_neighbors(_cuda(pred), _cuda(gt), transform=torch.from_numpy(T))
    dp, ip = re_.nearest_neighbors(_cuda(moved, torch.float64), _cuda(gt))
    assert np.abs(dt.cpu().numpy() - dp.cpu().numpy()).max() <= 1e-12 * max(1.0, scale)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_gpu_metrics_match_golden(i):
    from spann3r_b200 import recon_eval as re_
    gt, pred, _ = _case(i)
    g = GOLD["cases"][i]
    acc = re_.accuracy(_cuda(gt), _cuda(pred))
    comp = re_.completion(_cuda(gt), _cuda(pred))
    ratio = re_.completion_ratio(_cuda(gt), _cuda(pred), dist_th=g["dist_th"])
    assert all(isinstance(v, float) for v in acc + comp) and isinstance(ratio, float)
    assert math.isclose(acc[0], g["accuracy"][0], rel_tol=1e-12) and math.isclose(comp[0], g["completion"][0], rel_tol=1e-12)
    assert _ulp_close(acc[1], g["accuracy"][1]) and _ulp_close(comp[1], g["completion"][1])
    assert ratio == g["completion_ratio"]
    s = g["sample"]
    d, idx = re_.nearest_neighbors(_cuda(pred)[s["query"]], _cuda(gt))
    assert _ulp_close(d.cpu().numpy(), s["dist"]).all()
    print(f"case {i}: sampled indices equal to scipy's {float(np.mean(idx.cpu().numpy() == np.array(s['index']))):.3f}")


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_gpu_normals_match_oracle(i):
    from oracle import recon_eval_oracle as ro
    from spann3r_b200 import recon_eval as re_
    for cloud in _case(i)[:2]:
        n_gpu = re_.estimate_normals(_cuda(cloud)).cpu().numpy()
        n_orc, diag = ro.knn_normals(cloud.astype(np.float64), 30, return_diagnostics=True)
        assert np.abs(np.linalg.norm(n_gpu, axis=1) - 1).max() < 1e-12
        if diag is None:                     # fewer than 3 points
            assert np.array_equal(n_gpu, n_orc)
            continue
        dk, dk1, w = diag
        well = (dk1 - dk > 1e-12 * dk1) & (w[:, 1] - w[:, 0] > 1e-6 * np.abs(w[:, 1]))
        dots = np.abs(np.sum(n_gpu * n_orc, axis=1))
        print(f"case {i}: N={len(cloud)} normals excluded as ill-posed {1 - well.mean():.4f}, "
              f"min |dot| on the rest {dots[well].min() if well.any() else float('nan'):.15f}")
        assert (dots[well] >= 1 - 1e-9).all()


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_gpu_icp_matches_oracle(i):
    from oracle import recon_eval_oracle as ro
    from spann3r_b200 import recon_eval as re_
    gt, pred, T_true = _case(i)
    scale = synth.RECON_CASES[i][3]
    thr = 0.1 * scale
    reg = re_.registration_icp(_cuda(pred), _cuda(gt), thr)
    orc = ro.registration_icp(pred.astype(np.float64), gt.astype(np.float64), thr)
    T = reg.transformation.cpu().numpy()
    print(f"case {i}: passes {reg.passes} (oracle {orc['passes']}), fitness {reg.fitness:.6f}, rmse {reg.inlier_rmse:.6e}, "
          f"max |dT| {np.abs(T - orc['transformation']).max():.2e}")
    assert reg.passes == orc["passes"]
    assert np.abs(T[:3, :3] - orc["transformation"][:3, :3]).max() < 1e-9
    assert np.abs(T[:3, 3] - orc["transformation"][:3, 3]).max() < 1e-9 * max(1.0, scale)
    assert all(abs(a - b) <= 2 for a, b in zip(reg.pass_correspondences, orc["pass_correspondences"]))
    assert math.isclose(reg.inlier_rmse, orc["inlier_rmse"], rel_tol=1e-9, abs_tol=1e-300)
    assert abs(reg.fitness - orc["fitness"]) <= 2 / len(pred)
    if synth.RECON_CASES[i][4] == 0 and synth.RECON_CASES[i][5] == 0 and len(pred) > 100:    # clean: the known transform
        assert np.abs(T - T_true).max() < 1e-6 * max(1.0, scale)


@pytest.mark.gpu
def test_gpu_icp_without_correspondences_and_with_init():
    from spann3r_b200 import recon_eval as re_
    gt, pred, T_true = _case(0)
    far = _cuda(pred + 1000.0)
    reg = re_.registration_icp(far, _cuda(gt), 0.1)
    assert np.array_equal(reg.transformation.cpu().numpy(), np.eye(4))
    assert reg.fitness == 0.0 and reg.inlier_rmse == 0.0 and reg.passes == 2
    # max_iteration = 0: one pass at the initial transform
    reg = re_.registration_icp(_cuda(pred), _cuda(gt), 0.1, init=T_true, max_iteration=0)
    assert reg.passes == 1 and np.array_equal(reg.transformation.cpu().numpy(), T_true)


@pytest.mark.gpu
def test_gpu_evaluate_reconstruction_end_to_end():
    from oracle import recon_eval_oracle as ro
    from spann3r_b200 import recon_eval as re_
    pts, pts_gt, masks = synth.make_eval_scene()
    args = (_cuda(pts), _cuda(pts_gt), torch.from_numpy(masks).cuda())
    m1 = re_.evaluate_reconstruction(*args, threshold=0.1)
    m2 = re_.evaluate_reconstruction(*args, threshold=0.1)
    assert tuple(m1) == tuple(m2)                               # bitwise identical
    orc = ro.evaluate_reconstruction(pts, pts_gt, masks, 0.1)
    print("gpu   ", m1)
    print("oracle", {k: v for k, v in orc.items() if k != "icp"}, "icp passes", orc["icp"]["passes"])
    for k in ("acc", "comp", "acc_med", "comp_med"):
        assert math.isclose(getattr(m1, k), orc[k], rel_tol=1e-9), (k, getattr(m1, k), orc[k])
    for k in ("nc1", "nc2", "nc1_med", "nc2_med"):
        assert abs(getattr(m1, k) - orc[k]) <= 1e-6, (k, getattr(m1, k), orc[k])


@pytest.mark.gpu
def test_gpu_inputs_are_validated():
    from spann3r_b200 import recon_eval as re_
    good = torch.rand(100, 3, device="cuda")
    bad_inputs = [good.cpu(), torch.rand(100, 2, device="cuda"), torch.rand(10, 3, 1, device="cuda"),
                  good.half(), good.long(), torch.empty(0, 3, device="cuda"), good.cpu().numpy()]
    nan = good.clone()
    nan[5, 1] = float("nan")
    inf = good.clone()
    inf[7, 2] = float("inf")
    bad_inputs += [nan, inf]
    for bad in bad_inputs:
        for call in (lambda: re_.nearest_neighbors(bad, good), lambda: re_.nearest_neighbors(good, bad),
                     lambda: re_.estimate_normals(bad), lambda: re_.registration_icp(bad, good, 0.1),
                     lambda: re_.accuracy(good, bad), lambda: re_.completion(bad, good),
                     lambda: re_.completion_ratio(good, bad)):
            with pytest.raises(ValueError):
                call()
    with pytest.raises(ValueError):
        re_.estimate_normals(good, knn=33)
    with pytest.raises(ValueError):
        re_.nearest_neighbors(good, good, max_dist=-1.0)
    with pytest.raises(ValueError):
        re_.evaluate_reconstruction(good.view(10, 10, 3), good.view(10, 10, 3), torch.ones(10, 9, device="cuda"), 0.1)
