"""The post-path geometry on adversarial pointmaps: the focal estimate (`s3r_focal_weiszfeld` / `s3r_focal_median`) and
PnP-RANSAC (`s3r_pnp_ransac`) on NaN / +-inf / z = 0 / behind-camera points, degenerate shapes, subnormal products and
frames nothing can solve.  The frames are seeded builders in spann3r_b200/synth.py (FOCAL_ADV_CASES, PNP_ADV_CASES).

Focal: golden values from the REAL reference (tools/make_golden_focal_adv.py -> tests/golden/focal_adv.json) with the
fp64 weiszfeld value beside them.  The kernel's weiszfeld result is held to fp64 within 16 times the reference's own fp32
error (floor 1e-6 relative), NaN exactly where the reference is NaN; the median is an element of the vote set, so it is
held bit for bit.

PnP: no cv2 golden (its behaviour on NaN input is not a contract); instead every result is checked in fp64 against the
problem it claims to solve -- (a) the host build of the same header with the same seed, (b) the reported inlier count is
the returned mask's, (c) the reported RMS error is the masked points' error at the returned pose, (d) the pose is a
stationary point of the masked least-squares problem (scipy LM), (e) without refinement the mask is exactly the
threshold test at the RANSAC model, (f) R is a rotation and rvec its logarithm, (g) unsolvable frames fail cleanly
without disturbing their batch neighbours."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from spann3r_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = {c["name"]: c for c in json.load(open(os.path.join(GOLDEN, "focal_adv.json")))["cases"]}
FOCAL = list(synth.FOCAL_ADV_CASES)
HOST_PNP = [n for n in synth.PNP_ADV_CASES if n != "hd"]     # at most 512 x 384: the host loop runs in seconds
UNSOLVABLE = ("three_finite", "all_behind", "all_nan", "three_finite_dense")


def _pp(c):
    return (c["W"] / 2, c["H"] / 2)


def _nan_equal(got, want):
    """Value-level equality (-0.0 == 0.0) with NaN matching NaN only."""
    return all((math.isnan(a) and math.isnan(b)) or a == b for a, b in zip(got, want)) and len(got) == len(want)


def _clip0(f):   # the reference's clip(min=0, max=inf), NaN kept
    return f if math.isnan(f) else max(f, 0.0)


# ------------------------------------------------------------------------------------------------------------------
# focal: CPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FOCAL)
def test_focal_oracle_fp32_reproduces_reference_golden(name):
    from oracle.postprocess_oracle import focal_median, focal_weiszfeld
    c = GOLD[name]
    pts = synth.make_focal_adv_case(name)
    assert tuple(pts.shape) == (c["B"], c["H"], c["W"], 3)
    for a, g in zip(focal_weiszfeld(pts, _pp(c)).tolist(), c["focal"]):
        assert math.isnan(a) == math.isnan(g), (a, g)
        assert math.isnan(g) or abs(a - g) <= 2e-6 * abs(g), (a, g)
    assert _nan_equal(focal_median(pts, _pp(c)).tolist(), c["focal_median"])
    for a, g in zip(focal_weiszfeld(pts.double(), _pp(c)).tolist(), c["focal_f64"]):   # the fp64 yardstick
        assert math.isnan(a) == math.isnan(g) and (math.isnan(g) or abs(a - g) <= 1e-12 * abs(g)), (a, g)


@pytest.fixture(scope="module")
def focal_host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("focal") / "focal_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "focal_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.focal_median_host.restype = C.c_float
    L.focal_median_host.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float]
    return L


@pytest.mark.parametrize("name", FOCAL)
def test_focal_median_device_math_on_host_equals_golden(focal_host, name):
    """focal_math.cuh's votes and keys through the kernels' 4 x 8-bit radix select, on the host, then the reference's
    clip(min=0) -- the golden median on every frame, NaN where it is NaN."""
    c = GOLD[name]
    pts = synth.make_focal_adv_case(name)
    got = []
    for b in range(c["B"]):
        p = pts[b].contiguous()
        got.append(_clip0(focal_host.focal_median_host(p.data_ptr(), c["H"], c["W"], c["W"] / 2, c["H"] / 2)))
    assert _nan_equal(got, c["focal_median"]), (got, c["focal_median"])


def test_focal_golden_spans_the_adversarial_cases():
    """The frames do reach the edges they are named for, in the reference itself."""
    g = GOLD
    assert math.isnan(g["all_z0"]["focal"][0]) and g["all_z0"]["focal_median"] == [0.0]
    assert math.isnan(g["all_nan"]["focal"][0]) and math.isnan(g["all_nan"]["focal_median"][0])
    assert math.isnan(g["underflow"]["focal"][0]) and 1e23 < g["underflow"]["focal_f64"][0] < 1e24
    assert g["med_plus_inf"]["focal_median"] == [math.inf] and g["med_identical"]["focal_median"] == [64.0]
    m = g["mixed"]["focal"]
    assert math.isfinite(m[0]) and math.isnan(m[1]) and math.isnan(m[2]) and math.isfinite(m[3])
    for c in g.values():   # the reference's own fp32 error, the yardstick of the kernel bound
        for e, f in zip(c["ref_err"], c["focal_f64"]):
            assert math.isnan(e) or e <= 1e-6 * abs(f), (c["name"], e, f)


# ------------------------------------------------------------------------------------------------------------------
# focal: GPU
# ------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.contiguous().view(torch.int32).cpu().tolist()


def _subnormal_bound(pts, f64):
    """Relative error bound of the fp32 sum sum(w a.a) on a frame whose a.a terms are subnormal (`underflow`), at the
    fp64 solution: there each square, the w * (a.a) product and the running-sum addition round with an absolute error
    of up to 2^-150 (half the subnormal spacing) instead of a relative one, so the sum's error is at most
    sum(2 w + 2) * 2^-150, against sum(w a.a).  The ratio f = sum(w a.p) / sum(w a.a) inherits that relative error (the
    numerator's terms are normal).  On the `underflow` frame this is ~0.6: fp32 has no precision left there."""
    B, H, W, _ = pts.shape
    jj, ii = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    p = torch.stack((ii - W / 2, jj - H / 2), -1).reshape(-1, 2)
    a = (pts[..., :2].double() / pts[..., 2:3].double()).reshape(-1, 2).nan_to_num(posinf=0, neginf=0)
    w = 1 / (p - f64 * a).norm(dim=-1).clamp(min=1e-8)
    return float(((2 * w + 2) * 2.0 ** -150).sum() / (w * (a * a).sum(-1)).sum())


def _weiszfeld_ok(f, c, b, pts):
    """|f_gpu - f64| <= max(16 |f_ref32 - f64|, 1e-6 |f64|); NaN exactly where the reference is NaN.  On the `underflow`
    frame the reference's fp32 sum of subnormal a.a terms rounds to 0 (NaN) while the kernel's FMA keeps a tiny
    nonzero sum: there either NaN or a value within the subnormal rounding bound of fp64 is right."""
    ref, f64, err = c["focal"][b], c["focal_f64"][b], c["ref_err"][b]
    if math.isnan(ref) and not c["underflow"]:
        return math.isnan(f)
    if math.isnan(f):
        return math.isnan(ref)
    bound = max(16 * err, 1e-6 * abs(f64)) if not math.isnan(err) else 1e-6 * abs(f64)
    if c["underflow"]:
        bound = max(bound, _subnormal_bound(pts[b:b + 1], f64) * abs(f64))
    return math.isfinite(f) and abs(f - f64) <= bound


@pytest.mark.gpu
def test_cuda_focal_weiszfeld_adversarial():
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    bad = []
    for name in FOCAL:
        c = GOLD[name]
        pts = synth.make_focal_adv_case(name)
        f = estimate_focal_knowing_depth(pts.cuda(), _pp(c), focal_mode="weiszfeld").tolist()
        for b in range(c["B"]):
            print(f"{name}[{b}]: gpu {f[b]!r} ref32 {c['focal'][b]!r} f64 {c['focal_f64'][b]!r}")
            if not _weiszfeld_ok(f[b], c, b, pts):
                bad.append((name, b, f[b], c["focal"][b], c["focal_f64"][b]))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["weiszfeld", "median"])
def test_cuda_focal_batch_equals_single_frames(mode):
    """Every frame of a batch, valid or not, is bit-identical to its single-frame run."""
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    for name in ("mixed", "h1", "w1"):
        pts = synth.make_focal_adv_case(name).cuda()
        pp = _pp(GOLD[name])
        batch = estimate_focal_knowing_depth(pts, pp, focal_mode=mode)
        for b in range(pts.shape[0]):
            assert _bits(estimate_focal_knowing_depth(pts[b:b + 1], pp, focal_mode=mode)) == _bits(batch[b:b + 1]), (name, b)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["weiszfeld", "median"])
def test_cuda_focal_clip_keeps_nan(mode):
    """min_focal / max_focal clip the valid frames exactly like torch.clip and leave a NaN focal NaN."""
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    c = GOLD["mixed"]
    pts = synth.make_focal_adv_case("mixed").cuda()
    base = max(c["H"], c["W"]) / (2 * math.tan(math.radians(60) / 2))
    free = estimate_focal_knowing_depth(pts, _pp(c), focal_mode=mode).cpu()
    for lo, hi in ((0.5, 1.0), (2.0, math.inf), (0.0, 0.9), (1.0, 1.0)):
        f = estimate_focal_knowing_depth(pts, _pp(c), focal_mode=mode, min_focal=lo, max_focal=hi).cpu()
        want = free.clip(min=lo * base, max=hi * base)
        assert torch.isnan(f).tolist() == [False, True, mode == "weiszfeld", False], (lo, hi, f)
        assert _nan_equal(f.tolist(), want.tolist()), (lo, hi, f, want)


@pytest.mark.gpu
def test_cuda_focal_median_adversarial():
    from spann3r_b200.postprocess import estimate_focal_knowing_depth
    for name in FOCAL:
        c = GOLD[name]
        f = estimate_focal_knowing_depth(synth.make_focal_adv_case(name).cuda(), _pp(c), focal_mode="median").tolist()
        assert _nan_equal(f, c["focal_median"]), (name, f, c["focal_median"])


# ------------------------------------------------------------------------------------------------------------------
# PnP: fp64 checks shared by the host build and the CUDA path
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pnp_host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pnp") / "pnp_host_check.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "pnp_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.pnp_host_check.restype = C.c_int
    L.pnp_host_check.argtypes = ([C.c_void_p, C.c_void_p, C.c_longlong, C.c_int] + [C.c_double] * 5 +
                                 [C.c_int, C.c_int, C.c_ulonglong, C.c_void_p, C.c_void_p])
    return L


def _frame(name):
    pts, img, K = synth.make_pnp_adv_case(name)
    width = 0 if img is not None else pts.shape[1]
    return np.ascontiguousarray(pts.reshape(-1, 3)), None if img is None else np.ascontiguousarray(img), width, K


def _host(L, pts, img, width, K, thr=8.0, samples=100, iters=15, seed=0):
    out = np.zeros(18)
    mask = np.zeros(len(pts), np.uint8)
    ok = L.pnp_host_check(pts.ctypes.data, None if img is None else img.ctypes.data, len(pts), width, K[0, 0], K[1, 1],
                          K[0, 2], K[1, 2], thr, samples, iters, seed, out.ctypes.data, mask.ctypes.data)
    return ok, out, mask.astype(bool)


def _points(pts, img, width):
    """fp64 world points, their pixels and load_point's validity (finite, |x + y + z + u + v| < 1e30)."""
    X = pts.astype(np.float64)
    if img is None:
        i = np.arange(len(pts))
        uv = np.stack((i % width, i // width), -1).astype(np.float64)
    else:
        uv = img.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        s = X[:, 0] + X[:, 1] + X[:, 2] + uv[:, 0] + uv[:, 1]
        return X, uv, (s == s) & (np.abs(s) < 1e30)


def _err2(R, t, K, X, uv, valid):
    """Squared reprojection error at (R, t) in fp64; +inf for invalid points and points not in front of the camera."""
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        Xc = X @ R.T + t
        du = K[0, 0] * Xc[:, 0] / Xc[:, 2] + K[0, 2] - uv[:, 0]
        dv = K[1, 1] * Xc[:, 1] / Xc[:, 2] + K[1, 2] - uv[:, 1]
        e = du * du + dv * dv
    return np.where(valid & (Xc[:, 2] > 1e-12) & (e == e), e, np.inf)


def _rot(rv):
    th = np.linalg.norm(rv)
    if th < 1e-12:
        return np.eye(3)
    k = rv / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _check_result(tag, out, mask, pts, img, width, K, thr=8.0, refined=True):
    """Checks b, c, e (when not refined), f on one frame's result; d separately (it is the slow one)."""
    R, t, rvec = out[:9].reshape(3, 3), out[9:12], out[12:15]
    n_in = int(mask.sum())
    assert out[15] == n_in, (tag, "b: reported inliers", out[15], n_in)
    if out[17] == 0:
        assert n_in == 0 and out[16] == 0, (tag, "g: failed frame with a mask", n_in, out[16])
        return
    X, uv, valid = _points(pts, img, width)
    e2 = _err2(R, t, K, X, uv, valid)
    sse = float(e2[mask].sum())
    # 1e-9 relative, plus the rounding of the residuals themselves (~1e-12 px each) when the fit is exact
    tol = 1e-9 * sse + 4e-12 * math.sqrt(n_in * sse)
    assert abs(out[16] ** 2 * n_in - sse) <= tol, (tag, "c: RMS vs masked error", out[16] ** 2 * n_in, sse)
    if not refined:
        want = e2 < thr * thr
        near = np.abs(e2 - thr * thr) <= 1e-9 * thr * thr
        bad = int(((mask != want) & ~near).sum())
        assert bad == 0, (tag, "e: mask vs threshold test at T", bad)
    assert np.abs(R.T @ R - np.eye(3)).max() < 1e-12 and abs(np.linalg.det(R) - 1) < 1e-12, (tag, "f: R", R)
    assert np.abs(_rot(rvec) - R).max() < 1e-12, (tag, "f: rvec != log R", rvec)


def _check_stationary(tag, out, mask, pts, img, width, K):
    """d: scipy's LM from the returned pose, on the masked correspondences in fp64, finds nothing better."""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    if out[17] == 0 or mask.sum() > 200_000:
        return
    X, uv, _ = _points(pts, img, width)
    X, uv = X[mask], uv[mask]

    def res(p):
        Xc = X @ Rotation.from_rotvec(p[:3]).as_matrix().T + p[3:]
        return np.concatenate((K[0, 0] * Xc[:, 0] / Xc[:, 2] + K[0, 2] - uv[:, 0],
                               K[1, 1] * Xc[:, 1] / Xc[:, 2] + K[1, 2] - uv[:, 1]))

    p0 = np.concatenate((out[12:15], out[9:12]))
    c0 = 0.5 * float(np.sum(res(p0) ** 2))
    r = least_squares(res, p0, method="lm", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    assert r.cost >= c0 * (1 - 1e-8) - 1e-18, (tag, "d: LM lowers the cost", c0, r.cost)
    assert np.abs(r.x - p0).max() < 1e-6, (tag, "d: LM moves the pose", r.x - p0)


@pytest.mark.parametrize("name", HOST_PNP)
def test_pnp_device_math_on_host_adversarial(pnp_host, name):
    pts, img, width, K = _frame(name)
    ok, out, mask = _host(pnp_host, pts, img, width, K)
    print(f"{name}: success {ok} inliers {int(mask.sum())} rms {out[16]:.3e}")
    assert ok == (name not in UNSOLVABLE)
    _check_result(name, out, mask, pts, img, width, K)
    _check_stationary(name, out, mask, pts, img, width, K)
    for thr in (0.5, 8.0, 50.0):
        ok, out, mask = _host(pnp_host, pts, img, width, K, thr=thr, iters=0)
        _check_result(f"{name} thr {thr}", out, mask, pts, img, width, K, thr=thr, refined=False)


# ------------------------------------------------------------------------------------------------------------------
# PnP: GPU, through the C ABI (out[15] and out[16] are not in the Python API's result)
# ------------------------------------------------------------------------------------------------------------------
def _gpu(pts, img, width, K, thr=8.0, samples=100, iters=15, seed=0):
    """pts [B, n, 3] / img [B, n, 2] or None (numpy) -> out [B, 18], mask [B, n] bool."""
    from spann3r_b200 import _lib
    L = _lib.lib()
    B, n = pts.shape[:2]
    p = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    im = None if img is None else torch.from_numpy(np.ascontiguousarray(img)).cuda()
    ws = torch.empty(int(L.s3r_pnp_workspace_bytes(B, samples)), dtype=torch.uint8, device="cuda")
    out = torch.empty(B, 18, dtype=torch.float64, device="cuda")
    mask = torch.empty(B, n, dtype=torch.uint8, device="cuda")
    _lib.check(L.s3r_pnp_ransac(_lib.ptr(p), _lib.ptr(im), B, n, width, K[0, 0], K[1, 1], K[0, 2], K[1, 2], thr, samples,
                                iters, seed, _lib.ptr(ws), _lib.ptr(out), _lib.ptr(mask), _lib.stream_ptr()),
               "s3r_pnp_ransac")
    return out.cpu().numpy(), mask.cpu().numpy().astype(bool)


@pytest.mark.gpu
@pytest.mark.parametrize("name", synth.PNP_ADV_CASES)
def test_cuda_pnp_adversarial(pnp_host, name):
    pts, img, width, K = _frame(name)
    ib = None if img is None else img[None]
    out, mask = _gpu(pts[None], ib, width, K, seed=7)
    out, mask = out[0], mask[0]
    print(f"{name}: success {out[17]} inliers {out[15]} mask {int(mask.sum())} rms {out[16]:.3e}")
    _check_result(name, out, mask, pts, img, width, K)
    _check_stationary(name, out, mask, pts, img, width, K)
    assert (out[17] == 1) == (name not in UNSOLVABLE), (name, out[17])
    if name != "hd":   # a: the host build of the same header, same seed
        ok, hout, hmask = _host(pnp_host, pts, img, width, K, seed=7)
        assert ok == out[17]
        assert int((hmask != mask).sum()) <= 3, (name, "a: mask flips", int((hmask != mask).sum()))
        if ok:
            dpose = max(np.abs(hout[12:15] - out[12:15]).max(), np.abs(hout[9:12] - out[9:12]).max())
            assert dpose < 1e-6, (name, "a: pose vs host", dpose)
    for thr in (0.5, 8.0, 50.0):
        o, m = _gpu(pts[None], ib, width, K, thr=thr, iters=0, seed=7)
        _check_result(f"{name} thr {thr}", o[0], m[0], pts, img, width, K, thr=thr, refined=False)


@pytest.mark.gpu
@pytest.mark.parametrize("samples,iters", [(1, 0), (100, 15), (4096, 100)])
def test_cuda_pnp_unsolvable_frames_fail_cleanly_in_a_batch(samples, iters):
    """g: frames with no model of 4 inliers report failure, an empty mask and the identity pose, and the frames beside
    them in the batch are bit-identical to their single-frame runs."""
    names = ["valid_small", "all_nan", "valid_small", "three_finite_dense", "valid_small"]
    frames = [_frame(nm) for nm in names]
    K, width = frames[0][3], frames[0][2]
    pts = np.stack([f[0] for f in frames])
    pts[2] = synth.make_pnp_adv_case("valid_small")[0].reshape(-1, 3)[::-1]   # a different solvable frame
    pts[4] = pts[0] * np.float32(1.5)
    out, mask = _gpu(pts, None, width, K, samples=samples, iters=iters, seed=3)
    for b, nm in enumerate(names):
        one, m1 = _gpu(pts[b:b + 1], None, width, K, samples=samples, iters=iters, seed=3)
        assert np.array_equal(one[0].view(np.int64), out[b].view(np.int64)) and np.array_equal(m1[0], mask[b]), (nm, b)
        _check_result(f"{nm}[{b}]", out[b], mask[b], pts[b], None, width, K)
        if nm in UNSOLVABLE:
            assert out[b, 17] == 0 and not mask[b].any()
            assert np.array_equal(out[b, :9], np.eye(3).reshape(-1)) and not out[b, 9:17].any(), (nm, out[b])
    # the sparse unsolvable frames, alone
    for nm in ("three_finite", "all_behind"):
        p, im, w, Ks = _frame(nm)
        o, m = _gpu(p[None], im[None], w, Ks, samples=samples, iters=iters, seed=3)
        assert o[0, 17] == 0 and not m[0].any(), (nm, o[0])
        assert np.array_equal(o[0, :9], np.eye(3).reshape(-1)) and not o[0, 9:17].any(), (nm, o[0])
