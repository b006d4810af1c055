"""The point-cloud evaluation kernels (csrc/pointcloud.cu) held to their contract in include/spann3r_b200.h on clouds where
exact ties and degenerate boxes are the rule: integer lattices, exact duplicates, flat boxes, far outliers, clusters
tighter than the Morton grid, a 1e6 offset, and sizes around every bucket, leaf and sort-tile boundary.

Checkers:
  * oracle/pcl_brute.py: tie-exact brute-force 1-NN and k-NN in fp64, rounded exactly as pointcloud_math.cuh rounds, so
    distances and indices are compared bit for bit;
  * the device normal math compiled for the host (tests/native/recon_host_check.cpp), fed the brute-force neighbour lists;
  * numpy's median / sum and math.fsum for the statistics, numpy for |a . b|;
  * oracle.recon_eval_oracle.registration_icp with the brute-force index as its tree, for ICP.
"""
import ctypes as C
import math
import os
import subprocess
import zlib

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle.pcl_brute import BruteIndex, apply_rt
from spann3r_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
KS = (1, 2, 3, 4, 8, 30, 32)
DTYPES = {"f32": np.float32, "f64": np.float64}
SIZES = (1, 2, 31, 32, 33, 63, 64, 65, 4095, 4096, 4097, 8193, 2 ** 17 + 1)
FAR = np.array([[1e8, 0.0, 0.0], [-1e8, 5.0, 5.0], [3e8, -2e8, 1e8], [0.5, 0.5, -1e8]])


# ------------------------------------------------------------------------------------------------------------------
# cloud families: (points [n, 3], queries [m, 3]) in fp64, each in a shuffled order
# ------------------------------------------------------------------------------------------------------------------
def _shuffle(p, rng):
    return np.ascontiguousarray(p[rng.permutation(len(p))])


def _grid(m):
    g = np.arange(m, dtype=np.float64)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)


def lattice(m=24, seed=0):
    """m^3 integer lattice; queries at lattice points (unique), edge midpoints (2-way ties), face centres (4-way), cell
    centres (8-way) and random positions."""
    rng = np.random.default_rng(seed)
    pts = _shuffle(_grid(m), rng)
    base = rng.integers(0, m - 1, (500, 3)).astype(np.float64)     # every +0.5 step stays inside the lattice
    e = np.eye(3)[rng.integers(0, 3, 500)]
    f = 1.0 - np.eye(3)[rng.integers(0, 3, 500)]
    qs = [pts[rng.choice(len(pts), 500, replace=False)], base + 0.5 * e, base + 0.5 * f, base + 0.5,
          rng.uniform(-1, m, (1000, 3)), FAR]
    return pts, np.concatenate(qs)


def duplicates(seed=1):
    """3000 random points, each repeated 1-5 times at scattered indices."""
    rng = np.random.default_rng(seed)
    base = rng.uniform(-1, 1, (3000, 3))
    pts = _shuffle(np.repeat(base, rng.integers(1, 6, 3000), 0), rng)
    return pts, np.concatenate([base[:800], rng.uniform(-1.2, 1.2, (800, 3)), FAR])


def one_point(seed=2):
    """1000 copies of one point: every query ties with all of them."""
    rng = np.random.default_rng(seed)
    pts = np.tile([[0.375, -0.25, 0.625]], (1000, 1))
    return pts, np.concatenate([pts[:1], rng.uniform(-1, 1, (200, 3)), FAR])


def flat(seed=3):
    """Every point on z = 0.25 exactly: a zero box extent along z (inv_ext = 0)."""
    rng = np.random.default_rng(seed)
    pts = np.c_[rng.integers(-64, 64, (6000, 2)) / 64.0, np.full(6000, 0.25)]   # on a grid: many exact ties
    qs = np.c_[rng.integers(-130, 130, (800, 2)) / 128.0, np.full(800, 0.25)]
    return _shuffle(pts, rng), np.concatenate([qs, rng.uniform(-1, 1, (800, 3)), FAR])


def line_axis(seed=4):
    """Every point on one axis-parallel line: two zero extents."""
    rng = np.random.default_rng(seed)
    t = rng.integers(-500, 500, 3000) / 16.0
    pts = np.c_[t, np.full(3000, 0.5), np.full(3000, -1.25)]
    qs = np.c_[rng.integers(-1000, 1000, 600) / 32.0, rng.uniform(-1, 1, (600, 2))]
    return pts, np.concatenate([qs, pts[:200], FAR])


def line_diag(seed=5):
    """Every point on the diagonal x = y = z: all Morton keys on one curve."""
    rng = np.random.default_rng(seed)
    t = rng.integers(-500, 500, 3000) / 16.0
    return np.c_[t, t, t], np.concatenate([rng.uniform(-32, 32, (800, 3)), np.c_[t[:200], t[:200], t[:200]] + 1 / 32, FAR])


def single(seed=6):
    rng = np.random.default_rng(seed)
    return np.array([[0.5, -0.5, 2.0]]), np.concatenate([rng.uniform(-3, 3, (300, 3)), [[0.5, -0.5, 2.0]], FAR])


def outliers(seed=7):
    """99.9 % of the points in a unit cube, 20 at +-1e6: almost everything falls into one Morton cell."""
    rng = np.random.default_rng(seed)
    inner = rng.uniform(0, 1, (20000, 3))
    far = rng.choice([-1e6, 1e6], (20, 3)) + rng.uniform(-1, 1, (20, 3))
    pts = _shuffle(np.concatenate([inner, far]), rng)
    return pts, np.concatenate([rng.uniform(-0.1, 1.1, (1500, 3)), far + rng.uniform(-2, 2, (20, 3)), FAR])


def clusters(seed=8):
    """300 clusters of 20 points within 1e-9 of their centre: Morton keys tie, so the stable sort decides the order."""
    rng = np.random.default_rng(seed)
    centre = rng.uniform(-1, 1, (300, 3))
    pts = _shuffle((centre[:, None] + rng.uniform(-1e-9, 1e-9, (300, 20, 3))).reshape(-1, 3), rng)
    return pts, np.concatenate([centre, centre + rng.uniform(-2e-9, 2e-9, (300, 3)), rng.uniform(-1, 1, (600, 3)), FAR])


def offset(seed=9):
    """Unit-scale noise around 1e6 (fp64 only: fp32 cannot hold it)."""
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, (8000, 3)) + 1e6, rng.uniform(-1.5, 1.5, (1500, 3)) + 1e6


def sized(n, seed=10):
    rng = np.random.default_rng(seed + n)
    pts = rng.integers(-256, 256, (n, 3)) / 256.0                    # coarse grid: ties at every size
    return pts, np.concatenate([rng.uniform(-1.1, 1.1, (1500, 3)), pts[rng.integers(0, n, 500)], FAR])


FAMILIES = {"lattice": lattice, "duplicates": duplicates, "one_point": one_point, "flat": flat, "line_axis": line_axis,
            "line_diag": line_diag, "single": single, "outliers": outliers, "clusters": clusters, "offset": offset}
FAMILIES.update({f"n{n}": (lambda n=n: sized(n)) for n in SIZES})
CASES = [(f, d) for f in FAMILIES for d in DTYPES if not (f == "offset" and d == "f32")]


def _cloud(family, dtype):
    p, q = FAMILIES[family]()
    return np.ascontiguousarray(p, DTYPES[dtype]), np.ascontiguousarray(q, DTYPES[dtype])


def _rigid(seed, scale=1.0):
    rng = np.random.default_rng(seed)
    T = np.eye(4)
    T[:3, :3] = synth._rotation(rng.normal(0, 0.3, 3))
    T[:3, 3] = rng.normal(0, scale, 3)
    return T


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float64)).view(np.int64)


def _same(a, b):
    """Bitwise equality of two fp64 arrays (+0.0 and -0.0 differ; NaN payloads compare)."""
    return np.array_equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------------------------
# host harness: the device math header compiled with g++
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pcl") / "recon_host_check.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "recon_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.rc_dist2.argtypes = [C.c_void_p] * 2
    L.rc_dist2.restype = C.c_double
    L.rc_knn_normals_listed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p]
    return L


def host_normals(L, cloud, nb):
    """Normals of the pointcloud_math.cuh k-NN rule on the host, from neighbour lists nb [m, k] (original indices)."""
    cloud = np.ascontiguousarray(cloud, np.float64)
    nb = np.ascontiguousarray(nb, np.int64)
    out = np.zeros((len(nb), 3))
    L.rc_knn_normals_listed(cloud.ctypes.data, nb.ctypes.data, len(nb), nb.shape[1], out.ctypes.data)
    return out


def _eig_gap_ok(cloud, nb):
    """The smallest eigenvalue of the neighbour covariance is separated: the rule of test_gpu_normals_match_oracle, with
    the gap measured against the largest eigenvalue, so that the rounding noise of a rank-one covariance (collinear or
    duplicate neighbours, clusters far apart) does not pass for a separated pair."""
    p = np.asarray(cloud, np.float64)[nb]
    d = p - p.mean(1, keepdims=True)
    w = np.linalg.eigvalsh(np.einsum("nki,nkj->nij", d, d) / nb.shape[1])
    return (w[:, 1] - w[:, 0] > 1e-6 * np.abs(w[:, 1])) & (w[:, 1] - w[:, 0] > 1e-6 * w[:, 2])


# ------------------------------------------------------------------------------------------------------------------
# CPU: the brute force itself
# ------------------------------------------------------------------------------------------------------------------
def test_brute_distance_is_the_device_formula(host):
    rng = np.random.default_rng(0)
    for scale, shift in ((1.0, 0.0), (1e-3, 1e6), (1e4, -3e5)):
        p = rng.normal(0, scale, (300, 3)) + shift
        q = rng.normal(0, scale, (40, 3)) + shift
        d2 = BruteIndex(p, device="cpu").nearest_d2(q)[0].numpy()
        full = np.array([[host.rc_dist2(np.ascontiguousarray(a).ctypes.data, np.ascontiguousarray(b).ctypes.data)
                          for b in p] for a in q])
        assert _same(d2, full.min(1))
    T = _rigid(1, 5.0)
    x = rng.normal(0, 3, (500, 3))
    ref = np.stack([((T[r, 0] * x[:, 0] + T[r, 1] * x[:, 1]) + T[r, 2] * x[:, 2]) + T[r, 3] for r in range(3)], 1)
    assert _same(apply_rt(T, torch.from_numpy(x)).numpy(), ref)


def test_brute_nearest_agrees_with_scipy_on_recon_cases():
    for i in (0, 3, 5, 6):
        gt, pred, _ = synth.make_recon_case(*synth.RECON_CASES[i])
        q = pred[:2000].astype(np.float64)
        d, idx = BruteIndex(gt, device="cpu").nearest(q)
        ds, iss = cKDTree(gt.astype(np.float64)).query(q, k=min(2, len(gt)))
        ds, iss = ds.reshape(len(q), -1), iss.reshape(len(q), -1)
        d = d.numpy()                                     # scipy's own loop may round differently: 1 ulp
        assert (np.abs(d - ds[:, 0]) <= np.spacing(ds[:, 0])).all()
        unique = ds[:, 1] > ds[:, 0] * (1 + 1e-12) if ds.shape[1] > 1 else np.ones(len(q), bool)
        assert np.array_equal(idx.numpy()[unique], iss[unique, 0])


def test_brute_ties_and_knn_order_on_the_lattice():
    pts, qs = lattice(8)
    B = BruteIndex(pts, device="cpu")
    d2, idx = B.nearest_d2(qs[:2000])
    full = ((qs[:2000, None] - pts[None]) ** 2).sum(-1)              # exact: small integers and halves
    assert np.array_equal(d2.numpy(), full.min(1))
    tied = full == full.min(1, keepdims=True)
    assert np.array_equal(idx.numpy(), np.argmax(tied, 1))
    assert {1, 2, 4, 8} <= set(tied.sum(1).tolist())                  # the query kinds tie as designed
    for k in (1, 4, 8, 30):
        for rev in (False, True):
            nb = B.knn(qs[:500], k, reverse_ties=rev).numpy()
            key = np.where(rev, -1, 1) * np.arange(len(pts))
            ref = np.stack([np.lexsort((key, row))[:k] for row in full[:500]])
            if rev:                                                   # the same set; its order is not a rule
                nb, ref = np.sort(nb, 1), np.sort(ref, 1)
            assert np.array_equal(nb, ref), (k, rev)


def test_reversed_tie_rule_moves_lattice_normals(host):
    """The lattice normals test tells the two tie rules apart: many k-th-neighbour ties span different planes."""
    pts, _ = lattice(12)
    B = BruteIndex(pts, device="cpu")
    for k in (4, 30):
        fwd, rev = B.knn(pts, k).numpy(), B.knn(pts, k, reverse_ties=True).numpy()
        nf, nr = host_normals(host, pts, fwd), host_normals(host, pts, rev)
        split = _eig_gap_ok(pts, fwd) & (np.abs(np.sum(nf * nr, 1)) < 0.9)
        assert split.sum() >= 0.1 * len(pts), (k, int(split.sum()))


def test_rounding_sensitive_bounds_exist():
    """Among the lattice's random queries are distances d = sqrt(d2) with d * d < d2, where a bound of max_dist^2 would
    drop the point the query returns at max_dist = d."""
    pts, qs = lattice()
    d2 = BruteIndex(pts, device="cpu").nearest_d2(qs[2000:3000])[0].numpy()
    d = np.sqrt(d2)
    assert (d * d < d2).sum() >= 50


def test_brute_index_stands_in_for_the_oracle_tree():
    from oracle import recon_eval_oracle as ro
    gt, pred, _ = synth.make_recon_case(*synth.RECON_CASES[4])
    gt, pred = gt[::10], pred[::10]                                   # still exactly the moved ground truth
    a = ro.registration_icp(pred, gt, 0.1)
    b = ro.registration_icp(pred, gt, 0.1, target_tree=BruteIndex(gt, device="cpu"))
    assert a["passes"] == b["passes"] and a["pass_correspondences"] == b["pass_correspondences"]
    assert np.abs(a["transformation"] - b["transformation"]).max() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    return t.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(synth.RECON_CASES)))
def test_gpu_nearest_is_brute_force_on_recon_cases(i):
    from spann3r_b200 import recon_eval as re_
    gt, pred, _ = synth.make_recon_case(*synth.RECON_CASES[i])
    for pts, qs in ((gt, pred), (pred, gt)):
        d, idx = re_.nearest_neighbors(_dev(qs), _dev(pts))
        bd, bi = BruteIndex(_dev(pts)).nearest(_dev(qs))
        assert _same(_np(d), _np(bd)) and np.array_equal(_np(idx), _np(bi))


@pytest.mark.gpu
@pytest.mark.parametrize("family,dtype", CASES)
def test_gpu_nearest_is_brute_force(family, dtype):
    from spann3r_b200 import recon_eval as re_
    pts, qs = _cloud(family, dtype)
    index = re_.PointIndex(_dev(pts))
    B = BruteIndex(_dev(pts))
    qd = _dev(qs)
    d, idx = index.query(qd)
    d2, bi = B.nearest_d2(qd)
    d, idx, d2, bi = _np(d), _np(idx), _np(d2), _np(bi)
    bd = np.sqrt(d2)
    assert _same(d, bd), np.nonzero(~(d == bd))[0][:10]
    assert np.array_equal(idx, bi), np.nonzero(idx != bi)[0][:10]
    # under a rigid transform of the queries
    T = _rigid(zlib.crc32(family.encode()), scale=float(np.abs(pts).max()) * 0.01 + 0.1)
    dt, it = index.query(qd, transform=T)
    bdt, bit = B.nearest(qd, transform=T)
    assert _same(_np(dt), _np(bdt)) and np.array_equal(_np(it), _np(bit))
    # max_dist is inclusive on the returned distance: hit exactly where the brute-force distance is <= max_dist.  The
    # sample favours distances with fl(d * d) < d2, where a bound of max_dist^2 would drop the hit.
    rng = np.random.default_rng(len(qs))
    tight = np.nonzero(bd * bd < d2)[0]
    zero = np.nonzero(bd == 0)[0]
    sample = np.concatenate([rng.permutation(tight)[:12], rng.permutation(zero)[:3],
                             rng.choice(len(qs), 12, replace=False)])
    for m in sorted({float(bd[s]) for s in sample} | {math.nextafter(float(bd[s]), 0.0) for s in sample if bd[s] > 0}):
        dm, im = index.query(qd, max_dist=m)
        hit = bd <= m
        assert np.array_equal(_np(im), np.where(hit, bi, -1)), m
        assert _same(_np(dm), np.where(hit, bd, np.inf)), m
    if family == "offset":
        # the same cloud and queries stored in fp32 lose the unit-scale detail: the comparison must notice
        d32, i32 = re_.nearest_neighbors(_dev(qs.astype(np.float32)), _dev(pts.astype(np.float32)))
        assert not (_same(_np(d32), bd) and np.array_equal(_np(i32), bi))


@pytest.mark.gpu
def test_gpu_max_dist_zero_hits_exact_duplicates():
    from spann3r_b200 import recon_eval as re_
    for family in ("duplicates", "one_point", "lattice"):
        for dtype in DTYPES:
            pts, qs = _cloud(family, dtype)
            bd, bi = BruteIndex(_dev(pts)).nearest(_dev(qs))
            on = _np(bd) == 0
            assert on.sum() >= 1
            d, idx = re_.nearest_neighbors(_dev(qs), _dev(pts), max_dist=0.0)
            assert np.array_equal(_np(idx), np.where(on, _np(bi), -1)) and _same(_np(d), np.where(on, 0.0, np.inf))


NORMAL_FAMILIES = ["lattice", "duplicates", "one_point", "flat", "line_axis", "line_diag", "single", "outliers", "clusters",
                   "offset", "n2", "n33", "n4097", f"n{2 ** 17 + 1}"]


@pytest.mark.gpu
@pytest.mark.parametrize("family,dtype", [c for c in CASES if c[0] in NORMAL_FAMILIES])
def test_gpu_normals_follow_the_tie_rule(host, family, dtype):
    from spann3r_b200 import recon_eval as re_
    pts, _ = _cloud(family, dtype)
    p64 = pts.astype(np.float64)
    index = re_.PointIndex(_dev(pts))
    B = BruteIndex(_dev(pts))
    rows = np.random.default_rng(0).permutation(len(pts))[:4000]
    for k in KS:
        n_gpu = _np(index.normals(k))[rows]
        assert np.abs(np.linalg.norm(n_gpu, axis=1) - 1).max() < 1e-12, k
        ke = min(k, len(pts))
        nb = _np(B.knn(_dev(p64[rows]), k))
        n_host = host_normals(host, p64, nb)
        if ke < 3:
            assert np.array_equal(n_gpu, n_host) and (n_host == (0.0, 0.0, 1.0)).all(), k
            continue
        well = _eig_gap_ok(p64, nb)
        dots = np.abs(np.sum(n_gpu * n_host, 1))
        assert (dots[well] >= 1 - 1e-12).all(), (k, dots[well].min())
        if family == "lattice" and k in (4, 30):
            n_rev = host_normals(host, p64, _np(B.knn(_dev(p64[rows]), k, reverse_ties=True)))
            split = well & (np.abs(np.sum(n_host * n_rev, 1)) < 0.9)
            assert split.sum() >= 200, (k, int(split.sum()))
            assert (np.abs(np.sum(n_gpu * n_rev, 1))[split] < 0.9).all()


STAT_CASES = {
    "n1": [3.5], "n2": [1.0, 2.0], "n3": [2.0, 1.0, 3.0], "n2_equal": [7.0, 7.0],
    "all_equal": [0.125] * 1001, "ties_mid": [1.0] * 3 + [2.0] * 5 + [3.0] * 4,
    "ties_mid_odd": [5.0, 1.0, 5.0, 5.0, 9.0, 5.0, 0.0],
    "zeros_inf": [0.0, np.inf, 1.0, np.inf], "inf_middle": [np.inf, np.inf, 1.0], "with_zero": [0.0, 0.0, 4.0],
    "subnormal": [5e-324, 1e-310, 0.0, 2.2e-308, 1e-320, 3e-315],
    "neg_zero_3": [-0.0, 1.0, 2.0], "neg_zero_even": [3.0, -0.0, 1.0, -0.0, 4.0, 2.0], "neg_zero_mid": [2.0, -0.0, 0.0, 3.0, -0.0], "neg_zero_1": [-0.0],
}


def _nextafter_chain(x0, n):
    out = [x0]
    for _ in range(n - 1):
        out.append(math.nextafter(out[-1], math.inf))
    return out


def _stat_vectors():
    rng = np.random.default_rng(5)
    v = {k: np.array(x, np.float64) for k, x in STAT_CASES.items()}
    v["nextafter"] = rng.permutation(np.array(_nextafter_chain(1.0, 1000) + _nextafter_chain(1.0, 24)))
    v["nextafter_even"] = rng.permutation(np.array(_nextafter_chain(0.75, 4096)))
    v["wide_range"] = 10.0 ** rng.uniform(-300, 300, 5001)
    v["wide_range_even"] = 10.0 ** rng.uniform(-300, 300, 5000)
    v["grid_stride"] = rng.integers(0, 1000, 256 * 264 * 3 + 7).astype(np.float64) / 8.0
    v["grid_stride_even"] = rng.exponential(1.0, 256 * 264 * 2 + 10)
    v["neg_zero_many"] = rng.permutation(np.r_[np.full(40, -0.0), np.full(21, 0.0), np.arange(1.0, 40.0)])
    return v


@pytest.mark.gpu
def test_gpu_stats_median_and_count_are_exact():
    from spann3r_b200 import recon_eval as re_
    for name, x in _stat_vectors().items():
        xd = _dev(x)
        med = float(np.median(x))
        finite = x[np.isfinite(x)]
        for thr in sorted({0.0, float(x[len(x) // 3]), float(x[-1]), med, math.inf, 1.0}):
            out = torch.empty(3, dtype=torch.float64, device="cuda")
            re_._stats_into(xd, out, thr)
            o = _np(out)
            again = torch.empty(3, dtype=torch.float64, device="cuda")
            re_._stats_into(xd, again, thr)
            assert _same(o, _np(again)), name                         # reproducible to the bit
            if np.signbit(med) or (name.startswith("neg_zero") and med == 0):
                assert o[1] == med and not np.signbit(o[1]), (name, o[1], med)   # -0.0 is keyed as +0.0
            else:
                assert _same(o[1], med), (name, o[1], med)
            assert o[2] == np.count_nonzero(x < thr), (name, thr)
            if len(finite) == len(x):
                ref = math.fsum(x) / len(x)
                bound = len(x) * np.finfo(np.float64).eps * math.fsum(np.abs(x)) / len(x) + 1e-300
                assert abs(o[0] - ref) <= bound, (name, o[0], ref)
            else:
                assert o[0] == np.inf, name


@pytest.mark.gpu
def test_gpu_abs_dot_is_numpy():
    from spann3r_b200 import recon_eval as re_
    rng = np.random.default_rng(11)
    for n, m in ((1, 1), (257, 3), (5000, 1200)):
        a = rng.normal(0, 1, (n, 3)) * 10.0 ** rng.uniform(-3, 3, (n, 1))
        b = rng.normal(0, 1, (m, 3))
        b /= np.linalg.norm(b, axis=1, keepdims=True)
        idx = rng.integers(0, m, n)                                   # repeats: m < n
        idx[: n // 2] = idx[0]
        ref = np.abs((a[:, 0] * b[idx, 0] + a[:, 1] * b[idx, 1]) + a[:, 2] * b[idx, 2])
        assert _same(_np(re_._abs_dot(_dev(a), _dev(b), _dev(idx))), ref)


def _icp_check(src, tgt, thr, **kw):
    from oracle import recon_eval_oracle as ro
    from spann3r_b200 import recon_eval as re_
    reg = re_.registration_icp(_dev(src), _dev(tgt), thr, **kw)
    orc = ro.registration_icp(src.astype(np.float64), tgt.astype(np.float64), thr,
                              target_tree=BruteIndex(_dev(tgt)), **kw)
    T = _np(reg.transformation)
    scale = float(np.abs(tgt).max())
    assert reg.passes == orc["passes"], (reg.passes, orc["passes"])
    assert reg.pass_correspondences == orc["pass_correspondences"]
    assert np.abs(T[:3, :3] - orc["transformation"][:3, :3]).max() < 1e-9
    assert np.abs(T[:3, 3] - orc["transformation"][:3, 3]).max() < 1e-9 * max(1.0, scale)
    # near-zero residuals are rounding noise: 1e-9 relative, or 4 ulps of the cloud's extent
    assert math.isclose(reg.inlier_rmse, orc["inlier_rmse"], rel_tol=1e-9, abs_tol=4 * np.spacing(max(1.0, scale)))
    assert reg.fitness == orc["fitness"]
    return reg, T


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_gpu_icp_on_tied_targets(dtype):
    rng = np.random.default_rng(12)
    dt = DTYPES[dtype]
    # lattice target: sources at lattice points, edge midpoints, face and cell centres tie in the first pass
    pts, qs = lattice(12, seed=3)
    src = np.concatenate([qs[:2000], pts[:500] + rng.normal(0, 0.05, (500, 3))])
    _icp_check(src.astype(dt), pts.astype(dt), 0.9)
    # duplicate target
    pts, _ = duplicates(seed=13)
    T = _rigid(14, 0.01)
    T[:3, :3] = synth._rotation((0.01, -0.02, 0.015))
    src = (pts[:4000] - T[:3, 3]) @ T[:3, :3] + rng.normal(0, 0.002, (4000, 3))
    _icp_check(src.astype(dt), pts.astype(dt), 0.05)
    # planar target
    pts, _ = flat(seed=15)
    R = synth._rotation((0.0, 0.0, 0.03))
    src = (pts - (0.02, -0.01, 0.0)) @ R
    _icp_check(src.astype(dt), pts.astype(dt), 0.1)


@pytest.mark.gpu
def test_gpu_icp_of_a_cloud_onto_itself():
    pts, _ = lattice(12, seed=4)
    pts = np.concatenate([pts, pts[:300]])                            # with duplicates too
    reg, T = _icp_check(pts, pts, 0.5)
    assert reg.passes == 2 and reg.fitness == 1.0 and reg.inlier_rmse <= 1e-15 * 12
    assert np.abs(T - np.eye(4)).max() <= 1e-15 * 12


@pytest.mark.gpu
def test_gpu_icp_recovers_a_transform_at_a_1e6_offset():
    pts, _ = offset(seed=16)
    c = pts.mean(0)
    R = synth._rotation((0.002, -0.001, 0.0015))
    T_true = np.eye(4)
    T_true[:3, :3] = R
    T_true[:3, 3] = c - R @ c + (0.001, -0.002, 0.0005)                 # about the cloud, not about the origin
    src = (pts - T_true[:3, 3]) @ R                                   # tgt = T_true src
    reg, T = _icp_check(src, pts, 0.2)
    assert reg.fitness == 1.0
    assert np.abs(T[:3, :3] - R).max() < 1e-9
    assert np.abs(T[:3, 3] - T_true[:3, 3]).max() < 1e-9 * np.abs(T_true[:3, 3]).max()


# ---- stream contract: every C entry point enqueues on the caller's stream and never waits for the device -------------
def _pcl_pipeline(L, bufs, stream, after_each=lambda: None):
    """Index build, nearest (transformed), normals, ICP, stats of the distances and |n . n| on the C ABI, on `stream`."""
    P = lambda t: C.c_void_p(t.data_ptr())
    n, nq = bufs["pts"].shape[0], bufs["qs"].shape[0]
    s = C.c_void_p(stream)
    steps = [
        lambda: L.s3r_pcl_index_build(P(bufs["pts"]), 0, n, None, P(bufs["index"]), s),
        lambda: L.s3r_pcl_nearest(P(bufs["index"]), n, P(bufs["qs"]), 0, nq, P(bufs["T"]), math.inf, P(bufs["dist"]),
                                  P(bufs["idx"]), s),
        lambda: L.s3r_pcl_normals(P(bufs["index"]), n, 8, P(bufs["normals"]), s),
        lambda: L.s3r_pcl_icp(P(bufs["qs"]), 0, nq, P(bufs["index"]), n, 0.6, P(bufs["T"]), 30, 1e-6, 1e-6,
                              P(bufs["icp_ws"]), P(bufs["icp"]), s),
        lambda: L.s3r_pcl_stats(P(bufs["dist"]), nq, 0.25, P(bufs["stats_ws"]), P(bufs["stats"]), s),
        lambda: L.s3r_pcl_abs_dot(P(bufs["qnormals"]), P(bufs["normals"]), P(bufs["idx"]), nq, P(bufs["dots"]), s),
    ]
    for step in steps:
        assert step() == 0, L.s3r_last_error()
        after_each()


@pytest.mark.gpu
def test_gpu_entry_points_run_on_the_callers_stream():
    from spann3r_b200 import _lib
    L = _lib.lib()
    pts, qs = lattice(12, seed=5)
    rng = np.random.default_rng(17)
    qs = qs[:1500] + rng.normal(0, 0.01, (1500, 3))
    T = _rigid(18, 0.05)[:3]
    T[:, :3] = synth._rotation((0.01, 0.0, -0.01))
    qn = rng.normal(0, 1, (len(qs), 3))
    inputs = {"pts": _dev(pts.astype(np.float32)), "qs": _dev(qs.astype(np.float32)), "T": _dev(T), "qnormals": _dev(qn)}

    def fresh():
        b = {k: torch.zeros_like(v) for k, v in inputs.items()}
        b.update(index=torch.zeros(int(L.s3r_pcl_index_bytes(len(pts))), dtype=torch.uint8, device="cuda"),
                 dist=torch.zeros(len(qs), dtype=torch.float64, device="cuda"),
                 idx=torch.zeros(len(qs), dtype=torch.int64, device="cuda"),
                 normals=torch.zeros(len(pts), 3, dtype=torch.float64, device="cuda"),
                 icp_ws=torch.zeros(int(L.s3r_pcl_icp_workspace_bytes()), dtype=torch.uint8, device="cuda"),
                 icp=torch.zeros(19 + 2 * 31, dtype=torch.float64, device="cuda"),
                 stats_ws=torch.zeros(int(L.s3r_pcl_stats_workspace_bytes()), dtype=torch.uint8, device="cuda"),
                 stats=torch.zeros(3, dtype=torch.float64, device="cuda"),
                 dots=torch.zeros(len(qs), dtype=torch.float64, device="cuda"))
        return b

    outs = ("index", "dist", "idx", "normals", "icp", "stats", "dots")
    ref = fresh()
    for k, v in inputs.items():
        ref[k].copy_(v)
    torch.cuda.synchronize()
    _pcl_pipeline(L, ref, 0)                                          # the legacy default stream
    torch.cuda.synchronize()

    side = fresh()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(600_000_000)                                # ~0.3 s of device time ahead of everything
        for k, v in inputs.items():
            side[k].copy_(v, non_blocking=True)

        def still_busy():
            assert not s.query(), "a call waited for the device"

        _pcl_pipeline(L, side, s.cuda_stream, still_busy)
    s.synchronize()
    for k in outs:
        a, b = ref[k].cpu().numpy(), side[k].cpu().numpy()
        assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), k
