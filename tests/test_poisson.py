"""Screened Poisson reconstruction (spann3r_b200.mesh.create_from_point_cloud_poisson, csrc/poisson.cu): the numpy /
scipy oracle against quadrature and analytic shapes on the CPU, the host-compiled device math bit for bit against the
oracle, PLY I/O and the C ABI's argument checks without a device; on the GPU, every stage against the oracle, the mesh
against analytic surfaces, and render_dtu.py's get_mesh_from_ply -> render_dtu_scenes chain on a synthetic scan."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse.linalg as spla

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import poisson_oracle as po  # noqa: E402
from spann3r_b200 import mesh  # noqa: E402


# ----------------------------------------------------------------------------------------------------------------------
# shapes
# ----------------------------------------------------------------------------------------------------------------------
def sphere(n, seed=0, r=1.0, centre=(0.0, 0.0, 0.0)):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * r + np.asarray(centre), d


def torus(n, seed=0, R=1.0, r=0.4):
    rng = np.random.default_rng(seed)
    u, v = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
    ring = np.stack([np.cos(u), np.sin(u), 0 * u], 1)
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    return R * ring + r * nrm, nrm


def wavy(n, seed=0):
    """An open height field z = 0.1 sin(3x) cos(2y) over [-1, 1]^2, normals up."""
    rng = np.random.default_rng(seed)
    x, y = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    z = 0.1 * np.sin(3 * x) * np.cos(2 * y)
    nrm = np.stack([-0.3 * np.cos(3 * x) * np.cos(2 * y), 0.2 * np.sin(3 * x) * np.sin(2 * y), np.ones(n)], 1)
    return np.stack([x, y, z], 1), nrm


def nonuniform(n, seed=0):
    """A sphere sampled ten times more densely on its z < 0 half, with unnormalised normals of random length."""
    p, nrm = sphere(4 * n, seed)
    rng = np.random.default_rng(seed + 1)
    keep = (p[:, 2] < 0) | (rng.uniform(size=len(p)) < 0.1)
    p, nrm = p[keep][:n], nrm[keep][:n]
    return p, nrm * rng.uniform(0.2, 5.0, (len(p), 1))


def duplicates(n, seed=0):
    """A sphere whose every sample appears twice, plus one sample with a zero normal."""
    p, nrm = sphere(n // 2, seed)
    p, nrm = np.concatenate([p, p]), np.concatenate([nrm, nrm])
    nrm[0] = 0
    return p, nrm


def topology(v, f):
    """(Euler characteristic, every edge in exactly two faces, number of connected components)."""
    import scipy.sparse as sp
    E = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    u, cnt = np.unique(E, axis=0, return_counts=True)
    g = sp.coo_matrix((np.ones(len(u)), (u[:, 0], u[:, 1])), shape=(len(v), len(v)))
    ncomp = sp.csgraph.connected_components(g, directed=False)[0]
    return len(v) - len(u) + len(f), bool((cnt == 2).all()), ncomp


def face_normals(v, f):
    v = np.asarray(v, np.float64)
    return np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), (v[f[:, 0]] + v[f[:, 1]] + v[f[:, 2]]) / 3


def sphere_dist(v):
    return np.abs(np.linalg.norm(np.asarray(v, np.float64), axis=1) - 1.0)


def torus_dist(v, R=1.0, r=0.4):
    v = np.asarray(v, np.float64)
    q = np.sqrt(v[:, 0] ** 2 + v[:, 1] ** 2) - R
    return np.abs(np.sqrt(q ** 2 + v[:, 2] ** 2) - r)


def torus_outward(c, R=1.0):
    ring = c.copy()
    ring[:, 2] = 0
    ring *= R / np.linalg.norm(ring, axis=1, keepdims=True)
    return c - ring


def check_closed_shape(v, f, h, kind):
    """The bars of every closed reconstruction: Euler characteristic, two faces per edge, one component, outward faces,
    vertex distance to the analytic surface at most h and 0.25 h on average."""
    euler, manifold, ncomp = topology(v, f)
    assert euler == (2 if kind == "sphere" else 0) and manifold and ncomp == 1, (euler, manifold, ncomp)
    nrm, c = face_normals(v, f)
    out = c if kind == "sphere" else torus_outward(c)
    area = np.linalg.norm(nrm, axis=1)
    ok = area > 0
    assert ((nrm[ok] * out[ok]).sum(1) > 0).all()
    dist = sphere_dist(v) if kind == "sphere" else torus_dist(v)
    assert dist.max() <= h and dist.mean() <= 0.25 * h, (dist.max() / h, dist.mean() / h)


# ----------------------------------------------------------------------------------------------------------------------
# CPU: the oracle's discretisation
# ----------------------------------------------------------------------------------------------------------------------
def _gauss_hats(R, h):
    """[cells * 8 quadrature points] (node indices [.., 8], hat values [.., 8], gradients [.., 8, 3], weights) on an
    R^3 grid of spacing h by 2-point Gauss quadrature per axis (exact for trilinear products)."""
    g = 0.5 + np.array([-1, 1]) / (2 * np.sqrt(3))
    pts = np.array([[a, b, c] for c in g for b in g for a in g])
    rows = []
    for cz in range(R):
        for cy in range(R):
            for cx in range(R):
                for xi in pts:
                    nodes, val, grad = [], [], []
                    for q in range(8):
                        bit = [(q >> d) & 1 for d in range(3)]
                        w = [xi[d] if bit[d] else 1 - xi[d] for d in range(3)]
                        dw = [(1 if bit[d] else -1) / h for d in range(3)]
                        nodes.append(po.node_index(cx + bit[0], cy + bit[1], cz + bit[2], R))
                        val.append(w[0] * w[1] * w[2])
                        grad.append([dw[0] * w[1] * w[2], w[0] * dw[1] * w[2], w[0] * w[1] * dw[2]])
                    rows.append((nodes, val, grad))
    return rows, (h ** 3) / 8


def test_oracle_stencils_equal_quadrature():
    R, h = 3, 0.37
    n = (R + 1) ** 3
    K, D = np.zeros((n, n)), [np.zeros((n, n)) for _ in range(3)]
    rows, wq = _gauss_hats(R, h)
    for nodes, val, grad in rows:
        grad = np.asarray(grad)
        for p in range(8):
            for q in range(8):
                K[nodes[p], nodes[q]] += wq * grad[p] @ grad[q]
                for d in range(3):
                    D[d][nodes[p], nodes[q]] += wq * grad[p, d] * val[q]
    assert np.allclose(po._assemble(R, po.element_stiffness()).toarray() * h, K, rtol=0, atol=1e-14)
    for d in range(3):
        assert np.allclose(po._assemble(R, po.element_divergence(d)).toarray() * h * h, D[d], rtol=0, atol=1e-14)
    # the interior stencil is the 27-point one: 8/3 h at the centre, 0 across faces, -h/6 across edges, -h/12 corners
    Kd = po._assemble(4, po.element_stiffness()).toarray()
    c = po.node_index(2, 2, 2, 4)
    st = {0: 8 / 3, 1: 0.0, 2: -1 / 6, 3: -1 / 12}
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                j = po.node_index(2 + dx, 2 + dy, 2 + dz, 4)
                assert abs(Kd[c, j] - st[abs(dx) + abs(dy) + abs(dz)]) < 1e-15


def test_oracle_system_is_spd_and_matches_brute_force():
    p, n = sphere(300, seed=3)
    s = po.System(p, n, 3)
    A = s.A.toarray()
    assert np.abs(A - A.T).max() <= 1e-15 * np.abs(A).max()      # symmetric up to the order duplicates were summed
    assert np.linalg.eigvalsh(A).min() > 0
    # brute force: per-sample loops for v, S; b through quadrature of grad phi_i . V
    R, nn = s.R, (s.R + 1) ** 3
    u = po.unit_normals(n)
    S = np.zeros((nn, nn))
    v = np.zeros((nn, 3))
    for k in range(len(p)):
        g = (p[k] - s.origin) / s.h
        c = np.clip(np.floor(g), 0, R - 1).astype(int)
        f = g - c
        for a in range(8):
            ia = po.node_index(c[0] + (a & 1), c[1] + (a >> 1 & 1), c[2] + (a >> 2), R)
            wa = np.prod([f[d] if a >> d & 1 else 1 - f[d] for d in range(3)])
            v[ia] += s.a / s.h ** 3 * wa * u[k]
            for b in range(8):
                ib = po.node_index(c[0] + (b & 1), c[1] + (b >> 1 & 1), c[2] + (b >> 2), R)
                S[ia, ib] += wa * np.prod([f[d] if b >> d & 1 else 1 - f[d] for d in range(3)])
    b = np.zeros(nn)
    rows, wq = _gauss_hats(R, s.h)
    for nodes, val, grad in rows:
        V = np.asarray(val) @ v[nodes]
        for q in range(8):
            b[nodes[q]] += wq * np.asarray(grad[q]) @ V
    assert np.linalg.norm(s.S.toarray() - S) <= 1e-13 * np.linalg.norm(S)
    assert np.linalg.norm(s.b - b) <= 1e-12 * np.linalg.norm(b)
    blocks = s.blocks()
    assert len(blocks) == s.occupied
    assert np.isclose(sum(B.sum() for B in blocks.values()), len(p), rtol=1e-13)


def _oracle_mesh(p, n, depth):
    s = po.System(p, n, depth)
    chi = s.solve() if depth <= 4 else spla.cg(s.A, s.b, rtol=1e-12, maxiter=5000)[0]
    iso = s.iso(chi)
    v, f = po.extract(chi, iso, s.origin, s.h, s.R)
    return s, v, f


@pytest.mark.parametrize("kind,depth", [("sphere", 4), ("torus", 4), ("sphere", 5), ("torus", 5)])
def test_oracle_geometry_on_closed_shapes(kind, depth):
    p, n = sphere(8000, seed=1) if kind == "sphere" else torus(16000, seed=1)
    s, v, f = _oracle_mesh(p, n, depth)
    check_closed_shape(v, f, s.h, kind)


# ----------------------------------------------------------------------------------------------------------------------
# CPU: the device math, host-compiled, bit for bit against the oracle
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("poisson") / "poisson_host_check.so")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-std=c++17", "-x", "c++",
                           os.path.join(HERE, "native", "poisson_host_check.cpp"), "-o", so])
    L = C.CDLL(so)
    L.ph_geometry.argtypes = [C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p]
    L.ph_locate.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p,
                            C.c_void_p]
    L.ph_unit_normals.argtypes = [C.c_void_p, C.c_longlong, C.c_void_p]
    L.ph_tet.argtypes = [C.c_int, C.c_void_p]
    L.ph_case.argtypes = [C.c_int, C.c_void_p]
    L.ph_edge_vertices.argtypes = [C.c_void_p]
    L.ph_edge_points.argtypes = [C.c_void_p] * 4 + [C.c_double, C.c_longlong, C.c_void_p]
    L.ph_quantile.argtypes = [C.c_void_p, C.c_longlong, C.c_double]
    L.ph_quantile.restype = C.c_double
    return L


def test_host_geometry_and_weights_match_the_oracle(host_lib):
    rng = np.random.default_rng(5)
    for depth, scale in ((1, 1.0), (4, 1.1), (9, 1.1), (10, 1.37)):
        p = rng.normal(size=(500, 3)) * rng.uniform(0.1, 100, 3) + rng.normal(size=3) * 50
        lo, hi = p.min(0), p.max(0)
        out = np.zeros(5)
        host_lib.ph_geometry(lo.ctypes.data, hi.ctypes.data, scale, depth, out.ctypes.data)
        origin, L, h = po.geometry(p, depth, scale)
        assert np.array_equal(out, np.r_[origin, L, h])
        R = 1 << depth
        cells, f, w = np.zeros((500, 3), np.int64), np.zeros((500, 3)), np.zeros((500, 8))
        host_lib.ph_locate(p.ctypes.data, 500, origin.ctypes.data, h, R, cells.ctypes.data, f.ctypes.data, w.ctypes.data)
        oc, of = po.locate(p, origin, h, R)
        assert np.array_equal(cells, oc) and np.array_equal(f, of) and np.array_equal(w, po.corner_weights(of))
    n = rng.normal(size=(300, 3)) * rng.uniform(1e-3, 1e3, (300, 1))
    n[:3] = 0
    u = np.zeros_like(n)
    host_lib.ph_unit_normals(n.ctypes.data, len(n), u.ctypes.data)
    assert np.array_equal(u, po.unit_normals(n))


def test_host_tetrahedra_and_cases_match_the_oracle(host_lib):
    ev = np.zeros(12, np.int32)
    host_lib.ph_edge_vertices(ev.ctypes.data)
    assert [tuple(x) for x in ev.reshape(6, 2)] == po.TET_EDGES
    for t in range(6):
        c = np.zeros(4, np.int32)
        pos = host_lib.ph_tet(t, c.ctypes.data)
        assert c.tolist() == po.tet_corners(t) and bool(pos) == po.tet_positive(t)
    for code in range(16):
        e = np.zeros(6, np.int32)
        k = host_lib.ph_case(code, e.ctypes.data)
        assert e[:3 * k].reshape(-1, 3).tolist() == po.CASES[code]


def test_host_edge_points_and_quantile_match_the_oracle(host_lib):
    rng = np.random.default_rng(6)
    n = 20000
    xa = rng.normal(size=n) * 10
    xb = xa + rng.uniform(0.01, 1, n)
    va = rng.normal(size=n)
    iso = 0.03125
    vb = np.where(va > iso, iso - rng.uniform(0, 1, n), iso + rng.uniform(1e-300, 1, n))
    va[:50] = iso                                   # a node exactly at the iso value (t = 0)
    vb[:50] = iso + 1
    out = np.zeros(n, np.float32)
    host_lib.ph_edge_points(xa.ctypes.data, xb.ctypes.data, va.ctypes.data, vb.ctypes.data, iso, n, out.ctypes.data)
    expect = np.array([po.edge_point(*a, iso) for a in zip(xa, xb, va, vb)], np.float32)
    assert np.array_equal(out.view(np.uint32), expect.view(np.uint32))
    for size in (1, 2, 3, 10, 1001, 4096):
        x = np.sort(rng.exponential(size=size))
        x[size // 3: size // 3 + size // 4] = x[size // 3]         # ties at the quantile
        for q in (0.0, 0.1, 0.25, 0.5, 0.3333333333333333, 0.9, 0.999, 1.0, rng.uniform()):
            got = host_lib.ph_quantile(x.ctypes.data, size, q)
            assert np.float64(got).view(np.uint64) == np.quantile(x, q).view(np.uint64), (size, q)


# ----------------------------------------------------------------------------------------------------------------------
# CPU: PLY I/O
# ----------------------------------------------------------------------------------------------------------------------
def _cloud_ply(path, pts, nrm, fmt="binary", extra=True, normals=True, dtype="float"):
    props = [("x", dtype), ("y", dtype), ("z", dtype)]
    if normals:
        props += [("nx", dtype), ("ny", dtype), ("nz", dtype)]
    if extra:
        props = props[:3] + [("red", "uchar"), ("green", "uchar"), ("blue", "uchar"), ("quality", "short")] + props[3:] \
            + [("alpha", "double")]
    head = "ply\nformat " + ("ascii" if fmt == "ascii" else "binary_little_endian") + " 1.0\ncomment synthetic\n"
    head += f"element vertex {len(pts)}\n" + "".join(f"property {t} {a}\n" for a, t in props) + "end_header\n"
    np_t = {"float": "<f4", "double": "<f8", "uchar": "u1", "short": "<i2"}
    rec = np.zeros(len(pts), np.dtype([(a, np_t[t]) for a, t in props]))
    for i, a in enumerate("xyz"):
        rec[a] = pts[:, i]
        if normals:
            rec["n" + a] = nrm[:, i]
    if extra:
        rec["red"], rec["quality"], rec["alpha"] = 7, -3, 0.5
    with open(path, "wb") as fh:
        fh.write(head.encode())
        if fmt == "ascii":
            for r in rec:
                fh.write((" ".join(repr(float(x)) if isinstance(x, np.floating) else str(x) for x in r) + "\n").encode())
        else:
            fh.write(rec.tobytes())


def test_ply_mesh_round_trip_and_point_clouds(tmp_path):
    rng = np.random.default_rng(7)
    v = rng.normal(size=(100, 3)).astype(np.float32)
    v[0] = [np.float32(1e-38), -0.0, np.float32(3.4e38)]
    f = rng.integers(0, 100, (60, 3))
    path = str(tmp_path / "m.ply")
    mesh.write_ply_mesh(path, v, f)
    rv, rf = mesh.read_ply_mesh(path)
    assert np.array_equal(rv.view(np.uint32), v.view(np.uint32)) and np.array_equal(rf, f)
    mesh.write_ply_mesh(path, v, np.zeros((0, 3), np.int64))
    assert len(mesh.read_ply_mesh(path)[1]) == 0
    with pytest.raises(ValueError):
        mesh.write_ply_mesh(path, v, f + 100)
    p, n = rng.normal(size=(50, 3)), rng.normal(size=(50, 3))
    for fmt in ("ascii", "binary"):
        for dtype in ("float", "double"):
            for extra in (False, True):
                _cloud_ply(str(tmp_path / "c.ply"), p, n, fmt, extra, dtype=dtype)
                rp, rn = mesh.read_point_cloud(str(tmp_path / "c.ply"))
                cast = np.float32 if dtype == "float" else np.float64
                assert rp.dtype == np.float64 and np.array_equal(rp, p.astype(cast)) and np.array_equal(rn, n.astype(cast))
    _cloud_ply(str(tmp_path / "c.ply"), p, n, normals=False)
    with pytest.raises(ValueError, match="normals"):
        mesh.read_point_cloud(str(tmp_path / "c.ply"))
    _cloud_ply(str(tmp_path / "c.ply"), p, n)
    data = open(tmp_path / "c.ply", "rb").read()
    open(tmp_path / "t.ply", "wb").write(data[:-5])
    with pytest.raises(ValueError, match="truncated"):
        mesh.read_point_cloud(str(tmp_path / "t.ply"))
    _cloud_ply(str(tmp_path / "c.ply"), p, n, fmt="ascii")
    data = open(tmp_path / "c.ply", "rb").read()
    open(tmp_path / "t.ply", "wb").write(data[:data.rindex(b"\n", 0, len(data) - 1)])
    with pytest.raises(ValueError):
        mesh.read_point_cloud(str(tmp_path / "t.ply"))


def test_c_abi_rejects_bad_arguments_without_a_device():
    from spann3r_b200 import _lib
    L = _lib.lib()
    assert L.s3r_poisson_workspace_bytes(3, 5) == 0 and L.s3r_poisson_workspace_bytes(100, 0) == 0
    assert L.s3r_poisson_workspace_bytes(100, 11) == 0 and L.s3r_poisson_workspace_bytes(100, 5) > 0
    assert L.s3r_poisson_offset(100, 5, 8) == 2 ** 64 - 1 and L.s3r_poisson_offset(3, 5, 1) == 2 ** 64 - 1
    info = (C.c_double * 8)()
    assert L.s3r_poisson_setup(None, None, 0, 100, 5, 1.1, None, 0, info, None) == -1
    assert b"poisson_setup" in L.s3r_last_error()
    assert L.s3r_poisson_solve(100, 11, 1e-8, 10, None, 0, info, None) == -1
    assert L.s3r_poisson_extract_count(100, 5, None, 0, None, None) == -1
    assert L.s3r_poisson_extract(2, 5, None, 0, None, None, None, None) == -1
    assert L.s3r_pcl_quantile(None, 10, 0.5, None, None, None) == -1
    assert L.s3r_mesh_compact_workspace_bytes(0, 5) == 0
    assert L.s3r_mesh_compact_count(None, None, 10, 5, None, 0, None, None) == -1
    assert b"mesh_compact_count" in L.s3r_last_error()
    assert L.s3r_mesh_compact(None, None, 10, 5, None, 0, None, None, None) == -1


# ----------------------------------------------------------------------------------------------------------------------
# GPU
# ----------------------------------------------------------------------------------------------------------------------
CASES = {
    "sphere_d4": (lambda: sphere(6000, seed=11), 4),
    "torus_d5": (lambda: torus(20000, seed=12), 5),
    "wavy_d5": (lambda: wavy(15000, seed=13), 5),
    "nonuniform_d6": (lambda: nonuniform(30000, seed=14), 6),
    "duplicates_d4": (lambda: duplicates(6000, seed=15), 4),
}


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(np.asarray(b)), 1e-300))


@pytest.fixture(scope="module", params=sorted(CASES))
def solved(request):
    import torch
    make, depth = CASES[request.param]
    p, n = make()
    st = mesh._Poisson(torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda(), depth, 1.1)
    R = 1 << depth
    NN = (R + 1) ** 3
    b = st.view(1, torch.float64, NN).cpu().numpy()
    chi = st.view(2, torch.float64, NN).cpu().numpy()
    order = st.view(0, torch.int32, len(p)).cpu().numpy()
    lo = st.view(4, torch.int32, R ** 3).cpu().numpy()
    hi = st.view(5, torch.int32, R ** 3).cpu().numpy()
    blocks = st.view(3, torch.float64, 64 * len(p)).cpu().numpy().reshape(-1, 8, 8)
    v, f, d = (x.cpu().numpy() for x in st.extract())
    return dict(name=request.param, p=p, n=n, depth=depth, st=st, sys=po.System(p, n, depth), b=b, chi=chi,
                order=order, lo=lo, hi=hi, blocks=blocks, v=v, f=f, d=d)


@pytest.mark.gpu
def test_gpu_system_matches_the_oracle(solved):
    s, st = solved["sys"], solved["st"]
    assert np.array_equal(st.origin, s.origin) and st.L == s.L and st.h == s.h and st.occupied == s.occupied
    assert st.a == s.a and st.beta == s.beta
    assert _rel(solved["b"], s.b) <= 1e-12
    ids = s.cell_id[solved["order"]]
    assert np.all(np.diff(ids) >= 0)                                       # sorted by cell, stable within a cell
    assert all(np.all(np.diff(solved["order"][ids == c]) > 0) for c in np.unique(ids)[:50])
    want = s.blocks()
    got = np.stack([solved["blocks"][solved["lo"][c]] for c in want])
    assert all(solved["hi"][c] > solved["lo"][c] for c in want)
    assert _rel(got, np.stack(list(want.values()))) <= 1e-12


@pytest.mark.gpu
def test_gpu_solve_residual_and_iso(solved):
    s, chi = solved["sys"], solved["chi"]
    assert np.linalg.norm(s.b - s.A @ chi) <= 1e-8 * np.linalg.norm(s.b)
    assert solved["st"].residual <= 1e-8 and 0 < solved["st"].iterations < mesh.POISSON_MAX_ITER
    if solved["depth"] <= 4:
        assert _rel(chi, s.solve()) <= 1e-5
    iso = s.iso(chi)
    assert abs(solved["st"].iso - iso) <= 1e-12 * max(abs(iso), np.abs(chi).max() * 1e-6)


@pytest.mark.gpu
def test_gpu_extraction_and_densities_match_the_oracle(solved):
    s, st = solved["sys"], solved["st"]
    v, f = po.extract(solved["chi"], st.iso, st.origin, st.h, 1 << solved["depth"])
    assert np.array_equal(solved["v"].view(np.uint32), v.view(np.uint32))
    assert np.array_equal(solved["f"], f)
    assert _rel(solved["d"], s.densities(solved["v"])) <= 1e-12
    if solved["name"].startswith(("sphere", "duplicates")):
        check_closed_shape(solved["v"], solved["f"], st.h, "sphere")
    if solved["name"].startswith("torus"):
        check_closed_shape(solved["v"], solved["f"], st.h, "torus")


@pytest.mark.gpu
def test_gpu_quantile_trim_and_vertex_removal(solved):
    import torch
    d = torch.from_numpy(solved["d"]).cuda()
    for q in (0.0, 0.1, 0.25, 0.5, 0.77, 1.0):
        assert mesh.quantile(d, q).item() == np.quantile(solved["d"], q)
    ties = np.repeat(solved["d"][:40], 25)
    for q in (0.1, 0.5, 0.9):
        assert mesh.quantile(torch.from_numpy(ties).cuda(), q).item() == np.quantile(ties, q)
    thr = np.quantile(solved["d"], 0.1)
    mask = solved["d"] < thr
    v, f = mesh.remove_vertices_by_mask(torch.from_numpy(solved["v"]).cuda(), torch.from_numpy(solved["f"]).cuda(),
                                        torch.from_numpy(mask).cuda())
    ev, ef = po.remove_vertices_by_mask(solved["v"], solved["f"], mask)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), ev.view(np.uint32)) and np.array_equal(f.cpu().numpy(), ef)
    rng = np.random.default_rng(1)
    mask = rng.uniform(size=len(solved["v"])) < 0.5
    v, f = mesh.remove_vertices_by_mask(torch.from_numpy(solved["v"]).cuda(), torch.from_numpy(solved["f"]).cuda(),
                                        torch.from_numpy(mask).cuda())
    ev, ef = po.remove_vertices_by_mask(solved["v"], solved["f"], mask)
    assert np.array_equal(v.cpu().numpy().view(np.uint32), ev.view(np.uint32)) and np.array_equal(f.cpu().numpy(), ef)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sphere", "torus"])
def test_gpu_depth8_million_samples(kind):
    import torch
    p, n = sphere(1_000_000, seed=21) if kind == "sphere" else torus(1_000_000, seed=22)
    P, N = torch.from_numpy(p).float().cuda(), torch.from_numpy(n).float().cuda()
    v1, f1, d1 = mesh.create_from_point_cloud_poisson(P, N, depth=8)
    v2, f2, d2 = mesh.create_from_point_cloud_poisson(P, N, depth=8)
    assert torch.equal(v1.view(torch.int32), v2.view(torch.int32)) and torch.equal(f1, f2)
    assert torch.equal(d1.view(torch.int64), d2.view(torch.int64))
    h = 1.1 * float((P.amax(0) - P.amin(0)).max()) / 256
    check_closed_shape(v1.cpu().numpy(), f1.cpu().numpy(), h, kind)


@pytest.mark.gpu
def test_gpu_rejects_bad_input():
    import torch
    p, n = sphere(100)
    P, N = torch.from_numpy(p).cuda(), torch.from_numpy(n).cuda()
    bad = [(torch.from_numpy(p), N, 5), (P, N[:50], 5), (P[:, :2], N[:, :2], 5), (P.int(), N, 5), (P[:3], N[:3], 5),
           (P, N, 0), (P, N, 11), (P, N, 5.0), (P, N, True), (P * 0 + 1, N, 5)]
    Pn = P.clone()
    Pn[3, 1] = float("nan")
    Nn = N.clone()
    Nn[7, 0] = float("inf")
    bad += [(Pn, N, 5), (P, Nn, 5)]
    for args in bad:
        with pytest.raises(ValueError):
            mesh.create_from_point_cloud_poisson(*args)
    with pytest.raises(ValueError):
        mesh.create_from_point_cloud_poisson(P, N, 5, scale=0.5)
    v, f, _ = mesh.create_from_point_cloud_poisson(P.float(), N, 3)      # mixed dtypes run in fp64
    assert len(v) and len(f)


def _write_scan(root, pts, nrm, W=96, H=72, cams=4):
    import cv2
    scan = root / "scan1"
    (scan / "images").mkdir(parents=True)
    (scan / "cams").mkdir()
    _cloud_ply(str(scan / "stl001_total.ply"), pts, nrm, "binary", True, dtype="float")
    Es = []
    for i in range(cams):
        cv2.imwrite(str(scan / "images" / f"{i:08d}.jpg"), np.full((H, W, 3), 128, np.uint8))
        a = 0.3 * (i - cams / 2)
        Rm = np.array([[np.cos(a), 0, -np.sin(a)], [0, 1, 0], [np.sin(a), 0, np.cos(a)]])
        E = np.eye(4)
        E[:3, :3] = Rm
        E[:3, 3] = [0.05 * i, -0.03, 4.0]          # world -> camera: the sphere 4 units in front
        Es.append(E)
        text = "extrinsic\n" + "\n".join(" ".join(repr(float(x)) for x in r) for r in E) + "\n\nintrinsic\n" + \
            f"60 0 {W / 2}\n0 60 {H / 2}\n0 0 1\n\n425 2.5\n"
        (scan / "cams" / f"{i:08d}_cam.txt").write_text(text)
    return scan, Es


@pytest.mark.gpu
def test_gpu_get_mesh_from_ply_then_render_dtu_scenes(tmp_path):
    # the camera-facing half (z < 0 in the world) is sampled densely, so the trimmed low-density 10 % lies behind it
    p, n = sphere(400_000, seed=31)
    rng = np.random.default_rng(32)
    keep = (p[:, 2] < 0.2) | (rng.uniform(size=len(p)) < 0.2)
    p, n = p[keep], n[keep]
    scan, Es = _write_scan(tmp_path, p, n)
    before = set(sys.modules)
    v, f = mesh.get_mesh_from_ply(str(scan), depth=7)
    mesh.render_dtu_scenes(str(scan), method=None)
    assert not {m for m in set(sys.modules) - before if m.split(".")[0] in ("open3d", "trimesh", "pyrender")}
    rv, rf = mesh.read_ply_mesh(str(scan / "001_pcd.ply"))
    assert np.array_equal(rv, v.cpu().numpy()) and np.array_equal(rf, f.cpu().numpy())
    h = 1.1 * float((p.max(0) - p.min(0)).max()) / 128
    W, H = 96, 72
    for i, E in enumerate(Es):
        depth = np.load(scan / "depths" / f"{i:08d}.npy")
        assert depth.shape == (H, W) and depth.dtype == np.float32
        c, r = np.meshgrid(np.arange(W), np.arange(H))
        d = np.stack([(c + 0.5 - W / 2) / 60, (r + 0.5 - H / 2) / 60, np.ones_like(c, float)], -1)
        C0 = E[:3, 3]                                   # the sphere's centre (world origin) in camera coordinates
        bq = (d @ C0)
        aq = (d * d).sum(-1)
        disc = bq ** 2 - aq * (C0 @ C0 - 1.0)
        hit = disc > 0
        s = np.where(hit, (bq - np.sqrt(np.maximum(disc, 0))) / aq, 0)
        covered = depth > 0
        assert covered[hit].mean() >= 0.8, covered[hit].mean()
        # a surface distance of up to h reaches the depth along a ray as h / cos(incidence): grazing rays (cos < 0.35)
        # near the silhouette are left out of the depth bar
        pt = d * s[..., None]
        nrm = (pt - C0) / np.linalg.norm(pt - C0, axis=-1, keepdims=True)
        cos = np.abs((nrm * d).sum(-1)) / np.linalg.norm(d, axis=-1)
        both = covered & hit & (cos >= 0.35)
        assert both.sum() > 0.5 * hit.sum()
        assert np.abs(depth[both] - s[both]).max() <= h
