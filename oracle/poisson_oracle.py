"""Dense-grid screened Poisson surface reconstruction in numpy / scipy fp64: the discrete problem that csrc/poisson.cu
solves, restated for the tests (definitions in csrc/poisson_math.cuh's header comment).

Every value the device rounds in a fixed order (geometry, hat weights, edge points, quantile lerp) is computed here in
the same order, so the extractor fed the device's chi and iso reproduces its vertices and faces bit for bit; sums over
samples (b, S, density, iso) are held to the device within a relative tolerance instead.
"""
from __future__ import annotations

import itertools

import numpy as np
import scipy.sparse as sp

ALPHA = 4.0


# ----------------------------------------------------------------------------------------------------------------------
# grid
# ----------------------------------------------------------------------------------------------------------------------
def geometry(points, depth, scale=1.1):
    p = np.asarray(points, np.float64)
    lo, hi = p.min(0), p.max(0)
    m = 0.0
    for d in range(3):
        e = hi[d] - lo[d]
        m = e if e > m else m
    L = scale * m
    origin = np.array([(lo[d] + hi[d]) * 0.5 - L * 0.5 for d in range(3)])
    return origin, L, L / float(1 << depth)


def locate(points, origin, h, R):
    """-> cells [N, 3] int (x, y, z), local coordinates f [N, 3]."""
    g = (np.asarray(points, np.float64) - origin) / h
    c = np.clip(np.floor(g), 0, R - 1).astype(np.int64)
    return c, g - c


def corner_weights(f):
    """[N, 8] hat weights ((wx wy) wz) of the 8 cell corners (bit 0 = x, 1 = y, 2 = z)."""
    w = np.empty((len(f), 8))
    for q in range(8):
        wx = f[:, 0] if q & 1 else 1.0 - f[:, 0]
        wy = f[:, 1] if q & 2 else 1.0 - f[:, 1]
        wz = f[:, 2] if q & 4 else 1.0 - f[:, 2]
        w[:, q] = (wx * wy) * wz
    return w


def unit_normals(n):
    n = np.asarray(n, np.float64)
    nn = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    out = np.zeros_like(n)
    ok = nn > 0
    out[ok] = n[ok] / nn[ok, None]
    return out


def node_index(x, y, z, R):
    return (z * (R + 1) + y) * (R + 1) + x


def cell_index(x, y, z, R):
    return (z * R + y) * R + x


def corner_nodes(cells, R):
    """[M, 8] node indices of the corners of cells [M, 3]."""
    return np.stack([node_index(cells[:, 0] + (q & 1), cells[:, 1] + (q >> 1 & 1), cells[:, 2] + (q >> 2 & 1), R)
                     for q in range(8)], 1)


def stiffness(k):
    return (1.0 / 3.0, 0.0, -1.0 / 12.0, -1.0 / 12.0)[k]


def divergence(k):
    return (1.0 / 18.0, 1.0 / 36.0, 1.0 / 72.0)[k]


def element_stiffness():
    """[8, 8] int grad phi_p . grad phi_q over a unit cell (times h on a cell of side h)."""
    return np.array([[stiffness(bin(p ^ q).count("1")) for q in range(8)] for p in range(8)])


def element_divergence(d):
    """[8, 8] int d_d phi_p phi_q over a unit cell (times h^2 on a cell of side h)."""
    E = np.zeros((8, 8))
    for p in range(8):
        for q in range(8):
            k = sum(((p ^ q) >> e) & 1 for e in range(3) if e != d)
            E[p, q] = (1.0 if (p >> d) & 1 else -1.0) * divergence(k)
    return E


def _assemble(R, E):
    """Sparse (R+1)^3 square matrix summing the element matrix E over every cell."""
    c = np.stack(np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing="ij"), -1).reshape(-1, 3)[:, ::-1]
    cn = corner_nodes(c, R)
    rows = np.repeat(cn, 8, 1).reshape(-1)
    cols = np.tile(cn, (1, 8)).reshape(-1)
    vals = np.tile(E.reshape(-1), len(c))
    n = (R + 1) ** 3
    return sp.csr_matrix((vals, (rows, cols)), shape=(n, n))


class System:
    """The assembled problem of one cloud: geometry, a, beta, v, b, K, S (sparse), the screening blocks per occupied
    cell {cell index: [8, 8]}, and the solver's helpers."""

    def __init__(self, points, normals, depth, scale=1.1):
        self.points = np.asarray(points, np.float64)
        self.depth, self.R = depth, 1 << depth
        R = self.R
        self.origin, self.L, self.h = geometry(self.points, depth, scale)
        self.cells, self.f = locate(self.points, self.origin, self.h, R)
        self.w = corner_weights(self.f)
        self.cn = corner_nodes(self.cells, R)
        self.cell_id = cell_index(self.cells[:, 0], self.cells[:, 1], self.cells[:, 2], R)
        N = len(self.points)
        self.occupied = len(np.unique(self.cell_id))
        self.a = (self.occupied * (self.h * self.h)) / N
        self.beta = ALPHA * self.a
        n = unit_normals(normals)
        nn = (R + 1) ** 3
        coef = self.a / (self.h * self.h * self.h)
        self.v = np.zeros((3, nn))
        for d in range(3):
            np.add.at(self.v[d], self.cn.reshape(-1), (self.w * n[:, d:d + 1]).reshape(-1))
        self.v *= coef
        self.K = _assemble(R, element_stiffness()) * self.h
        self.D = [_assemble(R, element_divergence(d)) * (self.h * self.h) for d in range(3)]
        # b_i = sum_j v_j^d int d_d phi_i phi_j
        self.b = sum(self.D[d] @ self.v[d] for d in range(3))
        rows = np.repeat(self.cn, 8, 1).reshape(-1)
        cols = np.tile(self.cn, (1, 8)).reshape(-1)
        vals = (self.w[:, :, None] * self.w[:, None, :]).reshape(-1)
        self.S = sp.csr_matrix((vals, (rows, cols)), shape=(nn, nn))
        self.A = (self.K + self.beta * self.S).tocsr()

    def blocks(self):
        """{cell index: [8, 8] sum_s phi_p(s) phi_q(s) over the cell's samples}."""
        out = {}
        order = np.argsort(self.cell_id, kind="stable")
        ids = self.cell_id[order]
        starts = np.flatnonzero(np.r_[True, ids[1:] != ids[:-1]])
        ends = np.r_[starts[1:], len(ids)]
        for s, e in zip(starts, ends):
            w = self.w[order[s:e]]
            out[int(ids[s])] = w.T @ w
        return out

    def solve(self):
        from scipy.sparse.linalg import spsolve
        return spsolve(self.A.tocsc(), self.b)

    def iso(self, chi):
        return float(np.mean((self.w * chi[self.cn]).sum(1)))

    def density_grid(self):
        """Sample counts splatted on the grid of depth max(depth - 2, 1), over its cell volume: [(Rd + 1)^3]."""
        dd = max(self.depth - 2, 1)
        Rd, hd = 1 << dd, self.L / float(1 << dd)
        cc = self.cells // (self.R // Rd)
        g = (self.points - self.origin) / hd
        w = corner_weights(g - cc)
        D = np.zeros((Rd + 1) ** 3)
        np.add.at(D, corner_nodes(cc, Rd).reshape(-1), w.reshape(-1))
        return D / ((hd * hd) * hd), dd

    def densities(self, vertices):
        D, dd = self.density_grid()
        Rd, hd = 1 << dd, self.L / float(1 << dd)
        v = np.asarray(vertices, np.float32).astype(np.float64)
        c, f = locate(v, self.origin, hd, Rd)
        w = corner_weights(f)
        vals = D[corner_nodes(c, Rd)]
        out = np.zeros(len(v))
        for q in range(8):
            out = out + w[:, q] * vals[:, q]
        return out


# ----------------------------------------------------------------------------------------------------------------------
# marching tetrahedra on the Kuhn split
# ----------------------------------------------------------------------------------------------------------------------
PERMS = list(itertools.permutations(range(3)))
TET_EDGES = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def tet_corners(t):
    a, b, _ = PERMS[t]
    return [0, 1 << a, (1 << a) | (1 << b), 7]


def tet_positive(t):
    c = [np.array([(m >> i) & 1 for i in range(3)], float) for m in tet_corners(t)]
    return bool(np.linalg.det(np.stack([c[1] - c[0], c[2] - c[0], c[3] - c[0]])) > 0)


def case_table():
    """[16] lists of triangles (tet-local edge triples) for a positively oriented tetrahedron, derived geometrically:
    triangles on the edges that join inside (bit 0) and outside (bit 1) vertices, a quad split along its (ac, bd)
    diagonal, each triangle wound so that its normal points towards the outside vertices."""
    V = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], float)    # det > 0
    table = []
    for code in range(16):
        out = [k for k in range(4) if code >> k & 1]
        ins = [k for k in range(4) if not code >> k & 1]
        cross = lambda a, b: TET_EDGES.index((min(a, b), max(a, b)))   # noqa: E731
        if len(out) in (0, 4):
            tris = []
        elif len(out) in (1, 3):
            lone = out[0] if len(out) == 1 else ins[0]
            rest = [k for k in range(4) if k != lone]
            tris = [[cross(lone, r) for r in rest]]
        else:
            a, b = ins
            c, d = out
            tris = [[cross(a, c), cross(a, d), cross(b, d)], [cross(a, c), cross(b, d), cross(b, c)]]
        fixed = []
        towards = V[out].mean(0) - V[ins].mean(0) if out and ins else None
        for tri in tris:
            P = [0.5 * (V[TET_EDGES[e][0]] + V[TET_EDGES[e][1]]) for e in tri]
            nrm = np.cross(P[1] - P[0], P[2] - P[0])
            fixed.append(tri if nrm @ towards > 0 else [tri[0], tri[2], tri[1]])
        table.append(fixed)
    return table


CASES = case_table()


def edge_point(xa, xb, va, vb, iso):
    t = (iso - va) / (vb - va)
    return np.float32(xa + t * (xb - xa))


def extract(chi, iso, origin, h, R):
    """The device's extractor in numpy: (vertices [V, 3] fp32, faces [F, 3] int64).  Vertices node-major, then by edge
    direction 1..7; faces cell-major, then by Kuhn tetrahedron, then in table order."""
    n1 = R + 1
    X = np.asarray(chi, np.float64).reshape(n1, n1, n1)           # [z, y, x]
    out = X > iso
    NN = n1 ** 3
    cross = np.zeros((NN, 7), bool)
    for d in range(1, 8):
        dx, dy, dz = d & 1, d >> 1 & 1, d >> 2 & 1
        m = np.zeros((n1, n1, n1), bool)
        m[:n1 - dz, :n1 - dy, :n1 - dx] = out[:n1 - dz, :n1 - dy, :n1 - dx] != out[dz:, dy:, dx:]
        cross[:, d - 1] = m.reshape(-1)
    node, dm1 = np.nonzero(cross)
    d = dm1 + 1
    x0, y0, z0 = node % n1, node // n1 % n1, node // (n1 * n1)
    ia = [x0, y0, z0]
    ib = [x0 + (d & 1), y0 + (d >> 1 & 1), z0 + (d >> 2 & 1)]
    va = X.reshape(-1)[node]
    vb = X.reshape(-1)[node_index(ib[0], ib[1], ib[2], R)]
    verts = np.empty((len(node), 3), np.float32)
    t = (iso - va) / (vb - va)
    for a in range(3):
        xa = origin[a] + h * ia[a].astype(np.float64)
        xb = origin[a] + h * ib[a].astype(np.float64)
        verts[:, a] = (xa + t * (xb - xa)).astype(np.float32)
    vid = np.full((NN, 7), -1, np.int64)
    vid[node, dm1] = np.arange(len(node))
    faces = []
    o = out.reshape(-1)
    cz, cy, cx = np.meshgrid(np.arange(R), np.arange(R), np.arange(R), indexing="ij")
    cells = np.stack([cx.reshape(-1), cy.reshape(-1), cz.reshape(-1)], 1)
    cn = corner_nodes(cells, R)
    co = o[cn]                                                        # [NC, 8]
    busy = np.flatnonzero(co.any(1) & ~co.all(1))
    for c in busy:
        for t in range(6):
            K = tet_corners(t)
            code = sum(int(co[c, K[k]]) << k for k in range(4))
            for tri in CASES[code]:
                if not tet_positive(t):
                    tri = [tri[0], tri[2], tri[1]]
                face = []
                for e in tri:
                    u, w = K[TET_EDGES[e][0]], K[TET_EDGES[e][1]]
                    face.append(vid[cn[c, u], (w ^ u) - 1])
                faces.append(face)
    return verts, np.array(faces, np.int64).reshape(-1, 3)


def reconstruct(points, normals, depth, scale=1.1):
    """The whole pipeline on the CPU: (System, chi, iso, vertices, faces, densities)."""
    s = System(points, normals, depth, scale)
    chi = s.solve()
    iso = s.iso(chi)
    v, f = extract(chi, iso, s.origin, s.h, s.R)
    return s, chi, iso, v, f, s.densities(v)


def remove_vertices_by_mask(vertices, faces, mask):
    keep = ~np.asarray(mask, bool)
    new = np.cumsum(keep) - 1
    fk = keep[faces].all(1) if len(faces) else np.zeros(0, bool)
    return np.asarray(vertices)[keep], new[faces[fk]].astype(np.int64)
