"""Oracle of the Poisson mesher (include/patchmatch_b200.h "Poisson surface reconstruction"; beyond the reference, which has
no mesher): the keep test, grid, density, weights, right-hand side, an exact float64 solve, the iso-value, the band field,
marching cubes (mesh_oracle.marching_cubes) and the nearest-point colours (cKDTree), restated in numpy / scipy.  Node
arrays are [N+1]^3 indexed [z, y, x], the layout of the native fields.  Never imported by the product.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from oracle import mesh_oracle as mo

CORNERS = [(k & 1, (k >> 1) & 1, k >> 2) for k in range(8)]


def keep(xyz, normals):
    """-> (mask [n], normals divided by their float64 length [n,3])."""
    p = np.asarray(xyz, np.float32)
    n = np.asarray(normals, np.float32).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        length = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        m = np.isfinite(p).all(1) & np.isfinite(n).all(1) & (length > 0) & np.isfinite(length)
        unit = n / np.where(m, length, 1.0)[:, None]
    return m, unit


def quantile(v: np.ndarray, q: float) -> float:
    s = np.sort(np.asarray(v, np.float64))
    pos = q * (len(s) - 1)
    g = int(np.floor(pos))
    t = pos - np.floor(pos)
    return float(s[g] + t * (s[min(g + 1, len(s) - 1)] - s[g]))


def place(xyz_kept, depth: int, scale: float = 1.1, q: float = 0.0):
    """-> (N, h, I0 int64 [3], lo [3], hi [3])."""
    N = 1 << depth
    lo = np.array([quantile(xyz_kept[:, a], q) for a in range(3)])
    hi = np.array([quantile(xyz_kept[:, a], 1.0 - q) for a in range(3)])
    E = float((hi - lo).max())
    h = scale * E / N
    I0 = np.floor((0.5 * (lo + hi)) / h).astype(np.int64) - N // 2
    return N, h, I0, lo, hi


def grid_coords(xyz, h: float, I0) -> np.ndarray:
    return (np.asarray(xyz, np.float32).astype(np.float64) / h - 0.5) - I0.astype(np.float64)


def cells(u: np.ndarray, N: int):
    base = np.clip(np.floor(u).astype(np.int64), 0, N - 1)
    return base, u - base


def _corner(base, f, k):
    c = CORNERS[k]
    w = [np.where(c[a], f[:, a], 1.0 - f[:, a]) for a in range(3)]
    s = [1.0 if c[a] else -1.0 for a in range(3)]
    idx = (base[:, 2] + c[2], base[:, 1] + c[1], base[:, 0] + c[0])
    return idx, (w[0] * w[1]) * w[2], np.stack([(s[0] * w[1]) * w[2], (w[0] * s[1]) * w[2], (w[0] * w[1]) * s[2]], 1)


def density(u, N: int):
    """-> (rho [N+1]^3, w per point)."""
    base, f = cells(u, N)
    rho = np.zeros((N + 1,) * 3)
    for k in range(8):
        idx, wt, _ = _corner(base, f, k)
        np.add.at(rho, idx, wt)
    rp = np.zeros(len(u))
    for k in range(8):
        idx, wt, _ = _corner(base, f, k)
        rp += wt * rho[idx]
    return rho, 1.0 / rp


def rhs(u, unit_normals, w, N: int) -> np.ndarray:
    base, f = cells(u, N)
    b = np.zeros((N + 1,) * 3)
    for k in range(8):
        idx, _, g = _corner(base, f, k)
        np.add.at(b, idx, w * (unit_normals * g).sum(1))
    b[[0, -1], :, :] = 0
    b[:, [0, -1], :] = 0
    b[:, :, [0, -1]] = 0
    return b


def kron_matrix(n: int) -> sp.csr_matrix:
    """A over n interior nodes per axis: K(x)M(x)M + M(x)K(x)M + M(x)M(x)K."""
    K = sp.diags([-np.ones(n - 1), 2 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1])
    M = sp.diags([np.ones(n - 1) / 6, 4 * np.ones(n) / 6, np.ones(n - 1) / 6], [-1, 0, 1])
    return (sp.kron(sp.kron(K, M), M) + sp.kron(sp.kron(M, K), M) + sp.kron(sp.kron(M, M), K)).tocsr()


def prolongation(nc: int) -> sp.csr_matrix:
    """Trilinear prolongation from nc coarse interior nodes per axis to 2 nc + 1 fine ones."""
    P = sp.lil_matrix((2 * nc + 1, nc))
    for j in range(nc):
        P[2 * j + 1, j] = 1.0
        P[2 * j, j] = 0.5
        P[2 * j + 2, j] = 0.5
    P = P.tocsr()
    return sp.kron(sp.kron(P, P), P).tocsr()


def apply_A(chi: np.ndarray) -> np.ndarray:
    """A chi at the interior nodes of a full [N+1]^3 field (boundary values taken as they are, normally 0)."""
    N = chi.shape[0] - 1
    c = chi.astype(np.float64)
    out = np.zeros_like(c)
    inner = out[1:N, 1:N, 1:N]
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nz = (dx != 0) + (dy != 0) + (dz != 0)
                wgt = [8.0 / 3.0, 0.0, -1.0 / 6.0, -1.0 / 12.0][nz]
                if wgt:
                    inner += wgt * c[1 + dz : N + dz, 1 + dy : N + dy, 1 + dx : N + dx]
    return out


def relative_residual(b: np.ndarray, chi: np.ndarray) -> float:
    r = (b.astype(np.float64) - apply_A(chi))[1:-1, 1:-1, 1:-1]
    return float(np.sqrt((r * r).sum()) / np.sqrt((b.astype(np.float64) ** 2).sum()))


def solve(b: np.ndarray, exact: bool = True) -> np.ndarray:
    """chi over [N+1]^3 with zero boundary: spsolve (exact), or CG to a relative residual of 1e-12."""
    N = b.shape[0] - 1
    A = kron_matrix(N - 1)
    rhs_v = b[1:N, 1:N, 1:N].reshape(-1).astype(np.float64)
    chi = np.zeros((N + 1,) * 3)
    if not rhs_v.any():
        return chi
    if exact:
        x = spl.spsolve(A.tocsc(), rhs_v)
    else:
        x, info = spl.cg(A, rhs_v, rtol=1e-12, maxiter=20000)
        assert info == 0
    chi[1:N, 1:N, 1:N] = x.reshape(N - 1, N - 1, N - 1)
    return chi


def iso_value(u, w, chi, N: int) -> float:
    base, f = cells(u, N)
    c = np.zeros(len(u))
    for k in range(8):
        idx, wt, _ = _corner(base, f, k)
        c += wt * chi[idx].astype(np.float64)
    return float((w * c).sum() / w.sum())


def band_field(keys, I0, N: int, chi, iso: float):
    """(tsdf float32, weight float32) per voxel of the allocated blocks."""
    node = mo.voxel_coords(np.asarray(keys, np.uint64)) - I0[None, :]
    inside = ((node >= 1) & (node <= N - 1)).all(1)
    nd = np.where(inside[:, None], node, 1)
    vals = chi[nd[:, 2], nd[:, 1], nd[:, 0]].astype(np.float64)
    tsdf = np.where(inside, (vals - iso).astype(np.float32), np.float32(1.0)).astype(np.float32)
    return tsdf, inside.astype(np.float32)


def nearest_colours(vertices, points, rgb):
    """Colour of the nearest point (float64 distance; ties to the smaller index)."""
    from scipy.spatial import cKDTree

    P = np.asarray(points, np.float32).astype(np.float64)
    V = np.asarray(vertices, np.float32).astype(np.float64)
    tree = cKDTree(P)
    d, _ = tree.query(V, k=1)
    out = np.zeros((len(V), 3), np.uint8)
    for i, cand in enumerate(tree.query_ball_point(V, d * (1 + 1e-9) + 1e-300)):
        cand = np.array(sorted(cand))
        diff = P[cand] - V[i]
        dd = (diff[:, 0] * diff[:, 0] + diff[:, 1] * diff[:, 1]) + diff[:, 2] * diff[:, 2]
        out[i] = rgb[cand[np.flatnonzero(dd == dd.min())[0]]]
    return out


def poisson(xyz, normals, rgb=None, depth: int = 5, scale: float = 1.1, band: int = 2, q: float = 0.0, exact: bool = True):
    """The whole definition -> dict(N, h, I0, inside (mask over the input), u, rho, w, b, chi, iso, keys, tsdf, weight, pos,
    col, faces)."""
    m, unit = keep(xyz, normals)
    if not m.any():
        raise ValueError("no point is kept")
    x = np.asarray(xyz, np.float32)
    N, h, I0, lo, hi = place(x[m], depth, scale, q)
    u_all = grid_coords(np.where(m[:, None], x, 0), h, I0)
    inside = m & ((u_all >= 0) & (u_all <= N)).all(1)
    u = u_all[inside]
    rho, w = density(u, N)
    b = rhs(u, unit[inside], w, N)
    chi = solve(b, exact)
    iso = iso_value(u, w, chi, N)
    keys = mo.allocate(x[inside], h, band)
    tsdf, weight = band_field(keys, I0, N, chi, iso)
    pos, _, faces = mo.marching_cubes(keys, h, tsdf, weight, np.zeros((len(tsdf), 3), np.uint8))
    col = nearest_colours(pos, x[inside], np.asarray(rgb)[inside]) if rgb is not None and len(pos) else None
    return dict(N=N, h=h, I0=I0, inside=inside, u=u, rho=rho, w=w, b=b, chi=chi, iso=iso, keys=keys, tsdf=tsdf, weight=weight,
                pos=pos, col=col, faces=faces)
