"""Float64 numpy restatement of the surface sampler (include/patchmatch_b200.h, "Surface sampling of triangle meshes";
csrc/pm_sample.cu, pm_sample_math.cuh), operation for operation in the same order, each rounded on its own: the GPU and
this oracle agree bit for bit.  TEST INFRASTRUCTURE: never imported by the package.

    lattice_sizes     n = max(1, ceil(L / s)) per face (0: a corner is not finite; MAX_LATTICE: n >= 2^31)
    face_samples      (n + 1)(n + 2) / 2 - 3, none for n <= 1
    lattice_points    the k-th face sample's (i, j), in the order i ascending, j ascending, corners left out
    sample            the whole output: the referenced finite vertices, then every face's lattice points
    sample_at         chosen output rows only, for meshes whose whole output is too large for the host
"""
from __future__ import annotations

import numpy as np

MAX_LATTICE = 1 << 31


def _edge(p, q):
    d = q - p
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def lattice_sizes(xyz, faces, s: float) -> np.ndarray:
    """int64 [nf]: each face's lattice size n, 0 when a corner is not finite, MAX_LATTICE when n >= 2^31."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    A, B, C = (xyz[faces[:, k]].astype(np.float64) for k in range(3))
    fin = np.isfinite(A).all(1) & np.isfinite(B).all(1) & np.isfinite(C).all(1)
    with np.errstate(invalid="ignore", over="ignore"):
        L = np.maximum(np.maximum(_edge(A, B), _edge(B, C)), _edge(C, A))
        n = np.ceil(L / np.float64(s))
    out = np.zeros(faces.shape[0], np.int64)
    big = fin & ~(n < MAX_LATTICE)
    ok = fin & ~big
    out[ok] = np.maximum(n[ok], 1.0).astype(np.int64)
    out[big] = MAX_LATTICE
    return out


def face_samples(n) -> np.ndarray:
    n = np.asarray(n, np.int64)
    return np.where(n <= 1, 0, (n + 1) * (n + 2) // 2 - 3)


def lattice_points(n, k):
    """(i, j) int64 of the k-th face sample of lattices of size n (arrays broadcast), by exact integer row inversion."""
    n, k = np.broadcast_arrays(np.asarray(n, np.int64), np.asarray(k, np.int64))
    N = (n + 1) * (n + 2) // 2
    p = np.where(k < n - 1, k + 1, k + 2)
    q = N - 1 - p
    t = np.maximum(((np.sqrt(8.0 * q.astype(np.float64) + 1.0) - 1.0) * 0.5).astype(np.int64), 0)
    while True:
        hi = t * (t + 1) // 2 > q
        if not hi.any():
            break
        t = t - hi
    while True:
        lo = (t + 1) * (t + 2) // 2 <= q
        if not lo.any():
            break
        t = t + lo
    return n - t, t - (q - t * (t + 1) // 2)


def points_at(xyz, rgb, faces, n, f, i, j):
    """Points (float64 [m,3]) and colours (uint8 [m,3] or None) of lattice points (i, j) of faces f with sizes n[f]."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    fv = np.asarray(faces, np.int64).reshape(-1, 3)[f]
    nn = np.asarray(n, np.int64)[f].astype(np.float64)
    wa = (nn - i.astype(np.float64) - j.astype(np.float64))  # exact: integers below 2^53
    wa, wb, wc = wa / nn, i.astype(np.float64) / nn, j.astype(np.float64) / nn
    corners = [xyz[fv[:, k]].astype(np.float64) for k in range(3)]
    P = (wa[:, None] * corners[0] + wb[:, None] * corners[1]) + wc[:, None] * corners[2]
    if rgb is None:
        return P, None
    rgb = np.asarray(rgb, np.uint8).reshape(-1, 3)
    cc = [rgb[fv[:, k]].astype(np.float64) for k in range(3)]
    col = np.rint((wa[:, None] * cc[0] + wb[:, None] * cc[1]) + wc[:, None] * cc[2])
    return P, np.clip(col, 0, 255).astype(np.uint8)


def referenced_vertices(xyz, faces) -> np.ndarray:
    """The finite vertices some face (with valid indices) references, ascending."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    used = np.zeros(xyz.shape[0], bool)
    used[faces.reshape(-1)] = True
    return np.nonzero(used & np.isfinite(xyz).all(1))[0]


def counts(xyz, faces, s: float):
    """-> (vertex samples, int64 [nf] face sample counts); ValueError when a face has n >= 2^31."""
    n = lattice_sizes(xyz, faces, s)
    if (n >= MAX_LATTICE).any():
        raise ValueError(f"face {int(np.argmax(n >= MAX_LATTICE))} needs n >= 2^31")
    return int(referenced_vertices(xyz, faces).size), face_samples(n)


def sample(xyz, faces, s: float, rgb=None):
    """The sampler's whole output: (float64 [m,3], uint8 [m,3] or None)."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    n = lattice_sizes(xyz, faces, s)
    c = face_samples(n)
    f = np.repeat(np.arange(c.size), c)
    k = np.arange(f.size, dtype=np.int64) - np.repeat(np.cumsum(c) - c, c)
    i, j = lattice_points(n[f], k)
    P, col = points_at(xyz, rgb, faces, n, f, i, j)
    v = referenced_vertices(xyz, faces)
    P = np.concatenate([xyz[v].astype(np.float64), P])
    if rgb is not None:
        col = np.concatenate([np.asarray(rgb, np.uint8).reshape(-1, 3)[v], col])
    return P, col


def sample_at(xyz, faces, s: float, rows, rgb=None):
    """Rows `rows` (int64, each < the total) of sample(xyz, faces, s, rgb), without forming the rest."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    rows = np.asarray(rows, np.int64)
    v = referenced_vertices(xyz, faces)
    n = lattice_sizes(xyz, faces, s)
    c = face_samples(n)
    off = np.cumsum(c) - c
    P = np.empty((rows.size, 3))
    col = None if rgb is None else np.empty((rows.size, 3), np.uint8)
    isv = rows < v.size
    P[isv] = xyz[v[rows[isv]]]
    if rgb is not None:
        col[isv] = np.asarray(rgb, np.uint8).reshape(-1, 3)[v[rows[isv]]]
    o = rows[~isv] - v.size
    f = np.searchsorted(off, o, side="right") - 1
    i, j = lattice_points(n[f], o - off[f])
    Pf, cf = points_at(xyz, rgb, faces, n, f, i, j)
    P[~isv] = Pf
    if rgb is not None:
        col[~isv] = cf
    return P, col
