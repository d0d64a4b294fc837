"""Meshes for the simplifier's tests: a tilted bordered grid, hard inputs, floaters beside a sphere, and the invariants a
simplified mesh must keep."""
import numpy as np

def grid(n=20):
    """A tilted planar (n x n)-quad grid with an open rectangular border, away from the origin so that no coordinate is 0.
    Every coordinate is exact in float32, so the vertices lie exactly on the plane z = 0.5 (x - 3.25) + 0.25 (y + 7.5) + 1.75."""
    u, v = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij")
    u, v = u.ravel(), v.ravel()
    xyz = np.stack([u * 0.5 + 3.25, v * 0.5 - 7.5, 0.25 * u + 0.125 * v + 1.75], 1).astype(np.float32)
    idx = lambda i, j: i * (n + 1) + j
    f = []
    for i in range(n):
        for j in range(n):
            f += [[idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], [idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)]]
    corners = [idx(0, 0), idx(n, 0), idx(0, n), idx(n, n)]
    return xyz, np.array(f, np.int32), corners


def grid_plane_distance(p):
    """Distance of points to the grid's plane, in float64."""
    q = np.asarray(p, np.float64) - np.array([3.25, -7.5, 1.75])
    n = np.array([-0.5, -0.25, 1.0])
    return np.abs((q * n).sum(1)) / np.sqrt((n * n).sum())


def tetrahedron():
    xyz = np.array([[0.1, 0.2, 0.3], [1.1, 0.2, 0.3], [0.1, 1.2, 0.3], [0.1, 0.2, 1.3]], np.float32)
    return xyz, np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int32)


def strip():
    xyz = np.array([[0, 0, 0.5], [1, 0, 0.5], [0, 1, 0.5], [1, 1, 0.5]], np.float32)
    return xyz, np.array([[0, 1, 3], [0, 3, 2]], np.int32)


def fan(n=40):
    """A flat fan of n triangles around vertex 0: vertex 0 is locked (valence above the cap)."""
    a = np.linspace(0, 2 * np.pi, n, endpoint=False)
    xyz = np.concatenate([[[0.0, 0.0, 1.0]], np.stack([np.cos(a), np.sin(a), np.ones(n)], 1)]).astype(np.float32)
    return xyz, np.array([[0, 1 + i, 1 + (i + 1) % n] for i in range(n)], np.int32)


def non_manifold():
    """Three triangles on one edge (0, 1), plus a strip around them."""
    xyz, f, _ = grid(4)
    nv = len(xyz)
    extra = np.array([[0.0, 0.0, 9.0], [1.0, 2.0, -9.0]], np.float32) + xyz[5]
    e = f[10]
    return np.concatenate([xyz, extra]), np.concatenate([f, [[e[0], e[1], nv], [e[1], e[0], nv + 1]]]).astype(np.int32)


def slivers():
    """A grid with zero-area slivers, as marching cubes makes them where a tsdf is exactly 0: a few interior vertices sit
    exactly on a neighbour along u (distinct indices, identical coordinates), so the two faces on that edge have a zero
    cross product; nothing folds over."""
    xyz, f, _ = grid(8)
    xyz = xyz.copy()
    for v in (10, 32, 58):  # interior vertices, pairwise not adjacent
        xyz[v] = xyz[v + 9]
    return xyz, f


def zero_area(xyz, faces):
    """Faces whose float64 cross product (X1 - X0) x (X2 - X0) is exactly zero."""
    p = np.asarray(xyz, np.float64)[np.asarray(faces, np.int64)]
    n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    return (n == 0).all(1)


def floaters(sphere_xyz, sphere_faces):
    """The sphere plus floaters of 1, 4 and 40 faces, far from it; -> (xyz, faces, the floaters' smallest vertex ids)."""
    xyz, faces, first = [sphere_xyz], [sphere_faces], []
    nv = len(sphere_xyz)
    for n, off in ((1, 5.0), (4, 7.0), (40, 9.0)):
        k = int(np.ceil(np.sqrt(n / 2)))
        g, f, _ = grid(k)
        f = f[:n]
        first.append(nv)
        xyz.append(g + np.float32(off))
        faces.append(f + nv)
        nv += len(g)
    return np.concatenate(xyz).astype(np.float32), np.concatenate(faces).astype(np.int32), first


def check_invariants(xyz, faces, target=None):
    """No repeated indices, no duplicate faces (as vertex sets), no unreferenced vertices, indices in range."""
    f = np.asarray(faces, np.int64)
    if target is not None:
        assert len(f) <= target
    if len(f) == 0:
        assert len(xyz) == 0
        return
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all()
    s = np.sort(f, 1)
    assert len(np.unique(s, axis=0)) == len(s)
    assert f.min() >= 0 and f.max() < len(xyz)
    assert len(np.unique(f)) == len(xyz)
