"""Seeded clouds, meshes and cameras for the renderer's tests (test infrastructure)."""
from __future__ import annotations

import numpy as np

W, H = 320, 240
F = 300.0


def pinhole(f: float = F, w: int = W, h: int = H, E=None) -> np.ndarray:
    """float64 3 x 4 K [R | t]; E (4 x 4 world -> camera) defaults to the identity."""
    K = np.array([[f, 0.0, (w - 1) / 2.0 + 0.25], [0.0, f, (h - 1) / 2.0 - 0.125], [0.0, 0.0, 1.0]])
    E = np.eye(4) if E is None else np.asarray(E, np.float64)
    return K @ E[:3, :4]


def cloud(n: int, seed: int = 0, w: int = W, h: int = H, f: float = F):
    """(xyz float32 [n,3], rgb uint8 [n,3], normals float32 [n,3]) seen by pinhole(): most points in front of the camera and
    in the frame, some behind it, some outside the frame, exact duplicates of earlier points (depth ties at one pixel, the
    lower index wins), points at one depth a hair apart, and some zero normals."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.0, 8.0, n)
    z[rng.random(n) < 0.03] *= -1.0                        # behind the camera
    z[rng.random(n) < 0.01] = 0.0
    sx, sy = w / (2 * f) * 1.3, h / (2 * f) * 1.3         # about 30 % beyond the frame
    xyz = np.stack([rng.uniform(-sx, sx, n) * np.abs(z), rng.uniform(-sy, sy, n) * np.abs(z), z], 1).astype(np.float32)
    dup = rng.choice(n // 2, size=n // 50, replace=False)
    xyz[n // 2 + np.arange(dup.size)] = xyz[dup]            # exact ties, the copy has the larger index
    k = n // 2 + dup.size + np.arange(n // 100)
    xyz[k] = xyz[k - 1]
    xyz[k, 0] = np.nextafter(xyz[k - 1, 0], np.float32(np.inf))  # same depth, nearly the same place
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    nrm = rng.normal(size=(n, 3)).astype(np.float32)
    nrm[rng.random(n) < 0.05] = 0.0
    return xyz, rgb, nrm


def mesh(seed: int = 0, w: int = W, h: int = H, f: float = F):
    """(xyz float32 [nv,3], rgb uint8 [nv,3], faces int32 [nf,3]) seen by pinhole(): a wavy grid whose cells project to
    boxes on both sides of 16 x 16 pixels, a two-triangle quad behind it filling the whole frame, triangles of random size
    and orientation, degenerate triangles (a repeated vertex, collinear vertices), triangles with a vertex behind the near
    plane and with a vertex beyond 2^22 pixels."""
    rng = np.random.default_rng(seed)
    verts, faces = [], []

    def add(v, fc):
        base = sum(len(x) for x in verts)
        verts.append(np.asarray(v, np.float64))
        faces.append(np.asarray(fc, np.int64) + base)

    # wavy grid: cells of 10..30 pixels
    for g, (n, z0) in enumerate(((12, 3.0), (7, 2.5))):
        s = np.linspace(-0.9, 0.9, n)
        X, Y = np.meshgrid(s * (1.0 + 0.3 * g), s * 0.75)
        Z = z0 + 0.3 * np.sin(3 * X) * np.cos(2 * Y)
        v = np.stack([X.ravel() * Z.ravel() / 2.0, Y.ravel() * Z.ravel() / 2.0, Z.ravel()], 1)
        i = np.arange(n * n).reshape(n, n)
        q = np.stack([i[:-1, :-1].ravel(), i[:-1, 1:].ravel(), i[1:, 1:].ravel(), i[1:, :-1].ravel()], 1)
        add(v, np.concatenate([q[:, [0, 1, 2]], q[:, [0, 2, 3]]]))
    # a quad far behind everything, larger than the frame: the one-CTA-per-triangle path
    add([[-40, -30, 20], [40, -30, 20], [40, 30, 20], [-40, 30, 20]], [[0, 1, 2], [0, 2, 3]])
    # random triangles, both windings, sizes from a pixel to most of the frame
    m = 300
    c = np.stack([rng.uniform(-0.6, 0.6, m), rng.uniform(-0.45, 0.45, m), rng.uniform(1.5, 6.0, m)], 1)
    size = np.exp(rng.uniform(np.log(0.003), np.log(0.5), m))[:, None, None]
    tri = c[:, None, :] + size * rng.normal(size=(m, 3, 3)) * np.array([1.0, 1.0, 0.3])
    tri[:, :, :2] *= tri[:, :, 2:3] / 2.0
    add(tri.reshape(-1, 3), np.arange(3 * m).reshape(m, 3))
    # degenerate: a repeated vertex, collinear vertices
    add([[0, 0, 2], [0.1, 0, 2], [0.2, 0, 2], [0.1, 0.1, 2]], [[0, 1, 2], [0, 3, 3], [1, 1, 1]])
    # near plane: a vertex behind the camera, a vertex at z = 0; beyond 2^22 pixels in u
    add([[0, 0, 2], [0.3, 0.1, 2], [0.1, 0.2, -1], [0.0, 0.3, 0.0], [4e5, 0, 0.01]], [[0, 1, 2], [0, 1, 3], [0, 1, 4]])
    xyz = np.concatenate(verts).astype(np.float32)
    fc = np.concatenate(faces).astype(np.int32)
    rgb = rng.integers(0, 256, (len(xyz), 3), dtype=np.uint8)
    return xyz, rgb, fc


def fan(w: int = W, h: int = H, k: int = 11, centre=(100.0, 77.0)):
    """A fan of k triangles around a vertex exactly on pixel `centre`, its rim far outside the frame, at depth 1 through the
    camera [I | 0] (so u = x exactly): it covers the frame.  -> (xyz float32, faces int32, the 3 x 4 camera)."""
    P = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float64)
    ang = np.linspace(0, 2 * np.pi, k, endpoint=False) + 0.1
    rim = np.stack([centre[0] + 5000 * np.cos(ang), centre[1] + 5000 * np.sin(ang)], 1)
    xyz = np.concatenate([np.vstack([[centre], rim]), np.ones((k + 1, 1))], 1).astype(np.float32)
    faces = np.array([[0, 1 + i, 1 + (i + 1) % k] for i in range(k)], np.int32)
    return xyz, faces, P
