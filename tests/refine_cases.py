"""Analytic scenes for the mesh refinement tests (test infrastructure): the sphere of tests/mesh_cases seen by its cameras but
carrying a high-frequency albedo (a period of about 10 pixels, so there is detail to refine against), rendered exactly by
ray-sphere hits at the pixel centres; a textured plane; subdivided icosphere meshes and radial noise."""
from __future__ import annotations

import math

import numpy as np

from tests import mesh_cases as mc

PERIOD = 0.13  # world units: about 10 pixels at the sphere's front for mesh_cases.sphere_scene's cameras (f 170, distance 2.2)


def albedo(world: np.ndarray) -> np.ndarray:
    """float32 [...] grey in [0.1, 0.9]: products of sines of the world coordinates with a period of about PERIOD."""
    k = 2 * math.pi / PERIOD
    x, y, z = world[..., 0], world[..., 1], world[..., 2]
    s = 0.5 * np.sin(k * x + 0.7) * np.cos(1.1 * k * y) + 0.5 * np.sin(0.9 * k * z + 1.3 * np.sin(0.5 * k * x))
    return (0.5 + 0.4 * s).astype(np.float32)


def _render_sphere(K, E, H, W):
    depth, _ = mc.sphere_depth(K, E, H, W)
    K64, E64 = K.astype(np.float64), E.astype(np.float64)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    ray = np.linalg.inv(K64) @ np.stack([u.ravel(), v.ravel(), np.ones(H * W)])
    cam = ray * depth.astype(np.float64).ravel()
    world = (np.linalg.inv(E64) @ np.vstack([cam, np.ones(H * W)]))[:3].T
    g = np.where(depth.ravel() > 0, albedo(world), 0.0).reshape(H, W).astype(np.float32)
    return np.stack([g, g, g])


def sphere_views(n_views: int = 14, H: int = 120, W: int = 160, sizes=None):
    """mesh_cases.sphere_scene's cameras with the albedo's images -> (images, Ks, Es)."""
    scn = mc.sphere_scene(n_views=n_views, H=H, W=W, sizes=sizes, n_seeds=10)
    images = [_render_sphere(K, E, *d.shape) for K, E, d in zip(scn["Ks"], scn["Es"], scn["depths"])]
    return images, scn["Ks"], scn["Es"]


def icosphere(level: int, centre=mc.SPHERE_CENTRE, radius=mc.SPHERE_RADIUS):
    """(xyz float32 [nv,3], faces int32 [nf,3]) of the unit icosahedron subdivided `level` times, outward wound."""
    t = (1 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t], [t, 0, -1], [t, 0, 1],
         [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6], [7, 1, 8],
         [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10], [8, 6, 7], [9, 8, 1]]
    verts = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    faces = f
    for _ in range(level):
        mid = {}

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = verts[a] + verts[b]
                verts.append(p / np.linalg.norm(p))
                mid[k] = len(verts) - 1
            return mid[k]

        nf = []
        for a, b, c in faces:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        faces = nf
    xyz = np.asarray(centre) + radius * np.array(verts)
    return xyz.astype(np.float32), np.array(faces, np.int32)


def radial_noise(xyz: np.ndarray, amplitude: float, seed: int = 0) -> np.ndarray:
    """xyz moved along the radius from the sphere centre by a smooth random field with maximum |amplitude|."""
    rng = np.random.default_rng(seed)
    d = xyz.astype(np.float64) - mc.SPHERE_CENTRE
    n = d / np.linalg.norm(d, axis=1, keepdims=True)
    field = np.zeros(len(xyz))
    for _ in range(6):
        k = rng.normal(size=3) * 3.0
        field += np.sin(n @ k + rng.uniform(0, 2 * math.pi))
    field *= amplitude / np.abs(field).max()
    return (xyz.astype(np.float64) + field[:, None] * n).astype(np.float32)


def radial_error(xyz: np.ndarray) -> np.ndarray:
    return np.linalg.norm(xyz.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS


def sphere_pairs(Es, neighbours: int):
    """Per view, its `neighbours` nearest other views by camera centre: [(i, j)]."""
    C = np.array([-(np.asarray(E, np.float64)[:3, :3].T @ np.asarray(E, np.float64)[:3, 3]) for E in Es])
    out = []
    for i in range(len(Es)):
        d = np.linalg.norm(C - C[i], axis=1)
        d[i] = np.inf
        out += [(i, int(j)) for j in np.argsort(d, kind="stable")[:neighbours]]
    return out


def plane_case(H: int = 48, W: int = 64, n: int = 12):
    """A grid of 2 n^2 triangles on z = 4 (x, y in [-1, 1]) wound towards three cameras near the origin, with the albedo
    rendered by ray-plane hits -> (xyz, faces, images, Ks, Es)."""
    g = np.stack(np.meshgrid(np.linspace(-1, 1, n + 1), np.linspace(-1, 1, n + 1)), -1).reshape(-1, 2)
    xyz = np.concatenate([g, np.full((len(g), 1), 4.0)], 1).astype(np.float32)
    i = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).ravel()
    faces = np.concatenate([np.stack([i, i + n + 2, i + 1], 1), np.stack([i, i + n + 1, i + n + 2], 1)]).astype(np.int32)
    images, Ks, Es = [], [], []
    for cx in (-0.3, 0.0, 0.3):
        E = mc.look_at(np.array([cx, 0.1 * cx, 0.0]), np.array([0.0, 0.0, 4.0]))
        K = np.array([[60, 0, W / 2 - 0.5], [0, 60, H / 2 - 0.5], [0, 0, 1]], np.float32)
        K64, E64 = K.astype(np.float64), E.astype(np.float64)
        u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
        ray = np.linalg.inv(E64[:3, :3]) @ np.linalg.inv(K64) @ np.stack([u.ravel(), v.ravel(), np.ones(H * W)])
        C = -np.linalg.inv(E64[:3, :3]) @ E64[:3, 3]
        t = (4.0 - C[2]) / ray[2]
        world = (C[:, None] + ray * t).T
        gimg = albedo(world * np.array([0.2, 0.2, 0.0])).reshape(H, W)
        images.append(np.stack([gimg, gimg, gimg]).astype(np.float32))
        Ks.append(K)
        Es.append(E)
    return xyz, faces, images, Ks, Es
