"""Analytic scenes and mesh invariants for the TSDF mesher tests (test infrastructure).

sphere_scene: a sphere seen by cameras spread over a larger sphere around it, with exact depth maps (ray-sphere hits at
the pixel centres, 0 where a ray misses) and a colour that is a function of the world point; the seed points lie on the
sphere.  plane_scene: the tilted plane of tests/scene_cases seen by its row of cameras."""
from __future__ import annotations

import math

import numpy as np

from tests import scene_cases
from tests.geo_cases import plane_depth

SPHERE_CENTRE = np.array([0.013, -0.021, 0.007])
SPHERE_RADIUS = 1.0


def look_at(centre: np.ndarray, target: np.ndarray) -> np.ndarray:
    """float32 [4,4] world -> camera with z towards target (y down)."""
    z = target - centre
    z = z / np.linalg.norm(z)
    up = np.array([0.0, 0.0, 1.0]) if abs(z[2]) < 0.9 else np.array([0.0, 1.0, 0.0])
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    E = np.eye(4)
    E[:3, :3] = np.stack([x, y, z])
    E[:3, 3] = -E[:3, :3] @ centre
    return E.astype(np.float32)


def fibonacci(n: int) -> np.ndarray:
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    theta = math.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(theta) * np.sin(phi), np.sin(theta) * np.sin(phi), np.cos(phi)], -1)


def colour_of(world: np.ndarray) -> np.ndarray:
    """float32 [...,3] in [0,1]: a smooth function of the world point."""
    return (0.5 + 0.4 * np.stack([np.sin(3 * world[..., 0]), np.cos(2 * world[..., 1]), np.sin(world[..., 2] + 1)], -1)).astype(np.float32)


def sphere_depth(K: np.ndarray, E: np.ndarray, H: int, W: int, centre=SPHERE_CENTRE, radius=SPHERE_RADIUS):
    """(depth float32 [H,W], 0 off the sphere; image float32 [3,H,W])."""
    K64, E64 = K.astype(np.float64), E.astype(np.float64)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    ray = np.linalg.inv(K64) @ np.stack([u.ravel(), v.ravel(), np.ones(H * W)])  # camera frame, z = 1
    c = E64[:3, :3] @ centre + E64[:3, 3]  # sphere centre in the camera frame
    a = (ray * ray).sum(0)
    b = -2 * (ray * c[:, None]).sum(0)
    cc = c @ c - radius * radius
    disc = b * b - 4 * a * cc
    hit = disc >= 0
    t = np.where(hit, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
    depth = np.where(hit & (t > 0), t, 0.0)
    cam = ray * depth
    world = (np.linalg.inv(E64) @ np.vstack([cam, np.ones(H * W)]))[:3].T
    img = np.where(depth[:, None] > 0, colour_of(world), 0.0).T.reshape(3, H, W)
    return depth.reshape(H, W).astype(np.float32), img.astype(np.float32)


def sphere_scene(n_views: int = 14, H: int = 120, W: int = 160, distance: float = 3.2, f: float = 170.0, sizes=None, n_seeds: int = 4000):
    """-> dict(depths, images, Ks, Es, seeds float32 [n,3]).  `sizes` gives each view its own (H, W)."""
    dirs = fibonacci(n_views)
    depths, images, Ks, Es = [], [], [], []
    for v in range(n_views):
        h, w = sizes[v % len(sizes)] if sizes else (H, W)
        K = np.array([[f, 0, w / 2 - 0.3], [0, f, h / 2 + 0.2], [0, 0, 1]], dtype=np.float32)
        E = look_at(SPHERE_CENTRE + distance * dirs[v], SPHERE_CENTRE)
        d, img = sphere_depth(K, E, h, w)
        depths.append(d); images.append(img); Ks.append(K); Es.append(E)
    seeds = (SPHERE_CENTRE + SPHERE_RADIUS * fibonacci(n_seeds)).astype(np.float32)
    return {"depths": depths, "images": images, "Ks": Ks, "Es": Es, "seeds": seeds}


def plane_scene(n_views: int = 6, H: int = 96, W: int = 128):
    """The tilted plane of tests/scene_cases: exact depth maps, the scene's texture, seeds on the plane."""
    depths, images, Ks, Es, seeds = [], [], [], [], []
    for K, E in scene_cases.cameras(n_views, H, W):
        d = plane_depth(K, E, H, W, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float32)
        depths.append(d)
        images.append((scene_cases.texture(K, E, H, W).transpose(2, 0, 1) / 255.0).astype(np.float32))
        Ks.append(K); Es.append(E)
        u, v = np.meshgrid(np.arange(0, W, 4.0), np.arange(0, H, 4.0))
        cam = np.linalg.inv(K.astype(np.float64)) @ np.stack([u.ravel(), v.ravel(), np.ones(u.size)]) * d[v.astype(int), u.astype(int)].ravel()
        seeds.append((np.linalg.inv(E.astype(np.float64)) @ np.vstack([cam, np.ones(u.size)]))[:3].T)
    return {"depths": depths, "images": images, "Ks": Ks, "Es": Es, "seeds": np.concatenate(seeds).astype(np.float32)}


def plane_distance(p: np.ndarray) -> np.ndarray:
    """Distance of world points to the plane of tests/scene_cases (n . x = d0 in the first camera's frame = world)."""
    return np.abs(p.astype(np.float64) @ scene_cases.PLANE_N - scene_cases.PLANE_D0)


def check_closed_manifold(faces: np.ndarray, n_vertices: int) -> None:
    """Every directed edge appears once and its reverse once (a closed, consistently oriented 2-manifold), every vertex is
    referenced, and V - E + F = 2."""
    f = np.asarray(faces, np.int64)
    assert len(f) and (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    keys = directed[:, 0] * n_vertices + directed[:, 1]
    assert len(np.unique(keys)) == len(keys), "a directed edge is used twice"
    rev = directed[:, 1] * n_vertices + directed[:, 0]
    assert np.isin(rev, keys).all(), "an edge is not shared by two oppositely wound faces"
    assert len(np.unique(f)) == n_vertices, "unreferenced vertices"
    n_edges = len(keys) // 2
    assert n_vertices - n_edges + len(f) == 2, (n_vertices, n_edges, len(f))


def face_normals(pos: np.ndarray, faces: np.ndarray) -> np.ndarray:
    p = pos.astype(np.float64)
    f = np.asarray(faces, np.int64)
    return np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
