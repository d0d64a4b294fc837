"""Seeded synthetic ETH3D training scenes, written in ETH3D's layout: a box room with a square pillar, ray-cast by laser scanners
on an angular grid, each scan stored in its own rotated and translated frame, and a reconstruction with designed classes.

    <root>/gt/<scene>/dslr_scan_eval/scan_alignment.mlp    the scans' files and matrices (local -> scene)
    <root>/gt/<scene>/dslr_scan_eval/scan<k>.ply             binary PLYs (double x y z among other properties), the last ASCII
    <root>/outputs/<scene>/fused.ply                         the reconstruction (float32 x y z, uchar colours)

Reconstruction parts (make_scene's "labels"): 0 surface samples (ground-truth points plus Gaussian noise), 1 free-space
outliers (on the segment from a scanner to one of its points, more than 0.6 m from every surface: inaccurate at every
tolerance up to 0.5), 2 points behind the walls, 3 points inside the pillar's core, 4 points far outside the room (2-4: in
no beam, unobserved)."""
from __future__ import annotations

import math
import os

import numpy as np
import torch

from patchmatchnet_b200 import data_io

ROOM = np.array([[0.0, 0.0, 0.0], [8.0, 6.0, 3.0]])
PILLAR = np.array([[3.6, 2.4, 0.0], [5.2, 4.0, 3.0]])  # full height, 1.6 m square
SCANNERS = np.array([[1.6, 1.5, 1.5], [6.5, 1.4, 1.5], [1.7, 4.6, 1.4]])
MARGIN = 0.6  # designed points keep this far from every surface


def rotation(axis, angle) -> np.ndarray:
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    k = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + math.sin(angle) * k + (1 - math.cos(angle)) * (k @ k)


def ray_cast(origin, dirs) -> np.ndarray:
    """First hit of each ray from `origin` (inside the room, outside the pillar): the room's walls from inside, the pillar from
    outside.  -> distances [k]."""
    o = np.asarray(origin, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / dirs
        t_room = np.min(np.maximum((ROOM[0] - o) * inv, (ROOM[1] - o) * inv), axis=1)
        t0, t1 = (PILLAR[0] - o) * inv, (PILLAR[1] - o) * inv
        near = np.max(np.minimum(t0, t1), axis=1)
        far = np.min(np.maximum(t0, t1), axis=1)
    hit = (near <= far) & (near > 0)
    return np.where(hit, np.minimum(near, t_room), t_room)


def scan_directions(n_az: int, n_el: int, rng) -> np.ndarray:
    az = (np.arange(n_az) + rng.uniform(0, 1)) * (2 * math.pi / n_az) - math.pi
    el = np.linspace(-1.35, 1.45, n_el)
    a, e = np.meshgrid(az, el, indexing="ij")
    return np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)


def _away_from_surfaces(p) -> np.ndarray:
    """Distance from points to the nearest wall, floor, ceiling or pillar face (0 inside the pillar)."""
    walls = np.min(np.concatenate([p - ROOM[0], ROOM[1] - p], 1), 1)
    d = np.maximum(np.maximum(PILLAR[0] - p, p - PILLAR[1]), 0.0)
    pillar = np.sqrt((d * d).sum(1))
    inside = (p > PILLAR[0]).all(1) & (p < PILLAR[1]).all(1)
    return np.where(inside, 0.0, np.minimum(walls, pillar))


def make_scene(seed: int, n_az: int = 240, n_el: int = 100, n_surface: int = 6000, noise: float = 0.002, n_outliers: int = 200,
               n_hidden: int = 100, n_scanners: int = 3):
    """-> {"scans": [{"matrix", "points" (local), "scene" (ray-cast, scene frame), "origin"}], "rec" [n,3], "labels" [n]}."""
    rng = np.random.RandomState(seed)
    scans = []
    for k in range(n_scanners):
        o = SCANNERS[k]
        dirs = scan_directions(n_az, n_el, rng)
        pts = o + ray_cast(o, dirs)[:, None] * dirs
        r = rotation(rng.normal(size=3), rng.uniform(0, 2 * math.pi))
        m = np.eye(4)
        m[:3, :3], m[:3, 3] = r, o
        local = (pts - o) @ r  # R^T (p - o), row-wise
        scans.append({"matrix": m, "points": local, "scene": pts, "origin": o.copy()})
    gt = np.concatenate([s["scene"] for s in scans])
    parts, labels = [], []
    surf = gt[rng.choice(gt.shape[0], n_surface, replace=False)] + (rng.normal(0, noise, (n_surface, 3)) if noise else 0.0)
    parts.append(surf)
    labels.append(np.zeros(n_surface, np.int64))
    out = []
    while sum(len(x) for x in out) < n_outliers:
        s = scans[rng.randint(len(scans))]
        p = s["scene"][rng.randint(s["scene"].shape[0], size=4 * n_outliers)]
        lam = rng.uniform(0.05, 0.95, (p.shape[0], 1))
        q = s["origin"] + lam * (p - s["origin"])
        out.append(q[_away_from_surfaces(q) > MARGIN + 0.05])
    parts.append(np.concatenate(out)[:n_outliers] if out else np.zeros((0, 3)))
    labels.append(np.ones(n_outliers, np.int64))
    # behind the walls: outside the room's box by MARGIN .. 2 m along one axis
    axis = rng.randint(0, 3, n_hidden)
    side = rng.randint(0, 2, n_hidden)
    behind = rng.uniform(ROOM[0], ROOM[1], (n_hidden, 3))
    depth = rng.uniform(MARGIN, 2.0, n_hidden)
    behind[np.arange(n_hidden), axis] = np.where(side == 1, ROOM[1][axis] + depth, ROOM[0][axis] - depth)
    parts.append(behind)
    labels.append(np.full(n_hidden, 2))
    core = rng.uniform(PILLAR[0] + [MARGIN, MARGIN, 0.5], PILLAR[1] - [MARGIN, MARGIN, 0.5], (n_hidden, 3))
    parts.append(core)
    labels.append(np.full(n_hidden, 3))
    far = rng.uniform(-1, 1, (n_hidden, 3)) * 5 + [40.0, -30.0, 10.0]
    parts.append(far)
    labels.append(np.full(n_hidden, 4))
    rec = np.concatenate(parts)
    return {"scans": scans, "rec": rec.astype(np.float32).astype(np.float64), "labels": np.concatenate(labels)}


def mlp_text(names, matrices, sep: str = " ") -> str:
    rows = []
    for name, m in zip(names, matrices):
        mat = "\n".join(sep.join(f"{v:.17g}" for v in row) + sep for row in m)
        rows.append(f'  <MLMesh label="{name}" filename="{name}">\n   <MLMatrix44>\n{mat}\n</MLMatrix44>\n  </MLMesh>\n')
    return ("<!DOCTYPE MeshLabDocument>\n<MeshLabProject>\n <MeshGroup>\n" + "".join(rows) + " </MeshGroup>\n <RasterGroup/>\n"
            "</MeshLabProject>\n")


def write_scan_binary(path: str, pts, rng) -> None:
    """Binary little-endian PLY with extra properties around double x, y, z."""
    n = pts.shape[0]
    rows = np.empty(n, dtype=[("intensity", "<f4"), ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"),
                              ("blue", "u1"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")])
    rows["intensity"] = rng.uniform(0, 1, n)
    rows["x"], rows["y"], rows["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    for c in ("red", "green", "blue"):
        rows[c] = rng.randint(0, 256, n)
    for c in ("nx", "ny", "nz"):
        rows[c] = 0.0
    header = (f"ply\nformat binary_little_endian 1.0\ncomment synthetic laser scan\nelement vertex {n}\nproperty float intensity\n"
              "property double x\nproperty double y\nproperty double z\nproperty uchar red\nproperty uchar green\n"
              "property uchar blue\nproperty float nx\nproperty float ny\nproperty float nz\nend_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rows.tobytes())


def write_scan_ascii(path: str, pts) -> None:
    n = pts.shape[0]
    with open(path, "w") as f:
        f.write(f"ply\nformat ascii 1.0\nelement vertex {n}\nproperty double x\nproperty double y\nproperty double z\n"
                "property uchar intensity\nend_header\n")
        for p in pts:
            f.write(f"{p[0]:.17g} {p[1]:.17g} {p[2]:.17g} 7\n")


def save_reconstruction(path: str, pts) -> None:
    xyz = np.asarray(pts, np.float32).reshape(-1, 3)
    body = np.concatenate([xyz.view(np.uint8).reshape(-1, 12), np.full((len(xyz), 3), 128, np.uint8)], axis=1)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    data_io.save_ply(path, torch.from_numpy(np.ascontiguousarray(body)))


def write_tree(root: str, scenes, **kw):
    """root/gt/<scene>/dslr_scan_eval/ and root/outputs/<scene>/fused.ply for each scene.  -> {scene: make_scene(...)}."""
    out = {}
    for k, scene in enumerate(scenes):
        c = make_scene(200 + k, **kw)
        d = os.path.join(root, "gt", scene, "dslr_scan_eval")
        os.makedirs(os.path.join(d, "scans"), exist_ok=True)
        rng = np.random.RandomState(300 + k)
        names = []
        for i, s in enumerate(c["scans"]):
            name = f"scans/scan{i}.ply"
            if i == len(c["scans"]) - 1:
                write_scan_ascii(os.path.join(d, name), s["points"])
            else:
                write_scan_binary(os.path.join(d, name), s["points"], rng)
            names.append(name)
        with open(os.path.join(d, "scan_alignment.mlp"), "w") as f:
            f.write(mlp_text(names, [s["matrix"] for s in c["scans"]]))
        save_reconstruction(os.path.join(root, "outputs", scene, "fused.ply"), c["rec"])
        out[scene] = c
    return out
