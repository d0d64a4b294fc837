"""Synthetic scene folders in the reference's eval.py layout (pair.txt, images/%08d.jpg, cams/%08d_cam.txt), generated from a
seed (test and benchmark infrastructure).

The scene is the tilted plane of tests/geo_cases seen by a row of cameras.  Images are the plane's texture (a function of the
world point) rendered into every view, so the views are photo-consistent and the network has something to match.  Depth and
confidence maps for a fusion-only run are analytic renders of the plane, corrupted in blocks as geo_cases.make_scene does."""
from __future__ import annotations

import math
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np

from tests.geo_cases import _rot_x, _rot_y, plane_depth

PLANE_N = np.array([0.12, -0.08, 1.0]) / np.linalg.norm([0.12, -0.08, 1.0])
PLANE_D0 = 600.0
DEPTH_RANGE = (425.0, 935.0)


def cameras(n_views: int, H: int, W: int) -> List[Tuple[np.ndarray, np.ndarray]]:
    """(K float32 [3,3], E float32 [4,4] world -> camera) per view: small rotations and a baseline that grows with the index."""
    cams = []
    for i in range(n_views):
        K = np.array([[1.2 * W, 0, W / 2 + 1.5 * i], [0, 1.2 * W, H / 2], [0, 0, 1]], dtype=np.float32)
        E = np.eye(4, dtype=np.float64)
        if i:
            sgn = 1.0 if i % 2 else -1.0
            j = (i + 1) // 2
            E[:3, :3] = _rot_y(math.radians(1.0 * j) * sgn) @ _rot_x(math.radians(0.4 * j))
            E[:3, 3] = [12.0 * sgn * j, -5.0 * (i % 3), 2.0 * j]
        cams.append((K, E.astype(np.float32)))
    return cams


def texture(K: np.ndarray, E: np.ndarray, H: int, W: int) -> np.ndarray:
    """uint8 [H,W,3]: the plane's colour (smooth stripes plus a fine pattern, all a function of the world point) in this view."""
    d = plane_depth(K, E, H, W, PLANE_N, PLANE_D0).astype(np.float64)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    cam = np.linalg.inv(K.astype(np.float64)) @ np.stack((u.ravel(), v.ravel(), np.ones(H * W))) * d.ravel()
    world = (np.linalg.inv(E.astype(np.float64)) @ np.vstack((cam, np.ones(H * W))))[:3]
    x, y = world[0].reshape(H, W), world[1].reshape(H, W)
    chans = [np.sin(x / (2.1 + c)) * np.cos(y / (2.7 + 0.5 * c)) + 0.5 * np.sin((x + 2 * y) / 0.9 + c) for c in range(3)]
    return np.clip(127.5 + 80.0 * np.stack(chans, axis=-1), 0, 255).astype(np.uint8)


def cam_text(K: np.ndarray, E: np.ndarray, depth_range=DEPTH_RANGE) -> str:
    rows = ["extrinsic"] + [" ".join("%.9g" % v for v in r) for r in E] + ["", "intrinsic"]
    rows += [" ".join("%.9g" % v for v in r) for r in K] + [""]
    if depth_range is not None:
        rows.append("%.9g %.9g" % depth_range)
    return "\n".join(rows) + "\n"


def all_pairs(n_views: int, n_src: int) -> List[Tuple[int, List[int]]]:
    """Every view a reference; its sources the n_src nearest other views by index distance (ties: lower index first)."""
    out = []
    for r in range(n_views):
        others = sorted((v for v in range(n_views) if v != r), key=lambda v: (abs(v - r), v))
        out.append((r, others[:n_src]))
    return out


def pair_text(pairs: Sequence[Tuple[int, List[int]]]) -> str:
    lines = [str(len(pairs))]
    for r, src in pairs:
        lines += [str(r), " ".join([str(len(src))] + ["%d %.1f" % (s, 100.0 - k) for k, s in enumerate(src)])]
    return "\n".join(lines) + "\n"


def write_scene(root: str, n_views: int, H: int, W: int, n_src: int, quality: int = 95) -> Dict[str, object]:
    """pair.txt, cams and textured JPEG images of the plane scene under `root`.  -> {"cams", "pairs"}."""
    from PIL import Image

    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    os.makedirs(os.path.join(root, "cams"), exist_ok=True)
    cams = cameras(n_views, H, W)
    pairs = all_pairs(n_views, n_src)
    with open(os.path.join(root, "pair.txt"), "w") as f:
        f.write(pair_text(pairs))
    for v, (K, E) in enumerate(cams):
        with open(os.path.join(root, "cams", "%08d_cam.txt" % v), "w") as f:
            f.write(cam_text(K, E))
        Image.fromarray(texture(K, E, H, W)).save(os.path.join(root, "images", "%08d.jpg" % v), quality=quality)
    return {"cams": cams, "pairs": pairs}


def write_fusion_maps(out_dir: str, cams, H: int, W: int, seed: int, fmt: str = ".pfm") -> None:
    """depth_est / confidence maps of every view: the plane's analytic depth, corrupted in blocks (relative errors of 0.5-5 %)
    with a little noise, and a seeded confidence in [0.4, 1)."""
    from patchmatchnet_b200 import data_io

    rng = np.random.default_rng(seed)
    os.makedirs(os.path.join(out_dir, "depth_est"), exist_ok=True)
    os.makedirs(os.path.join(out_dir, "confidence"), exist_ok=True)
    for v, (K, E) in enumerate(cams):
        d = plane_depth(K, E, H, W, PLANE_N, PLANE_D0)
        for _ in range(3):
            y0, x0 = int(rng.integers(0, H - 16)), int(rng.integers(0, W - 24))
            d[y0:y0 + 16, x0:x0 + 24] *= np.float32(1.0 + rng.choice([-1, 1]) * rng.uniform(0.005, 0.05))
        d += rng.normal(0, 0.05, size=(H, W)).astype(np.float32)
        conf = rng.uniform(0.4, 1.0, size=(H, W)).astype(np.float32)
        data_io.save_map(os.path.join(out_dir, "depth_est", "%08d%s" % (v, fmt)), d.astype(np.float32))
        data_io.save_map(os.path.join(out_dir, "confidence", "%08d%s" % (v, fmt)), conf)
