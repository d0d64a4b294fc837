"""Synthetic multi-view scenes for the geometric-consistency tests (test infrastructure): a tilted plane seen by a
reference camera and a few source cameras, per-view depth maps rendered analytically, then corrupted in places so that
every branch of the filter (out-of-image taps, pixel-distance failures, depth failures, low confidence) is exercised."""
from __future__ import annotations

import math

import numpy as np


def _rot_y(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)


def _rot_x(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=np.float64)


def plane_depth(K, E, H, W, n, d0):
    """z-depth of the plane n.X = d0 (world) along every pixel ray of camera (K, E: world -> camera)."""
    R, t = E[:3, :3].astype(np.float64), E[:3, 3].astype(np.float64)
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    rays = np.linalg.inv(K.astype(np.float64)) @ np.stack((u.ravel(), v.ravel(), np.ones(H * W)))
    num = d0 + n @ (R.T @ t)
    den = n @ (R.T @ rays)
    return (num / den).reshape(H, W).astype(np.float32)


def source_pose(i):
    """[R | t] (3x4) of source camera i >= 1.  Sources past the fourth repeat the first four baselines (their principal
    points and corruptions still differ), so that every source of a scene with many sources overlaps the reference."""
    k = (i - 1) % 4 + 1
    sgn = 1.0 if k % 2 else -1.0
    return np.concatenate([_rot_y(math.radians(2.0 * k) * sgn) @ _rot_x(math.radians(0.7 * k)),
                           np.array([[40.0 * sgn * k], [-15.0 * (k % 3)], [5.0 * k]])], axis=1)


def make_scene(H=96, W=128, n_src=4, seed=0):
    rng = np.random.default_rng(seed)
    K = np.array([[1.2 * W, 0, W / 2], [0, 1.2 * W, H / 2], [0, 0, 1]], dtype=np.float32)
    n = np.array([0.12, -0.08, 1.0])
    n = n / np.linalg.norm(n)
    d0 = 600.0
    cams = []
    for i in range(n_src + 1):
        E = np.eye(4, dtype=np.float64)
        if i:
            E[:3, :] = source_pose(i)
        Ki = K.copy()
        Ki[0, 2] += 1.5 * i
        cams.append((Ki, E.astype(np.float32)))
    depths = [plane_depth(k, e, H, W, n, d0) for k, e in cams]
    # corrupt: block-wise relative errors in the source maps, a wrong-depth band in the reference map
    for i in range(1, n_src + 1):
        for _ in range(3):
            y0, x0 = int(rng.integers(0, H - 16)), int(rng.integers(0, W - 24))
            depths[i][y0:y0 + 16, x0:x0 + 24] *= np.float32(1.0 + rng.choice([-1, 1]) * rng.uniform(0.005, 0.05))
        depths[i] += rng.normal(0, 0.05, size=(H, W)).astype(np.float32)
    depths[0][H // 3: H // 3 + 6, :] *= np.float32(1.03)
    conf = rng.uniform(0.5, 1.0, size=(H, W)).astype(np.float32)
    return dict(ref_depth=depths[0], ref_K=cams[0][0], ref_E=cams[0][1], src_depths=depths[1:],
                src_Ks=[c[0] for c in cams[1:]], src_Es=[c[1] for c in cams[1:]], confidence=conf)
