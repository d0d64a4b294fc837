"""CPU restatement of the surface normals of pmb200_depth_normals and of the oriented fused.ply records of
pmb200_fuse_points_oriented.  The reference has no normals; the definition is this project's own
(include/patchmatch_b200.h).

TEST INFRASTRUCTURE ONLY: nothing under patchmatchnet_b200/ imports this file.  It states the definition in numpy float64
with batched np.linalg.eigh instead of the kernel's closed-form 3x3 solve:

    P(q)      = D(q) K^-1 (x_q, y_q, 1), float64, K^-1 the float32 inverse of the float32 intrinsics, widened
    valid     D finite and > 0
    inliers   the valid q of the (2r+1)^2 window around p, clipped at the image border, with |D(q) - D(p)| <= t D(p)
    zero      p invalid, fewer than m inliers, or lambda_mid <= 1e-6 lambda_max of the inliers' covariance
    normal    the eigenvector of lambda_min, flipped so that n . P(p) < 0

The covariance is taken about the centroid of the points shifted by P(p).  The depth map may be float64 (analytic tests) or
float32 (what the kernel reads); it is widened, never rounded.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

DEGENERATE = 1e-6
ORIENTED_VERTEX = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                            ("red", "u1"), ("green", "u1"), ("blue", "u1")])


def kinv64(K: np.ndarray) -> np.ndarray:
    """K^-1 as the kernel takes it: numpy's float32 inverse of the float32 intrinsics, widened to float64."""
    return np.linalg.inv(np.asarray(K, dtype=np.float32)).astype(np.float64)


def rays(K: np.ndarray, H: int, W: int) -> np.ndarray:
    """[H,W,3] float64: K^-1 (x, y, 1) at every pixel; P(p) = D(p) * rays[p]."""
    u, v = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    return np.einsum("ij,jhw->hwi", kinv64(K), np.stack([u, v, np.ones_like(u)]))


def estimate_normals(depth: np.ndarray, K: np.ndarray, radius: int = 3, depth_thres: float = 0.01,
                     min_inliers: int = 6) -> Tuple[np.ndarray, np.ndarray]:
    """depth [H,W], K [3,3] -> (normals float64 [H,W,3], gap float64 [H,W]).  gap is (lambda_mid - lambda_min) / lambda_max
    where a normal was estimated and 0 elsewhere: the conditioning of the eigenvector, for tolerances."""
    d = np.asarray(depth, dtype=np.float64)
    H, W = d.shape
    r = int(radius)
    kinv = kinv64(K)
    valid = np.isfinite(d) & (d > 0)
    dpad = np.full((H + 2 * r, W + 2 * r), np.nan)
    dpad[r:r + H, r:r + W] = np.where(valid, d, np.nan)  # outside the image and invalid pixels: never inliers
    u, v = np.meshgrid(np.arange(-r, W + r, dtype=np.float64), np.arange(-r, H + r, dtype=np.float64))
    rays = np.einsum("ij,jhw->hwi", kinv, np.stack([u, v, np.ones_like(u)]))
    ppad = dpad[..., None] * rays  # [H+2r, W+2r, 3]
    dp, pp = dpad[r:r + H, r:r + W], ppad[r:r + H, r:r + W]
    tol = depth_thres * dp
    offsets = [(dy, dx) for dy in range(-r, r + 1) for dx in range(-r, r + 1)]

    def window(dy, dx):
        dq = dpad[r + dy:r + dy + H, r + dx:r + dx + W]
        with np.errstate(invalid="ignore"):
            inl = np.abs(dq - dp) <= tol  # NaN (invalid or outside) compares false
        return inl, ppad[r + dy:r + dy + H, r + dx:r + dx + W] - pp

    n = np.zeros((H, W), dtype=np.int64)
    s = np.zeros((H, W, 3))
    for dy, dx in offsets:
        inl, e = window(dy, dx)
        n += inl
        s += np.where(inl[..., None], e, 0.0)
    c = s / np.maximum(n, 1)[..., None]
    cov = np.zeros((H, W, 3, 3))
    for dy, dx in offsets:
        inl, e = window(dy, dx)
        e = np.where(inl[..., None], e - c, 0.0)
        cov += e[..., :, None] * e[..., None, :]
    normals = np.zeros((H, W, 3))
    gap = np.zeros((H, W))
    cand = valid & (n >= min_inliers)
    if cand.any():
        lam, vec = np.linalg.eigh(cov[cand] / n[cand][:, None, None])
        ok = lam[:, 1] > DEGENERATE * lam[:, 2]
        nv = vec[:, :, 0]
        flip = np.einsum("ni,ni->n", nv, pp[cand]) > 0
        nv = np.where(flip[:, None], -nv, nv)
        normals[cand] = np.where(ok[:, None], nv, 0.0)
        gap[cand] = np.where(ok, (lam[:, 1] - lam[:, 0]) / lam[:, 2], 0.0)
    return normals, gap


def world_normals(normals_cam: np.ndarray, E: np.ndarray) -> np.ndarray:
    """Camera-frame normals [..., 3] -> world frame, float32: the rotation block of the float32 inverse of the extrinsics
    (compose_fusion_camera's), in float64; zero normals stay zero."""
    rot = np.linalg.inv(np.asarray(E, dtype=np.float32)).astype(np.float64)[:3, :3]
    n = np.asarray(normals_cam, dtype=np.float64)
    out = np.einsum("ij,...j->...i", rot, n)
    return np.where((n == 0).all(axis=-1, keepdims=True), 0.0, out).astype(np.float32)


def oriented_records(positions: np.ndarray, normals: np.ndarray, colours: np.ndarray) -> np.ndarray:
    """uint8 [n,27]: float32 x, y, z, nx, ny, nz, uint8 red, green, blue little endian, the vertex of COLMAP's fused.ply."""
    rec = np.empty(len(positions), dtype=ORIENTED_VERTEX)
    for i, k in enumerate(("x", "y", "z")):
        rec[k] = positions[:, i]
    for i, k in enumerate(("nx", "ny", "nz")):
        rec[k] = normals[:, i]
    for i, k in enumerate(("red", "green", "blue")):
        rec[k] = colours[:, i]
    return rec.view(np.uint8).reshape(-1, 27)


def split_oriented(records: np.ndarray) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """uint8 [n,27] -> (positions float32 [n,3], normals float32 [n,3], colours uint8 [n,3])."""
    rec = np.ascontiguousarray(records).view(ORIENTED_VERTEX).reshape(-1)
    return (np.stack([rec[k] for k in ("x", "y", "z")], 1), np.stack([rec[k] for k in ("nx", "ny", "nz")], 1),
            np.stack([rec[k] for k in ("red", "green", "blue")], 1))
