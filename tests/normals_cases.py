"""Depth maps with known normals for the normal estimation tests (test and benchmark infrastructure), and the comparison
of an estimate against oracle/normals_oracle.py.

Planes are camera-frame planes n . X = c (c < 0: the plane faces the camera) rendered by ray / plane intersection with the
oracle's own rays, so a float64 map back-projects onto the plane to rounding."""
from __future__ import annotations

from typing import Dict, Tuple

import numpy as np

from oracle import normals_oracle as no

TILT_N = np.array([0.3, -0.2, -1.0]) / np.linalg.norm([0.3, -0.2, -1.0])
STEP_N = np.array([-0.25, 0.1, -1.0]) / np.linalg.norm([-0.25, 0.1, -1.0])


def intrinsics(H: int, W: int) -> np.ndarray:
    """A focal length of 2000 pixels whatever the size (DTU's is ~1.8 widths at 1600 x 1200): a plane's depth changes by
    well under depth_thres across a window, so every window pixel of a plane is an inlier."""
    return np.array([[2000.0, 0, W / 2 + 0.5], [0, 2000.0, H / 2 - 0.25], [0, 0, 1]], dtype=np.float32)


def plane(K: np.ndarray, H: int, W: int, n: np.ndarray, c: float) -> np.ndarray:
    """float64 [H,W]: the depth D with D * K^-1 (x, y, 1) on the plane n . X = c."""
    return c / (no.rays(K, H, W) @ n)


def fronto(H: int, W: int) -> Dict[str, np.ndarray]:
    K = intrinsics(H, W)
    return {"K": K, "depth": np.full((H, W), 500.0), "want": np.broadcast_to([0.0, 0.0, -1.0], (H, W, 3))}


def tilted(H: int, W: int) -> Dict[str, np.ndarray]:
    K = intrinsics(H, W)
    return {"K": K, "depth": plane(K, H, W, TILT_N, -600.0), "want": np.broadcast_to(TILT_N, (H, W, 3))}


def step(H: int, W: int) -> Dict[str, np.ndarray]:
    """Two planes meeting at column W // 2, the right one ~25 % deeper: each side keeps its own normal up to the edge."""
    K = intrinsics(H, W)
    left = np.arange(W)[None, :] < W // 2
    depth = np.where(left, plane(K, H, W, TILT_N, -600.0), plane(K, H, W, STEP_N, -750.0))
    want = np.where(left[..., None], TILT_N, STEP_N) * np.ones((H, W, 1))
    return {"K": K, "depth": depth, "want": want}


def holes(H: int, W: int, seed: int = 0) -> Tuple[Dict[str, np.ndarray], np.ndarray]:
    """The tilted plane with zero, negative, NaN and infinite depths at seeded pixels -> (case, the invalid pixels)."""
    case = tilted(H, W)
    rng = np.random.default_rng(seed)
    bad = rng.random((H, W)) < 0.08
    depth = case["depth"].copy()
    depth[bad] = rng.choice([0.0, -3.0, np.nan, np.inf], size=int(bad.sum()))
    return dict(case, depth=depth), bad


def noisy(H: int, W: int, seed: int = 1, sigma: float = 0.05) -> Dict[str, np.ndarray]:
    """float32: the step scene plus seeded Gaussian depth noise (mm)."""
    case = step(H, W)
    rng = np.random.default_rng(seed)
    return dict(case, depth=(case["depth"] + rng.normal(0, sigma, (H, W))).astype(np.float32))


def angle(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Angle between unit vectors [..., 3], accurate near 0."""
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=-1), np.einsum("...i,...i->...", a, b))


def check_against_oracle(got: np.ndarray, depth: np.ndarray, K: np.ndarray, *, angle_tol: float = 1e-5, **kw) -> None:
    """An estimate [H,W,3] against the oracle on the same (float32) map: zero / non-zero classification may differ on at most
    1e-4 of the pixels (thresholds met within rounding); where both are non-zero and the oracle's eigen gap is >= 1e-3
    lambda_max the angle is <= angle_tol; every non-zero normal has unit length to 1e-6 and faces the camera.

    A normal seen edge-on (|n . P(p)| < 1e-6 |P(p)|, e.g. when every inlier lies on one image row, whose points share a plane
    through the camera centre) has its orientation decided by rounding: there the angle is taken up to sign, and facing the
    camera means n . P(p) < 1e-6 |P(p)|."""
    want, gap = no.estimate_normals(depth, K, **kw)
    H, W = depth.shape
    zg, zw = (got == 0).all(-1), (want == 0).all(-1)
    assert (zg != zw).sum() <= int(1e-4 * H * W), ((zg != zw).sum(), H, W)
    p = np.asarray(depth, dtype=np.float64)[..., None] * no.rays(K, H, W)
    with np.errstate(invalid="ignore", divide="ignore"):
        ph = p / np.linalg.norm(p, axis=-1, keepdims=True)
    both = ~zg & ~zw & (gap >= 1e-3)
    if both.any():
        err = angle(got[both].astype(np.float64), want[both])
        edge_on = np.abs(np.einsum("ni,ni->n", want[both], ph[both])) < 1e-6
        err = np.where(edge_on, np.minimum(err, np.pi - err), err)
        assert err.max() <= angle_tol, (err.max(), int(edge_on.sum()))
    nz = got[~zg].astype(np.float64)
    assert np.abs(np.linalg.norm(nz, axis=-1) - 1).max(initial=0) <= 1e-6
    facing = np.einsum("ni,ni->n", nz, ph[~zg])
    assert (facing < 1e-6).all(), facing.max()
