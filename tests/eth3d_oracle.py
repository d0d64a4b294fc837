"""The ETH3D evaluation protocol (INTEGRATION.md "ETH3D evaluation (beyond the reference)") restated with numpy and scipy, as
the CPU reference the GPU path is checked against.  Test infrastructure only.

Every float64 operation is the protocol's, in its order (numpy's elementwise operations round each product and sum on their
own): scan transforms ((m00 x + m01 y) + m02 z) + m03, dot products ((x0 y0 + x1 y1) + x2 y2), the beam predicate evaluated by
brute force over every (query, scan point) pair, nearest distances from cKDTree's neighbour re-measured with
((dx^2 + dy^2) + dz^2), and the voxels from np.unique."""
from __future__ import annotations

import math

import numpy as np
from scipy.spatial import cKDTree

TOLERANCES = (0.01, 0.02, 0.05, 0.1, 0.2, 0.5)


def transform(points, m) -> np.ndarray:
    p = np.asarray(points, np.float64).reshape(-1, 3)
    m = np.asarray(m, np.float64)
    out = np.empty_like(p)
    for r in range(3):
        out[:, r] = ((m[r, 0] * p[:, 0] + m[r, 1] * p[:, 1]) + m[r, 2] * p[:, 2]) + m[r, 3]
    return out


def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def in_free_beam(a, b, r0: float, t: float) -> np.ndarray:
    """The predicate for broadcast a = p - o and b = q - o: 0 < t' < a.a and |a x b|^2 <= (r0 r + t' T)^2."""
    tp = _dot(a, b)
    aa = _dot(a, a)
    r = np.sqrt(aa)
    c0 = a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1]
    c1 = a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2]
    c2 = a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]
    cc = (c0 * c0 + c1 * c1) + c2 * c2
    w = r0 * r + tp * t
    with np.errstate(invalid="ignore", over="ignore"):
        return (0.0 < tp) & (tp < aa) & (cc <= w * w)


def beam_observed(queries, scan_points, origin, r0: float, t: float, chunk: int = 1 << 22) -> np.ndarray:
    """observed[i]: query i lies in the free beam of some scan point (scene-frame points, scan origin).  Brute force."""
    q = np.asarray(queries, np.float64).reshape(-1, 3)
    o = np.asarray(origin, np.float64).reshape(3)
    a = np.asarray(scan_points, np.float64).reshape(-1, 3) - o
    b = q - o
    out = np.zeros(q.shape[0], dtype=bool)
    if a.shape[0] == 0:
        return out
    step = max(1, chunk // a.shape[0])
    for s in range(0, q.shape[0], step):
        out[s:s + step] = in_free_beam(a[None, :, :], b[s:s + step, None, :], r0, t).any(1)
    return out


def nearest_distance(to_points, from_points) -> np.ndarray:
    """Exact distance from each `from` point to the nearest `to` point (inf when `to` is empty)."""
    frm = np.asarray(from_points, np.float64).reshape(-1, 3)
    to = np.asarray(to_points, np.float64).reshape(-1, 3)
    if to.shape[0] == 0:
        return np.full(frm.shape[0], np.inf)
    if frm.shape[0] == 0:
        return np.zeros(0)
    _, j = cKDTree(to).query(frm)
    d = frm - to[j]
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def voxel_score(points, dist, tau: float, observed=None):
    """(good, bad, excluded, voxels, sum over voxels of good / (good + bad)); voxel floor(x / tau), anchored at the origin."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    d = np.asarray(dist, np.float64)
    good = d <= tau
    bad = ~good if observed is None else (~good & np.asarray(observed, bool))
    counted = good | bad
    if not counted.any():
        return int(good.sum()), int(bad.sum()), int((~counted).sum()), 0, 0.0
    keys = np.floor(p[counted] / tau).astype(np.int64)
    _, inv = np.unique(keys, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    g = np.bincount(inv, weights=good[counted].astype(np.float64))
    tot = np.bincount(inv).astype(np.float64)
    return int(good.sum()), int(bad.sum()), int((~counted).sum()), int(tot.size), float(np.sum(g / tot))


def evaluate(rec, scans, tolerances=TOLERANCES, r0: float = 0.001125, halfangle_deg: float = 0.011):
    """scans: [{"matrix" [4,4], "points" local [m,3]}] -> (per-tau dicts, d_acc, d_comp, observed)."""
    rec = np.asarray(rec, np.float64).reshape(-1, 3)
    moved = [transform(s["points"], s["matrix"]) for s in scans]
    gt = np.concatenate(moved) if moved else np.zeros((0, 3))
    d_acc = nearest_distance(gt, rec)
    d_comp = nearest_distance(rec, gt)
    t = math.tan(math.radians(halfangle_deg))
    need = d_acc > min(tolerances)
    observed = np.zeros(rec.shape[0], dtype=bool)
    for s, g in zip(scans, moved):
        todo = need & ~observed
        observed[todo] |= beam_observed(rec[todo], g, np.asarray(s["matrix"], np.float64)[:3, 3], r0, t)
    out = []
    for tau in tolerances:
        a = voxel_score(rec, d_acc, tau, observed)
        c = voxel_score(gt, d_comp, tau)
        acc = a[4] / a[3] if a[3] else 0.0
        comp = c[4] / c[3] if c[3] else 0.0
        out.append({"tolerance": tau, "accuracy": acc, "completeness": comp,
                    "f1": 2 * acc * comp / (acc + comp) if acc + comp > 0 else 0.0,
                    "accurate": a[0], "inaccurate": a[1], "unobserved": a[2], "covered": c[0], "gt_points": gt.shape[0],
                    "accuracy_voxels": a[3], "completeness_voxels": c[3]})
    return out, d_acc, d_comp, observed
