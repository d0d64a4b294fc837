"""DTU evaluation inputs at the sizes and densities of real scans, generated from seeds (no DTU data is needed or stored).

A fused DTU cloud comes from 49 views of 1600x1200: tens of millions of points, every surface patch seen by many views, so
a point has tens to hundreds of neighbours within the thinning distance of 0.2 mm.  The rows model that with sheets: each
view's points lie on its own copy of the surface (dtu_cases.height), offset along z by a per-sheet bias, plus noise.  All
coordinates are float32-representable, because PLY files store float32.

    sheets    20M data points (above 2^24) on a 250 x 250 mm patch, about 320 per mm^2, 1% outliers over the widened box;
              3M STL samples of the exact surface; bb, obs_mask, res, plane as dtu_cases.make_scan builds them
    literal   300k points at the density of `sheets`: small enough for the sequential oracle, dtu_oracle.thin
    stack     200k points at 10 000 per mm^2 (hundreds of neighbours), 10% of them exact duplicates of others
    lattice   100^3 points exactly 0.25 apart around 1000 with dst = 0.25: every neighbour is at exactly dst
    chain     3000 points 0.9 dst apart on a line, visited along it (or against it): each decision waits for the one
              before, so a synchronous thinning needs about one round per point, beyond the native bound of 256
"""
from __future__ import annotations

import numpy as np

from oracle import dtu_oracle as do
from patchmatchnet_b200 import dtu_eval
from tests import dtu_cases

DST = 0.2
THIN_ROUND_BOUND = 256   # rounds of the native thinning (csrc/pm_cloud.cu, kThinMaxRounds)
SHEETS = 49              # views of a DTU scan
SHEET_SIGMA = 0.1        # mm: spread of the per-sheet z bias
NOISE = 0.03             # mm: per-point noise on every axis
SIDE = 250.0             # mm: the sheets row's patch
N_DATA = 20_000_000
N_STL = 3_000_000
DENSITY = N_DATA / SIDE ** 2  # points per mm^2 of the sheets row


def _f32(p: np.ndarray) -> np.ndarray:
    return p.astype(np.float32).astype(np.float64)


def layered(rng: np.random.RandomState, n: int, side: float) -> np.ndarray:
    """n points on SHEETS offset copies of the surface over a side x side patch centred at the origin, z around 600."""
    x = rng.uniform(-side / 2, side / 2, n)
    y = rng.uniform(-side / 2, side / 2, n)
    bias = rng.normal(0.0, SHEET_SIGMA, SHEETS)[rng.randint(0, SHEETS, n)]
    p = np.stack([x, y, dtu_cases.height(x, y) + 600.0 + bias], axis=1)
    p += rng.normal(0.0, NOISE, (n, 3))
    return _f32(p)


def _row(points, dst, seed):
    return {"points": points, "dst": dst, "order": dtu_eval.visiting_order(points.shape[0], seed)}


def sheets(seed: int):
    """-> {"data", "stl", "obs_mask", "bb", "res", "plane"}, the layout of dtu_cases.make_scan."""
    rng = np.random.RandomState(seed)
    stl = dtu_cases.surface(rng, N_STL, SIDE)
    data = layered(rng, N_DATA, SIDE)
    lo = stl.min(axis=0) - 40.0
    hi = stl.max(axis=0) + 40.0
    n_out = N_DATA // 100
    data[:n_out] = _f32(rng.uniform(lo - 40.0, hi + 40.0, (n_out, 3)))  # some fall outside BB and its blocks
    data = data[rng.permutation(N_DATA)]
    return {"data": data, "stl": stl, **dtu_cases.scan_truth(stl, lo, hi, 4.0)}


def literal(seed: int):
    n = 300_000
    return _row(layered(np.random.RandomState(seed), n, float(np.sqrt(n / DENSITY))), DST, seed)


def stack(seed: int, n: int = 200_000):
    rng = np.random.RandomState(seed)
    p = layered(rng, n, float(np.sqrt(n / 10_000.0)))
    m = n // 10
    p[:m] = p[rng.randint(m, n, m)]  # exact duplicates
    return _row(p[rng.permutation(n)], DST, seed)


def lattice(seed: int):
    g = np.arange(100) * 0.25
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3) + 1000.0
    return _row(p, 0.25, seed)


def chain(decreasing: bool = False):
    n = 3000
    step = 0.9 * DST * np.array([3.0, 2.0, 1.0]) / np.sqrt(14.0)
    p = _f32(np.array([-150.0, -100.0, 550.0]) + np.arange(n)[:, None] * step)
    order = np.arange(n)[::-1].copy() if decreasing else np.arange(n)
    return {"points": p, "dst": DST, "order": order}


def neighbour_counts(points: np.ndarray, dst: float, lo, hi) -> np.ndarray:
    """Points within dst (dtu_oracle's exact test, the point itself not counted) of each point inside the box [lo, hi)."""
    lo, hi = np.asarray(lo, dtype=np.float64), np.asarray(hi, dtype=np.float64)
    near = np.nonzero(((points >= lo - 2 * dst) & (points < hi + 2 * dst)).all(axis=1))[0]
    inner = ((points[near] >= lo) & (points[near] < hi)).all(axis=1)
    pairs = do.thin_pairs(points[near], dst)
    return np.bincount(pairs.ravel(), minlength=near.size)[inner]
