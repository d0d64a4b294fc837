"""CPU restatement of the DTU point-cloud evaluation protocol (reference evaluations/dtu/*.m) in numpy + scipy's cKDTree.

TEST INFRASTRUCTURE ONLY: nothing under patchmatchnet_b200/ imports this file; only tests/ and tools/ may.  It follows the
MATLAB scripts step by step, in float64:

    thin              reducePts_haa.m: the literal sequential loop over the visiting order -- a point still in the set
                      removes every point within distance <= dst of it, then puts itself back
    max_dist_cp       MaxDistCP.m: the literal loop over the max_dist blocks of BB, a nearest-neighbour search per block into
                      the "to" points of the block widened by max_dist, max_dist where that set is empty or the point is in
                      no block (values above max_dist are kept, as the script keeps them)
    data_in_mask      PointCompareMain.m:31-41 (MATLAB round: half away from zero)
    stl_above_plane   PointCompareMain.m:53
    side_stats        BaseEvalMain_web.m:62-75 / ComputeStat_web.m:52-68: count, mean, median, var (N - 1) of the values < 20

"distance <= dst" is sqrt((dx*dx + dy*dy) + dz*dz) <= dst evaluated in that order; the kd-tree only proposes candidates
(radius widened by 1e-9 relative) and this exact test decides.  MATLAB and the DTU data are not available to pin these
functions against; tests/test_dtu_eval.py pins them with small cases whose answers are worked out by hand.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
from scipy.spatial import cKDTree


def _dist(points: np.ndarray, p: np.ndarray) -> np.ndarray:
    dx = points[:, 0] - p[0]
    dy = points[:, 1] - p[1]
    dz = points[:, 2] - p[2]
    return np.sqrt((dx * dx + dy * dy) + dz * dz)


def thin(points: np.ndarray, order: np.ndarray, dst: float) -> np.ndarray:
    """reducePts_haa.m with the visiting order `order` (point indices, first visited first) -> keep mask bool [n]."""
    points = np.asarray(points, dtype=np.float64)
    n = points.shape[0]
    keep = np.ones(n, dtype=bool)
    if n == 0:
        return keep
    candidates = cKDTree(points).query_ball_point(points, dst * (1 + 1e-9), workers=-1)
    for i in np.asarray(order):
        if keep[i]:
            c = np.asarray(candidates[i], dtype=np.int64)
            keep[c[_dist(points[c], points[i]) <= dst]] = False
            keep[i] = True
    return keep


def max_dist_cp(q_to: np.ndarray, q_from: np.ndarray, bb: np.ndarray, max_dist: float) -> np.ndarray:
    """MaxDistCP.m: per-block nearest distance from each q_from point to q_to (points as rows)."""
    q_to = np.asarray(q_to, dtype=np.float64)
    q_from = np.asarray(q_from, dtype=np.float64)
    bb = np.asarray(bb, dtype=np.float64).reshape(2, 3)
    dist = np.full(q_from.shape[0], float(max_dist))
    rng = np.floor((bb[1] - bb[0]) / max_dist)
    if (rng < 0).any():
        return dist
    for x in range(int(rng[0]) + 1):
        for y in range(int(rng[1]) + 1):
            for z in range(int(rng[2]) + 1):
                low = bb[0] + np.array([x, y, z], dtype=np.float64) * max_dist
                high = low + max_dist
                idx_f = np.nonzero(((q_from >= low) & (q_from < high)).all(axis=1))[0]
                if idx_f.size == 0:
                    continue
                low = low - max_dist
                high = high + max_dist
                idx_t = np.nonzero(((q_to >= low) & (q_to < high)).all(axis=1))[0]
                if idx_t.size == 0:
                    dist[idx_f] = max_dist
                else:
                    dist[idx_f] = cKDTree(q_to[idx_t]).query(q_from[idx_f], k=1, workers=-1)[0]
    return dist


def matlab_round(v: np.ndarray) -> np.ndarray:
    t = np.trunc(v)
    return t + np.sign(v) * (np.abs(v - t) >= 0.5)


def data_in_mask(q: np.ndarray, obs_mask: np.ndarray, bb: np.ndarray, res: float) -> np.ndarray:
    """PointCompareMain.m:31-41."""
    bb = np.asarray(bb, dtype=np.float64).reshape(2, 3)
    qv = matlab_round((np.asarray(q, dtype=np.float64) - bb[0]) / res + 1)
    size = np.array(obs_mask.shape)
    inside = ((qv > 0) & (qv <= size)).all(axis=1)
    out = np.zeros(q.shape[0], dtype=bool)
    iv = qv[inside].astype(np.int64) - 1
    out[np.nonzero(inside)[0]] = np.asarray(obs_mask)[iv[:, 0], iv[:, 1], iv[:, 2]] != 0
    return out


def stl_above_plane(q_stl: np.ndarray, plane: np.ndarray) -> np.ndarray:
    """PointCompareMain.m:53."""
    p = np.asarray(plane, dtype=np.float64).reshape(4)
    q = np.asarray(q_stl, dtype=np.float64)
    return ((p[0] * q[:, 0] + p[1] * q[:, 1]) + p[2] * q[:, 2]) + p[3] > 0


def side_stats(d: np.ndarray) -> Dict[str, float]:
    """MATLAB's length / mean / median / var of one side's filtered distances."""
    d = np.asarray(d, dtype=np.float64)
    n = d.size
    if n == 0:
        return {"count": 0, "mean": math.nan, "median": math.nan, "var": math.nan}
    return {"count": n, "mean": float(np.mean(d)), "median": float(np.median(d)), "var": float(np.var(d, ddof=1)) if n > 1 else 0.0}


def evaluate_scan(data_points, stl_points, obs_mask, bb, res, plane, order, *, dst=0.2, search_dist=60.0, outlier_dist=20.0):
    """PointCompareMain.m + the per-scan statistics, with the thinning's visiting order given."""
    data = np.asarray(data_points, dtype=np.float64).reshape(-1, 3)
    stl = np.asarray(stl_points, dtype=np.float64).reshape(-1, 3)
    thinned = data[thin(data, order, dst)]
    d_data = max_dist_cp(stl, thinned, bb, search_dist)
    d_stl = max_dist_cp(thinned, stl, bb, search_dist)
    acc = d_data[data_in_mask(thinned, obs_mask, bb, res)]
    comp = d_stl[stl_above_plane(stl, plane)]
    out = {"n_data": int(data.shape[0]), "n_thinned": int(thinned.shape[0]), "n_stl": int(stl.shape[0])}
    for name, d in (("acc", acc[acc < outlier_dist]), ("comp", comp[comp < outlier_dist])):
        for k, v in side_stats(d).items():
            out[f"{name}_{k}"] = v
    return out
