"""CPU restatement of the DTU point-cloud evaluation protocol (reference evaluations/dtu/*.m) in numpy + scipy's cKDTree.

TEST INFRASTRUCTURE ONLY: nothing under patchmatchnet_b200/ imports this file; only tests/ and tools/ may.  It follows the
MATLAB scripts step by step, in float64:

    thin              reducePts_haa.m: the literal sequential loop over the visiting order -- a point still in the set
                      removes every point within distance <= dst of it, then puts itself back
    thin_violations   a vectorised check of a keep mask against `thin` for clouds too big for its Python loop
    thin_sync_rounds  the rounds a synchronous parallel thinning needs, and its keep mask
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


# thin's result is the one set in which a point is kept iff no kept point u != v with dist(u, v) <= dst comes before it in the
# visiting order: the loop's result has that property, and by induction over the order no other set does.  So a mask equals
# thin's iff every point passes that local test, which needs only the kept points' neighbourhoods.

def rank_of(order: np.ndarray) -> np.ndarray:
    """Visiting order (point indices, first visited first) -> rank[i], the position at which point i is visited."""
    order = np.asarray(order, dtype=np.int64)
    rank = np.empty(order.size, dtype=np.int64)
    rank[order] = np.arange(order.size, dtype=np.int64)
    return rank


def _exact_within(points: np.ndarray, a: np.ndarray, b: np.ndarray, dst: float) -> np.ndarray:
    """_dist's expression on index pairs (any matching shapes): dist(points[a], points[b]) <= dst."""
    d = points[a] - points[b]
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]) <= dst


THIN_CHECK_K = 24     # kept points are pairwise more than dst apart: at most 13 fit in a ball of radius dst (12 + centre)
THIN_CHECK_CHUNK = 1 << 20


def thin_violations(points: np.ndarray, rank: np.ndarray, keep: np.ndarray, dst: float) -> np.ndarray:
    """Indices v where keep[v] differs from "no kept u != v within dst has rank[u] < rank[v]" (rank[i]: visiting position of
    point i).  Empty iff keep == thin(points, order, dst) for the order whose ranks these are."""
    points = np.asarray(points, dtype=np.float64)
    rank = np.asarray(rank, dtype=np.int64)
    keep = np.asarray(keep, dtype=bool)
    n = points.shape[0]
    kept = np.nonzero(keep)[0]
    if kept.size == 0:
        return np.arange(n) if n else np.zeros(0, dtype=np.int64)
    tree = cKDTree(points[kept])
    bad = []
    for a in range(0, n, THIN_CHECK_CHUNK):
        v = np.arange(a, min(n, a + THIN_CHECK_CHUNK))
        d, j = tree.query(points[v], k=THIN_CHECK_K, distance_upper_bound=dst * (1 + 1e-9), workers=-1)
        # a saturated query could hide a neighbour; only a mask keeping points within dst of each other saturates
        if np.isfinite(d[:, -1]).any():
            raise AssertionError(f"thin_violations: more than {THIN_CHECK_K - 1} kept points within dst of one point")
        u = kept[np.where(np.isfinite(d), j, 0)]
        nb = np.isfinite(d) & (u != v[:, None]) & _exact_within(points, u, v[:, None], dst)
        earlier = (nb & (rank[u] < rank[v][:, None])).any(axis=1)
        bad.append(v[keep[v] == earlier])
    return np.concatenate(bad)


def thin_pairs(points: np.ndarray, dst: float) -> np.ndarray:
    """Every unordered pair [i, j] (i < j) with dist <= dst in _dist's expression -> int64 [m, 2]."""
    points = np.asarray(points, dtype=np.float64)
    if points.shape[0] < 2:
        return np.zeros((0, 2), dtype=np.int64)
    pairs = cKDTree(points).query_pairs(dst * (1 + 1e-9), output_type="ndarray").astype(np.int64)
    return pairs[_exact_within(points, pairs[:, 0], pairs[:, 1], dst)]


def thin_sync_rounds(points: np.ndarray, rank: np.ndarray, dst: float):
    """The thinning as synchronous rounds: in each, an undecided point is rejected if an earlier neighbour is accepted and
    accepted if every earlier neighbour is decided, all reading the state the round started with.  -> (rounds, keep).
    keep equals thin's.  A parallel thinning whose points also read decisions made earlier in the same round, decisions
    being final, needs at most `rounds` rounds."""
    points = np.asarray(points, dtype=np.float64)
    rank = np.asarray(rank, dtype=np.int64)
    n = points.shape[0]
    pairs = thin_pairs(points, dst)
    first = rank[pairs[:, 0]] < rank[pairs[:, 1]]
    early = np.where(first, pairs[:, 0], pairs[:, 1])
    late = np.where(first, pairs[:, 1], pairs[:, 0])
    undecided, accepted, rejected = 0, 1, 2
    state = np.full(n, undecided, dtype=np.int8)
    rounds = 0
    while (state == undecided).any():
        rounds += 1
        s = state[early]
        blocked = np.zeros(n, dtype=bool)
        blocked[late[s == undecided]] = True
        hit = np.zeros(n, dtype=bool)
        hit[late[s == accepted]] = True
        open_ = state == undecided
        state[open_ & hit] = rejected
        state[open_ & ~hit & ~blocked] = accepted
    return rounds, state == accepted


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
