"""CPU restatement of the Tanks and Temples evaluation (patchmatchnet_b200/tnt_eval.py) in numpy + scipy, float64.

TEST INFRASTRUCTURE ONLY: nothing under patchmatchnet_b200/ imports this file.  Each function states the definition it
implements (the same one include/patchmatch_b200.h and INTEGRATION.md give) in the plainest form:

    transform            x' = ((m00 x + m01 y) + m02 z) + m03 per row
    crop                 SelectionPolygonVolume: axis bounds, then an odd count of polygon crossings strictly below p_u
    voxel_downsample     origin min - s/2, voxel floor((p - o) / s), mean per voxel in original order, voxels ascending
    uniform_downsample   every k-th point, k = round(n / 4 * 2^20) when n > 4 * 2^20
    correspondences      nearest target point within distance <= r, ties to the smallest target index (cKDTree proposes,
                         the exact float64 distance decides)
    umeyama / icp        Eigen::umeyama with scaling on centred points; Open3D's registration_icp loop
    ransac               the per-sample loop of trajectory alignment over given index samples, then the refit
    score                uncapped cKDTree distances, precision / recall / F, np.histogram curves

The literal forms loop in Python over points and voxels; they are the definition.  The *_v forms below compute the same
results with whole-array numpy and batched cKDTree queries, so that the oracle runs at the sizes of real scenes (tens of
millions of points); tests/test_tnt_scale_oracle.py shows them equal to the literal forms bit for bit and index for index.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.spatial import cKDTree


def transform(points: np.ndarray, t) -> np.ndarray:
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    m = np.asarray(t, dtype=np.float64).reshape(4, 4)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((m[r, 0] * x + m[r, 1] * y) + m[r, 2] * z) + m[r, 3] for r in range(3)], axis=1)


def crop(points: np.ndarray, crop_volume) -> np.ndarray:
    """Keep mask of SelectionPolygonVolume, evaluated point by point with Python floats (IEEE float64, no contraction)."""
    w = crop_volume["orthogonal_axis"]
    u, v = {0: (1, 2), 1: (0, 2), 2: (0, 1)}[w]
    poly = np.asarray(crop_volume["polygon"], dtype=np.float64).reshape(-1, 3)
    pu_, pv_ = poly[:, u].tolist(), poly[:, v].tolist()
    nv = len(pu_)
    keep = np.zeros(len(points), dtype=bool)
    for i, p in enumerate(np.asarray(points, dtype=np.float64).reshape(-1, 3).tolist()):
        if not (crop_volume["axis_min"] <= p[w] <= crop_volume["axis_max"]):
            continue
        inside = False
        for a in range(nv):
            b = (a + 1) % nv
            if (pv_[a] < p[v] <= pv_[b]) or (pv_[b] < p[v] <= pv_[a]):
                c = pu_[a] + (p[v] - pv_[a]) / (pv_[b] - pv_[a]) * (pu_[b] - pu_[a])
                if c < p[u]:
                    inside = not inside
        keep[i] = inside
    return keep


def voxel_downsample(points: np.ndarray, s: float) -> np.ndarray:
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if p.shape[0] == 0:
        return p.copy()
    o = p.min(0) - s * 0.5
    idx = np.floor((p - o) / s).astype(np.int64)
    order = np.lexsort((np.arange(p.shape[0]), idx[:, 2], idx[:, 1], idx[:, 0]))
    si = idx[order]
    start = np.ones(p.shape[0], dtype=bool)
    start[1:] = (si[1:] != si[:-1]).any(1)
    bounds = np.append(np.nonzero(start)[0], p.shape[0])
    out = np.empty((bounds.size - 1, 3))
    sp = p[order]
    for k in range(bounds.size - 1):
        acc = np.zeros(3)
        for q in sp[bounds[k]:bounds[k + 1]]:
            acc = acc + q
        out[k] = acc / (bounds[k + 1] - bounds[k])
    return out


def uniform_downsample(points: np.ndarray, max_points: int = 4 * 2 ** 20) -> np.ndarray:
    n = len(points)
    return points if n <= max_points else points[:: max(int(round(n / max_points)), 1)]


def correspondences(src: np.ndarray, tgt: np.ndarray, r: float):
    """-> (index int64 [n] (-1 = none), squared distance [n])."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    idx = np.full(len(src), -1, dtype=np.int64)
    d2 = np.full(len(src), np.inf)
    if len(src) == 0 or len(tgt) == 0:
        return idx, d2
    tree = cKDTree(tgt)
    d0, _ = tree.query(src, k=1, distance_upper_bound=r * (1 + 1e-9))
    for i in np.nonzero(np.isfinite(d0))[0]:
        c = np.asarray(tree.query_ball_point(src[i], d0[i] * (1 + 1e-9) + 1e-300), dtype=np.int64)
        dx, dy, dz = tgt[c, 0] - src[i, 0], tgt[c, 1] - src[i, 1], tgt[c, 2] - src[i, 2]
        e = (dx * dx + dy * dy) + dz * dz
        best = e.min()
        if math.sqrt(best) <= r:
            idx[i] = c[e == best].min()
            d2[i] = best
    return idx, d2


def umeyama(src: np.ndarray, dst: np.ndarray) -> np.ndarray:
    """Eigen::umeyama(src^T, dst^T, with_scaling=true) -> [4,4]; the identity for no points."""
    src, dst = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(dst, np.float64).reshape(-1, 3)
    if len(src) == 0:
        return np.eye(4)
    ms, md = src.mean(0), dst.mean(0)
    cs, cd = src - ms, dst - md
    sigma = cd.T @ cs / len(src)
    u, d, vt = np.linalg.svd(sigma)
    s = np.ones(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        s[2] = -1
    r = u @ np.diag(s) @ vt
    c = (d @ s) / ((cs ** 2).sum() / len(src))
    t = np.eye(4)
    t[:3, :3] = c * r
    t[:3, 3] = md - c * r @ ms
    return t


def icp(src, tgt, r, max_iteration=30, init=None, relative_fitness=1e-6, relative_rmse=1e-6):
    """Open3D's registration_icp loop with the composed transform applied to the original source each time."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    t = np.eye(4) if init is None else np.asarray(init, np.float64).copy()

    def evaluate(t):
        p = transform(src, t)
        idx, d2 = correspondences(p, tgt, r)
        ok = idx >= 0
        n = int(ok.sum())
        return p, idx, n, (n / len(src) if len(src) else 0.0), (math.sqrt(d2[ok].sum() / n) if n else 0.0), float(d2[ok].sum())

    p, idx, n, fit, rmse, s2 = evaluate(t)
    history = [(n, s2)]
    it = 0
    for _ in range(max_iteration):
        ok = idx >= 0
        t = umeyama(p[ok], tgt[idx[ok]]) @ t
        p, idx, n, f2, r2, s2 = evaluate(t)
        history.append((n, s2))
        it += 1
        done = abs(fit - f2) < relative_fitness and abs(rmse - r2) < relative_rmse
        fit, rmse = f2, r2
        if done:
            break
    return {"transformation": t, "fitness": fit, "inlier_rmse": rmse, "iterations": it, "correspondences": n,
            "history": history, "correspondence_set": idx}


def ransac(source, target, samples, inlier_dist=0.2):
    """The per-sample loop of trajectory alignment over the given samples [iterations, 6], then the refit."""
    source, target = np.asarray(source, np.float64), np.asarray(target, np.float64)
    best = (-1, math.inf, -1)
    with np.errstate(all="ignore"):
        for k, smp in enumerate(samples):
            t = umeyama(source[smp], target[smp])
            d2 = ((transform(source, t) - target) ** 2).sum(1)
            inl = d2 < inlier_dist * inlier_dist
            n = int(inl.sum())
            rmse = math.sqrt(d2[inl].sum() / n) if n else 0.0
            if n > best[0] or (n == best[0] and rmse < best[1]):
                best = (n, rmse, k)
    t = umeyama(source[samples[best[2]]], target[samples[best[2]]])
    inl = ((transform(source, t) - target) ** 2).sum(1) < inlier_dist * inlier_dist
    return umeyama(source[inl], target[inl]), best


def refine(rec, gt, crop_volume, init, tau, max_iteration=20):
    t = np.asarray(init, np.float64)
    rounds = []
    for method, voxel, dist in (("voxel", tau, 80 * tau), ("voxel", tau / 2, 20 * tau), ("uniform", None, 2 * tau)):
        s = transform(rec, t)
        s = s[crop(s, crop_volume)]
        g = gt[crop(gt, crop_volume)]
        s, g = (voxel_downsample(s, voxel), voxel_downsample(g, voxel)) if method == "voxel" else (uniform_downsample(s), uniform_downsample(g))
        r = icp(s, g, dist, max_iteration=max_iteration)
        t = r["transformation"] @ t
        rounds.append({"n_source": len(s), "n_target": len(g), "iterations": r["iterations"], "correspondences": r["correspondences"],
                       "fitness": r["fitness"], "history": r["history"], "transformation": t})
    return t, rounds


def score(rec, gt, crop_volume, t, tau):
    s = transform(rec, t)
    s = voxel_downsample(s[crop(s, crop_volume)], tau / 2)
    g = voxel_downsample(gt[crop(gt, crop_volume)], tau / 2)
    d1 = cKDTree(g).query(s, k=1)[0] if len(g) else np.full(len(s), np.inf)
    d2 = cKDTree(s).query(g, k=1)[0] if len(s) else np.full(len(g), np.inf)
    p = float((d1 < tau).mean()) if len(d1) else 0.0
    r = float((d2 < tau).mean()) if len(d2) else 0.0
    f = 2 * p * r / (p + r) if p + r > 0 else 0.0
    edges = np.arange(0, 5 * tau, tau / 100)
    cum = [np.cumsum(np.histogram(d, edges)[0]) / max(len(d), 1) for d in (d1, d2)]
    return {"precision": p, "recall": r, "fscore": f, "n_source_scored": len(s), "n_gt_scored": len(g),
            "precision_count": int((d1 < tau).sum()), "recall_count": int((d2 < tau).sum()),
            "cum_precision": cum[0], "cum_recall": cum[1]}


def evaluate_scene(rec, gt, crop_volume, init, tau, max_iteration=20):
    rec, gt = np.asarray(rec, np.float64).reshape(-1, 3), np.asarray(gt, np.float64).reshape(-1, 3)
    t, rounds = refine(rec, gt, crop_volume, init, tau, max_iteration)
    out = {"transformation": t, "rounds": rounds, "fitness": rounds[-1]["fitness"]}
    out.update(score(rec, gt, crop_volume, t, tau))
    return out


# ---- vectorised forms (same results as the literal ones above, at scene sizes) ---------------------------------------------

CANDIDATES = 8  # correspondences_v: nearest candidates per source point proposed by one batched cKDTree query


def crop_v(points: np.ndarray, crop_volume) -> np.ndarray:
    """crop over all points at once: one pass per polygon edge with crop's float64 expression in crop's order,
    pu_a + ((pv - pv_a) / (pv_b - pv_a)) * (pu_b - pu_a), and its strict / non-strict comparisons.  numpy rounds every
    operation on its own (no contraction), so the mask is crop's bit for bit."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    w = crop_volume["orthogonal_axis"]
    u, v = {0: (1, 2), 1: (0, 2), 2: (0, 1)}[w]
    poly = np.asarray(crop_volume["polygon"], dtype=np.float64).reshape(-1, 3)
    pu_, pv_ = poly[:, u].tolist(), poly[:, v].tolist()
    nv = len(pu_)
    keep = (crop_volume["axis_min"] <= p[:, w]) & (p[:, w] <= crop_volume["axis_max"])
    sel = np.nonzero(keep)[0]
    pu, pv = p[sel, u], p[sel, v]
    inside = np.zeros(sel.size, dtype=bool)
    for a in range(nv):
        b = (a + 1) % nv
        m = ((pv_[a] < pv) & (pv <= pv_[b])) | ((pv_[b] < pv) & (pv <= pv_[a]))
        c = pu_[a] + (pv[m] - pv_[a]) / (pv_[b] - pv_[a]) * (pu_[b] - pu_[a])
        inside[m] ^= c < pu[m]
    keep[sel] = inside
    return keep


def voxel_downsample_v(points: np.ndarray, s: float) -> np.ndarray:
    """voxel_downsample without the per-voxel loop.  The order argument: voxel_downsample sorts by (x, y, z, original index)
    with one lexsort, so its voxels come out in ascending (x, y, z) order and the points of a voxel in their original order;
    this form uses the same lexsort.  Its sum then runs over the voxels together, one point position at a time: step j adds
    the j-th point of every voxel that has more than j points, to that voxel's running sum from 0.0.  Each voxel thus sees
    voxel_downsample's additions in voxel_downsample's order, and the mean is the same division, so every output is the
    literal one's bits (np.add.reduceat would sum pairwise, a different rounding)."""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    if p.shape[0] == 0:
        return p.copy()
    o = p.min(0) - s * 0.5
    idx = np.floor((p - o) / s).astype(np.int64)
    order = np.lexsort((np.arange(p.shape[0]), idx[:, 2], idx[:, 1], idx[:, 0]))
    si = idx[order]
    start = np.ones(p.shape[0], dtype=bool)
    start[1:] = (si[1:] != si[:-1]).any(1)
    first = np.nonzero(start)[0]
    count = np.diff(np.append(first, p.shape[0]))
    sp = p[order]
    acc = np.zeros((first.size, 3))
    live = np.arange(first.size)
    j = 0
    while live.size:
        acc[live] = acc[live] + sp[first[live] + j]
        j += 1
        live = live[count[live] > j]
    return acc / count[:, None]


def correspondences_v(src: np.ndarray, tgt: np.ndarray, r: float, tree=None, k: int = CANDIDATES):
    """correspondences with one batched query: cKDTree proposes the k nearest target points within r (1 + 1e-9); their exact
    distances ((dx dx + dy dy) + dz dz) are recomputed, the minimum is taken, then the smallest index at the minimum.
    correspondences' candidates are the points within R = d0 (1 + 1e-9) + 1e-300 of the query, d0 the tree's nearest
    distance; when the k-th proposal lies beyond R every such point is among the proposals and none of the others can reach
    the minimum, so the result is correspondences'.  Otherwise (k points tie within R) that row falls back to
    correspondences' own ball query.  `tree`: a cKDTree over tgt to reuse.  -> (index int64 [n] (-1 = none), d^2 [n])."""
    src, tgt = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(tgt, np.float64).reshape(-1, 3)
    idx = np.full(len(src), -1, dtype=np.int64)
    d2 = np.full(len(src), np.inf)
    if len(src) == 0 or len(tgt) == 0:
        return idx, d2
    tree = cKDTree(tgt) if tree is None else tree
    k = min(k, len(tgt))
    dk, ik = tree.query(src, k=k, distance_upper_bound=r * (1 + 1e-9), workers=-1)
    dk, ik = dk.reshape(len(src), k), ik.reshape(len(src), k)
    found = np.isfinite(dk[:, 0])
    rows = np.nonzero(found)[0]
    c = ik[rows]
    ok = c < len(tgt)
    cc = np.where(ok, c, 0)
    q = src[rows]
    dx, dy, dz = tgt[cc, 0] - q[:, 0:1], tgt[cc, 1] - q[:, 1:2], tgt[cc, 2] - q[:, 2:3]
    e = np.where(ok, (dx * dx + dy * dy) + dz * dz, np.inf)
    best = e.min(1)
    pick = np.where(e == best[:, None], cc, np.iinfo(np.int64).max).min(1)
    hit = np.sqrt(best) <= r
    idx[rows[hit]] = pick[hit]
    d2[rows[hit]] = best[hit]
    ball = dk[rows, 0] * (1 + 1e-9) + 1e-300
    for t in np.nonzero(dk[rows, k - 1] <= ball)[0]:  # k proposals within the literal ball: it may hold more
        i = rows[t]
        cb = np.asarray(tree.query_ball_point(src[i], ball[t]), dtype=np.int64)
        ex, ey, ez = tgt[cb, 0] - src[i, 0], tgt[cb, 1] - src[i, 1], tgt[cb, 2] - src[i, 2]
        eb = (ex * ex + ey * ey) + ez * ez
        b = eb.min()
        idx[i], d2[i] = (cb[eb == b].min(), b) if math.sqrt(b) <= r else (-1, np.inf)
    return idx, d2


def icp_v(src, tgt, r, max_iteration=30, init=None, relative_fitness=1e-6, relative_rmse=1e-6):
    """icp on correspondences_v, the target tree built once.  The sums over the correspondences are the literal ones'
    (numpy sums of the same arrays), so every record is icp's."""
    src, tgt = np.asarray(src, np.float64).reshape(-1, 3), np.asarray(tgt, np.float64).reshape(-1, 3)
    t = np.eye(4) if init is None else np.asarray(init, np.float64).copy()
    tree = cKDTree(tgt) if len(tgt) else None

    def evaluate(t):
        p = transform(src, t)
        idx, d2 = correspondences_v(p, tgt, r, tree)
        ok = idx >= 0
        n = int(ok.sum())
        return p, idx, n, (n / len(src) if len(src) else 0.0), (math.sqrt(d2[ok].sum() / n) if n else 0.0), float(d2[ok].sum())

    p, idx, n, fit, rmse, s2 = evaluate(t)
    history = [(n, s2)]
    deltas = []
    it = 0
    for _ in range(max_iteration):
        ok = idx >= 0
        t = umeyama(p[ok], tgt[idx[ok]]) @ t
        p, idx, n, f2, r2, s2 = evaluate(t)
        history.append((n, s2))
        it += 1
        deltas.append((abs(fit - f2), abs(rmse - r2)))
        done = abs(fit - f2) < relative_fitness and abs(rmse - r2) < relative_rmse
        fit, rmse = f2, r2
        if done:
            break
    return {"transformation": t, "fitness": fit, "inlier_rmse": rmse, "iterations": it, "correspondences": n,
            "history": history, "correspondence_set": idx, "deltas": deltas}


def refine_v(rec, gt, crop_volume, init, tau, max_iteration=20, keep_inputs=False):
    """refine on the vectorised pieces.  keep_inputs: each round's record also holds its down-sampled clouds ("source",
    "target") and the estimate it started from ("start")."""
    t = np.asarray(init, np.float64)
    rounds = []
    for method, voxel, dist in (("voxel", tau, 80 * tau), ("voxel", tau / 2, 20 * tau), ("uniform", None, 2 * tau)):
        s = transform(rec, t)
        s = s[crop_v(s, crop_volume)]
        g = gt[crop_v(gt, crop_volume)]
        n_cropped = len(s)
        s, g = (voxel_downsample_v(s, voxel), voxel_downsample_v(g, voxel)) if method == "voxel" else (uniform_downsample(s), uniform_downsample(g))
        r = icp_v(s, g, dist, max_iteration=max_iteration)
        rec_ = {"n_source": len(s), "n_target": len(g), "iterations": r["iterations"], "correspondences": r["correspondences"],
                "fitness": r["fitness"], "history": r["history"], "deltas": r["deltas"], "transformation": r["transformation"] @ t,
                "n_source_cropped": n_cropped}
        if keep_inputs:
            rec_.update(source=s, target=g, start=t, icp=r["transformation"])
        t = rec_["transformation"]
        rounds.append(rec_)
    return t, rounds


def score_v(rec, gt, crop_volume, t, tau):
    """score on the vectorised pieces, the distances from multi-threaded cKDTree queries."""
    s = transform(rec, t)
    s = voxel_downsample_v(s[crop_v(s, crop_volume)], tau / 2)
    g = voxel_downsample_v(gt[crop_v(gt, crop_volume)], tau / 2)
    d1 = cKDTree(g).query(s, k=1, workers=-1)[0] if len(g) else np.full(len(s), np.inf)
    d2 = cKDTree(s).query(g, k=1, workers=-1)[0] if len(s) else np.full(len(g), np.inf)
    p = float((d1 < tau).mean()) if len(d1) else 0.0
    r = float((d2 < tau).mean()) if len(d2) else 0.0
    f = 2 * p * r / (p + r) if p + r > 0 else 0.0
    edges = np.arange(0, 5 * tau, tau / 100)
    cum = [np.cumsum(np.histogram(d, edges)[0]) / max(len(d), 1) for d in (d1, d2)]
    return {"precision": p, "recall": r, "fscore": f, "n_source_scored": len(s), "n_gt_scored": len(g),
            "precision_count": int((d1 < tau).sum()), "recall_count": int((d2 < tau).sum()),
            "cum_precision": cum[0], "cum_recall": cum[1]}


def evaluate_scene_v(rec, gt, crop_volume, init, tau, max_iteration=20, keep_inputs=False):
    rec, gt = np.asarray(rec, np.float64).reshape(-1, 3), np.asarray(gt, np.float64).reshape(-1, 3)
    t, rounds = refine_v(rec, gt, crop_volume, init, tau, max_iteration, keep_inputs)
    out = {"transformation": t, "rounds": rounds, "fitness": rounds[-1]["fitness"]}
    out.update(score_v(rec, gt, crop_volume, t, tau))
    return out
