"""CPU restatement of the view selection of the reference's colmap_input.py (:318-373): depth ranges, view scores and the
per-row selection, with the reference's own numpy calls (np.matmul, np.dot, np.linalg.norm, np.arccos, np.exp) in its order.
Membership in obs_j is a set lookup instead of the reference's list scan, so test-sized models take seconds; the sum still runs
over obs_i in order.  Test infrastructure: never imported by the product.

Two documented differences from the reference, shared with the GPU path: the cosine is clamped to [-1, 1], and a point on
either camera centre contributes 0."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np


def depth_ranges(extrinsics: Sequence[np.ndarray], obs: Sequence[Sequence[int]], xyz: np.ndarray) -> List[Tuple[float, float]]:
    """obs[i]: dense point indices of image i (no -1), in order."""
    out = []
    for e, ids in zip(extrinsics, obs):
        zs = sorted(np.matmul(e, [xyz[p][0], xyz[p][1], xyz[p][2], 1])[2].item() for p in ids)
        out.append((zs[int(len(zs) * .01)], zs[int(len(zs) * .99)]))
    return out


def view_scores(centers: np.ndarray, obs: Sequence[Sequence[int]], xyz: np.ndarray, theta0: float = 5.0, sigma1: float = 1.0,
                sigma2: float = 10.0) -> np.ndarray:
    n = len(obs)
    sets = [set(int(p) for p in ids) for ids in obs]
    score = np.zeros((n, n))
    for i in range(n):
        for j in range(i + 1, n):
            ci, cj = centers[i], centers[j]
            s = 0.0
            for p in obs[i]:
                if int(p) not in sets[j]:
                    continue
                x = xyz[int(p)]
                na, nb = np.linalg.norm(ci - x), np.linalg.norm(cj - x)
                if na == 0 or nb == 0:
                    continue
                c = np.dot(ci - x, cj - x) / na / nb
                theta = (180 / np.pi) * np.arccos(min(max(c, -1.0), 1.0))
                s += np.exp(-(theta - theta0) * (theta - theta0) / (2 * (sigma1 if theta <= theta0 else sigma2) ** 2))
            score[i, j] = s
            score[j, i] = s
    return score
