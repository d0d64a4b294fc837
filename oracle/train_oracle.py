"""CPU restatement (NumPy, float64 accumulation) of the reference's per-step training arithmetic: create_stage_images
(train.py:174-180), patchmatchnet_loss with its depth-map gradients (models/net.py:321-342) and the two metrics
(utils.py:187-221).  The checker of the K-L kernels (pm_train.cu).

`elem` selects the dtype of each per-pixel term: float64 restates the reference evaluated on float64 tensors; float32 forms
every term as torch forms it on float32 tensors (the kernels' definition), and the sums stay float64 either way."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np


def stage_images(image: np.ndarray) -> List[np.ndarray]:
    """[B,...,H,W] -> the four levels F.interpolate(scale_factor=0.5**l, mode="nearest") gives: pixel (y, x) of level l is
    pixel (y << l, x << l), size (H >> l, W >> l)."""
    H, W = image.shape[-2:]
    return [image[..., : (H >> l) << l: 1 << l, : (W >> l) << l: 1 << l] for l in range(4)]


def _smooth_l1(diff: np.ndarray) -> np.ndarray:
    z = np.abs(diff)
    half = diff.dtype.type(0.5)
    return np.where(z < 1, half * z * z, z - half)


def loss_terms(maps: Sequence[np.ndarray], levels: Sequence[int], depth_gt: np.ndarray, mask: np.ndarray,
               elem=np.float64) -> np.ndarray:
    """float64 [n_maps + 4]: per map the sum of smooth-L1(d - gt) over the masked pixels of its level, then the counts."""
    gts, masks = stage_images(depth_gt), stage_images(mask.astype(bool))
    out = []
    for m, l in zip(maps, levels):
        sel = masks[l]
        d = np.asarray(m, dtype=elem).reshape(gts[l].shape)[sel]
        out.append(np.sum(_smooth_l1(d - gts[l].astype(elem)[sel]).astype(np.float64)))
    out += [float(np.count_nonzero(masks[l])) for l in range(4)]
    return np.array(out, dtype=np.float64)


def loss_and_grads(maps: Sequence[np.ndarray], levels: Sequence[int], depth_gt: np.ndarray, mask: np.ndarray,
                   elem=np.float64) -> Tuple[float, List[np.ndarray]]:
    """patchmatchnet_loss = sum over maps of the mean smooth-L1 over the level's masked pixels, and d loss / d map
    (clamp(d - gt, -1, 1) / count on the masked pixels, 0 elsewhere), each of its map's shape."""
    terms = loss_terms(maps, levels, depth_gt, mask, elem)
    n = len(maps)
    with np.errstate(invalid="ignore", divide="ignore"):
        loss = float(sum(terms[m] / terms[n + l] for m, l in enumerate(levels)))
    gts, masks = stage_images(depth_gt), stage_images(mask.astype(bool))
    grads = []
    for m, l in zip(maps, levels):
        d = np.asarray(m, dtype=elem).reshape(gts[l].shape)
        diff = np.clip((d - gts[l].astype(elem)).astype(np.float64), -1.0, 1.0)
        with np.errstate(invalid="ignore", divide="ignore"):
            grads.append(np.where(masks[l], diff / terms[n + l], 0.0).reshape(np.shape(m)))
    return loss, grads


def abs_error_per_image(est: np.ndarray, depth_gt: np.ndarray, mask: np.ndarray) -> np.ndarray:
    """absolute_depth_error_metrics before the batch mean: per image, the mean |d - gt| over the masked pixels (float64)."""
    out = []
    for b in range(est.shape[0]):
        sel = mask[b].astype(bool)
        with np.errstate(invalid="ignore"):
            out.append(np.mean(np.abs(est[b].astype(np.float64)[sel] - depth_gt[b].astype(np.float64)[sel])))
    return np.array(out)


def threshold_rate_per_image(est: np.ndarray, depth_gt: np.ndarray, mask: np.ndarray, threshold: float) -> np.ndarray:
    """threshold_metrics before the batch mean: per image, float32 (count of float32 |d - gt| > t) / float32 (masked
    pixels): the reference's mean(err_mask.float()) on the CPU, where a float32 mean is a float32 sum then a division."""
    out = []
    for b in range(est.shape[0]):
        sel = mask[b].astype(bool)
        err = np.abs(est[b][sel] - depth_gt[b][sel]).astype(np.float32)
        with np.errstate(invalid="ignore", divide="ignore"):
            out.append(np.float32(np.count_nonzero(err > np.float32(threshold))) / np.float32(err.size))
    return np.array(out, dtype=np.float32)


def metrics(per_level: Dict[int, np.ndarray], depth_gt: np.ndarray, mask: np.ndarray,
            thresholds=(1, 2, 4, 8)) -> Dict[str, np.ndarray]:
    """Per-image values of the scalars train.py:161-169 logs: depth-error-stage-{l} and threshold-{t}mm-error."""
    gts, masks = stage_images(depth_gt), stage_images(mask)
    out = {f"depth-error-stage-{l}": abs_error_per_image(per_level[l], gts[l], masks[l]) for l in range(4)}
    for t in thresholds:
        out[f"threshold-{t}mm-error"] = threshold_rate_per_image(per_level[0], gts[0], masks[0], float(t))
    return out
