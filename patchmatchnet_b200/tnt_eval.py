"""Tanks and Temples evaluation on the GPU: precision, recall and F-score of a reconstruction against a training scene's
ground truth at the scene's distance threshold tau, the protocol of the public T&T toolbox (run.py, registration.py,
evaluation.py), restated here in full and computed in float64 throughout (INTEGRATION.md, "Tanks and Temples evaluation").

Inputs of one scene, ground-truth folder <gt>/<Scene>/: <Scene>.ply (GT points), <Scene>.json (crop volume),
<Scene>_trans.txt (COLMAP SfM frame -> GT frame) and <Scene>_COLMAP_SfM.log (camera-to-world poses).

    1. initial alignment   --init trajectory: RANSAC similarity from the scene folder's camera centres (cams/%08d_cam.txt)
                           to the log's camera centres mapped through _trans.txt, then one refit on the best sample's
                           inliers; --init trans: _trans.txt as it is
    2. refinement          three ICP rounds (point to point, with scaling), each on the cropped and down-sampled clouds:
                           voxel tau / 80 tau, voxel tau/2 / 20 tau, uniform / 2 tau (down-sampling / max distance)
    3. scoring             crop, voxel down-sample at tau/2, nearest distances both ways (ops.nearest_distance capped at
                           5 tau, without MaxDistCP's blocks), precision = mean(d1 < tau), recall = mean(d2 < tau), F = 2PR / (P + R), and the
                           cumulative histograms over np.arange(0, 5 tau, tau / 100)

Kernels: ops.crop_points, ops.voxel_downsample, ops.icp and ops.nearest_distance (csrc/pm_cloud.cu).  The host runs the
RANSAC over the few hundred camera centres and the 3 x 3 SVD of each ICP update.

Command line:
    python -m patchmatchnet_b200.tnt_eval --gt-path TrainingSet --outputs outputs --scenes Ignatius Barn --json tnt.json

With --surface the reconstruction is a triangle mesh scored as a surface: its samples (ops.sample_mesh) instead of its
vertices, taken in the reconstruction's frame before the alignment at spacing (tau / 4) / c, c the scale of the initial
similarity (surface_spacing), so that every point of the surface lies within half the tau / 2 scoring voxel of a sample.
"""
from __future__ import annotations

import argparse
import glob
import json
import math
import os
import re
import sys
import time
from typing import Dict, Optional

import numpy as np
import torch

from . import data_io, ops, sample

# distance threshold tau of each training scene (T&T toolbox, run.py / setup)
SCENE_TAU = {"Barn": 0.01, "Caterpillar": 0.005, "Church": 0.025, "Courthouse": 0.025, "Ignatius": 0.003,
             "Meetingroom": 0.01, "Truck": 0.005}
AXES = {"X": 0, "Y": 1, "Z": 2}
UNIFORM_MAX_POINTS = 4 * 2 ** 20  # round 3 keeps every k-th point, k = round(n / this), when a cloud has more points
RANSAC_SAMPLE = 6


# ---- readers --------------------------------------------------------------------------------------------------------------

def read_crop_json(path: str) -> Dict[str, object]:
    """Open3D's SelectionPolygonVolume JSON -> {"orthogonal_axis" 0/1/2, "axis_min", "axis_max", "polygon" float64 [k,3]}."""
    with open(path) as f:
        j = json.load(f)
    axis = str(j["orthogonal_axis"]).upper()
    if axis not in AXES:
        raise ValueError(f"{path}: orthogonal_axis must be X, Y or Z, got {j['orthogonal_axis']!r}")
    poly = np.asarray(j["bounding_polygon"], dtype=np.float64).reshape(-1, 3)
    return {"orthogonal_axis": AXES[axis], "axis_min": float(j["axis_min"]), "axis_max": float(j["axis_max"]), "polygon": poly}


def read_log(path: str) -> np.ndarray:
    """A trajectory .log: per frame one `i j k` line, then 4 rows of the 4 x 4 camera-to-world pose -> float64 [N,4,4]."""
    with open(path) as f:
        rows = [line.split() for line in f if line.strip()]
    if len(rows) % 5:
        raise ValueError(f"{path}: expected 5 lines per frame, got {len(rows)} non-empty lines")
    poses = np.array([[[float(v) for v in rows[5 * i + 1 + r]] for r in range(4)] for i in range(len(rows) // 5)], dtype=np.float64)
    return poses.reshape(-1, 4, 4)


def read_trans(path: str) -> np.ndarray:
    """_trans.txt: a 4 x 4 matrix, 4 rows of 4 numbers -> float64 [4,4]."""
    m = np.loadtxt(path, dtype=np.float64)
    if m.shape != (4, 4):
        raise ValueError(f"{path}: expected a 4 x 4 matrix, got shape {m.shape}")
    return m


def camera_centres(scene_dir: str) -> np.ndarray:
    """Camera centres -R^T t of a scene folder's cams/%08d_cam.txt (world -> camera extrinsics), in view order -> [N,3]."""
    files = sorted(glob.glob(os.path.join(scene_dir, "cams", "*_cam.txt")),
                   key=lambda p: int(re.match(r"(\d+)", os.path.basename(p)).group(1)))
    out = []
    for p in files:
        e = data_io.read_cam_file(p)[1].astype(np.float64)
        out.append(-e[:3, :3].T @ e[:3, 3])
    return np.array(out, dtype=np.float64).reshape(-1, 3)


def load_scene_truth(gt_path: str, scene: str) -> Dict[str, object]:
    """<gt_path>/<scene>/: {"points" float64 [m,3], "crop" (read_crop_json), "trans" [4,4], "log" [N,4,4]}."""
    d = os.path.join(gt_path, scene)
    return {"points": data_io.read_ply_points(os.path.join(d, f"{scene}.ply")),
            "crop": read_crop_json(os.path.join(d, f"{scene}.json")),
            "trans": read_trans(os.path.join(d, f"{scene}_trans.txt")),
            "log": read_log(os.path.join(d, f"{scene}_COLMAP_SfM.log"))}


# ---- initial alignment ----------------------------------------------------------------------------------------------------

def umeyama(src: np.ndarray, dst: np.ndarray) -> np.ndarray:
    """Similarity with scaling mapping src onto dst, batched: [..., k, 3] x2 -> [..., 4, 4] (ops.umeyama_from_moments'
    definition, evaluated on centred points)."""
    src, dst = np.asarray(src, np.float64), np.asarray(dst, np.float64)
    mu_s, mu_d = src.mean(-2), dst.mean(-2)
    cs, cd = src - mu_s[..., None, :], dst - mu_d[..., None, :]
    k = src.shape[-2]
    sigma = np.einsum("...ka,...kb->...ab", cd, cs) / k
    var_s = (cs * cs).sum((-2, -1)) / k
    u, d, vt = np.linalg.svd(sigma)
    s = np.ones(d.shape)
    s[..., 2] = np.where(np.linalg.det(u) * np.linalg.det(vt) < 0, -1.0, 1.0)
    r = (u * s[..., None, :]) @ vt
    c = (d * s).sum(-1) / var_s
    out = np.zeros(src.shape[:-2] + (4, 4))
    out[..., :3, :3] = c[..., None, None] * r
    out[..., :3, 3] = mu_d - np.einsum("...ab,...b->...a", out[..., :3, :3], mu_s)
    out[..., 3, 3] = 1.0
    return out


def ransac_samples(n: int, iterations: int, seed: int) -> np.ndarray:
    """RANSAC's index samples: `iterations` rows of 6 distinct indices in 0..n-1 from numpy's legacy seeded generator.  Row
    entry j is drawn uniformly from the n - j indices not yet in the row (drawn in [0, n - j), then moved past the row's
    earlier entries in ascending order)."""
    rng = np.random.RandomState(seed)
    out = np.empty((iterations, RANSAC_SAMPLE), dtype=np.int64)
    for j in range(RANSAC_SAMPLE):
        r = rng.randint(0, n - j, size=iterations).astype(np.int64)
        if j:
            for c in np.sort(out[:, :j], axis=1).T:
                r += r >= c
        out[:, j] = r
    return out


def trajectory_alignment(source: np.ndarray, target: np.ndarray, seed: int = 0, iterations: int = 100000,
                         inlier_dist: float = 0.2, chunk: int = 4096) -> Dict[str, object]:
    """RANSAC similarity from matched point pairs (source[i] <-> target[i]): each sample of 6 pairs gives a Umeyama
    similarity; its inliers are the pairs with |T s - t|^2 < inlier_dist^2 and its RMSE is over those.  The best sample has
    the most inliers, then the lowest RMSE, then the lowest sample number; the result is its similarity refitted once on its
    inliers.  -> {"transformation" [4,4], "inliers", "rmse", "best_sample"}."""
    source, target = np.asarray(source, np.float64).reshape(-1, 3), np.asarray(target, np.float64).reshape(-1, 3)
    n = source.shape[0]
    if n != target.shape[0]:
        raise ValueError(f"trajectory alignment: {n} camera centres in the scene folder but {target.shape[0]} poses in the "
                         "log; frame i must be view i (use --init trans for a reconstruction already in the T&T COLMAP frame)")
    if n < RANSAC_SAMPLE:
        raise ValueError(f"trajectory alignment needs at least {RANSAC_SAMPLE} cameras, got {n}")
    samples = ransac_samples(n, iterations, seed)
    thr2 = inlier_dist * inlier_dist
    best = (-1, math.inf, -1)
    with np.errstate(all="ignore"):
        for c0 in range(0, iterations, chunk):
            idx = samples[c0:c0 + chunk]
            t = umeyama(source[idx], target[idx])
            mapped = np.einsum("bij,nj->bni", t[:, :3, :3], source) + t[:, None, :3, 3]
            d2 = ((mapped - target[None]) ** 2).sum(-1)
            inl = d2 < thr2
            cnt = inl.sum(1)
            rmse = np.sqrt(np.where(inl, d2, 0.0).sum(1) / np.maximum(cnt, 1))
            order = np.lexsort((np.arange(cnt.size), rmse, -cnt))[0]
            if cnt[order] > best[0] or (cnt[order] == best[0] and rmse[order] < best[1]):
                best = (int(cnt[order]), float(rmse[order]), c0 + int(order))
    if best[0] <= 0:
        raise ValueError("trajectory alignment: no RANSAC sample has an inlier; try --init trans")
    t = umeyama(source[samples[best[2]]], target[samples[best[2]]])
    d2 = (((source @ t[:3, :3].T + t[:3, 3]) - target) ** 2).sum(-1)
    inliers = d2 < thr2
    final = umeyama(source[inliers], target[inliers])
    return {"transformation": final, "inliers": int(inliers.sum()), "rmse": best[1], "best_sample": best[2]}


# ---- refinement and scoring -------------------------------------------------------------------------------------------------

def crop(points: torch.Tensor, crop_volume: Dict[str, object], transform=None) -> torch.Tensor:
    """The points of `points` (after `transform`) inside the crop volume, in their order."""
    out, keep = ops.crop_points(points, crop_volume["orthogonal_axis"], crop_volume["axis_min"], crop_volume["axis_max"],
                                crop_volume["polygon"], transform)
    return out[keep]


def uniform_downsample(points: torch.Tensor, max_points: int = UNIFORM_MAX_POINTS) -> torch.Tensor:
    """Every k-th point from the first, k = round(n / max_points) (round half to even), when n > max_points."""
    n = points.shape[0]
    if n <= max_points:
        return points
    return points[:: max(int(round(n / max_points)), 1)]


def _down(points, method, voxel):
    return ops.voxel_downsample(points, voxel) if method == "voxel" else uniform_downsample(points)


def refine(rec: torch.Tensor, gt: torch.Tensor, crop_volume, init: np.ndarray, tau: float, max_iteration: int = 20):
    """The three ICP rounds: each transforms the reconstruction by the current estimate, crops and down-samples both clouds,
    runs ICP from the identity and composes its result onto the estimate.  -> (transform, per-round records)."""
    t = np.asarray(init, dtype=np.float64)
    rounds = []
    for method, voxel, dist in (("voxel", tau, 80 * tau), ("voxel", tau / 2, 20 * tau), ("uniform", None, 2 * tau)):
        s = _down(crop(rec, crop_volume, t), method, voxel)
        g = _down(crop(gt, crop_volume), method, voxel)
        r = ops.icp(s, g, dist, max_iteration=max_iteration)
        t = r["transformation"] @ t
        rounds.append({"down_sample": method, "voxel_size": voxel, "max_dist": dist, "n_source": int(s.shape[0]),
                       "n_target": int(g.shape[0]), "fitness": r["fitness"], "inlier_rmse": r["inlier_rmse"],
                       "iterations": r["iterations"], "correspondences": r["correspondences"], "transformation": t.tolist()})
    return t, rounds


def histogram_edges(tau: float, device) -> torch.Tensor:
    return torch.as_tensor(np.arange(0, 5 * tau, tau / 100), device=device)


def cumulative_histogram(d: torch.Tensor, edges: torch.Tensor) -> np.ndarray:
    """np.histogram(d, edges) (bins closed on the left, the last one on both sides), cumulated, divided by len(d)."""
    nb = edges.numel() - 1
    b = torch.searchsorted(edges, d, right=True) - 1
    b = torch.where(d == edges[-1], torch.full_like(b, nb - 1), b)
    ok = (b >= 0) & (b < nb)
    counts = torch.bincount(b[ok], minlength=nb)[:nb]
    # divided on the host: torch divides a CUDA tensor by a scalar as a product with its reciprocal, not an IEEE division
    return torch.cumsum(counts, 0).cpu().numpy() / max(d.numel(), 1)


def score(rec: torch.Tensor, gt: torch.Tensor, crop_volume, transform: np.ndarray, tau: float) -> Dict[str, object]:
    """Precision, recall, F-score and the cumulative curves of the aligned reconstruction (toolbox EvaluateHisto and
    get_f1_score_histo2)."""
    s_crop, g_crop = crop(rec, crop_volume, transform), crop(gt, crop_volume)
    s, g = ops.voxel_downsample(s_crop, tau / 2), ops.voxel_downsample(g_crop, tau / 2)
    cap = 5 * tau
    both = [c for c in (s, g) if c.shape[0]]
    if both:
        allp = torch.cat(both)
        box = [(allp.min(0).values - cap).cpu().tolist(), (allp.max(0).values + cap).cpu().tolist()]
    else:
        box = [[0.0] * 3, [1.0] * 3]
    # plain capped distances (compute_point_cloud_distance has no blocks); the box only sizes the search cell
    d1 = ops.nearest_distance(g, s, box, cap, blocks=False)  # reconstruction -> GT
    d2 = ops.nearest_distance(s, g, box, cap, blocks=False)  # GT -> reconstruction
    n1, n2 = int(d1.numel()), int(d2.numel())
    c1, c2 = int((d1 < tau).sum()) if n1 else 0, int((d2 < tau).sum()) if n2 else 0
    precision = c1 / n1 if n1 else 0.0
    recall = c2 / n2 if n2 else 0.0
    f = 2 * precision * recall / (precision + recall) if precision + recall > 0 else 0.0
    edges = histogram_edges(tau, s.device)
    return {"precision": precision, "recall": recall, "fscore": f, "n_source_cropped": int(s_crop.shape[0]),
            "n_gt_cropped": int(g_crop.shape[0]), "n_source_scored": n1, "n_gt_scored": n2,
            "precision_count": c1, "recall_count": c2, "edges": edges.cpu().tolist(),
            "cum_precision": cumulative_histogram(d1, edges).tolist(), "cum_recall": cumulative_histogram(d2, edges).tolist()}


def evaluate_scene(rec_points, gt_points, crop_volume, init_transform, tau: float, *, max_iteration: int = 20,
                   device="cuda") -> Dict[str, object]:
    """Refinement and scoring of one scene, from an initial alignment `init_transform` (reconstruction frame -> GT frame).
    rec_points [n,3], gt_points [m,3]: array-likes, widened to float64."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("tnt_eval runs on a CUDA device; there is no CPU path")
    rec = torch.as_tensor(np.asarray(rec_points, dtype=np.float64).reshape(-1, 3)).to(dev)
    gt = torch.as_tensor(np.asarray(gt_points, dtype=np.float64).reshape(-1, 3)).to(dev)
    t, rounds = refine(rec, gt, crop_volume, init_transform, tau, max_iteration)
    out = {"tau": tau, "n_source": int(rec.shape[0]), "n_gt": int(gt.shape[0]),
           "init_transformation": np.asarray(init_transform, dtype=np.float64).tolist(), "rounds": rounds,
           "transformation": t.tolist(), "fitness": rounds[-1]["fitness"]}
    out.update(score(rec, gt, crop_volume, t, tau))
    return out


def surface_spacing(tau: float, init: np.ndarray) -> float:
    """The default --surface spacing in the reconstruction's frame: (tau / 4) / c, c = cbrt(det) of the initial similarity's
    3 x 3 part (its scale).  ICP's later change of scale is not included; it is small once the initial alignment holds."""
    det = float(np.linalg.det(np.asarray(init, np.float64)[:3, :3]))
    if not (det > 0 and math.isfinite(det)):
        raise ValueError(f"--surface: the initial alignment's 3 x 3 part has determinant {det}; it is not a similarity")
    return (tau / 4) / (det ** (1.0 / 3.0))


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.tnt_eval", description=__doc__.split("\n\n")[0])
    ap.add_argument("--gt-path", required=True, help="T&T ground-truth folder holding <Scene>/<Scene>.ply, .json, _trans.txt, .log")
    ap.add_argument("--outputs", default="outputs", help="folder substituted for {outputs} in --ply-template")
    ap.add_argument("--ply-template", default="{outputs}/{scene}/fused.ply", help="path of a scene's reconstruction")
    ap.add_argument("--input", default="scenes", help="folder substituted for {input} in --scene-template")
    ap.add_argument("--scene-template", default="{input}/{scene}", help="scene folder whose cams/ give the camera centres")
    ap.add_argument("--scenes", nargs="+", required=True)
    ap.add_argument("--init", choices=("trajectory", "trans"), default="trajectory")
    ap.add_argument("--tau", type=float, default=None, help="distance threshold (required for scenes without a known one)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the trajectory alignment's RANSAC")
    ap.add_argument("--json", default=None, help="write the per-scene results to this file")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--surface", action="store_true",
                    help="score the mesh at --ply-template as a surface: its samples instead of its vertices")
    ap.add_argument("--surface-spacing", type=float, default=None,
                    help="sample spacing of --surface in the reconstruction's frame (default (tau / 4) / the initial scale)")
    args = ap.parse_args(argv)
    if args.surface_spacing is not None and not args.surface:
        raise ValueError("--surface-spacing needs --surface")
    sample.check_spacing(args.surface_spacing, "--surface-spacing")
    if not torch.cuda.is_available() or torch.device(args.device).type != "cuda":
        raise RuntimeError("tnt_eval needs a CUDA device; there is no CPU path")
    for scene in args.scenes:
        if args.tau is None and scene not in SCENE_TAU:
            raise ValueError(f"no known tau for scene {scene!r}; pass --tau")

    results = []
    for scene in args.scenes:
        t0 = time.perf_counter()
        tau = args.tau if args.tau is not None else SCENE_TAU[scene]
        truth = load_scene_truth(args.gt_path, scene)
        align: Optional[Dict[str, object]] = None
        if args.init == "trajectory":
            centres = camera_centres(args.scene_template.format(input=args.input, scene=scene))
            target = np.einsum("ij,nj->ni", truth["trans"][:3, :3], truth["log"][:, :3, 3]) + truth["trans"][:3, 3]
            align = trajectory_alignment(centres, target, seed=args.seed)
            init = align["transformation"]
        else:
            init = truth["trans"]
        path = args.ply_template.format(outputs=args.outputs, scene=scene)
        surface = None
        if args.surface:
            spacing = surface_spacing(tau, init) if args.surface_spacing is None else args.surface_spacing
            pts, surface = sample.mesh_samples(path, spacing, args.device)
            rec = pts.cpu().numpy()
            del pts
        else:
            rec = data_io.read_ply_points(path)
        r = evaluate_scene(rec, truth["points"], truth["crop"], init, tau, device=args.device)
        r["scene"] = scene
        r["init"] = args.init
        if align is not None:
            r["alignment"] = {"inliers": align["inliers"], "rmse": align["rmse"], "best_sample": align["best_sample"]}
        r["seconds"] = time.perf_counter() - t0
        if surface is not None:
            r["surface"] = surface
        results.append(r)
        print(f"{scene}: precision {r['precision']:.4f}  recall {r['recall']:.4f}  f-score {r['fscore']:.4f}  tau {tau:g}  "
              f"fitness {r['fitness']:.4f}  ({r['seconds']:.1f} s)", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"init": args.init, "seed": args.seed, "scenes": results}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
