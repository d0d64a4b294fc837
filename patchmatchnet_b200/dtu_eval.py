"""DTU point-cloud evaluation on the GPU: accuracy / completeness / overall in mm of fused point clouds against the DTU
ground truth, the protocol of the reference's MATLAB scripts (evaluations/dtu: BaseEvalMain_web.m, PointCompareMain.m,
reducePts_haa.m, MaxDistCP.m, ComputeStat_web.m) in float64 throughout.

    thinning      ops.thin_points (csrc/pm_cloud.cu), visiting order drawn from `seed`
    distances     ops.nearest_distance, both directions, capped at `search_dist`
    mask, plane   tensor gathers on the device
    statistics    count, mean, median, variance (N - 1) of the distances below `outlier_dist`

Two documented differences from a MATLAB run (INTEGRATION.md, "DTU evaluation"):
  - the thinning visits the points in an order drawn from a seeded generator instead of MATLAB's randperm, so a result
    differs from a MATLAB run only by which random order was drawn, as two MATLAB runs differ from each other;
  - a distance that MaxDistCP reports above 60 mm (a nearest point found inside the widened block but farther than 60) is 60
    here.  The statistics keep only distances below 20 mm, so they are unaffected.

Command line:
    python -m patchmatchnet_b200.dtu_eval --data-path "SampleSet/MVS Data" --outputs outputs --json dtu.json

With --surface the reconstruction is a triangle mesh scored as a surface: its samples (ops.sample_mesh, every point of the
surface within --surface-spacing of one, default the thinning distance 0.2 mm) go through the unchanged thinning, instead of
its vertices (INTEGRATION.md, "Surface sampling of meshes (beyond the reference)").
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time
from typing import Dict, Sequence

import numpy as np
import torch

from . import data_io, ops, sample

# BaseEvalMain_web.m:23
DTU_EVAL_SCANS = (1, 4, 9, 10, 11, 12, 13, 15, 23, 24, 29, 32, 33, 34, 48, 49, 62, 75, 77, 110, 114, 118)
MASK_MARGIN = 10  # PointCompareMain.m: ObsMask{scan}_10.mat
THIN_DST = 0.2  # BaseEvalMain_web.m: dst, the thinning distance (mm); also the default --surface-spacing


def visiting_order(n: int, seed: int) -> np.ndarray:
    """The thinning's visiting order: a permutation of 0..n-1 from numpy's legacy seeded generator, whose stream is fixed
    across numpy versions and machines (same seed, same order, same kept set)."""
    return np.random.RandomState(seed).permutation(n)


def matlab_round(v: torch.Tensor) -> torch.Tensor:
    """MATLAB's round: half away from zero (not round-half-even).  v - trunc(v) is exact, so the tie test is too."""
    t = torch.trunc(v)
    return t + torch.sign(v) * ((v - t).abs() >= 0.5).to(v.dtype)


def data_in_mask(points: torch.Tensor, obs_mask: torch.Tensor, bb_lo: torch.Tensor, res: float) -> torch.Tensor:
    """PointCompareMain.m: Qv = round((q - BB(1,:)) / Res + 1) (1-based voxel), inside size(ObsMask) and ObsMask(Qv) true."""
    qv = matlab_round((points - bb_lo) / res + 1.0)
    size = torch.tensor(obs_mask.shape, dtype=qv.dtype, device=qv.device)
    inside = ((qv >= 1) & (qv <= size)).all(dim=1)
    idx = (qv.clamp(min=1) - 1).to(torch.int64)
    idx = torch.minimum(idx, (size - 1).to(torch.int64))
    return inside & obs_mask[idx[:, 0], idx[:, 1], idx[:, 2]]


def above_plane(points: torch.Tensor, plane: torch.Tensor) -> torch.Tensor:
    """PointCompareMain.m: P(1) x + P(2) y + P(3) z + P(4) > 0."""
    return ((plane[0] * points[:, 0] + plane[1] * points[:, 1]) + plane[2] * points[:, 2]) + plane[3] > 0


def side_stats(d: torch.Tensor) -> Dict[str, float]:
    """count, mean, median (even count: mean of the two middle values), variance with N - 1 -- MATLAB's mean / median / var,
    including NaN for an empty set and a variance of 0 for a single value."""
    n = int(d.numel())
    if n == 0:
        return {"count": 0, "mean": math.nan, "median": math.nan, "var": math.nan}
    s = torch.sort(d).values
    med = s[n // 2] if n % 2 else (s[n // 2 - 1] + s[n // 2]) / 2
    mean = d.mean()
    var = ((d - mean) ** 2).sum() / (n - 1) if n > 1 else d.new_zeros(())
    return {"count": n, "mean": float(mean), "median": float(med), "var": float(var)}


def evaluate_scan(data_points, stl_points, obs_mask, bb, res, plane, *, dst: float = THIN_DST, search_dist: float = 60.0,
                  outlier_dist: float = 20.0, seed: int = 0, device="cuda") -> Dict[str, float]:
    """One scan (PointCompareMain.m + the per-scan statistics of BaseEvalMain_web.m / ComputeStat_web.m).

    data_points [n,3], stl_points [m,3]: the fused cloud and the DTU STL points (array-likes, widened to float64);
    obs_mask [X,Y,Z] (non-zero = observed), bb [2,3], res: ObsMask{scan}_10.mat; plane [4]: Plane{scan}.mat.
    -> {"n_data", "n_thinned", "n_stl", "acc_count", "acc_mean", "acc_median", "acc_var", "comp_count", ...}"""
    dev = torch.device(device)
    data = torch.as_tensor(np.asarray(data_points, dtype=np.float64).reshape(-1, 3)).to(dev)
    stl = torch.as_tensor(np.asarray(stl_points, dtype=np.float64).reshape(-1, 3)).to(dev)
    bb_np = np.asarray(bb, dtype=np.float64).reshape(2, 3)
    mask = torch.as_tensor(np.asarray(obs_mask) != 0).to(dev)
    plane_t = torch.as_tensor(np.asarray(plane, dtype=np.float64).reshape(4)).to(dev)

    rank = torch.empty(data.shape[0], dtype=torch.int32)
    rank[torch.as_tensor(visiting_order(data.shape[0], seed))] = torch.arange(data.shape[0], dtype=torch.int32)
    keep = ops.thin_points(data, rank.to(dev), dst)
    thinned = data[keep]

    d_data = ops.nearest_distance(stl, thinned, bb_np, search_dist)  # accuracy side: thinned data -> STL
    d_stl = ops.nearest_distance(thinned, stl, bb_np, search_dist)  # completeness side: STL -> thinned data
    in_mask = data_in_mask(thinned, mask, torch.as_tensor(bb_np[0]).to(dev), float(res))
    above = above_plane(stl, plane_t)
    acc = d_data[in_mask]
    comp = d_stl[above]
    out = {"n_data": int(data.shape[0]), "n_thinned": int(thinned.shape[0]), "n_stl": int(stl.shape[0])}
    for name, d in (("acc", acc[acc < outlier_dist]), ("comp", comp[comp < outlier_dist])):
        for k, v in side_stats(d).items():
            out[f"{name}_{k}"] = v
    return out


def summarize(per_scan: Sequence[Dict[str, float]]) -> Dict[str, float]:
    """BaseEvalMain_web.m:98-99: acc and comp are the means over scans of the per-scan means; overall = (acc + comp) / 2."""
    acc = float(np.mean([r["acc_mean"] for r in per_scan])) if per_scan else math.nan
    comp = float(np.mean([r["comp_mean"] for r in per_scan])) if per_scan else math.nan
    return {"acc": acc, "comp": comp, "overall": (acc + comp) / 2}


def load_scan_truth(data_path: str, scan: int) -> Dict[str, object]:
    """The ground truth of one scan under DTU's `SampleSet/MVS Data` folder:
    Points/stl/stl%03d_total.ply, ObsMask/ObsMask{scan}_10.mat (ObsMask, BB, Res) and ObsMask/Plane{scan}.mat (P).
    -> {"stl_points" float64 [m,3], "obs_mask" bool [X,Y,Z], "bb" float64 [2,3], "res" float, "plane" float64 [4]}"""
    from scipy.io import loadmat  # only the evaluation needs scipy

    stl = data_io.read_ply_points(os.path.join(data_path, "Points", "stl", "stl%03d_total.ply" % scan))
    m = loadmat(os.path.join(data_path, "ObsMask", f"ObsMask{scan}_{MASK_MARGIN}.mat"))
    p = loadmat(os.path.join(data_path, "ObsMask", f"Plane{scan}.mat"))
    return {
        "stl_points": stl,
        "obs_mask": np.asarray(m["ObsMask"]) != 0,  # savemat writes logicals back as uint8
        "bb": np.asarray(m["BB"], dtype=np.float64).reshape(2, 3),
        "res": float(np.asarray(m["Res"], dtype=np.float64).squeeze()),  # loadmat returns a scalar as [[x]]
        "plane": np.asarray(p["P"], dtype=np.float64).reshape(4),
    }


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.dtu_eval", description=__doc__.split("\n\n")[0])
    ap.add_argument("--data-path", required=True, help="DTU `SampleSet/MVS Data` folder (Points/stl, ObsMask)")
    ap.add_argument("--outputs", default="outputs", help="folder substituted for {outputs} in --ply-template")
    ap.add_argument("--ply-template", default="{outputs}/scan{scan}/fused.ply", help="path of a scan's fused cloud")
    ap.add_argument("--scans", type=int, nargs="+", default=list(DTU_EVAL_SCANS))
    ap.add_argument("--seed", type=int, default=0, help="seed of the thinning's visiting order")
    ap.add_argument("--json", default=None, help="write the per-scan and final results to this file")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--surface", action="store_true",
                    help="score the mesh at --ply-template as a surface: its samples instead of its vertices")
    ap.add_argument("--surface-spacing", type=float, default=None,
                    help=f"sample spacing of --surface in mm (default {THIN_DST:g}, the thinning distance)")
    args = ap.parse_args(argv)
    if args.surface_spacing is not None and not args.surface:
        raise ValueError("--surface-spacing needs --surface")
    sample.check_spacing(args.surface_spacing, "--surface-spacing")
    spacing = THIN_DST if args.surface_spacing is None else args.surface_spacing

    per_scan = []
    for scan in args.scans:
        t0 = time.perf_counter()
        truth = load_scan_truth(args.data_path, scan)
        path = args.ply_template.format(outputs=args.outputs, scan=scan)
        surface = None
        if args.surface:
            pts, surface = sample.mesh_samples(path, spacing, args.device)
            data = pts.cpu().numpy()
            del pts
        else:
            data = data_io.read_ply_points(path)
        r = evaluate_scan(data, truth["stl_points"], truth["obs_mask"], truth["bb"], truth["res"], truth["plane"],
                          seed=args.seed, device=args.device)
        r["scan"] = scan
        r["seconds"] = time.perf_counter() - t0
        if surface is not None:
            r["surface"] = surface
        per_scan.append(r)
        print(f"scan{scan}: acc. mean/median {r['acc_mean']:.6f}/{r['acc_median']:.6f}  comp. mean/median "
              f"{r['comp_mean']:.6f}/{r['comp_median']:.6f}  ({r['n_data']} -> {r['n_thinned']} points, {r['seconds']:.1f} s)",
              flush=True)
    final = summarize(per_scan)
    print(f"final evaluation result on {len(per_scan)} scans: acc.: {final['acc']:.6f}, comp.: {final['comp']:.6f}, "
          f"overall: {final['overall']:.6f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"seed": args.seed, "scans": per_scan, "final": final}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
