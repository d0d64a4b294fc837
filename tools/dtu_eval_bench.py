"""DTU evaluation kernels (csrc/pm_cloud.cu) on synthetic clouds of DTU-like size, beside the CPU oracle's cKDTree path.

    python tools/dtu_eval_bench.py [--data 10000000] [--stl 2500000] [--outliers 0.01] [--reps 3] > dtu_eval_bench.json

Clouds: a smooth 300 x 300 mm surface (tests/dtu_cases.height), STL = `--stl` samples of it, data = `--data` samples with
0.3 mm Gaussian noise plus a fraction `--outliers` spread uniformly over the box widened by 80 mm; the real DTU point counts
are not measured here.  GPU: CUDA events on the current stream around ops.thin_points (dst = 0.2), the data -> STL and the
STL -> data distance passes (max_dist = 60), each after one warm-up call, median of `--reps`.  CPU: the oracle's cKDTree
path on the same clouds -- tree build + nearest query (workers=-1, the global nearest distance that MaxDistCP's block loop
reduces to below 60 mm), and the thinning's radius search (count of pairs within dst) -- one pass each.
Algorithmic work: points of each pass and, for thinning, the pairs within dst (the edges its rounds resolve)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import dtu_eval, ops  # noqa: E402
from tests.dtu_cases import height  # noqa: E402


def clouds(n_data, n_stl, outliers, seed=0):
    rng = np.random.RandomState(seed)

    def surf(n):
        x, y = rng.uniform(-150, 150, n), rng.uniform(-150, 150, n)
        return np.stack([x, y, height(x, y) + 600.0], axis=1)

    stl = surf(n_stl).astype(np.float32).astype(np.float64)
    data = surf(n_data) + rng.normal(0.0, 0.3, (n_data, 3))
    lo, hi = stl.min(0) - 40.0, stl.max(0) + 40.0
    k = int(outliers * n_data)
    data[:k] = rng.uniform(lo - 40.0, hi + 40.0, (k, 3))
    return data.astype(np.float32).astype(np.float64), stl, np.stack([lo, hi])


def gpu_time(fn, reps):
    fn()  # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", type=int, default=10_000_000)
    ap.add_argument("--stl", type=int, default=2_500_000)
    ap.add_argument("--outliers", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dtu_eval_bench needs a CUDA device")
    dev = "cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    data, stl, bb = clouds(args.data, args.stl, args.outliers)
    d_data = torch.as_tensor(data, device=dev)
    d_stl = torch.as_tensor(stl, device=dev)
    rank = torch.empty(args.data, dtype=torch.int32)
    rank[torch.as_tensor(dtu_eval.visiting_order(args.data, 0))] = torch.arange(args.data, dtype=torch.int32)
    rank = rank.to(dev)

    t_thin, keep = gpu_time(lambda: ops.thin_points(d_data, rank, 0.2), args.reps)
    thinned = d_data[keep]
    t_acc, acc = gpu_time(lambda: ops.nearest_distance(d_stl, thinned, bb, 60.0), args.reps)
    t_comp, comp = gpu_time(lambda: ops.nearest_distance(thinned, d_stl, bb, 60.0), args.reps)
    n_thin = int(thinned.shape[0])
    th = thinned.cpu().numpy()

    t0 = time.perf_counter()
    tree = cKDTree(data)
    pairs = (int(tree.count_neighbors(tree, 0.2)) - args.data) // 2  # unordered pairs within dst (self pairs removed)
    t_cpu_thin_search = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref_acc = cKDTree(stl).query(th, k=1, distance_upper_bound=60.0, workers=-1)[0]
    t_cpu_acc = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref_comp = cKDTree(th).query(stl, k=1, distance_upper_bound=60.0, workers=-1)[0]
    t_cpu_comp = time.perf_counter() - t0
    # agreement where both are below the cap (outside MaxDistCP's blocks the GPU reports 60 by definition)
    a, c = acc.cpu().numpy(), comp.cpu().numpy()
    ok_a, ok_c = (ref_acc < 60) & (a < 60), (ref_comp < 60) & (c < 60)
    max_rel = max(float(np.max(np.abs(a[ok_a] - ref_acc[ok_a]) / np.maximum(ref_acc[ok_a], 1e-300), initial=0.0)),
                  float(np.max(np.abs(c[ok_c] - ref_comp[ok_c]) / np.maximum(ref_comp[ok_c], 1e-300), initial=0.0)))
    print(json.dumps({
        "device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi,
        "cpu_cores": os.cpu_count(),
        "clouds": {"data": args.data, "stl": args.stl, "outlier_fraction": args.outliers, "thinned": n_thin},
        "gpu_ms": {"thin": t_thin, "dist_data_to_stl": t_acc, "dist_stl_to_data": t_comp, "total": t_thin + t_acc + t_comp},
        "cpu_ckdtree_s": {"thin_radius_search_count": t_cpu_thin_search, "dist_data_to_stl": t_cpu_acc,
                          "dist_stl_to_data": t_cpu_comp,
                          "note": "tree build + query; the sequential greedy loop of the thinning is not included"},
        "work": {"thin_points": args.data, "thin_pairs_within_dst": pairs, "dist_data_to_stl_queries": n_thin,
                 "dist_stl_to_data_queries": args.stl},
        "max_rel_diff_vs_ckdtree_below_cap": max_rel,
    }))


if __name__ == "__main__":
    main()
