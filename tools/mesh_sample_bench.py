"""Times of the surface sampler (ops.sample_mesh) on the scene-size TSDF rows of tests/test_gpu_mesh_at_scene_sizes.py and
their 1 % simplifications, at each evaluation's default spacing, and of a whole dtu_eval.evaluate_scan with sampling on a
triangulation of the real-scan-sized synthetic DTU case (tests/dtu_scale_cases.sheets).

    python tools/mesh_sample_bench.py [--out mesh_sample_bench.json] [--rows dtu,tnt,eth3d]

The count pass (ops.sample_mesh_count: workspace, count kernel, two scans, one read) and the whole call (count and emit,
output allocated) are timed with CUDA events after a warm-up; emit = whole - count.  Bytes written per second counts the
output alone, 27 bytes per sample (float64 xyz, uint8 rgb), next to the H100 SXM's 3.35 TB/s.  The card's name, power limit
and maximum SM clock are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from patchmatchnet_b200 import dtu_eval, ops  # noqa: E402

SPACING = {"dtu": 0.2, "tnt": 0.01 / 4, "eth3d": 0.005}  # DTU dst (mm); T&T tau/4 at tau = 0.01 m; ETH3D 0.01 / 2 (m)
HBM_TBS = 3.35


def _time(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(reps):
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
        del out
    return best


def sample_row(name, xyz, rgb, faces, s):
    n = ops.sample_mesh_count(xyz, faces, s)
    t_count = _time(lambda: ops.sample_mesh_count(xyz, faces, s))
    t_all = _time(lambda: ops.sample_mesh(xyz, faces, s, rgb))
    emit = t_all - t_count
    return {"row": name, "faces": int(faces.shape[0]), "samples": n, "spacing": s, "count_ms": t_count, "emit_ms": emit,
            "total_ms": t_all, "write_TBps": 27 * n / (emit * 1e-3) / 1e12 if emit > 0 else None}


def dtu_scan_seconds():
    from tests import dtu_cases, dtu_scale_cases as dsc

    c = dsc.sheets(0)
    t = np.arange(-dsc.SIDE / 2, dsc.SIDE / 2 + 0.25, 0.5)
    x, y = np.meshgrid(t, t, indexing="ij")
    xyz = np.stack([x.ravel(), y.ravel(), dtu_cases.height(x.ravel(), y.ravel()) + 600.0], 1).astype(np.float32)
    m = len(t)
    v = np.arange(m * m).reshape(m, m)
    a, b, cc, d = v[:-1, :-1].ravel(), v[1:, :-1].ravel(), v[:-1, 1:].ravel(), v[1:, 1:].ravel()
    faces = np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, cc], 1)]).astype(np.int32)
    x_d, f_d = torch.from_numpy(xyz).cuda(), torch.from_numpy(faces).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pts, _ = ops.sample_mesh(x_d, f_d, dtu_eval.THIN_DST)
    t1 = time.perf_counter()
    r = dtu_eval.evaluate_scan(pts.cpu().numpy(), c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"], device="cuda")
    t2 = time.perf_counter()
    return {"faces": int(faces.shape[0]), "samples": int(pts.shape[0]), "n_thinned": r["n_thinned"], "sample_s": t1 - t0,
            "evaluate_scan_s": t2 - t1, "total_s": t2 - t0}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--rows", default="dtu,tnt,eth3d")
    args = ap.parse_args()
    from tests import test_gpu_mesh_at_scene_sizes as ms

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    res = {"card": card[0] if card else "unknown", "rows": []}
    for name in args.rows.split(","):
        sc = ms.build_scene(name, "cuda")
        verts, faces = ops.tsdf_mesh(sc["seeds"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], ms.TRUNC, 1)
        del sc
        xyz = verts[:, :12].contiguous().view(torch.float32).view(-1, 3)
        rgb = verts[:, 12:].contiguous()
        res["rows"].append(sample_row(name, xyz, rgb, faces, SPACING[name]))
        print(json.dumps(res["rows"][-1]), flush=True)
        body, f, _ = ops.simplify_mesh(xyz, rgb, faces, faces.shape[0] // 100)
        del verts, faces, xyz, rgb
        res["rows"].append(sample_row(name + " 1%", body[:, :12].contiguous().view(torch.float32).view(-1, 3),
                                      body[:, 12:].contiguous(), f, SPACING[name]))
        print(json.dumps(res["rows"][-1]), flush=True)
        del body, f
        torch.cuda.empty_cache()
    res["dtu_scan"] = dtu_scan_seconds()
    print(json.dumps({"card": res["card"], "dtu_scan": res["dtu_scan"]}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
