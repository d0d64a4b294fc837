"""Surface normals and oriented fusion (pmb200_depth_normals, pmb200_fuse_points_oriented) on the GPU.

    python tools/normals_bench.py [--height 1200] [--width 1600] [--reps 30] [--views 49] [--sources 10] [--scene-reps 2]

* `ops.estimate_normals` on a seeded 1600x1200 depth map (tests/normals_cases.noisy: two tilted planes with Gaussian
  depth noise), at the default radius 3 and at the largest radius 7.  CUDA events around each call, median of `--reps`
  after warm-up; bytes are the kernel's compulsory traffic, 4 read + 12 written per pixel.
* `ops.fuse_points` plain against oriented on the same size (half the pixels survive), alternated, median of `--reps`; the
  times include the wrapper's allocations and its one read of the vertex count.
* `reconstruct` fusion seconds without and with --normals on tools/reconstruct_bench.py's seeded scene (49 views at
  1600x1200, 10 sources in pair.txt, geo mask 3, photo 0.8): one depth run, then --output-type fusion alternated plain /
  --normals `--scene-reps` times each; host wall clock around work that ends in a device synchronisation, and the size of
  each fused.ply.
The GPU's name, power limit and maximum SM clock are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops, reconstruct  # noqa: E402
from tests import normals_cases, scene_cases  # noqa: E402

WEIGHTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "weights_000007.pt")


def timed(fn, reps, warmup=5):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--sources", type=int, default=10)
    ap.add_argument("--scene-reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("normals_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    dev = "cuda:0"
    H, W = args.height, args.width
    case = normals_cases.noisy(H, W)
    depth = torch.from_numpy(case["depth"]).to(dev)
    result = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi, "size": [H, W]}
    for r in (3, 7):
        ms = timed(lambda: ops.estimate_normals(depth, case["K"], radius=r), args.reps)
        result[f"estimate_normals_r{r}_ms"] = ms
        result[f"estimate_normals_r{r}_gbs"] = H * W * 16 / (ms * 1e-3) / 1e9
    normals = ops.estimate_normals(depth, case["K"])
    result["nonzero_normals"] = float((normals != 0).any(-1).float().mean())

    rng = np.random.default_rng(0)
    mask = torch.from_numpy(rng.random((H, W)) < 0.5).to(dev)
    avg = torch.from_numpy(rng.uniform(400, 900, (H, W))).to(dev)
    img = torch.from_numpy(rng.random((H, W, 3), dtype=np.float32)).to(dev)
    cam = ops.compose_fusion_camera(case["K"], np.eye(4, dtype=np.float32))
    plain, oriented = [], []
    for _ in range(3):  # alternate the two forms
        plain.append(timed(lambda: ops.fuse_points(mask, avg, img, cam), args.reps // 3 or 1))
        oriented.append(timed(lambda: ops.fuse_points(mask, avg, img, cam, normals), args.reps // 3 or 1))
    result["fuse_points_plain_ms"] = float(np.median(plain))
    result["fuse_points_oriented_ms"] = float(np.median(oriented))
    result["fuse_points_points"] = int(mask.sum())

    with tempfile.TemporaryDirectory() as tmp:
        scene, out = os.path.join(tmp, "scene"), os.path.join(tmp, "out")
        scene_cases.write_scene(scene, args.views, H, W, args.sources)
        common = ["--input-folder", scene, "--output-folder", out, "--checkpoint-path", WEIGHTS, "--num-views", "5",
                  "--geo-mask-thres", "3", "--photo-thres", "0.8"]
        depth_stats = reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-type", "depth"]), log=lambda *a: None)
        runs = {"plain": [], "normals": []}
        sizes = {}
        for _ in range(args.scene_reps):
            for name, extra in (("plain", []), ("normals", ["--normals"])):
                stats = reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-type", "fusion"] + extra), log=lambda *a: None)
                runs[name].append(stats["fusion_seconds"])
                sizes[name] = os.path.getsize(os.path.join(out, "fused.ply"))
                result["scene_points"] = stats["points"]
    result["scene"] = {"views": args.views, "height": H, "width": W, "sources_in_pair": args.sources,
                       "depth_seconds": depth_stats["depth_seconds"]}
    result["fusion_seconds"] = runs
    result["fused_ply_bytes"] = sizes
    print(json.dumps(result))


if __name__ == "__main__":
    main()
