"""End-to-end scene reconstruction (patchmatchnet_b200.reconstruct) on a seeded synthetic DTU-sized scene.

    python tools/reconstruct_bench.py [--views 49] [--height 1200] [--width 1600] [--sources 10] [--num-views 5] [--reps 2]

The scene (tests/scene_cases.write_scene: a textured plane seen by a row of cameras, JPEG images, cams with a depth range,
`--sources` sources per view in pair.txt) is written into a temporary folder, and the command's library call runs on it with
--output-type both and the DTU thresholds of eval.sh (geo mask 3, photo 0.8), `--reps` times, each run building its engines
anew.  Times are host wall clock around work that ends in a device synchronisation: depth stage (decode + upload, engine
set-up and graph capture, network, map files), fusion stage (filter, masks, fusion, fused.ply), end to end.  Host baseline:
the CPU oracle's filter and fusion (oracle/geo_oracle.py: fuse_reference_view + fuse_points) for ONE reference view with all
its sources, timed once and not extrapolated.  The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import geo_oracle as go  # noqa: E402
from patchmatchnet_b200 import data_io, reconstruct  # noqa: E402
from tests import scene_cases  # noqa: E402

WEIGHTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "weights_000007.pt")


def host_baseline(scene: str, out: str, ref: int, srcs, fmt: str) -> float:
    """Seconds of the oracle's filter + fusion for one reference view, maps and cams read beforehand (not timed)."""
    def cam(v):
        img, oh, ow = data_io.read_image(os.path.join(scene, "images", f"{v:08d}.jpg"))
        k, e, _ = data_io.read_cam_file(os.path.join(scene, "cams", f"{v:08d}_cam.txt"))
        return img, data_io.scale_intrinsics(k, img.shape[:2], oh, ow), e

    read = lambda kind, v: data_io.read_map(os.path.join(out, kind, f"{v:08d}{fmt}"))[..., 0]
    img, K, E = cam(ref)
    cams = [cam(s) for s in srcs]
    ref_depth, conf, src_depths = read("depth_est", ref), read("confidence", ref), [read("depth_est", s) for s in srcs]
    t0 = time.perf_counter()
    with np.errstate(divide="ignore", invalid="ignore"):
        _, _, final, avg = go.fuse_reference_view(ref_depth, K, E, src_depths, [c[1] for c in cams], [c[2] for c in cams], conf,
                                                  1.0, 0.01, 0.8, 3)
        go.fuse_points(final, avg, img, K, E)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--height", type=int, default=1200)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--sources", type=int, default=10)
    ap.add_argument("--num-views", type=int, default=5)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--file-format", default=".pfm", choices=[".pfm", ".bin"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reconstruct_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    H, W, V = args.height, args.width, args.views
    with tempfile.TemporaryDirectory() as tmp:
        scene = os.path.join(tmp, "scene")
        t0 = time.perf_counter()
        sc = scene_cases.write_scene(scene, V, H, W, args.sources)
        t_write = time.perf_counter() - t0
        runs = []
        for r in range(args.reps):
            out = os.path.join(tmp, f"out{r}")
            cli = ["--input-folder", scene, "--output-folder", out, "--checkpoint-path", WEIGHTS, "--num-views",
                   str(args.num_views), "--file-format", args.file_format, "--geo-mask-thres", "3", "--photo-thres", "0.8"]
            torch.cuda.reset_peak_memory_stats()
            stats = reconstruct.reconstruct(reconstruct.parse_args(cli), log=lambda *a: None)
            stats["peak_allocated_gb"] = torch.cuda.max_memory_allocated() / 1e9
            runs.append(stats)
        same = open(os.path.join(tmp, "out0", "fused.ply"), "rb").read() == open(os.path.join(out, "fused.ply"), "rb").read()
        ref, srcs = sc["pairs"][0]
        t_host = host_baseline(scene, out, ref, srcs, args.file_format)
    last = runs[-1]
    print(json.dumps({
        "device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi, "cpu_cores": os.cpu_count(),
        "scene": {"views": V, "height": H, "width": W, "sources_in_pair": args.sources, "num_views": args.num_views,
                  "file_format": args.file_format, "write_seconds": t_write},
        "depth_seconds": last["depth_seconds"], "fusion_seconds": last["fusion_seconds"], "end_to_end_seconds": last["total_seconds"],
        "engine_setup_seconds": last["engine_setup_seconds"], "points": last["points"], "runs": runs,
        "fused_ply_identical_across_runs": same,
        "banks_gb": {"images": V * 3 * H * W * 4 / 1e9, "maps": V * 2 * H * W * 4 / 1e9},
        "host_oracle_one_view_seconds": t_host,
        "host_oracle_note": "oracle filter + fusion of one reference view with its %d sources; not extrapolated" % len(srcs),
    }))


if __name__ == "__main__":
    main()
