"""The TSDF mesher (pmb200_tsdf_alloc / _integrate / _mesh_count / _mesh_write) on the GPU.

    python tools/mesh_bench.py [--height 1200] [--width 1600] [--views 49] [--sources 10] [--reps 10] [--scene-reps 2]

On tools/reconstruct_bench.py's seeded scene (49 views at 1600x1200, 10 sources in pair.txt, geo mask 3, photo 0.8): one
depth run, then `reconstruct --output-type fusion` alternated without and with --mesh, `--scene-reps` times each (host wall
clock around work that ends in a device synchronisation).  The mesher's inputs of the last --mesh run (the kept
final-masked depths, the image bank, the cameras, the fused points and the default voxel size) are captured and each phase
is timed on them with CUDA events, median of `--reps` after warm-up: allocation (including its one host synchronisation),
integration, and extraction (count, scans, the read of the counts, write).  Also: blocks, voxels, vertices, faces, and the
peak of device memory allocated by one ops.tsdf_mesh call above what was allocated before it.
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
from tests import scene_cases  # noqa: E402

WEIGHTS = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "weights_000007.pt")


def timed(fn, reps, warmup=2):
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
    ap.add_argument("--views", type=int, default=49)
    ap.add_argument("--sources", type=int, default=10)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--scene-reps", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    H, W = args.height, args.width
    result = {"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi}
    captured = {}
    original = reconstruct.mesh_scan

    def capture(rargs, bank, refs, depths, bodies, path):
        out = original(rargs, bank, refs, depths, bodies, path)
        Ks = [bank.intrinsics[r] for r in refs]
        captured.update(depths=list(depths), images=[bank.images[r] for r in refs], Ks=Ks, Es=[bank.extrinsics[r] for r in refs],
                        seeds=torch.cat([b[:, :12] for b in bodies]).contiguous().view(torch.float32).view(-1, 3),
                        s=reconstruct.default_mesh_voxel_size(depths, Ks))
        return out

    reconstruct.mesh_scan = capture
    with tempfile.TemporaryDirectory() as tmp:
        scene, out = os.path.join(tmp, "scene"), os.path.join(tmp, "out")
        scene_cases.write_scene(scene, args.views, H, W, args.sources)
        common = ["--input-folder", scene, "--output-folder", out, "--checkpoint-path", WEIGHTS, "--num-views", "5",
                  "--geo-mask-thres", "3", "--photo-thres", "0.8"]
        depth_stats = reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-type", "depth"]), log=lambda *a: None)
        runs = {"plain": [], "mesh": []}
        mesh_stats = {}
        for _ in range(args.scene_reps):
            for name, extra in (("plain", []), ("mesh", ["--mesh"])):
                stats = reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-type", "fusion"] + extra), log=lambda *a: None)
                runs[name].append(stats["fusion_seconds"])
                if name == "mesh":
                    mesh_stats = {k: stats[k] for k in ("mesh_vertices", "mesh_faces", "mesh_seconds")}
                    result["mesh_ply_bytes"] = os.path.getsize(os.path.join(out, "mesh.ply"))
                result["scene_points"] = stats["points"]
        reconstruct.mesh_scan = original

        c = captured
        s = c["s"]
        keys = ops.tsdf_allocate(c["seeds"], s, 3)
        vol = ops.tsdf_integrate(keys, c["depths"], c["images"], c["Ks"], c["Es"], s, 3)
        verts, faces = ops.tsdf_extract(keys, *vol, s, 1)
        result["voxel_size"] = s
        result["seed_points"] = int(c["seeds"].shape[0])
        result["blocks"] = int(keys.shape[0])
        result["voxels"] = int(keys.shape[0]) * 512
        result["observed_voxels"] = int((vol[1] > 0).sum())
        result["vertices"], result["faces"] = int(verts.shape[0]), int(faces.shape[0])
        result["allocation_ms"] = timed(lambda: ops.tsdf_allocate(c["seeds"], s, 3), args.reps)
        result["integration_ms"] = timed(lambda: ops.tsdf_integrate(keys, c["depths"], c["images"], c["Ks"], c["Es"], s, 3), args.reps)
        result["extraction_ms"] = timed(lambda: ops.tsdf_extract(keys, *vol, s, 1), args.reps)
        del vol, verts, faces, keys
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ops.tsdf_mesh(c["seeds"], c["depths"], c["images"], c["Ks"], c["Es"], s)
        torch.cuda.synchronize()
        result["tsdf_mesh_peak_bytes_above_inputs"] = torch.cuda.max_memory_allocated() - before
        result["kept_depth_bytes"] = sum(d.numel() * 4 for d in c["depths"])
    result["scene"] = {"views": args.views, "height": H, "width": W, "sources_in_pair": args.sources,
                       "depth_seconds": depth_stats["depth_seconds"]}
    result["fusion_seconds"] = runs
    result["reconstruct_mesh_stats"] = mesh_stats
    print(json.dumps(result))


if __name__ == "__main__":
    main()
