"""Seconds per ops.simplify_mesh call, round count and milliseconds per round, on a synthetic TSDF sphere mesh and on the
scene-size rows of tests/test_gpu_mesh_at_scene_sizes.py, simplified to 10 % and 1 % of their faces.  Reads the card's
name and power limit in the same run.

    python tools/simplify_bench.py [--rows eth3d big] [--repeats 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from patchmatchnet_b200 import ops  # noqa: E402
from tests import mesh_cases as mc  # noqa: E402
from tests.test_gpu_mesh_at_scene_sizes import build_scene  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def sphere_mesh():
    sc = mc.sphere_scene(H=480, W=640, f=680.0)
    d = [torch.from_numpy(x).to(DEV) for x in sc["depths"]]
    i = [torch.from_numpy(x).to(DEV) for x in sc["images"]]
    return ops.tsdf_mesh(torch.from_numpy(sc["seeds"]).to(DEV), d, i, sc["Ks"], sc["Es"], 0.0125)


def row_mesh(name):
    row = build_scene(name, DEV)
    return ops.tsdf_mesh(row["seeds"], row["depths"], row["images"], row["Ks"], row["Es"], row["s"])


def measure(name, verts, faces, repeats):
    xyz = verts[:, :12].contiguous().view(torch.float32)
    rgb = verts[:, 12:].contiguous()
    out = []
    for share in (0.1, 0.01):
        target = int(faces.shape[0] * share)
        ops.simplify_mesh(xyz, rgb, faces, target)  # warm-up: module load, CUB tuning, allocator
        torch.cuda.synchronize()
        times = []
        for _ in range(repeats):
            t0 = time.perf_counter()
            body, f, rounds = ops.simplify_mesh(xyz, rgb, faces, target)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        s = min(times)
        r = {"mesh": name, "vertices": int(verts.shape[0]), "faces": int(faces.shape[0]), "target": target,
             "faces_out": int(f.shape[0]), "rounds": rounds, "seconds": round(s, 4), "ms_per_round": round(1e3 * s / max(rounds, 1), 3),
             "seconds_all": [round(t, 4) for t in times]}
        print(json.dumps(r), flush=True)
        out.append(r)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", nargs="*", default=["dtu", "tnt", "eth3d", "big"])
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    verts, faces = sphere_mesh()
    measure("sphere", verts, faces, args.repeats)
    del verts, faces
    for name in args.rows:
        verts, faces = row_mesh(name)
        measure(name, verts, faces, args.repeats)
        del verts, faces
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
