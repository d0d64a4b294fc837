"""Seconds of photometric mesh refinement on the scene-size rows of tests/test_gpu_mesh_at_scene_sizes.py (dtu: 49 views at
1600 x 1200, tnt: 100 at 1920 x 1080, eth3d: 24 at 2688 x 1792 in both orientations), each row's TSDF mesh simplified to
10 % and 1 % and refined against the row's own views, each view paired with its 4 neighbours in the row's order.  Per case:
seconds per iteration and per stage (z-buffers, pixel passes, update, from CUDA events inside the call), and pixel-pairs per
second (reference pixels over all pairs, per second of the whole iteration).  Prints one JSON line per case with the card's
name and power limit read in the same run.

    python tools/refine_bench.py [--rows dtu tnt eth3d] [--iterations 3] [--out results/refine_bench.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops  # noqa: E402
from tests.test_gpu_mesh_at_scene_sizes import build_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def neighbour_pairs(V, k=4):
    offs = [1, -1, 2, -2, 3, -3][:k]
    return [(i, (i + d) % V) for i in range(V) for d in offs if (i + d) % V != i]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", nargs="+", default=["dtu", "tnt", "eth3d"])
    ap.add_argument("--shares", nargs="+", type=float, default=[0.1, 0.01])
    ap.add_argument("--iterations", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gpu = card()
    lines = []
    for name in args.rows:
        row = build_scene(name, "cuda:0")
        verts, faces = ops.tsdf_mesh(row["seeds"], row["depths"], row["images"], row["Ks"], row["Es"], row["s"])
        xyz, rgb = verts[:, :12].contiguous().view(torch.float32), verts[:, 12:].contiguous()
        images, Ks, Es = row["images"], row["Ks"], row["Es"]
        del row["depths"]
        pairs = neighbour_pairs(len(images), ops.REFINE_NEIGHBOURS)
        for share in args.shares:
            body, sf, _ = ops.simplify_mesh(xyz, rgb, faces, int(faces.shape[0] * share))
            sx = body[:, :12].contiguous().view(torch.float32)
            ops.refine_mesh(sx, sf, images, Ks, Es, pairs, iterations=1)  # warm-up: module load and the caching allocator
            _, st = ops.refine_mesh(sx, sf, images, Ks, Es, pairs, iterations=args.iterations)
            it = st["iterations"]
            per_it = (st["zbuffer_seconds"] + st["pixel_seconds"] + st["update_seconds"]) / it
            rec = {"row": name, "share": share, "faces": int(sf.shape[0]), "vertices": int(sx.shape[0]), "views": len(images),
                   "pairs": len(pairs), "iterations": it, "seconds_per_iteration": round(per_it, 4),
                   "zbuffer_seconds_per_iteration": round(st["zbuffer_seconds"] / it, 4),
                   "pixel_seconds_per_iteration": round(st["pixel_seconds"] / it, 4),
                   "update_seconds_per_iteration": round(st["update_seconds"] / it, 5),
                   "call_seconds": round(st["seconds"], 3), "pixel_pairs_per_iteration": st["pixel_pairs"] // it,
                   "gpixel_pairs_per_second": round(st["pixel_pairs"] / it / per_it / 1e9, 3), "gpu": gpu}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del verts, faces, xyz, rgb, images, row
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.writelines(json.dumps(r) + "\n" for r in lines)


if __name__ == "__main__":
    main()
