"""Seconds of mesh texturing on the scene-size rows of tests/test_gpu_mesh_at_scene_sizes.py (dtu: 49 views at 1600 x 1200,
tnt: 100 at 1920 x 1080, eth3d: 24 at 2688 x 1792 in both orientations), each row's TSDF mesh simplified to 10 % and 1 %
and textured from the row's own views.  Stages: the selection call (pmb200_texture_mesh: visibility of every view, labels
and charts; also given per view), the whole ops.texture_mesh (selection, host packing, page fill and coordinates), the
host packing alone, the download of coordinates and pages, and the PNG encoding of the pages (data_io.save_obj).  Prints
one JSON line per case with the atlas fill and page count, and the card's name and power limit read in the same run.

    python tools/texture_bench.py [--rows dtu tnt eth3d] [--out results/texture_bench.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import data_io, ops  # noqa: E402
from tests.test_gpu_mesh_at_scene_sizes import build_scene  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", nargs="+", default=["dtu", "tnt", "eth3d"])
    ap.add_argument("--shares", nargs="+", type=float, default=[0.1, 0.01])
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
        for share in args.shares:
            body, sf, _ = ops.simplify_mesh(xyz, rgb, faces, int(faces.shape[0] * share))
            sx, sc = body[:, :12].contiguous().view(torch.float32), body[:, 12:].contiguous()
            ops.texture_mesh(sx, sc, sf, images, Ks, Es)  # warm-up: module load and the caching allocator
            (_, table, _, _), t_sel = timed(lambda: ops.texture_labels(sx, sf, images, Ks, Es))
            tab = table.cpu().numpy()
            (uv, page, pages, st), t_all = timed(lambda: ops.texture_mesh(sx, sc, sf, images, Ks, Es))
            n_cells = st["untextured_faces"]
            t0 = time.perf_counter()
            ops.texture_pack(tab[:, 4:6], n_cells)
            t_pack = time.perf_counter() - t0
            (_, t_down) = timed(lambda: (uv.cpu(), page.cpu(), pages.cpu(), sx.cpu(), sf.cpu()))
            with tempfile.TemporaryDirectory() as d:
                t0 = time.perf_counter()
                data_io.save_obj(os.path.join(d, "m"), sx, sf, uv, page, pages)
                t_write = time.perf_counter() - t0
            rec = {"row": name, "share": share, "faces": int(sf.shape[0]), "views": len(images), "select_seconds": round(t_sel, 4),
                   "select_seconds_per_view": round(t_sel / len(images), 5), "texture_mesh_seconds": round(t_all, 4),
                   "pack_seconds": round(t_pack, 4), "fill_and_uv_seconds": round(max(t_all - t_sel - t_pack, 0.0), 4),
                   "download_seconds": round(t_down, 4), "obj_png_write_seconds": round(t_write, 4), "charts": st["charts"],
                   "pages": st["pages"], "page_side": st["page_side"], "atlas_fill": round(st["atlas_fill"], 4),
                   "untextured": st["untextured_faces"], "entries": st["entries"], "gpu": gpu}
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
