"""Texture a triangle mesh from a scene's views on the GPU: per face the view that sees it best (occlusion-aware), charts of
neighbouring faces with one view cut from that view's image and packed into square PNG pages, and a textured OBJ
(ops.texture_mesh; definition in include/patchmatch_b200.h).

    python -m patchmatchnet_b200.texture --ply outputs/scan1/mesh_simplified.ply --input-folder scene --output out/mesh_textured

Writes <output>.obj, <output>.mtl and <output>_NN.png (data_io.save_obj).  Views default to every view with a cams file;
images are decoded with data_io.read_image (scaled by --image-max-dim as reconstruct scales them) and uploaded one at a
time, with intrinsics scaled to the decoded size."""
from __future__ import annotations

import argparse
import glob
import os
import time
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import data_io, ops


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.texture", description="Texture a triangle mesh from a scene's views")
    ap.add_argument("--ply", required=True, help="input PLY with a face element")
    ap.add_argument("--input-folder", required=True, help="scene folder with cams/ and images/")
    ap.add_argument("--views", nargs="+", type=int, default=None, help="texturing views (default: every view with a cams file)")
    ap.add_argument("--image-max-dim", type=int, default=-1, help="max image dimension, as reconstruct's option")
    ap.add_argument("--output", required=True, help="output stem: writes <output>.obj, .mtl and _NN.png")
    return ap


def scene_views(scene: str) -> List[int]:
    return sorted(int(os.path.basename(p)[:8]) for p in glob.glob(os.path.join(scene, "cams", "*_cam.txt")))


def check_args(args: argparse.Namespace) -> List[int]:
    """ValueError for inconsistent arguments, before anything is read or written; -> the views."""
    if not os.path.isfile(args.ply):
        raise ValueError(f"--ply: no such file {args.ply!r}")
    if not os.path.isdir(args.input_folder):
        raise ValueError(f"--input-folder: no such folder {args.input_folder!r}")
    views = args.views if args.views is not None else scene_views(args.input_folder)
    if not views:
        raise ValueError(f"--input-folder {args.input_folder!r} has no cams/*_cam.txt")
    for v in views:
        for path in (os.path.join(args.input_folder, "cams", "{:0>8}_cam.txt".format(v)),
                     os.path.join(args.input_folder, "images", "{:0>8}.jpg".format(v))):
            if not os.path.isfile(path):
                raise ValueError(f"view {v}: no such file {path!r}")
    out_dir = os.path.dirname(os.path.abspath(args.output))
    if not os.path.isdir(out_dir):
        raise ValueError(f"--output: the folder {out_dir!r} does not exist")
    return list(views)


def load_views(scene: str, views: Sequence[int], max_dim: int, device):
    """(images float32 [3,H,W] on the device, K float32 [3,3] scaled to the decoded size, E float32 [4,4]) per view, as
    reconstruct.SceneBank decodes them."""
    images, Ks, Es = [], [], []
    for v in views:
        img, oh, ow = data_io.read_image(os.path.join(scene, "images", "{:0>8}.jpg".format(v)), max_dim)
        k, e, _ = data_io.read_cam_file(os.path.join(scene, "cams", "{:0>8}_cam.txt".format(v)))
        Ks.append(data_io.scale_intrinsics(k, img.shape[:2], oh, ow))
        Es.append(e)
        images.append(torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).to(device))
    return images, Ks, Es


def texture_and_save(xyz: torch.Tensor, rgb: Optional[torch.Tensor], faces: torch.Tensor, images, Ks, Es, stem: str) -> dict:
    """ops.texture_mesh, then data_io.save_obj -> the texture stats with texture_seconds and texture_write_seconds."""
    t0 = time.perf_counter()
    uv, page, pages, stats = ops.texture_mesh(xyz, rgb, faces, images, Ks, Es)
    torch.cuda.synchronize(xyz.device)
    t1 = time.perf_counter()
    data_io.save_obj(stem, xyz, faces, uv, page, pages)
    stats = {"texture_" + k: v for k, v in stats.items()}
    stats.update({"texture_seconds": t1 - t0, "texture_write_seconds": time.perf_counter() - t1})
    return stats


def main(argv: Optional[Sequence[str]] = None, device: str = "cuda:0") -> dict:
    args = build_parser().parse_args(argv)
    views = check_args(args)
    xyz, rgb, _, faces = data_io.read_ply(args.ply)
    if faces is None:
        raise ValueError(f"{args.ply} has no faces: texture needs a triangle mesh")
    if not torch.cuda.is_available():
        raise RuntimeError("texture needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    images, Ks, Es = load_views(args.input_folder, views, args.image_max_dim, dev)
    xyz_d = torch.from_numpy(xyz).to(dev)
    rgb_d = None if rgb is None else torch.from_numpy(rgb).to(dev)
    stats = texture_and_save(xyz_d, rgb_d, torch.from_numpy(faces).to(dev), images, Ks, Es, args.output)
    print(f"{args.ply}: {len(faces)} faces, {len(views)} views -> {args.output}.obj: {stats['texture_charts']} charts on "
          f"{stats['texture_pages']} pages of {stats['texture_page_side']}^2, {stats['texture_untextured_faces']} faces untextured")
    return stats


if __name__ == "__main__":
    main()
