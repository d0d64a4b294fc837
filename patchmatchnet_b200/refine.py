"""Refine a triangle mesh's vertices on the GPU by multi-view photo-consistency (ops.refine_mesh; definition in
include/patchmatch_b200.h): windowed ZNCC between each reference view and its pair.txt sources reprojected through the mesh,
gradient steps along the vertex normals and thin-plate smoothing, coarse to fine.

    python -m patchmatchnet_b200.refine --ply outputs/scan1/mesh_simplified.ply --input-folder scene --output mesh_refined.ply

Writes the input's vertex layout (colours kept when present) with the refined positions, and its faces.  Views default to
every reference view of pair.txt with a cams file; each takes its first --neighbours sources among the views used.  Images
are decoded as reconstruct decodes them (texture.load_views)."""
from __future__ import annotations

import argparse
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import data_io, ops
from .texture import load_views


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.refine", description="Refine a triangle mesh by photo-consistency")
    ap.add_argument("--ply", required=True, help="input PLY with a face element")
    ap.add_argument("--input-folder", required=True, help="scene folder with cams/, images/ and pair.txt")
    ap.add_argument("--output", required=True, help="output PLY")
    ap.add_argument("--views", nargs="+", type=int, default=None, help="views to use (default: every reference view of pair.txt)")
    ap.add_argument("--neighbours", type=int, default=ops.REFINE_NEIGHBOURS, help="source views per reference view, from pair.txt")
    ap.add_argument("--iterations", type=int, default=ops.REFINE_ITERATIONS, help="iterations per level")
    ap.add_argument("--levels", type=int, default=ops.REFINE_LEVELS, help="image levels, coarse to fine (1..16)")
    ap.add_argument("--smoothness", type=float, default=ops.REFINE_SMOOTHNESS, help="thin-plate smoothing weight lambda")
    ap.add_argument("--image-max-dim", type=int, default=-1, help="max image dimension, as reconstruct's option")
    return ap


def pairs_among(entries, views: Sequence[int], neighbours: int) -> List[Tuple[int, int]]:
    """(i, j) indices into `views`: each view's first `neighbours` sources among `views`, from pair.txt entries
    [(reference, [sources])] (data_io.read_pair_file)."""
    index = {v: k for k, v in enumerate(views)}
    srcs = {ref: s for ref, s in entries}
    out = []
    for v in views:
        mine = [index[s] for s in srcs.get(v, []) if s in index and s != v][:neighbours]
        out += [(index[v], j) for j in mine]
    return out


def scene_pairs(pair_file: str, views: Sequence[int], neighbours: int) -> List[Tuple[int, int]]:
    """pairs_among of a pair.txt file."""
    return pairs_among(data_io.read_pair_file(pair_file), views, neighbours)


def check_args(args: argparse.Namespace) -> List[int]:
    """ValueError for inconsistent arguments, before anything is read or written; -> the views."""
    if not os.path.isfile(args.ply):
        raise ValueError(f"--ply: no such file {args.ply!r}")
    if not os.path.isdir(args.input_folder):
        raise ValueError(f"--input-folder: no such folder {args.input_folder!r}")
    pair_file = os.path.join(args.input_folder, "pair.txt")
    if not os.path.isfile(pair_file):
        raise ValueError(f"--input-folder {args.input_folder!r} has no pair.txt")
    if args.neighbours < 1:
        raise ValueError(f"--neighbours must be >= 1, got {args.neighbours}")
    if args.iterations < 0:
        raise ValueError(f"--iterations must be >= 0, got {args.iterations}")
    if not 1 <= args.levels <= 16:
        raise ValueError(f"--levels must be 1..16, got {args.levels}")
    if not (0.0 <= args.smoothness < float("inf")):
        raise ValueError(f"--smoothness must be finite and >= 0, got {args.smoothness}")
    views = args.views if args.views is not None else [ref for ref, _ in data_io.read_pair_file(pair_file)]
    if not views:
        raise ValueError(f"{pair_file!r} lists no reference views")
    for v in views:
        for path in (os.path.join(args.input_folder, "cams", "{:0>8}_cam.txt".format(v)),
                     os.path.join(args.input_folder, "images", "{:0>8}.jpg".format(v))):
            if not os.path.isfile(path):
                raise ValueError(f"view {v}: no such file {path!r}")
    if not scene_pairs(pair_file, views, args.neighbours):
        raise ValueError(f"no view among {list(views)} has a pair.txt source among them: without a pair there is no photometric "
                         "term, only smoothing")
    out_dir = os.path.dirname(os.path.abspath(args.output))
    if not os.path.isdir(out_dir):
        raise ValueError(f"--output: the folder {out_dir!r} does not exist")
    return list(views)


def refine_and_save(xyz: torch.Tensor, rgb: Optional[torch.Tensor], faces: torch.Tensor, images, Ks, Es, pairs, path: str,
                    **kw) -> Tuple[torch.Tensor, dict]:
    """ops.refine_mesh, then data_io.save_ply with the input's colours -> (refined xyz, stats)."""
    out, stats = ops.refine_mesh(xyz, faces, images, Ks, Es, pairs, **kw)
    body = out.contiguous().view(torch.uint8)
    if rgb is not None:
        body = torch.cat([body, rgb.to(torch.uint8)], 1)
    data_io.save_ply(path, body, faces)
    return out, stats


def main(argv: Optional[Sequence[str]] = None, device: str = "cuda:0") -> dict:
    args = build_parser().parse_args(argv)
    views = check_args(args)
    xyz, rgb, _, faces = data_io.read_ply(args.ply)
    if faces is None:
        raise ValueError(f"{args.ply} has no faces: refine needs a triangle mesh")
    if not torch.cuda.is_available():
        raise RuntimeError("refine needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    pairs = scene_pairs(os.path.join(args.input_folder, "pair.txt"), views, args.neighbours)
    images, Ks, Es = load_views(args.input_folder, views, args.image_max_dim, dev)
    _, stats = refine_and_save(torch.from_numpy(np.ascontiguousarray(xyz)).to(dev), None if rgb is None else torch.from_numpy(rgb).to(dev),
                               torch.from_numpy(faces).to(dev), images, Ks, Es, pairs, args.output, iterations=args.iterations,
                               levels=args.levels, smoothness=args.smoothness)
    e = stats["energy"]
    print(f"{args.ply}: {len(faces)} faces, {len(views)} views, {len(pairs)} pairs -> {args.output}: energy "
          f"{e[0] if e else 0:.1f} -> {e[-1] if e else 0:.1f} in {stats['seconds']:.2f} s")
    return stats


if __name__ == "__main__":
    main()
