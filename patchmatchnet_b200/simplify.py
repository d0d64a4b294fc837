"""Simplify a triangle mesh on the GPU: quadric edge collapse to a target face count, with optional removal of small
connected pieces (ops.simplify_mesh; definition in include/patchmatch_b200.h).

    python -m patchmatchnet_b200.simplify --ply outputs/scan1/mesh.ply --output mesh_small.ply --target-faces 200000

Reads any triangle PLY data_io.read_ply reads, uploads it once, simplifies and writes the result with data_io.save_ply
(x, y, z, and red, green, blue when the input has colours; normals are dropped, since they would be stale)."""
from __future__ import annotations

import argparse
import time
from typing import Optional, Sequence

import torch

from . import data_io, ops


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="Simplify a triangle mesh on the GPU (quadric edge collapse)")
    ap.add_argument("--ply", required=True, help="input PLY with a face element")
    ap.add_argument("--output", required=True, help="output PLY")
    ap.add_argument("--target-faces", type=int, required=True, help="at most this many faces in the result")
    ap.add_argument("--min-component-faces", type=int, default=0,
                    help="first remove connected pieces with fewer faces than this (default 0: none)")
    return ap


def main(argv: Optional[Sequence[str]] = None, device: str = "cuda:0") -> dict:
    args = build_parser().parse_args(argv)
    if args.target_faces < 0 or args.min_component_faces < 0:
        raise ValueError("--target-faces and --min-component-faces must be >= 0")
    xyz, rgb, _, faces = data_io.read_ply(args.ply)
    if faces is None:
        raise ValueError(f"{args.ply} has no faces: simplify needs a triangle mesh")
    if not torch.cuda.is_available():
        raise RuntimeError("simplify needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    xyz_d = torch.as_tensor(xyz).contiguous().to(dev)
    rgb_d = None if rgb is None else torch.as_tensor(rgb).contiguous().to(dev)
    faces_d = torch.as_tensor(faces).contiguous().to(dev)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    body, out_faces, rounds = ops.simplify_mesh(xyz_d, rgb_d, faces_d, args.target_faces, args.min_component_faces)
    torch.cuda.synchronize(dev)
    seconds = time.perf_counter() - t0
    data_io.save_ply(args.output, body, out_faces)
    stats = {"vertices_in": len(xyz), "faces_in": len(faces), "vertices_out": int(body.shape[0]),
             "faces_out": int(out_faces.shape[0]), "rounds": rounds, "seconds": seconds}
    print(f"{args.ply}: {stats['vertices_in']} vertices, {stats['faces_in']} faces -> {args.output}: {stats['vertices_out']} "
          f"vertices, {stats['faces_out']} faces in {rounds} rounds, {seconds:.3f} s")
    return stats


if __name__ == "__main__":
    main()
