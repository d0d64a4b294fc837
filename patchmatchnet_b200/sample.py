"""Sample a triangle mesh's surface on the GPU: a regular barycentric lattice on every face, at most --spacing apart along
its edges, so that every point of the surface lies within --spacing of a sample (ops.sample_mesh; definition in
include/patchmatch_b200.h).

    python -m patchmatchnet_b200.sample --ply outputs/scan1/mesh_simplified.ply --spacing 0.2 --output samples.ply

Reads a PLY mesh through data_io.read_ply or this project's textured OBJ through data_io.read_obj, and writes the samples
with data_io.save_ply as float x, y, z, with red, green, blue when the input has vertex colours.  The output feeds the T&T
toolbox, ETH3D's evaluation program, any viewer, or `render --ply samples.ply`.  The evaluations sample meshes themselves
with --surface (mesh_samples below)."""
from __future__ import annotations

import argparse
import math
import time
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import data_io, ops


def read_mesh(path: str) -> Tuple[np.ndarray, Optional[np.ndarray], np.ndarray]:
    """A triangle mesh from a .ply (data_io.read_ply) or this project's .obj (data_io.read_obj; it has no vertex colours)
    -> (xyz float32 [nv,3], rgb uint8 [nv,3] or None, faces int32 [nf,3]).  ValueError naming the file when it has no faces."""
    if path.lower().endswith(".obj"):
        xyz, faces = data_io.read_obj(path)[:2]
        rgb = None
    else:
        xyz, rgb, _, faces = data_io.read_ply(path)
    if faces is None or len(faces) == 0:
        raise ValueError(f"{path} has no faces: surface sampling needs a triangle mesh")
    return xyz, rgb, faces


def check_spacing(spacing, what: str) -> None:
    if spacing is not None and not (math.isfinite(spacing) and spacing > 0):
        raise ValueError(f"{what} must be finite and > 0, got {spacing}")


def mesh_samples(path: str, spacing: float, device) -> Tuple[torch.Tensor, Dict[str, object]]:
    """The surface samples of the mesh at `path` on `device` (float64 [n,3]) and the record the evaluations add to their
    JSON: {"spacing", "n_faces", "n_samples"}.  ValueError naming the file when it has no faces."""
    xyz, _, faces = read_mesh(path)
    dev = torch.device(device)
    pts, _ = ops.sample_mesh(torch.as_tensor(xyz).contiguous().to(dev), torch.as_tensor(faces).contiguous().to(dev), spacing)
    return pts, {"spacing": float(spacing), "n_faces": int(len(faces)), "n_samples": int(pts.shape[0])}


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.sample",
                                 description="Sample a triangle mesh's surface on the GPU (regular barycentric lattice per face)")
    ap.add_argument("--ply", required=True, help="input mesh: a PLY with a face element, or this project's textured OBJ")
    ap.add_argument("--spacing", type=float, required=True, help="largest lattice edge, in the mesh's units")
    ap.add_argument("--output", required=True, help="output PLY of the samples")
    return ap


def main(argv: Optional[Sequence[str]] = None, device: str = "cuda:0") -> dict:
    args = build_parser().parse_args(argv)
    check_spacing(args.spacing, "--spacing")
    xyz, rgb, faces = read_mesh(args.ply)
    if not torch.cuda.is_available():
        raise RuntimeError("sample needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    xyz_d = torch.as_tensor(xyz).contiguous().to(dev)
    rgb_d = None if rgb is None else torch.as_tensor(rgb).contiguous().to(dev)
    faces_d = torch.as_tensor(faces).contiguous().to(dev)
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    pts, col = ops.sample_mesh(xyz_d, faces_d, args.spacing, rgb_d)
    torch.cuda.synchronize(dev)
    seconds = time.perf_counter() - t0
    body = pts.float().view(torch.uint8).view(-1, 12)
    data_io.save_ply(args.output, body if col is None else torch.cat([body, col], 1))
    stats = {"vertices": len(xyz), "faces": len(faces), "samples": int(pts.shape[0]), "spacing": args.spacing, "seconds": seconds}
    print(f"{args.ply}: {stats['vertices']} vertices, {stats['faces']} faces -> {args.output}: {stats['samples']} samples at "
          f"spacing {args.spacing:g} in {seconds:.3f} s")
    return stats


if __name__ == "__main__":
    main()
