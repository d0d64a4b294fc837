"""Mesh an oriented point cloud on the GPU by Poisson surface reconstruction: a multigrid solve on a dense grid and marching
cubes trimmed to a band around the points (ops.poisson_mesh; definition in include/patchmatch_b200.h).

    python -m patchmatchnet_b200.poisson --ply outputs/scan1/fused.ply --output mesh_poisson.ply --depth 9

Reads any PLY with normals that data_io.read_ply reads (this project's oriented fused.ply from reconstruct --normals,
COLMAP's fused.ply, a scan with normals), uploads it once, and writes the mesh with data_io.save_ply: x, y, z, and red,
green, blue (the nearest input point's) when the input has colours."""
from __future__ import annotations

import argparse
import time
from typing import Optional, Sequence

import torch

from . import data_io, ops


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description="Mesh an oriented point cloud on the GPU (Poisson surface reconstruction)")
    ap.add_argument("--ply", required=True, help="input PLY with nx, ny, nz per vertex")
    ap.add_argument("--output", required=True, help="output PLY")
    ap.add_argument("--depth", type=int, default=9, help="grid of 2^depth cells per axis, 5..10 (default 9)")
    ap.add_argument("--scale", type=float, default=1.1, help="grid extent over the box's largest extent, >= 1 (default 1.1)")
    ap.add_argument("--band", type=int, default=2, help="mesh only within this many voxels of a point, 1..4 (default 2)")
    ap.add_argument("--bbox-quantile", type=float, default=0.0,
                    help="box from this quantile to 1 minus it per axis, dropping outliers (default 0: the exact box)")
    ap.add_argument("--tol", type=float, default=1e-5, help="relative residual at which the multigrid stops (default 1e-5)")
    ap.add_argument("--max-cycles", type=int, default=50, help="at most this many multigrid cycles (default 50)")
    return ap


def mesh_cloud(xyz: torch.Tensor, normals: torch.Tensor, rgb: Optional[torch.Tensor], output: str, **kw) -> dict:
    """ops.poisson_mesh on device tensors and data_io.save_ply of the result -> the stats plus vertices, faces and seconds."""
    dev = xyz.device
    torch.cuda.synchronize(dev)
    t0 = time.perf_counter()
    verts, faces, stats = ops.poisson_mesh(xyz, normals, rgb, **kw)
    torch.cuda.synchronize(dev)
    stats = dict(stats, vertices=int(verts.shape[0]), faces=int(faces.shape[0]), seconds=time.perf_counter() - t0)
    data_io.save_ply(output, verts, faces)
    return stats


def main(argv: Optional[Sequence[str]] = None, device: str = "cuda:0") -> dict:
    args = build_parser().parse_args(argv)
    kw = dict(depth=args.depth, scale=args.scale, band=args.band, bbox_quantile=args.bbox_quantile, tol=args.tol,
              max_cycles=args.max_cycles)
    ops._poisson_args(**kw, what="poisson")
    xyz, rgb, normals, _ = data_io.read_ply(args.ply)
    if normals is None:
        raise ValueError(f"{args.ply} has no normals (nx, ny, nz): Poisson reconstruction needs an oriented cloud")
    if not torch.cuda.is_available():
        raise RuntimeError("poisson needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    stats = mesh_cloud(torch.as_tensor(xyz).to(dev), torch.as_tensor(normals).to(dev),
                       None if rgb is None else torch.as_tensor(rgb).to(dev), args.output, **kw)
    print(f"{args.ply}: {stats['kept']} of {stats['points']} points, N = {stats['N']}, {stats['cycles']} cycles to residual "
          f"{stats['residual']:.2e} -> {args.output}: {stats['vertices']} vertices, {stats['faces']} faces, {stats['seconds']:.3f} s")
    return stats


if __name__ == "__main__":
    main()
