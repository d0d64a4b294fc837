"""Per-stage times of the Poisson mesher (ops.poisson_mesh) on seeded synthetic clouds: points on a unit sphere with outward
normals and colours, at depth 8, 9 and 10 with 1M, 5M and 20M points.

    python tools/poisson_bench.py [--out poisson_bench.json] [--rows DEPTH:POINTS,...]

Stages are timed with CUDA events around the C ABI calls: setup, density, rhs, solve (the multigrid and the iso-value),
band, extraction (pmb200_tsdf_alloc, _mesh_count, _mesh_write) and colours.  The multigrid's rate is a model figure: 12 bytes
per node per stencil sweep (read chi and b, write chi) over the 6 stencil sweeps of each level in a V(2,2) cycle plus the
final residual, divided by the solve time, next to the H100 SXM's 3.35 TB/s.  The card's name and power limit are read in the
same run."""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import _native, ops  # noqa: E402


def cloud(n: int, seed: int = 0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = torch.randn((n, 3), generator=g, device="cuda", dtype=torch.float64)
    d /= d.norm(dim=1, keepdim=True)
    rgb = ((d * 0.5 + 0.5) * 255).round().to(torch.uint8)
    return d.float().contiguous(), d.float().contiguous(), rgb.contiguous()


def run(depth: int, n: int) -> dict:
    xyz, nrm, rgb = cloud(n)
    lib = _native.lib()
    need = ops.poisson_mesh_bytes(depth, n)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    g, r = _native.PoissonGrid(), _native.PoissonResult()
    st = torch.cuda.current_stream().cuda_stream
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
    torch.cuda.synchronize()
    ev[0].record()
    _native.check(lib.pmb200_poisson_setup(xyz.data_ptr(), nrm.data_ptr(), rgb.data_ptr(), n, depth, 1.1, 0.0, ctypes.byref(g),
                                           ws.data_ptr(), need, st), "setup")
    ev[1].record()
    _native.check(lib.pmb200_poisson_density(ctypes.byref(g), None, None, ws.data_ptr(), need, st), "density")
    ev[2].record()
    _native.check(lib.pmb200_poisson_rhs(ctypes.byref(g), None, ws.data_ptr(), need, st), "rhs")
    ev[3].record()
    _native.check(lib.pmb200_poisson_solve(ctypes.byref(g), 1e-5, 50, ctypes.byref(r), None, ws.data_ptr(), need, st), "solve")
    ev[4].record()
    off, m = int(g.points_offset), int(g.n_inside)
    keys = ops.tsdf_allocate(ws[off: off + 12 * m].view(torch.float32).view(m, 3), g.h, 2)
    nb = keys.shape[0]
    tsdf = torch.empty(nb * 512, dtype=torch.float32, device="cuda")
    weight = torch.empty_like(tsdf)
    ev[5].record()
    _native.check(lib.pmb200_poisson_band(ctypes.byref(g), r.iso, keys.data_ptr(), nb, tsdf.data_ptr(), weight.data_ptr(), ws.data_ptr(),
                                          need, st), "band")
    colour = torch.zeros((nb * 512, 4), dtype=torch.uint8, device="cuda")
    verts, faces = ops.tsdf_extract(keys, tsdf, weight, colour, g.h, 1)
    ev[6].record()
    _native.check(lib.pmb200_poisson_colours(ctypes.byref(g), verts.data_ptr(), verts.shape[0], ws.data_ptr(), need, st), "colours")
    ev[7].record()
    torch.cuda.synchronize()
    t = [ev[i].elapsed_time(ev[i + 1]) / 1e3 for i in range(7)]
    N = 2 ** depth
    nodes = sum((N // 2 ** k + 1) ** 3 for k in range(depth))
    model_bytes = 12 * (nodes * 6 * r.cycles + (N + 1) ** 3 * 2)
    return {"depth": depth, "points": n, "cycles": r.cycles, "residual": r.residual, "converged": bool(r.converged), "iso": r.iso,
            "blocks": nb, "vertices": int(verts.shape[0]), "faces": int(faces.shape[0]), "workspace_gib": need / 2 ** 30,
            "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
            "seconds": dict(zip(("setup", "density", "rhs", "solve", "alloc", "band_extract", "colours"), t)),
            "multigrid_model_tb_s": model_bytes / t[3] / 1e12, "hbm_tb_s": 3.35}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--rows", default="8:1000000,9:5000000,10:20000000")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    run(7, 100000)  # warm-up: module load and the CUB passes
    rows = []
    for item in args.rows.split(","):
        d, n = (int(v) for v in item.split(":"))
        torch.cuda.reset_peak_memory_stats()
        rows.append(run(d, n))
        print(json.dumps(rows[-1]), flush=True)
        torch.cuda.empty_cache()
    res = {"card": card, "rows": rows}
    print(json.dumps({"card": card}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
