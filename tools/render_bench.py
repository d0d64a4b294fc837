"""Time the renderer (ops.render_points / ops.render_mesh) on the GPU: ms per frame with CUDA events over many frames after a
warm-up, each kernel's mean time from torch.profiler in a separate pass, and the upload of the PLY arrays.  Prints one JSON
object, with the card's name and power limit read in the same run.

    python tools/render_bench.py --frames 50 --json render_bench.json

Workloads (seeded, synthetic): clouds of 10 M and 50 M points at 1920 x 1080 (point size 1 and 3); a TSDF-sized grid mesh
of about 4 M faces at 1920 x 1080 and 3840 x 2160; the same mesh seen from close up, where the visible faces span about
20 pixels, larger than the 16 x 16 box of the one-thread-per-face pass, so the one-CTA-per-face pass carries them."""
from __future__ import annotations

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


def camera(w, h, eye, target, f_scale=0.9):
    z = np.asarray(target, float) - eye
    z /= np.linalg.norm(z)
    y = np.cross(z, [1.0, 0.0, 0.0])
    y /= np.linalg.norm(y)
    x = np.cross(y, z)
    R = np.stack([x, y, z])
    K = np.array([[f_scale * w, 0, (w - 1) / 2], [0, f_scale * w, (h - 1) / 2], [0, 0, 1]])
    return K @ np.hstack([R, (-R @ eye)[:, None]])


def cloud(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    xyz = torch.rand((n, 3), generator=g, device="cuda") * 2 - 1
    xyz[:, 2] = 0.2 * torch.sin(4 * xyz[:, 0]) * torch.cos(3 * xyz[:, 1])  # a wavy sheet
    rgb = torch.randint(0, 256, (n, 3), generator=g, device="cuda", dtype=torch.uint8)
    return xyz.contiguous(), rgb


def grid_mesh(side):
    s = torch.linspace(-1, 1, side, device="cuda")
    Y, X = torch.meshgrid(s, s, indexing="ij")
    Z = 0.2 * torch.sin(4 * X) * torch.cos(3 * Y)
    xyz = torch.stack([X, Y, Z], -1).reshape(-1, 3).contiguous()
    i = torch.arange(side * side, device="cuda", dtype=torch.int32).reshape(side, side)
    a, b, c, d = i[:-1, :-1].reshape(-1), i[:-1, 1:].reshape(-1), i[1:, 1:].reshape(-1), i[1:, :-1].reshape(-1)
    faces = torch.cat([torch.stack([a, b, c], 1), torch.stack([a, c, d], 1)]).contiguous()
    rgb = ((xyz * 0.5 + 0.5) * 255).to(torch.uint8).contiguous()
    return xyz, rgb, faces


def timed(fn, frames, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(frames):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / frames


def kernel_means(fn, frames):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(frames):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("splat_kernel", "resolve_points_kernel", "project_kernel", "raster_small_kernel", "raster_large_kernel",
                  "resolve_mesh_kernel", "Memset"):
            if k in e.key:
                out[k] = out.get(k, 0.0) + e.device_time_total / 1e3 / frames  # ms per frame
    return out


def upload_seconds(n_bytes_arrays):
    host = [np.random.default_rng(0).integers(0, 255, n, dtype=np.uint8) for n in n_bytes_arrays]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dev = [torch.from_numpy(h).to("cuda") for h in host]
    torch.cuda.synchronize()
    del dev
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", type=str, default="")
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    res = {"device": torch.cuda.get_device_name(0), "nvidia_smi": smi, "frames": args.frames, "workloads": []}
    eye = np.array([0.0, -0.4, -2.6])
    for n in (10_000_000, 50_000_000):
        xyz, rgb = cloud(n, 1)
        for ps in (1, 3):
            P = camera(1920, 1080, eye, [0, 0, 0])
            fn = lambda: ops.render_points(xyz, rgb, None, P, 1920, 1080, 1e-3, point_size=ps)
            ms = timed(fn, args.frames, args.warmup)
            res["workloads"].append({"what": f"points {n / 1e6:.0f} M, point size {ps}, 1920x1080", "ms_per_frame": ms,
                                     "kernels_ms": kernel_means(fn, 5),
                                     "upload_seconds": upload_seconds([n * 15])})  # the 15-byte records of fused.ply
        del xyz, rgb
        torch.cuda.empty_cache()
    xyz, rgb, faces = grid_mesh(1415)  # 2.0 M vertices, 4.0 M faces
    nf = faces.shape[0]
    for (w, h), e, label in (((1920, 1080), eye, "whole"), ((3840, 2160), eye, "whole"), ((1920, 1080), np.array([0.0, -0.02, -0.12]), "close-up")):
        P = camera(w, h, e, [0, 0, 0])
        fn = lambda: ops.render_mesh(xyz, rgb, faces, P, w, h, 1e-3, shade=True, check_faces=False)
        ms = timed(fn, args.frames, args.warmup)
        res["workloads"].append({"what": f"mesh {nf / 1e6:.1f} M faces, {label}, {w}x{h}", "ms_per_frame": ms, "kernels_ms": kernel_means(fn, 5),
                                 "upload_seconds": upload_seconds([xyz.shape[0] * 15, nf * 13])})
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
