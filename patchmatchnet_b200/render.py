"""Headless rendering of a PLY point cloud or mesh to PNG images on the GPU -- the counterpart of the reference's
visualize_ply.py, which opens an Open3D window and so needs a display.

    python -m patchmatchnet_b200.render --ply results/fused.ply --input-folder scene --views 0 5 --depth --output-folder renders
    python -m patchmatchnet_b200.render --ply results/mesh.ply --orbit 8 --shade --output-folder renders
    python -m patchmatchnet_b200.render --ply results/fused.ply --viewpoint viewpoint.json --point-size 3 --output-folder renders

The PLY is read once (data_io.read_ply) and uploaded once; a file with faces renders as a mesh (ops.render_mesh), any other
as points (ops.render_points).  Cameras, which may be combined:
  --views ID ...     the views' cams/%08d_cam.txt under --input-folder, intrinsics scaled to the image size as reconstruct
                     scales them (with --image-max-dim); image sizes come from the image headers.  -> view_%08d.png
  --orbit N          N frames on a circle around the centre of the per-axis 1st-99th percentile box of the vertices, at
                     --elevation degrees above its plane, vertical field of view 40 degrees, at the distance where the box's
                     bounding sphere fits the frame; --width x --height.  The up direction is --up, else the mean image-up
                     of the scene's cameras with --input-folder, else -Y.  -> orbit_%04d.png
  --viewpoint FILE   an Open3D PinholeCameraParameters JSON (visualize_ply.py --use_viewpoint's file).  -> viewpoint.png
--depth also writes each frame's depth (0 where nothing was drawn) as .pfm next to its PNG, through data_io.save_map.
The default near plane is 1e-3 times the distance from the camera centre to the box centre.  Definition and differences
from Open3D: include/patchmatch_b200.h and INTEGRATION.md "Rendering (beyond the reference)".
"""
from __future__ import annotations

import argparse
import glob
import json
import math
import os
import sys
import time
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import data_io, ops

ORBIT_FOV_Y = 40.0  # degrees
DEFAULT_UP = (0.0, -1.0, 0.0)


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.render", description="Render a PLY cloud or mesh to PNG images")
    ap.add_argument("--ply", type=str, required=True, help="PLY point cloud or triangle mesh")
    ap.add_argument("--output-folder", type=str, default="renders", help="where the images go")
    ap.add_argument("--input-folder", type=str, default="", help="scene folder (cams/, images/) for --views and the default up")
    ap.add_argument("--views", nargs="+", type=int, default=[], help="render from these scene views")
    ap.add_argument("--image-max-dim", type=int, default=-1, help="max image dimension, as reconstruct's option")
    ap.add_argument("--orbit", type=int, default=0, help="render N frames around the cloud")
    ap.add_argument("--elevation", type=float, default=20.0, help="orbit elevation in degrees")
    ap.add_argument("--up", nargs=3, type=float, default=None, help="orbit up direction X Y Z")
    ap.add_argument("--viewpoint", type=str, default="", help="Open3D PinholeCameraParameters JSON file")
    ap.add_argument("--width", type=int, default=1280, help="orbit frame width")
    ap.add_argument("--height", type=int, default=960, help="orbit frame height")
    ap.add_argument("--point-size", type=int, default=1, help="square splat size in pixels, odd, 1..15")
    ap.add_argument("--shade", action="store_true", help="headlight Lambert shading (point normals, face normals)")
    ap.add_argument("--background", nargs=3, type=int, default=[255, 255, 255], help="background colour R G B")
    ap.add_argument("--depth", action="store_true", help="also write each frame's depth as .pfm")
    ap.add_argument("--near", type=float, default=None, help="near plane depth (default: 1e-3 x distance to the box centre)")
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return build_parser().parse_args(argv)


def check_args(args: argparse.Namespace) -> None:
    """ValueError for inconsistent arguments, before anything is read or written."""
    if not os.path.isfile(args.ply):
        raise ValueError(f"--ply: no such file {args.ply!r}")
    if not args.views and args.orbit <= 0 and not args.viewpoint:
        raise ValueError("give at least one camera: --views, --orbit N or --viewpoint")
    if args.views and not (args.input_folder and os.path.isdir(args.input_folder)):
        raise ValueError("--views needs --input-folder, a scene folder with cams/ and images/")
    if args.orbit < 0:
        raise ValueError(f"--orbit must be >= 0, got {args.orbit}")
    if args.viewpoint and not os.path.isfile(args.viewpoint):
        raise ValueError(f"--viewpoint: no such file {args.viewpoint!r}")
    if not (1 <= args.width <= 16384 and 1 <= args.height <= 16384):
        raise ValueError(f"--width and --height must be 1..16384, got {args.width} x {args.height}")
    if not (1 <= args.point_size <= 15 and args.point_size % 2 == 1):
        raise ValueError(f"--point-size must be odd, 1..15, got {args.point_size}")
    if any(not 0 <= c <= 255 for c in args.background):
        raise ValueError(f"--background values must be 0..255, got {args.background}")
    if args.up is not None and not (np.isfinite(args.up).all() and np.linalg.norm(args.up) > 0):
        raise ValueError(f"--up must be a finite non-zero vector, got {args.up}")
    if args.near is not None and not (0 < args.near < float("inf")):
        raise ValueError(f"--near must be positive and finite, got {args.near}")


# ---- cameras --------------------------------------------------------------------------------------------------------------


def percentile_box(xyz: torch.Tensor) -> Tuple[np.ndarray, np.ndarray]:
    """Per axis the k-th and (n-1-k)-th smallest coordinates, k = floor(0.01 (n - 1)): the 1st-99th percentile box, so
    outliers do not set the framing.  xyz float32 [n,3] (any device) -> (lo, hi) float64 [3]."""
    n = xyz.shape[0]
    if n == 0:
        return np.zeros(3), np.zeros(3)
    k = int(0.01 * (n - 1))
    lo, hi = np.zeros(3), np.zeros(3)
    for a in range(3):
        s = torch.sort(xyz[:, a]).values
        lo[a], hi[a] = float(s[k]), float(s[n - 1 - k])
    return lo, hi


def look_at(eye: np.ndarray, target: np.ndarray, up: np.ndarray) -> np.ndarray:
    """float64 [4,4] world -> camera with z towards target, x right and y down, image-up along `up` (projected)."""
    z = target - eye
    z = z / np.linalg.norm(z)
    y = -(up - np.dot(up, z) * z)
    if np.linalg.norm(y) < 1e-9 * np.linalg.norm(up):  # looking along up: any perpendicular will do
        y = np.cross(z, [1.0, 0.0, 0.0] if abs(z[0]) < 0.9 else [0.0, 1.0, 0.0])
    y = y / np.linalg.norm(y)
    x = np.cross(y, z)
    E = np.eye(4)
    E[:3, :3] = np.stack([x, y, z])
    E[:3, 3] = -E[:3, :3] @ eye
    return E


def orbit_intrinsics(width: int, height: int, fov_y: float = ORBIT_FOV_Y) -> np.ndarray:
    f = (height / 2.0) / math.tan(math.radians(fov_y) / 2.0)
    return np.array([[f, 0.0, (width - 1) / 2.0], [0.0, f, (height - 1) / 2.0], [0.0, 0.0, 1.0]])


def orbit_cameras(centre, radius: float, n: int, elevation: float, up, width: int, height: int) -> List[np.ndarray]:
    """n float64 3 x 4 cameras K [R | t] on a circle around `centre` at `elevation` degrees above the plane normal to `up`,
    looking at the centre, at the distance where a sphere of `radius` fits the frame (vertical field of view 40 degrees)."""
    centre, up = np.asarray(centre, np.float64), np.asarray(up, np.float64)
    up = up / np.linalg.norm(up)
    K = orbit_intrinsics(width, height)
    half_y = math.radians(ORBIT_FOV_Y) / 2.0
    half_x = math.atan(math.tan(half_y) * width / height)
    dist = max(radius, 1e-12) / math.sin(min(half_x, half_y))
    a0 = np.cross(up, [1.0, 0.0, 0.0] if abs(up[0]) < 0.9 else [0.0, 1.0, 0.0])
    a0 /= np.linalg.norm(a0)
    b0 = np.cross(up, a0)
    el = math.radians(elevation)
    cams = []
    for k in range(n):
        phi = 2.0 * math.pi * k / n
        d = math.cos(el) * (math.cos(phi) * a0 + math.sin(phi) * b0) + math.sin(el) * up
        E = look_at(centre + dist * d, centre, up)
        cams.append(K @ E[:3, :4])
    return cams


def read_viewpoint(path: str) -> Tuple[np.ndarray, int, int]:
    """An Open3D PinholeCameraParameters JSON -> (float64 3 x 4 camera K [R | t], width, height).  Open3D writes its Eigen
    matrices column-major: intrinsic.intrinsic_matrix (3 x 3) and extrinsic (4 x 4, world -> camera)."""
    with open(path) as f:
        doc = json.load(f)
    try:
        intr = doc["intrinsic"]
        K = np.asarray(intr["intrinsic_matrix"], np.float64).reshape(3, 3, order="F")
        E = np.asarray(doc["extrinsic"], np.float64).reshape(4, 4, order="F")
        width, height = int(intr["width"]), int(intr["height"])
    except (KeyError, TypeError, ValueError) as e:
        raise ValueError(f"{path}: not an Open3D PinholeCameraParameters file ({e})") from None
    if width < 1 or height < 1 or not np.isfinite(K).all() or not np.isfinite(E).all():
        raise ValueError(f"{path}: the camera needs a positive size and finite matrices")
    return K @ E[:3, :4], width, height


def image_size(scene: str, view: int, max_dim: int) -> Tuple[int, int, int, int]:
    """(H, W) of a view's image as data_io.read_image would return it, and its original (H, W), from the image header
    alone."""
    from PIL import Image

    with Image.open(os.path.join(scene, "images", "{:0>8}.jpg".format(view))) as im:
        w, h = im.size
    scale = max_dim / max(h, w)
    if 0 < scale < 1:
        return int(scale * h), int(scale * w), h, w
    return h, w, h, w


def view_camera(scene: str, view: int, max_dim: int) -> Tuple[np.ndarray, int, int]:
    """(float64 3 x 4 camera, W, H) of a scene view: its cam file's intrinsics scaled to the image size."""
    h, w, oh, ow = image_size(scene, view, max_dim)
    k, e, _ = data_io.read_cam_file(os.path.join(scene, "cams", "{:0>8}_cam.txt".format(view)))
    K = data_io.scale_intrinsics(k, (h, w), oh, ow)
    return K.astype(np.float64) @ e.astype(np.float64)[:3, :4], w, h


def scene_up(scene: str) -> Optional[np.ndarray]:
    """The mean image-up (minus the camera y axis, in the world) over the scene's cam files, or None without any."""
    ups = []
    for path in sorted(glob.glob(os.path.join(scene, "cams", "*_cam.txt"))):
        _, e, _ = data_io.read_cam_file(path)
        ups.append(-e[1, :3].astype(np.float64))
    if not ups:
        return None
    m = np.mean(ups, axis=0)
    return m / np.linalg.norm(m) if np.linalg.norm(m) > 0 else None


def camera_centre(P: np.ndarray) -> np.ndarray:
    return -np.linalg.solve(P[:, :3], P[:, 3])


def frames(args: argparse.Namespace, box: Tuple[np.ndarray, np.ndarray]) -> List[Tuple[str, np.ndarray, int, int]]:
    """(file stem, float64 3 x 4 camera, W, H) of every requested frame."""
    out = []
    for v in args.views:
        P, w, h = view_camera(args.input_folder, v, args.image_max_dim)
        out.append(("view_{:0>8}".format(v), P, w, h))
    if args.orbit > 0:
        lo, hi = box
        up = np.asarray(args.up, np.float64) if args.up is not None else None
        if up is None and args.input_folder:
            up = scene_up(args.input_folder)
        if up is None:
            up = np.asarray(DEFAULT_UP)
        cams = orbit_cameras((lo + hi) / 2.0, 0.5 * float(np.linalg.norm(hi - lo)), args.orbit, args.elevation, up, args.width, args.height)
        out += [("orbit_{:0>4}".format(k), P, args.width, args.height) for k, P in enumerate(cams)]
    if args.viewpoint:
        P, w, h = read_viewpoint(args.viewpoint)
        out.append(("viewpoint", P, w, h))
    return out


# ---- command --------------------------------------------------------------------------------------------------------------


def render(args: argparse.Namespace, *, device: str = "cuda:0", log=print) -> Dict[str, float]:
    """The command's library call.  -> seconds of reading the PLY, uploading it, rendering (kernels and the device-to-host
    copies) and writing the files, end to end, and the frame count.  Raises ValueError before it writes anything when the
    arguments are invalid."""
    check_args(args)
    if not torch.cuda.is_available():
        raise RuntimeError("render needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    stats = {"read_seconds": 0.0, "upload_seconds": 0.0, "render_seconds": 0.0, "write_seconds": 0.0}
    t_start = time.perf_counter()
    xyz, rgb, normals, faces = data_io.read_ply(args.ply)
    t0 = time.perf_counter()
    stats["read_seconds"] = t0 - t_start
    with torch.cuda.device(dev):
        d_xyz = torch.from_numpy(xyz).to(dev)
        d_rgb = torch.from_numpy(rgb).to(dev) if rgb is not None else None
        d_nrm = torch.from_numpy(normals).to(dev) if normals is not None else None
        d_faces = torch.from_numpy(faces).to(dev) if faces is not None else None
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        stats["upload_seconds"] = t1 - t0
        box = percentile_box(d_xyz)
        todo = frames(args, box)
        os.makedirs(args.output_folder, exist_ok=True)
        centre = (box[0] + box[1]) / 2.0
        for stem, P, w, h in todo:
            t1 = time.perf_counter()
            near = args.near if args.near is not None else 1e-3 * max(float(np.linalg.norm(camera_centre(P) - centre)), 1e-30)
            if d_faces is not None:
                img, depth = ops.render_mesh(d_xyz, d_rgb, d_faces, P, w, h, near, shade=args.shade, background=args.background,
                                             check_faces=False)  # read_ply checked the indices
            else:
                img, depth = ops.render_points(d_xyz, d_rgb, d_nrm, P, w, h, near, point_size=args.point_size, shade=args.shade,
                                               background=args.background)
            img_h, depth_h = img.cpu().numpy(), depth.cpu().numpy()
            t2 = time.perf_counter()
            stats["render_seconds"] += t2 - t1
            path = os.path.join(args.output_folder, stem + ".png")
            data_io.save_image(path, img_h)
            if args.depth:
                data_io.save_map(os.path.join(args.output_folder, stem + ".pfm"), depth_h)
            stats["write_seconds"] += time.perf_counter() - t2
            log("rendered", path)
    stats["frames"] = len(todo)
    stats["total_seconds"] = time.perf_counter() - t_start
    return stats


def main(argv: Optional[Sequence[str]] = None) -> int:
    render(parse_args(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
