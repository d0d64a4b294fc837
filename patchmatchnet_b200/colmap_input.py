"""COLMAP sparse model -> scene folder (pair.txt, cams/%08d_cam.txt, images/%08d.jpg): the counterpart of the reference's
colmap_input.py, with view selection and depth ranges on the GPU.

    python -m patchmatchnet_b200.colmap_input --input-folder project --undistort
    python -m patchmatchnet_b200.reconstruct --input-folder project --checkpoint-path model.pt

Input: <input folder>/sparse/{cameras,images,points3D}.bin (or .txt when there is no .bin) and <input folder>/images/<name>.
The view index of an image is its position in the images file, as in the reference.  --sparse-folder NAME reads the model
from <input folder>/NAME instead; an image name may hold subfolders.  So an ETH3D training scene (dslr_calibration_undistorted/
and images/dslr_images_undistorted/*.JPG) converts in place with --sparse-folder dslr_calibration_undistorted.

Host side (reference expressions, so the text written from them is byte-identical): the readers, the rotation of each
quaternion, the intrinsics of all 11 COLMAP camera models (without --undistort, distortion parameters are ignored, as in the
reference, with a warning: undistort first), the extrinsics and the camera centres -R^T t.
Device side (csrc/pm_colmap.cu through ops.view_scores / ops.depth_ranges): the pairwise view scores, whose cost follows the
co-visibility of the model instead of the reference's N^2 x obs^2 list scans, and the per-image depth ranges.

--undistort (beyond the reference; INTEGRATION.md "Undistortion (beyond the reference)"): every camera with a non-zero
distortion parameter becomes the PINHOLE camera of COLMAP's UndistortCamera (border extents on the GPU, ops.undistort_extents;
scale on the host, ops.undistorted_camera), and each of its images is resampled on the GPU (ops.undistort_image) and written
in its source's codec (PNG stays PNG, JPEG is written at quality 95 with 4:4:4 chroma, anything else becomes PNG).  Cameras
without distortion keep the byte-for-byte copy.  cams/ gets the new intrinsics; pair.txt and the depth ranges do not change.

Differences from the reference (INTEGRATION.md "COLMAP interop"): the cosine of the triangulation angle is clamped to [-1, 1]
and a point on a camera centre contributes 0 (the reference writes nan); ties between scores are ordered by descending view
index (a stable argsort, reversed); a point ID missing from points3D and an image without observations are ValueErrors that
name the image; the .txt model is read when there is no .bin; --convert-format and the debug prints are left out, and
there is no requirement that a camera with ID 1 exists.  There is no CPU path: without a CUDA device the command raises before
it writes anything.
"""
from __future__ import annotations

import argparse
import os
import shutil
import struct
import sys
import time
from typing import Callable, Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

# COLMAP camera models: id -> (name, number of parameters)
CAMERA_MODELS: Dict[int, Tuple[str, int]] = {
    0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
    5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4), 9: ("RADIAL_FISHEYE", 5),
    10: ("THIN_PRISM_FISHEYE", 12),
}

# parameter names per model (COLMAP's src/base/camera_models.h); the first ones are the pinhole part, the rest distortion
PARAM_TYPE: Dict[str, List[str]] = {
    "SIMPLE_PINHOLE": ["f", "cx", "cy"],
    "PINHOLE": ["fx", "fy", "cx", "cy"],
    "SIMPLE_RADIAL": ["f", "cx", "cy", "k"],
    "SIMPLE_RADIAL_FISHEYE": ["f", "cx", "cy", "k"],
    "RADIAL": ["f", "cx", "cy", "k1", "k2"],
    "RADIAL_FISHEYE": ["f", "cx", "cy", "k1", "k2"],
    "OPENCV": ["fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2"],
    "OPENCV_FISHEYE": ["fx", "fy", "cx", "cy", "k1", "k2", "k3", "k4"],
    "FULL_OPENCV": ["fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "k4", "k5", "k6"],
    "FOV": ["fx", "fy", "cx", "cy", "omega"],
    "THIN_PRISM_FISHEYE": ["fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3", "k4", "sx1", "sy1"],
}
_PINHOLE_PARAMS = {"f", "fx", "fy", "cx", "cy"}


class Camera(NamedTuple):
    id: int
    model: str
    width: int
    height: int
    params: List[float]


class Image(NamedTuple):
    """One registered image.  point3d_ids: int64 [number of 2D points], the point ID of every 2D point in file order (-1: none)."""
    id: int
    qvec: Sequence[float]
    tvec: Sequence[float]
    camera_id: int
    name: str
    point3d_ids: np.ndarray


class Points3D(NamedTuple):
    """The points of a model as arrays, in file order (tracks are skipped: view selection does not use them)."""
    ids: np.ndarray    # uint64 [P]
    xyz: np.ndarray    # float64 [P,3]
    rgb: np.ndarray    # uint8 [P,3]
    error: np.ndarray  # float64 [P]


# ---- readers ------------------------------------------------------------------------------------------------------------------

def _text_lines(path: str):
    with open(path, "r") as f:
        for line in f:
            line = line.strip()
            if line and line[0] != "#":
                yield line


def read_cameras_text(path: str) -> Dict[int, Camera]:
    cams: Dict[int, Camera] = {}
    for line in _text_lines(path):
        e = line.split()
        cams[int(e[0])] = Camera(int(e[0]), e[1], int(e[2]), int(e[3]), [float(v) for v in e[4:]])
    return cams


def read_cameras_binary(path: str) -> Dict[int, Camera]:
    cams: Dict[int, Camera] = {}
    with open(path, "rb") as f:
        data = f.read()
    (n,), off = struct.unpack_from("<Q", data, 0), 8
    for _ in range(n):
        cam_id, model_id, width, height = struct.unpack_from("<iiQQ", data, off)
        off += 24
        if model_id not in CAMERA_MODELS:
            raise ValueError(f"{path}: camera {cam_id} has unknown model id {model_id}")
        name, n_params = CAMERA_MODELS[model_id]
        params = list(struct.unpack_from("<" + "d" * n_params, data, off))
        off += 8 * n_params
        cams[cam_id] = Camera(cam_id, name, width, height, params)
    return cams


def read_images_text(path: str) -> List[Image]:
    images: List[Image] = []
    with open(path, "r") as f:
        while True:
            line = f.readline()
            if not line:
                break
            line = line.strip()
            if not line or line[0] == "#":
                continue
            e = line.split()
            points = f.readline().split()
            ids = np.array([int(v) for v in points[2::3]], dtype=np.int64)
            images.append(Image(int(e[0]), [float(v) for v in e[1:5]], [float(v) for v in e[5:8]], int(e[8]), e[9], ids))
    return images


_POINT2D = np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<i8")])


def read_images_binary(path: str) -> List[Image]:
    images: List[Image] = []
    with open(path, "rb") as f:
        data = f.read()
    (n,), off = struct.unpack_from("<Q", data, 0), 8
    for _ in range(n):
        props = struct.unpack_from("<idddddddi", data, off)
        off += 64
        end = data.index(b"\x00", off)
        name = data[off:end].decode("utf-8")
        off = end + 1
        (n2d,) = struct.unpack_from("<Q", data, off)
        off += 8
        pts = np.frombuffer(data, dtype=_POINT2D, count=n2d, offset=off)
        off += 24 * n2d
        images.append(Image(props[0], props[1:5], props[5:8], props[8], name, pts["id"].astype(np.int64)))
    return images


def read_points3d_text(path: str) -> Points3D:
    ids, xyz, rgb, err = [], [], [], []
    for line in _text_lines(path):
        e = line.split(maxsplit=8)
        ids.append(int(e[0]))
        xyz.append((float(e[1]), float(e[2]), float(e[3])))
        rgb.append((int(e[4]), int(e[5]), int(e[6])))
        err.append(float(e[7]))
    return Points3D(np.array(ids, dtype=np.uint64), np.array(xyz, dtype=np.float64).reshape(-1, 3),
                    np.array(rgb, dtype=np.uint8).reshape(-1, 3), np.array(err, dtype=np.float64))


def read_points3d_binary(path: str) -> Points3D:
    with open(path, "rb") as f:
        data = f.read()
    (n,) = struct.unpack_from("<Q", data, 0)
    head = struct.Struct("<QdddBBBdQ")  # the 43-byte point record and its track length; the track itself is skipped
    ids = np.empty(n, dtype=np.uint64)
    xyz = np.empty((n, 3), dtype=np.float64)
    rgb = np.empty((n, 3), dtype=np.uint8)
    err = np.empty(n, dtype=np.float64)
    off = 8
    unpack = head.unpack_from
    for k in range(n):
        r = unpack(data, off)
        ids[k] = r[0]
        xyz[k] = r[1:4]
        rgb[k] = r[4:7]
        err[k] = r[7]
        off += 51 + 8 * r[8]
    return Points3D(ids, xyz, rgb, err)


def model_ext(path: str) -> str:
    """'.bin' when the three .bin files are there, else '.txt' when the three .txt files are; FileNotFoundError otherwise."""
    for ext in (".bin", ".txt"):
        if all(os.path.isfile(os.path.join(path, name + ext)) for name in ("cameras", "images", "points3D")):
            return ext
    raise FileNotFoundError(f"no COLMAP model in {path}: expected cameras, images and points3D as .bin or .txt")


def read_model(path: str, ext: Optional[str] = None) -> Tuple[Dict[int, Camera], List[Image], Points3D]:
    """(cameras by ID, images in file order, points) of the sparse model in `path`: the .bin form when present, else .txt."""
    ext = ext or model_ext(path)
    if ext == ".bin":
        return (read_cameras_binary(os.path.join(path, "cameras.bin")), read_images_binary(os.path.join(path, "images.bin")),
                read_points3d_binary(os.path.join(path, "points3D.bin")))
    return (read_cameras_text(os.path.join(path, "cameras.txt")), read_images_text(os.path.join(path, "images.txt")),
            read_points3d_text(os.path.join(path, "points3D.txt")))


# ---- host math (the reference's expressions) ----------------------------------------------------------------------------------

def quaternion_to_rotation_matrix(qvec: Sequence[float]) -> np.ndarray:
    w, x, y, z = qvec[0], qvec[1], qvec[2], qvec[3]
    return np.array([
        [1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
        [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
        [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def intrinsic_matrix(cam: Camera) -> np.ndarray:
    """[[fx, 0, cx], [0, fy, cy], [0, 0, 1]] float64 from the camera's pinhole parameters (f for both when the model has one)."""
    names = PARAM_TYPE[cam.model]
    p = dict(zip(names, cam.params))
    if "f" in names:
        p["fx"] = p["fy"] = p["f"]
    return np.array([[p["fx"], 0, p["cx"]], [0, p["fy"], p["cy"]], [0, 0, 1]])


def has_distortion(cam: Camera) -> bool:
    return any(v != 0 for k, v in zip(PARAM_TYPE[cam.model], cam.params) if k not in _PINHOLE_PARAMS)


def extrinsic_matrix(image: Image) -> np.ndarray:
    e = np.zeros((4, 4))
    e[:3, :3] = quaternion_to_rotation_matrix(image.qvec)
    e[:3, 3] = image.tvec
    e[3, 3] = 1
    return e


def camera_center(extrinsic: np.ndarray) -> np.ndarray:
    return -np.matmul(extrinsic[:3, :3].transpose(), extrinsic[:3, 3:4])[:, 0]


class SceneModel(NamedTuple):
    """A sparse model ready for the device: dense point indices, observations in CSR form, and the host-composed cameras."""
    intrinsics: List[np.ndarray]  # float64 [3,3] per image
    extrinsics: np.ndarray        # float64 [N,4,4]
    centers: np.ndarray           # float64 [N,3]
    xyz: np.ndarray               # float64 [P,3]
    obs_offsets: np.ndarray       # int32 [N+1]
    obs_points: np.ndarray        # int32 [M]


def prepare(cameras: Dict[int, Camera], images: List[Image], points: Points3D) -> SceneModel:
    """Host half of the conversion.  Raises ValueError for an image that names a point missing from points3D, an image
    without a valid observation, or an image whose camera is missing."""
    if not images:
        raise ValueError("the model has no images")
    if len(images) >= 65536:
        raise ValueError(f"the model has {len(images)} images; at most 65535 are supported")
    order = np.argsort(points.ids, kind="stable")
    sorted_ids = points.ids[order]
    counts, chunks = [], []
    for i, im in enumerate(images):
        if im.camera_id not in cameras:
            raise ValueError(f"image {i} ({im.name}): camera {im.camera_id} is not in the model")
        ids = im.point3d_ids[im.point3d_ids != -1]
        if ids.size == 0:
            raise ValueError(f"image {i} ({im.name}) has no valid observation: no depth range can be computed for it")
        key = ids.astype(np.uint64)
        pos = np.searchsorted(sorted_ids, key)
        found = pos < sorted_ids.size
        found[found] = sorted_ids[pos[found]] == key[found]
        if not found.all():
            raise ValueError(f"image {i} ({im.name}) observes point {int(key[~found][0])}, which is not in points3D")
        chunks.append(order[pos].astype(np.int32))
        counts.append(ids.size)
    offsets = np.zeros(len(images) + 1, dtype=np.int64)
    np.cumsum(counts, out=offsets[1:])
    if offsets[-1] >= 2 ** 31:
        raise ValueError(f"the model has {offsets[-1]} observations; fewer than 2^31 are supported")
    extrinsics = np.stack([extrinsic_matrix(im) for im in images])
    return SceneModel(
        intrinsics=[intrinsic_matrix(cameras[im.camera_id]) for im in images],
        extrinsics=extrinsics,
        centers=np.stack([camera_center(e) for e in extrinsics]),
        xyz=np.ascontiguousarray(points.xyz, dtype=np.float64),
        obs_offsets=offsets.astype(np.int32),
        obs_points=np.concatenate(chunks),
    )


def gpu_scores_and_ranges(model: SceneModel, theta0: float, sigma1: float, sigma2: float, device="cuda:0"):
    """(scores float64 [N,N], depth ranges float64 [N,2]) on the device (ops.view_scores, ops.depth_ranges)."""
    import torch

    from . import ops

    dev = torch.device(device)
    xyz = torch.from_numpy(model.xyz).to(dev)
    offs = torch.from_numpy(model.obs_offsets).to(dev)
    pts = torch.from_numpy(model.obs_points).to(dev)
    scores = ops.view_scores(xyz, offs, pts, torch.from_numpy(model.centers).to(dev), theta0, sigma1, sigma2)
    ranges = ops.depth_ranges(xyz, offs, pts, torch.from_numpy(model.extrinsics).to(dev))
    return scores, ranges


def select_views(scores: np.ndarray, num_src_images: int) -> List[List[Tuple[int, float]]]:
    """Per row: (view, score) by descending score, ties by descending view index; the first num_src_images (all when < 0),
    the view itself (score 0) included as in the reference."""
    n = scores.shape[0]
    keep = n if num_src_images < 0 else num_src_images
    out = []
    for i in range(n):
        order = np.argsort(scores[i], kind="stable")[::-1]
        out.append([(k, scores[i, k]) for k in order[:keep]])
    return out


def cam_text(extrinsic: np.ndarray, intrinsic: np.ndarray, depth_range: Tuple[float, float]) -> str:
    parts = ["extrinsic\n"]
    for j in range(4):
        parts.append("".join(str(extrinsic[j, k]) + " " for k in range(4)) + "\n")
    parts.append("\nintrinsic\n")
    for j in range(3):
        parts.append("".join(str(intrinsic[j, k]) + " " for k in range(3)) + "\n")
    parts.append("\n%f %f \n" % (depth_range[0], depth_range[1]))
    return "".join(parts)


def pair_text(view_sel: List[List[Tuple[int, float]]]) -> str:
    parts = ["%d\n" % len(view_sel)]
    for i, row in enumerate(view_sel):
        parts.append("%d\n%d " % (i, len(row)))
        parts.append("".join("%d %f " % (k, s) for k, s in row))
        parts.append("\n")
    return "".join(parts)


def write_scene(output_folder: str, model: SceneModel, depth_ranges: Sequence[Tuple[float, float]],
                view_sel: List[List[Tuple[int, float]]]) -> None:
    """cams/%08d_cam.txt and pair.txt."""
    cam_dir = os.path.join(output_folder, "cams")
    os.makedirs(cam_dir, exist_ok=True)
    for i, (e, k) in enumerate(zip(model.extrinsics, model.intrinsics)):
        with open(os.path.join(cam_dir, "%08d_cam.txt" % i), "w") as f:
            f.write(cam_text(e, k, depth_ranges[i]))
    with open(os.path.join(output_folder, "pair.txt"), "w") as f:
        f.write(pair_text(view_sel))


def copy_images(input_folder: str, output_folder: str, images: List[Image], skip: Sequence[int] = ()) -> None:
    """images/<name> -> images/%08d.jpg, byte for byte (reconstruct decodes by content, whatever the extension says), except
    the view indices in `skip`."""
    out_dir = os.path.join(output_folder, "images")
    os.makedirs(out_dir, exist_ok=True)
    skip = set(skip)
    for i, im in enumerate(images):
        if i not in skip:
            shutil.copyfile(os.path.join(input_folder, "images", im.name), os.path.join(out_dir, "%08d.jpg" % i))


# ---- undistortion -------------------------------------------------------------------------------------------------------------

UNDISTORT_JPEG_QUALITY = 95


def undistortion_plan(input_folder: str, cameras: Dict[int, Camera], images: List[Image], blank_pixels: float,
                      device="cuda:0") -> Dict[int, Camera]:
    """The PINHOLE camera of every camera with distortion, by camera ID (ops.undistort_extents, ops.undistorted_camera).
    Raises ValueError, naming the image or camera, for blank_pixels outside [0, 1], an image of such a camera that is not RGB
    or whose size differs from its camera's, and a camera whose scale is not finite.  Reads image headers only; writes
    nothing."""
    from PIL import Image as PILImage

    from . import ops

    if not 0.0 <= blank_pixels <= 1.0:
        raise ValueError(f"--blank-pixels must be in [0, 1], got {blank_pixels}")
    distorted = [cameras[c] for c in sorted(cameras) if has_distortion(cameras[c])]
    if not distorted:
        return {}
    ids = {c.id for c in distorted}
    for i, im in enumerate(images):
        if im.camera_id not in ids:
            continue
        cam = cameras[im.camera_id]
        with PILImage.open(os.path.join(input_folder, "images", im.name)) as f:
            size, mode = f.size, f.mode
        if mode != "RGB":
            raise ValueError(f"image {i} ({im.name}) is {mode}, not RGB: it cannot be undistorted")
        if size != (cam.width, cam.height):
            raise ValueError(f"image {i} ({im.name}) is {size[0]} x {size[1]}, but its camera {cam.id} is {cam.width} x {cam.height}")
    extents = ops.undistort_extents(distorted, device).cpu().numpy()
    return {c.id: ops.undistorted_camera(c, e, blank_pixels) for c, e in zip(distorted, extents)}


def _decode_pinned(path: str):
    """(uint8 [H,W,3] pinned host tensor, source format) of an RGB image file."""
    import torch
    from PIL import Image as PILImage

    with PILImage.open(path) as f:
        fmt = f.format
        arr = np.asarray(f)
    host = torch.empty(arr.shape, dtype=torch.uint8, pin_memory=True)
    host.numpy()[...] = arr
    return host, fmt


def _encode(arr: np.ndarray, fmt: str, path: str) -> None:
    """PNG stays lossless, JPEG is written at quality 95 with 4:4:4 chroma, any other source format as PNG."""
    from PIL import Image as PILImage

    img = PILImage.fromarray(arr, "RGB")
    if fmt == "JPEG":
        img.save(path, format="JPEG", quality=UNDISTORT_JPEG_QUALITY, subsampling=0)
    else:
        img.save(path, format="PNG")


def undistort_images(input_folder: str, output_folder: str, images: List[Image], cameras: Dict[int, Camera],
                     plan: Dict[int, Camera], device="cuda:0", workers: Optional[int] = None) -> int:
    """images/<name> -> images/%08d.jpg for every image whose camera is in `plan`: decode on the host, pinned upload, one warp
    launch (ops.undistort_image), download, encode in the source's codec.  Decoding and encoding run in a thread pool of
    `workers` threads with at most `workers` decoded and `workers` warped images in flight, so the host codec overlaps the
    GPU and memory stays bounded.  -> the number of images written."""
    import collections
    from concurrent.futures import ThreadPoolExecutor

    import torch

    from . import ops

    workers = workers or max(1, min(4, os.cpu_count() or 1))
    out_dir = os.path.join(output_folder, "images")
    os.makedirs(out_dir, exist_ok=True)
    todo = [(i, im) for i, im in enumerate(images) if im.camera_id in plan]
    dev = torch.device(device)
    with ThreadPoolExecutor(max_workers=workers) as pool, torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev)
        decoded = collections.deque()
        encoded = collections.deque()
        nxt = 0
        for i, im in todo:
            while nxt < len(todo) and len(decoded) < workers:
                decoded.append(pool.submit(_decode_pinned, os.path.join(input_folder, "images", todo[nxt][1].name)))
                nxt += 1
            src, fmt = decoded.popleft().result()
            out = ops.undistort_image(src.to(dev, non_blocking=True), cameras[im.camera_id], plan[im.camera_id])
            host = torch.empty(out.shape, dtype=torch.uint8, pin_memory=True)
            host.copy_(out, non_blocking=True)
            stream.synchronize()
            encoded.append(pool.submit(_encode, host.numpy(), fmt, os.path.join(out_dir, "%08d.jpg" % i)))
            while len(encoded) > workers:
                encoded.popleft().result()
        for f in encoded:
            f.result()
    return len(todo)


# ---- command ------------------------------------------------------------------------------------------------------------------

def build_parser() -> argparse.ArgumentParser:
    """colmap_input.py's options in this project's hyphen style, same defaults; without --convert-format."""
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.colmap_input",
                                 description="Convert colmap results into input for PatchmatchNet")
    ap.add_argument("--input-folder", type=str, help="Project input dir.")
    ap.add_argument("--output-folder", type=str, default="", help="Project output dir.")
    ap.add_argument("--num-src-images", type=int, default=-1, help="Related images")
    ap.add_argument("--theta0", type=float, default=5)
    ap.add_argument("--sigma1", type=float, default=1)
    ap.add_argument("--sigma2", type=float, default=10)
    ap.add_argument("--sparse-folder", type=str, default="sparse",
                    help="folder under the input folder that holds the sparse model (ETH3D: dslr_calibration_undistorted)")
    ap.add_argument("--undistort", action="store_true",
                    help="resample the images of every camera with distortion into COLMAP's undistorted PINHOLE camera, on the GPU")
    ap.add_argument("--blank-pixels", type=float, default=0.0,
                    help="with --undistort: 0 keeps only valid pixels, 1 keeps the whole view (blank borders); in [0, 1]")
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return build_parser().parse_args(argv)


def check_args(args: argparse.Namespace) -> None:
    """colmap_input.py's checks and messages; sets the default output folder."""
    if not args.output_folder:
        args.output_folder = args.input_folder
    if args.input_folder is None or not os.path.isdir(args.input_folder):
        raise Exception("Invalid input folder")
    if args.output_folder is None or not os.path.isdir(args.output_folder):
        raise Exception("Invalid output folder")


def convert(args: argparse.Namespace, *, device: str = "cuda:0", log: Callable[..., None] = print) -> Dict[str, float]:
    """The command's library call.  `args` as parse_args returns it.  -> seconds per phase and counts.  Raises before it writes
    anything when the arguments or the model are invalid or there is no CUDA device."""
    import torch

    check_args(args)
    if not torch.cuda.is_available():
        raise RuntimeError("colmap_input needs a CUDA device (H100); there is no CPU fallback")
    undistort = getattr(args, "undistort", False)
    t0 = time.perf_counter()
    cameras, images, points = read_model(os.path.join(args.input_folder, getattr(args, "sparse_folder", "sparse")))
    t1 = time.perf_counter()
    if not undistort:
        for cam_id in sorted(cameras):
            if has_distortion(cameras[cam_id]):
                log(f"warning: camera {cam_id} ({cameras[cam_id].model}) has distortion parameters, which are ignored; "
                    "run COLMAP's image_undistorter first")
    model = prepare(cameras, images, points)
    plan: Dict[int, Camera] = {}
    if undistort:
        with torch.cuda.device(torch.device(device)):
            plan = undistortion_plan(args.input_folder, cameras, images, args.blank_pixels, device)
        model = model._replace(intrinsics=[intrinsic_matrix(plan.get(im.camera_id, cameras[im.camera_id])) for im in images])
    t2 = time.perf_counter()
    with torch.cuda.device(torch.device(device)):
        scores, ranges = gpu_scores_and_ranges(model, args.theta0, args.sigma1, args.sigma2, device)
        scores_h, ranges_h = scores.cpu().numpy(), ranges.cpu().tolist()
    t3 = time.perf_counter()
    write_scene(args.output_folder, model, ranges_h, select_views(scores_h, args.num_src_images))
    warped = [i for i, im in enumerate(images) if im.camera_id in plan]
    copy_images(args.input_folder, args.output_folder, images, skip=warped)
    if plan:
        undistort_images(args.input_folder, args.output_folder, images, cameras, plan, device)
    t4 = time.perf_counter()
    log(f"colmap_input: {len(images)} images, {points.ids.size} points, {model.obs_points.size} observations -> {args.output_folder}")
    stats = {"read_seconds": t1 - t0, "prepare_seconds": t2 - t1, "gpu_seconds": t3 - t2, "write_seconds": t4 - t3,
             "total_seconds": t4 - t0, "images": len(images), "points": int(points.ids.size), "observations": int(model.obs_points.size)}
    if undistort:
        log(f"colmap_input: undistorted {len(warped)} images of {len(plan)} cameras")
        stats.update(undistorted_cameras=len(plan), undistorted_images=len(warped))
    return stats


def main(argv: Optional[Sequence[str]] = None) -> int:
    convert(parse_args(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
