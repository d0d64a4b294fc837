"""Scene folder + reconstruct results -> COLMAP dense workspace: the counterpart of the reference's colmap_output.py.

    python -m patchmatchnet_b200.reconstruct --input-folder scene --output-folder outputs --checkpoint-path model.pt
    python -m patchmatchnet_b200.colmap_output --input-folder scene --results-folder outputs --output-folder workspace --normals
    colmap stereo_fusion --workspace_path workspace --input_type geometric --output_path workspace/fused.ply
    colmap poisson_mesher --input_path workspace/fused.ply --output_path workspace/meshed-poisson.ply

Writes, under the output folder: images/ (a copy of the scene's images), stereo/depth_maps/<image>.geometric.bin and
stereo/confidence_maps/<image>.geometric.bin (.bin results are copied, .pfm results converted through data_io.read_map /
save_map), stereo/patch-match.cfg and stereo/fusion.cfg from pair.txt, and sparse/{cameras,images,points3D}.txt with one
PINHOLE camera per view and the quaternion of each rotation from the reference's eigen-decomposition.  The empty
consistency_graphs/ folder COLMAP expects is created too, and normal_maps/, which stays empty without --normals.

COLMAP's stereo_fusion skips every image whose stereo/normal_maps/<image>.geometric.bin is missing, and its
max_normal_error test reads those maps.  With --normals (off by default; it needs a CUDA device and changes no other
file) each image's normal map is estimated on the GPU from its depth map (ops.estimate_normals: camera-frame unit normals,
(0, 0, 0) where there is no estimate) with the cam file's intrinsics scaled to the depth map's size, and written there as
a 3-channel COLMAP .bin at the depth map's size.  Without the flag the command runs on the host only, as before.

Difference from the reference: cameras and images are listed in ascending view ID (the reference lists them in os.listdir
order, which depends on the file system), and the map extension is taken from the first depth map in sorted order.
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import data_io
from .colmap_input import Camera, Image


def rotation_matrix_to_quaternion(rot: np.ndarray) -> List[float]:
    """[qw, qx, qy, qz] with qw >= 0: the eigenvector of the largest eigenvalue of the symmetric 4x4 matrix K of the rotation
    (Bar-Itzhack's construction, as the reference computes it; the dtype of `rot` is kept)."""
    rxx, ryx, rzx, rxy, ryy, rzy, rxz, ryz, rzz = rot.flat
    k = np.array([
        [rxx - ryy - rzz, 0, 0, 0],
        [ryx + rxy, ryy - rxx - rzz, 0, 0],
        [rzx + rxz, rzy + ryz, rzz - rxx - ryy, 0],
        [ryz - rzy, rzx - rxz, rxy - ryx, rxx + ryy + rzz]]) / 3.0
    values, vectors = np.linalg.eigh(k)
    q = vectors[[3, 0, 1, 2], np.argmax(values)]
    if q[0] < 0:
        q *= -1
    return [q[0], q[1], q[2], q[3]]


def create_output_dirs(path: str) -> None:
    for sub in ("", "images", "sparse", "stereo", os.path.join("stereo", "confidence_maps"), os.path.join("stereo", "consistency_graphs"),
                os.path.join("stereo", "depth_maps"), os.path.join("stereo", "normal_maps")):
        os.makedirs(os.path.join(path, sub), exist_ok=True)


def copy_maps(input_path: str, results_path: str, output_path: str) -> None:
    """images/ and, per image of the scene, its depth and confidence maps as <image file>.geometric.bin."""
    shutil.copytree(os.path.join(input_path, "images"), os.path.join(output_path, "images"), dirs_exist_ok=True)
    depth_files = sorted(os.listdir(os.path.join(results_path, "depth_est")))
    if not depth_files:
        raise FileNotFoundError(f"no depth maps in {os.path.join(results_path, 'depth_est')}")
    ext = os.path.splitext(depth_files[0])[1]
    for image_file in sorted(os.listdir(os.path.join(input_path, "images"))):
        name = os.path.splitext(image_file)[0]
        for kind, out_kind in (("depth_est", "depth_maps"), ("confidence", "confidence_maps")):
            src = os.path.join(results_path, kind, name + ext)
            dst = os.path.join(output_path, "stereo", out_kind, image_file + ".geometric.bin")
            if ext == ".bin":
                shutil.copy(src, dst)
            else:
                data_io.save_map(dst, data_io.read_map(src))


def write_normal_maps(input_path: str, results_path: str, output_path: str, device: str = "cuda:0") -> None:
    """stereo/normal_maps/<image file>.geometric.bin per image of the scene: ops.estimate_normals on its depth map, with the
    intrinsics of cams/<name>_cam.txt scaled from the image's size to the depth map's (reconstruct --image-max-dim writes
    smaller maps)."""
    from PIL import Image as PilImage

    from . import ops

    ext = os.path.splitext(sorted(os.listdir(os.path.join(results_path, "depth_est")))[0])[1]
    for image_file in sorted(os.listdir(os.path.join(input_path, "images"))):
        name = os.path.splitext(image_file)[0]
        depth = data_io.read_map_to_device(os.path.join(results_path, "depth_est", name + ext), device)[..., 0]
        with PilImage.open(os.path.join(input_path, "images", image_file), "r") as img:
            width, height = img.width, img.height
        k, _, _ = data_io.read_cam_file(os.path.join(input_path, "cams", name + "_cam.txt"))
        normals = ops.estimate_normals(depth, data_io.scale_intrinsics(k, tuple(depth.shape), height, width))
        data_io.save_map_from_device(os.path.join(output_path, "stereo", "normal_maps", image_file + ".geometric.bin"), normals)


def read_reconstruction(path: str) -> Tuple[List[Camera], List[Image], List[Tuple[int, List[int]]]]:
    """One PINHOLE camera and one image per cams/%08d_cam.txt, in ascending view ID, and the pairs of pair.txt."""
    from PIL import Image as PilImage

    cameras, images = [], []
    cam_files = sorted(os.listdir(os.path.join(path, "cams")), key=lambda f: (int(f.split("_")[0]), f))
    for cam_file in cam_files:
        prefix = cam_file.split("_")[0]
        im_id, im_file = int(prefix), prefix + ".jpg"
        with PilImage.open(os.path.join(path, "images", im_file), "r") as img:
            width, height = img.width, img.height
        k, e, _ = data_io.read_cam_file(os.path.join(path, "cams", cam_file))
        cameras.append(Camera(im_id, "PINHOLE", width, height, [k[0, 0], k[1, 1], k[0, 2], k[1, 2]]))
        images.append(Image(im_id, rotation_matrix_to_quaternion(e[0:3, 0:3]), list(e[0:3, 3]), im_id, im_file, np.empty(0, np.int64)))
    return cameras, images, data_io.read_pair_file(os.path.join(path, "pair.txt"))


def write_patch_match_config(path: str, images: List[Image], pairs: List[Tuple[int, List[int]]]) -> None:
    names: Dict[int, str] = {im.id: im.name for im in images}
    with open(path, "w") as f:
        for ref, srcs in pairs:
            f.write(names[ref] + "\n")
            f.write(", ".join(names[s] for s in srcs) + "\n")


def write_fusion_config(path: str, images: List[Image], pairs: List[Tuple[int, List[int]]]) -> None:
    names: Dict[int, str] = {im.id: im.name for im in images}
    with open(path, "w") as f:
        f.writelines(",".join(names[v] for v in [ref] + srcs) + "\n" for ref, srcs in pairs)


def write_sparse(path: str, cameras: List[Camera], images: List[Image]) -> None:
    """COLMAP text model: cameras.txt, images.txt (no 2D points) and an empty points3D.txt."""
    with open(os.path.join(path, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n")
        f.write("#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        f.write("# Number of cameras: {}\n".format(len(cameras)))
        f.writelines("{} {} {} {} {} {} {} {}\n".format(c.id, c.model, c.width, c.height, *c.params[:4]) for c in cameras)
    with open(os.path.join(path, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n")
        f.write("#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n")
        f.write("#   POINTS2D[] as (X, Y, POINT3D_ID)\n")
        f.write("# Number of images: {}, mean observations per image: 0\n".format(len(images)))
        f.writelines("{} {} {} {} {} {} {} {} {} {}\n\n".format(i.id, *i.qvec[:4], *i.tvec[:3], i.camera_id, i.name) for i in images)
    with open(os.path.join(path, "points3D.txt"), "w") as f:
        f.write("# 3D point list with one line of data per point:\n")
        f.write("#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n")
        f.write("# Number of points: 0, mean track length: 0")


def build_parser() -> argparse.ArgumentParser:
    """colmap_output.py's options in this project's hyphen style, same defaults."""
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.colmap_output",
                                 description="Convert PatchMatchNet results into a COLMAP dense workspace")
    ap.add_argument("--input-folder", type=str, help="Input PatchMatchNet reconstruction dir")
    ap.add_argument("--results-folder", type=str, default="", help="Input PatchMatchNet results dir")
    ap.add_argument("--output-folder", type=str, default="", help="Output ColMap MVS workspace")
    ap.add_argument("--normals", action="store_true",
                    help="estimate a normal map per image on the GPU and write it to stereo/normal_maps (COLMAP's "
                         "stereo_fusion needs them)")
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return build_parser().parse_args(argv)


def check_args(args: argparse.Namespace) -> None:
    """colmap_output.py's checks and messages; sets the default results and output folders."""
    if not args.results_folder:
        args.results_folder = args.input_folder
    if not args.output_folder:
        args.output_folder = args.input_folder
    if args.input_folder is None or not os.path.isdir(args.input_folder):
        raise Exception("Invalid input folder")
    if args.results_folder is None or not os.path.isdir(args.results_folder):
        raise Exception("Invalid results folder")
    if args.output_folder is None or not os.path.isdir(args.output_folder):
        raise Exception("Invalid output folder")


def export(args: argparse.Namespace) -> None:
    """The command's library call.  With --normals it raises before it writes anything when there is no CUDA device."""
    check_args(args)
    if args.normals:
        import torch

        if not torch.cuda.is_available():
            raise RuntimeError("colmap_output --normals needs a CUDA device (H100); there is no CPU fallback")
    create_output_dirs(args.output_folder)
    copy_maps(args.input_folder, args.results_folder, args.output_folder)
    if args.normals:
        write_normal_maps(args.input_folder, args.results_folder, args.output_folder)
    cameras, images, pairs = read_reconstruction(args.input_folder)
    write_patch_match_config(os.path.join(args.output_folder, "stereo", "patch-match.cfg"), images, pairs)
    write_fusion_config(os.path.join(args.output_folder, "stereo", "fusion.cfg"), images, pairs)
    write_sparse(os.path.join(args.output_folder, "sparse"), cameras, images)


def main(argv: Optional[Sequence[str]] = None) -> int:
    export(parse_args(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
