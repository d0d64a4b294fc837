"""Convert the DTU training set from its original layout to the layout `train` reads -- the counterpart of the reference's
convert_dtu_dataset.py, writing the same bytes.

    python -m patchmatchnet_b200.convert_dtu --input-folder dtu_training --output-folder dtu_train --scan-list lists/dtu/train.txt

Input: Cameras_1/pair.txt, Cameras_1/train/%08d_cam.txt, Depths_raw/<scan>/depth_map_%04d.pfm and depth_visual_%04d.png,
Rectified/<scan>_train/rect_%03d_<light>_r5000.png.  Output per scan: pair.txt (copied), cams/ (intrinsic rows 1-2 times
4, the training images being 4x the cameras' resolution), depth_gt/%08d.pfm (the raw map read at max dimension 800 and
cropped to [44:556, 80:720]), masks/%08d.png (the visual map, read and cropped alike, > 0.04) and images/<light>/%08d.jpg
for the 7 lights.
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys
from typing import Optional, Sequence

import numpy as np

from . import data_io


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.convert_dtu",
                                 description="Convert DTU training dataset to standard input format")
    ap.add_argument("--input-folder", type=str, help="Input training data")
    ap.add_argument("--output-folder", type=str, help="Output converted training data")
    ap.add_argument("--scan-list", type=str, help="Input scan list for conversion")
    return ap


def _scaled_row(line: str) -> str:
    """An intrinsic row times 4 in float32, printed as the reference prints it (numpy float32 str)."""
    tmp = np.fromstring(line, dtype=np.float32, sep=" ") * 4.0
    return "{} {} {}".format(tmp[0], tmp[1], tmp[2])


def convert(input_folder: str, output_folder: str, scan_list: str) -> None:
    """convert_dtu_dataset.py:16-80, with its checks and messages."""
    if input_folder is None or not os.path.isdir(input_folder):
        raise Exception("Invalid input folder")
    if output_folder is None or not os.path.isdir(output_folder):
        raise Exception("Invalid output folder")
    if scan_list is None or not os.path.isfile(scan_list):
        raise Exception("Invalid input scan list")
    from PIL import Image

    with open(scan_list) as f:
        scans = [line.rstrip() for line in f.readlines()]
    cam_dir = os.path.join(input_folder, "Cameras_1", "train")
    for scan in scans:
        scan_path = os.path.join(output_folder, scan)
        paths = {k: os.path.join(scan_path, k) for k in ("cams", "depth_gt", "images", "masks")}
        for p in [scan_path] + list(paths.values()):
            os.makedirs(p, exist_ok=True)
        shutil.copy(os.path.join(input_folder, "Cameras_1", "pair.txt"), os.path.join(scan_path, "pair.txt"))
        for cam_file in os.listdir(cam_dir):
            view_id = int(cam_file.split("_")[0])
            with open(os.path.join(cam_dir, cam_file)) as f:
                lines = [line.rstrip() for line in f.readlines()]
            lines[7] = _scaled_row(lines[7])
            lines[8] = _scaled_row(lines[8])
            with open(os.path.join(paths["cams"], cam_file), "w") as f:
                for line in lines:
                    f.write(line + "\n")
            raw = os.path.join(input_folder, "Depths_raw", scan)
            depth = data_io.read_map(os.path.join(raw, "depth_map_{:0>4}.pfm".format(view_id)), 800)[44:556, 80:720]
            data_io.save_map(os.path.join(paths["depth_gt"], "{:0>8}.pfm".format(view_id)), depth)
            mask = data_io.read_image(os.path.join(raw, "depth_visual_{:0>4}.png".format(view_id)), 800)[0]
            data_io.save_image(os.path.join(paths["masks"], "{:0>8}.png".format(view_id)), mask[44:556, 80:720] > 0.04)
            for light in range(7):
                light_path = os.path.join(paths["images"], str(light))
                os.makedirs(light_path, exist_ok=True)
                image = Image.open(os.path.join(input_folder, "Rectified", "{}_train".format(scan),
                                                "rect_{:0>3}_{}_r5000.png".format(view_id + 1, light)))
                image.save(os.path.join(light_path, "{:0>8}.jpg".format(view_id)))


def main(argv: Optional[Sequence[str]] = None) -> int:
    args = build_parser().parse_args(argv)
    convert(args.input_folder, args.output_folder, args.scan_list)
    return 0


if __name__ == "__main__":
    sys.exit(main())
