"""Convert the ETH3D training set from its pre-processed layout to the layout `train` reads -- the counterpart of the
reference's convert_eth3d_dataset.py, writing the same bytes.

    python -m patchmatchnet_b200.convert_eth3d --input-folder eth3d_training --output-folder eth3d_train --scan-list lists/eth3d/train.txt
    python -m patchmatchnet_b200.train --input-folder eth3d_train --image-extension .png ...

Input per scan: cams/index2prefix.txt ("<count>" then "<id> <image name>" lines), cams/pair.txt, cams/%08d_cam.txt,
images/<image name> and depths/<image name without "_undistorted", extension .pfm>.  Output per scan: pair.txt and cams/
(copied), images/%08d.png (copied: the ETH3D images are PNG files), depth_gt/%08d.pfm (copied) and masks/%08d.png
(depth_gt > 0, written by data_io.save_image).  ETH3D's views differ in size between scenes and cameras, so the converted
data usually trains with one sample per rank.
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys
from typing import Optional, Sequence

from . import data_io


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.convert_eth3d",
                                 description="Convert ETH 3D training dataset to standard input format")
    ap.add_argument("--input-folder", type=str, help="Input training data")
    ap.add_argument("--output-folder", type=str, help="Output converted training data")
    ap.add_argument("--scan-list", type=str, help="Input scan list for conversion")
    return ap


def convert(input_folder: str, output_folder: str, scan_list: str) -> None:
    """convert_eth3d_dataset.py:15-68, with its checks and messages."""
    if input_folder is None or not os.path.isdir(input_folder):
        raise Exception("Invalid input folder")
    if output_folder is None or not os.path.isdir(output_folder):
        raise Exception("Invalid output folder")
    if scan_list is None or not os.path.isfile(scan_list):
        raise Exception("Invalid input scan list")

    with open(scan_list) as f:
        scans = [line.rstrip() for line in f.readlines()]
    for scan in scans:
        scan_path = os.path.join(output_folder, scan)
        paths = {k: os.path.join(scan_path, k) for k in ("cams", "depth_gt", "images", "masks")}
        for p in [scan_path] + list(paths.values()):
            os.makedirs(p, exist_ok=True)
        input_cam_path = os.path.join(input_folder, scan, "cams")
        image_index = data_io.read_image_dictionary(os.path.join(input_cam_path, "index2prefix.txt"))
        shutil.copy(os.path.join(input_cam_path, "pair.txt"), os.path.join(scan_path, "pair.txt"))
        for cam_file in os.listdir(input_cam_path):
            if cam_file == "index2prefix.txt" or cam_file == "pair.txt":
                continue
            view_id = int(cam_file.split("_")[0])
            shutil.copy(os.path.join(input_cam_path, cam_file), os.path.join(paths["cams"], cam_file))
            image_filename = os.path.join(input_folder, scan, "images", image_index[view_id])
            shutil.copy(image_filename, os.path.join(paths["images"], "{:0>8}.png".format(view_id)))
            depth_gt_filename = os.path.join(input_folder, scan, "depths", image_index[view_id])
            depth_gt_filename = os.path.splitext(depth_gt_filename.replace("_undistorted", ""))[0] + ".pfm"
            shutil.copy(depth_gt_filename, os.path.join(paths["depth_gt"], "{:0>8}.pfm".format(view_id)))
            mask = (data_io.read_map(depth_gt_filename) > 0.0).squeeze(2).astype(bool)
            data_io.save_image(os.path.join(paths["masks"], "{:0>8}.png".format(view_id)), mask)


def main(argv: Optional[Sequence[str]] = None) -> int:
    args = build_parser().parse_args(argv)
    convert(args.input_folder, args.output_folder, args.scan_list)
    return 0


if __name__ == "__main__":
    sys.exit(main())
