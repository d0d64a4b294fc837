"""Generate tests/golden/multisize_case.pt from the UNMODIFIED reference: requests whose views differ in size.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet) and cv2; tests/golden/weights_000007.pt must exist
(make_golden.py writes it):

    python tests/golden/make_multisize_golden.py <path to the reference checkout>

Two parts, inputs from tests/multisize_cases.py:
    net   PatchmatchNet.forward (CPU, eval) on a 1 + 4 view request with three distinct sizes after adjust_image_dims, a
          portrait source and a source whose size is not a multiple of 8: depth, confidence and the per-stage maps, plus
          the checksum of the inputs.
    geo   check_geometric_consistency (eval.py:149-190, executed from eval.py's own source text as make_geo_golden.py does)
          of one reference view against source depth maps of three sizes, and filter_depth's accumulation (eval.py:226-256)
          on top: per-view masks and reprojected depths, geo_mask_sum, photo / final masks, averaged depth.
"""
import os
import sys
import warnings
from typing import Tuple

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
REFERENCE = os.path.abspath(sys.argv[1])
sys.path.insert(0, REFERENCE)
warnings.filterwarnings("ignore")

from models.net import PatchmatchNet as RefNet  # noqa: E402

from tests import multisize_cases, pm_cases  # noqa: E402


def net_part():
    weights = torch.load(os.path.join(HERE, "weights_000007.pt"), map_location="cpu")
    net = RefNet(**pm_cases.NET_KWARGS)
    net.load_state_dict(weights, strict=True)
    net.eval()
    inp = multisize_cases.make_net_inputs()
    with torch.no_grad():
        torch.manual_seed(multisize_cases.NET_SEED + 1000)
        depth, conf, per_stage = net([im.clone() for im in inp["images"]], inp["intrinsics"].clone(), inp["extrinsics"].clone(),
                                     inp["depth_min"], inp["depth_max"])
    print("net", tuple(depth.shape), float(depth.mean()), float(conf.mean()))
    return {"checksum": pm_cases.checksum(inp), "depth": depth.clone(), "confidence": conf.clone(),
            "per_stage": {k: [d.clone() for d in v] for k, v in per_stage.items()}}


def geo_part():
    src = open(os.path.join(REFERENCE, "eval.py")).read()
    ns = {"np": np, "cv2": cv2, "Tuple": Tuple}
    exec(src[src.index("def reproject_with_depth("):src.index("def filter_depth(")], ns)
    sc = multisize_cases.make_geo_scene(seed=0)
    geo_mask_sum = 0
    all_src, masks = [], []
    for d, k, e in zip(sc["src_depths"], sc["src_Ks"], sc["src_Es"]):
        geo_mask, depth_reprojected = ns["check_geometric_consistency"](sc["ref_depth"], sc["ref_K"], sc["ref_E"], d, k, e, 1.0, 0.01)
        geo_mask_sum += geo_mask.astype(np.int32)      # eval.py:248
        all_src.append(depth_reprojected)              # eval.py:249
        masks.append(geo_mask)
    depth_est_averaged = (sum(all_src) + sc["ref_depth"]) / (geo_mask_sum + 1)  # eval.py:252
    photo_mask = sc["confidence"] > 0.8                # eval.py:220
    final_mask = np.logical_and(photo_mask, geo_mask_sum >= 3)                  # eval.py:254-255
    print("geo: mask sum histogram", np.bincount(geo_mask_sum.ravel()), "final mask mean", final_mask.mean())
    t = torch.from_numpy
    return {"geo_mask_sum": t(geo_mask_sum), "photo_mask": t(photo_mask), "final_mask": t(final_mask),
            "depth_est_averaged": t(depth_est_averaged), "per_view_masks": [t(m) for m in masks],
            "per_view_depths": [t(d) for d in all_src]}


if __name__ == "__main__":
    torch.set_num_threads(8)
    torch.save({"net": net_part(), "geo": geo_part()}, os.path.join(HERE, "multisize_case.pt"))
    print("multisize_case.pt", os.path.getsize(os.path.join(HERE, "multisize_case.pt")))
