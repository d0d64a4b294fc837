"""Generate tests/golden/geo_case.npz from the UNMODIFIED reference's geometric-consistency code.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet) and cv2:

    python tests/golden/make_geo_golden.py <path to the reference checkout>

`eval.py` itself cannot be imported here (it imports `plyfile`, which is absent), so the two functions are executed from
its own source text -- `reproject_with_depth` and `check_geometric_consistency`, eval.py:86-190, byte for byte -- and
the per-view accumulation of `filter_depth` (eval.py:226-256) is applied on top exactly as written there.  Inputs come
from tests/geo_cases.make_scene(seed=0) and are stored with the outputs.
"""
import os
import sys
from typing import Tuple

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
from tests import geo_cases  # noqa: E402

if len(sys.argv) != 2:
    raise SystemExit(__doc__)
src = open(os.path.join(sys.argv[1], "eval.py")).read()
ns = {"np": np, "cv2": cv2, "Tuple": Tuple}
exec(src[src.index("def reproject_with_depth("):src.index("def filter_depth(")], ns)

sc = geo_cases.make_scene(seed=0)
geo_mask_sum = 0
all_src = []
per_view_masks = []
for d, k, e in zip(sc["src_depths"], sc["src_Ks"], sc["src_Es"]):
    geo_mask, depth_reprojected = ns["check_geometric_consistency"](sc["ref_depth"], sc["ref_K"], sc["ref_E"], d, k, e, 1.0, 0.01)
    geo_mask_sum += geo_mask.astype(np.int32)          # eval.py:248
    all_src.append(depth_reprojected)                  # eval.py:249
    per_view_masks.append(geo_mask)
depth_est_averaged = (sum(all_src) + sc["ref_depth"]) / (geo_mask_sum + 1)   # eval.py:252
photo_mask = sc["confidence"] > 0.8                    # eval.py:220
final_mask = np.logical_and(photo_mask, geo_mask_sum >= 3)                   # eval.py:254-255
np.savez_compressed(
    os.path.join(HERE, "geo_case.npz"), ref_depth=sc["ref_depth"], ref_K=sc["ref_K"], ref_E=sc["ref_E"],
    src_depths=np.stack(sc["src_depths"]), src_Ks=np.stack(sc["src_Ks"]), src_Es=np.stack(sc["src_Es"]),
    confidence=sc["confidence"], geo_mask_sum=geo_mask_sum, photo_mask=photo_mask, final_mask=final_mask,
    depth_est_averaged=depth_est_averaged, per_view_masks=np.stack(per_view_masks), per_view_depths=np.stack(all_src))
print("wrote geo_case.npz; geo mask sum histogram", np.bincount(geo_mask_sum.ravel()), "final mask mean", final_mask.mean())
