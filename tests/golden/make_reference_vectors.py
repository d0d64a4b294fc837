"""Record what the UNMODIFIED reference computes for the tests that compare the oracles with it directly, so that those
comparisons run from this repository alone.  Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet) and cv2:

    python tests/golden/make_reference_vectors.py <path to the reference checkout>

Writes
    reference_vectors.pt    differentiable_warping and PatchMatch.get_grid outputs (tests/test_oracle_vs_reference.py)
    geo_reference.npz       eval.py's reproject_with_depth / check_geometric_consistency on a 72x100 scene with 3 source
                            views, and the body of filter_depth's fusion loop on the same scene (tests/test_geo.py)
    maps/reference_io.npz   bytes datasets/data_io.py writes for ragged maps and PFM scales, the arrays it reads back, and
                            the errors it raises on malformed PFM files (tests/test_mapio.py)
"""
import os
import sys
import warnings
from typing import Tuple

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
warnings.filterwarnings("ignore")

from tests import geo_cases, pm_cases  # noqa: E402
from tests.test_geo import _fusion_case  # noqa: E402
from tests.test_mapio import BAD_PFMS, SCALES, _cases  # noqa: E402


def warp_and_grids(ref_pm, ref_mod):
    case = pm_cases.make_stage_inputs(pm_cases.STAGE_CASES["stage2_small"])
    B, C, H, W = case["ref_feature"].shape
    depth, offsets = pm_cases.warp_case_inputs(B, H, W)
    warped = ref_mod.differentiable_warping(case["src_features"][0], case["src_projs"][0], case["ref_proj"], depth)
    mod = ref_pm.PatchMatch(**pm_cases.stage_ctor_kwargs(3))
    grids = {kind: mod.get_grid(gid, B, H, W, offsets[kind], offsets[kind].device) for kind, gid in (("propagation", 1), ("evaluation", 2))}
    return {"checksum": pm_cases.checksum({"depth": depth, **offsets}), "warped": warped, "grids": grids, "dilation": mod.dilation}


def geo(reference):
    import cv2

    src = open(os.path.join(reference, "eval.py")).read()
    ns = {"np": np, "cv2": cv2, "Tuple": Tuple}
    exec(src[src.index("def reproject_with_depth("):src.index("def filter_depth(")], ns)  # eval.py:86-190, unmodified
    out = {}
    sc = geo_cases.make_scene(seed=3, H=72, W=100, n_src=3)
    for i, (d, k, e) in enumerate(zip(sc["src_depths"], sc["src_Ks"], sc["src_Es"])):
        m, dd = ns["check_geometric_consistency"](sc["ref_depth"], sc["ref_K"], sc["ref_E"], d, k, e, 1.0, 0.01)
        out[f"mask{i}"], out[f"depth_diff{i}"] = m, dd
        for j, a in enumerate(ns["reproject_with_depth"](sc["ref_depth"], sc["ref_K"], sc["ref_E"], d, k, e)):
            out[f"reproject{i}_{j}"] = a
    lines = src.split("\n")
    snippet = "\n".join(line[8:] for line in lines[272:281])  # eval.py:273-281, the body of filter_depth's loop, de-indented
    assert snippet.lstrip().startswith("height, width = depth_est_averaged.shape[:2]") and "vertex_colors.append" in snippet
    fs, final, avg, img = _fusion_case(72, 100, 3, 3)
    fns = dict(np=np, depth_est_averaged=avg, final_mask=final, ref_img=img, ref_intrinsics=fs["ref_K"], ref_extrinsics=fs["ref_E"],
               vertices=[], vertex_colors=[])
    exec(snippet, fns)
    out["fusion_vertices"], out["fusion_colors"] = fns["vertices"][0], fns["vertex_colors"][0]
    return out


def mapio(data_io, tmp):
    out = {}
    for tag, arr in _cases():
        for ext in ("pfm", "bin"):
            p = os.path.join(tmp, f"{tag}.{ext}")
            data_io.save_map(p, arr)
            out[f"{tag}.{ext}.bytes"] = np.frombuffer(open(p, "rb").read(), dtype=np.uint8)
            out[f"{tag}.{ext}.read"] = np.ascontiguousarray(data_io.read_map(p))
    arr = list(_cases())[-1][1]
    p = os.path.join(tmp, "scaled.pfm")
    for i, scale in enumerate(SCALES):
        data_io.save_pfm(p, arr, scale)
        out[f"scaled{i}.bytes"] = np.frombuffer(open(p, "rb").read(), dtype=np.uint8)
        out[f"scaled{i}.scale"] = np.float64(data_io.read_pfm(p)[1])
    for i, blob in enumerate(BAD_PFMS):
        p = os.path.join(tmp, "bad.pfm")
        open(p, "wb").write(blob)
        try:
            data_io.read_pfm(p)
            raise AssertionError("the reference accepted a malformed PFM")
        except Exception as e:  # noqa: BLE001
            out[f"bad{i}.type"], out[f"bad{i}.text"] = np.array(type(e).__name__), np.array(str(e))
    return out


def main() -> None:
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    reference = os.path.abspath(sys.argv[1])
    sys.path.insert(0, reference)
    import models.module as ref_mod
    import models.patchmatch as ref_pm
    from datasets import data_io

    torch.save(warp_and_grids(ref_pm, ref_mod), os.path.join(HERE, "reference_vectors.pt"))
    np.savez_compressed(os.path.join(HERE, "geo_reference.npz"), **geo(reference))
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        np.savez_compressed(os.path.join(HERE, "maps", "reference_io.npz"), **mapio(data_io, tmp))
    for f in ("reference_vectors.pt", "geo_reference.npz", os.path.join("maps", "reference_io.npz")):
        print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
