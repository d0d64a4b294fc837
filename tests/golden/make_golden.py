"""Generate the golden fixtures in this directory from the UNMODIFIED reference.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet), checkpoints included:

    python tests/golden/make_golden.py <path to the reference checkout>

Writes
    weights_000007.pt   the reference's shipped weights (checkpoints/params_000007.ckpt["model"],
                        'module.' prefix stripped, optimizer state dropped)
    stage_cases.pt      reference PatchMatch outputs for small stage-3/2/1 problems (B=2, odd sizes)
    net_case.pt         reference PatchmatchNet outputs for a 1+2-view 64x80 image pair set
    config1_case.pt     BASELINE.json configs[0]: 1 ref + 2 src, 160x128 image, single stage-1
                        PatchMatch, 8 hypotheses (inputs are re-derived from the seed; outputs stored)

Inputs that are cheap to store are stored; large ones are regenerated from the recorded seed by
``tests/pm_cases.py`` (same torch build -> same CPU RNG stream) and guarded by a checksum.
"""
import os
import sys
import warnings

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
from models.patchmatch import PatchMatch as RefPatchMatch  # noqa: E402

from tests import pm_cases  # noqa: E402


def main() -> None:
    torch.set_num_threads(8)
    ck = torch.load(os.path.join(REFERENCE, "checkpoints", "params_000007.ckpt"), map_location="cpu", weights_only=False)["model"]
    weights = {k[len("module."):]: v.clone() for k, v in ck.items()}
    torch.save(weights, os.path.join(HERE, "weights_000007.pt"))

    # ---- stage cases -------------------------------------------------------------------
    stage_out = {}
    for name, spec in pm_cases.STAGE_CASES.items():
        case = pm_cases.make_stage_inputs(spec)
        mod = RefPatchMatch(**pm_cases.stage_ctor_kwargs(spec["stage"]))
        mod.load_state_dict(pm_cases.stage_state(weights, spec["stage"]), strict=True)
        mod.eval()
        with torch.no_grad():
            torch.manual_seed(spec["seed"] + 1000)  # the reference draws torch.rand internally
            depths, score, vw = mod(
                ref_feature=case["ref_feature"], src_features=case["src_features"], ref_proj=case["ref_proj"],
                src_projs=case["src_projs"], depth_min=case["depth_min"], depth_max=case["depth_max"],
                depth=case["depth"], view_weights=case["view_weights"],
            )
        stage_out[name] = {
            "checksum": pm_cases.checksum(case),
            "depths": [d.clone() for d in depths],
            "score": score.clone(),
            "view_weights": vw.clone(),
        }
        print(name, [tuple(d.shape) for d in depths], tuple(score.shape), float(depths[-1].mean()))
    torch.save(stage_out, os.path.join(HERE, "stage_cases.pt"))

    # ---- config 1 of BASELINE.json -------------------------------------------------------
    spec = pm_cases.CONFIG1
    case = pm_cases.make_stage_inputs(spec)
    mod = RefPatchMatch(**pm_cases.stage_ctor_kwargs(1))
    mod.load_state_dict(pm_cases.stage_state(weights, 1), strict=True)
    mod.eval()
    with torch.no_grad():
        depths, score, vw = mod(
            ref_feature=case["ref_feature"], src_features=case["src_features"], ref_proj=case["ref_proj"],
            src_projs=case["src_projs"], depth_min=case["depth_min"], depth_max=case["depth_max"],
            depth=case["depth"], view_weights=case["view_weights"],
        )
    torch.save(
        {"checksum": pm_cases.checksum(case), "depths": [d.clone() for d in depths], "score": score.clone()},
        os.path.join(HERE, "config1_case.pt"),
    )
    print("config1", tuple(depths[-1].shape), float(depths[-1].mean()))

    # ---- full network ------------------------------------------------------------------
    net = RefNet(**pm_cases.NET_KWARGS)
    net.load_state_dict(weights, strict=True)
    net.eval()
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    with torch.no_grad():
        torch.manual_seed(pm_cases.NET_CASE["seed"] + 1000)
        depth, conf, per_stage = net(
            [im.clone() for im in inp["images"]], inp["intrinsics"].clone(), inp["extrinsics"].clone(),
            inp["depth_min"], inp["depth_max"],
        )
    torch.save(
        {
            "checksum": pm_cases.checksum(inp),
            "depth": depth.clone(),
            "confidence": conf.clone(),
            "per_stage": {k: [d.clone() for d in v] for k, v in per_stage.items()},
        },
        os.path.join(HERE, "net_case.pt"),
    )
    print("net", tuple(depth.shape), float(depth.mean()), float(conf.mean()))
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".pt"):
            print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
