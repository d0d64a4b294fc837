"""Pin the oracle bit for bit against what the UNMODIFIED reference computed on the same seeded inputs: its PatchMatch
stages and network (tests/golden/stage_cases.pt, net_case.pt, written by tests/golden/make_golden.py with the reference's
torch.rand stream seeded) and its warping / sampling-grid helpers (tests/golden/reference_vectors.pt, written by
tests/golden/make_reference_vectors.py)."""
import os

import pytest
import torch

from oracle import pm_oracle
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state
from tests import pm_cases

VECTORS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_vectors.pt")


def _oracle_stage(weights, stage):
    mod = pm_oracle.PatchMatchOracle(**pm_cases.stage_ctor_kwargs(stage))
    missing, unexpected = mod.load_state_dict(pm_cases.stage_state(weights, stage), strict=True)
    assert not missing and not unexpected
    return mod.eval()


@pytest.mark.parametrize("name", list(pm_cases.STAGE_CASES))
def test_stage_bit_identical(golden_stage_cases, golden_weights, name):
    gold = golden_stage_cases[name]
    spec = pm_cases.STAGE_CASES[name]
    case = pm_cases.make_stage_inputs(spec)
    assert pm_cases.checksum(case) == gold["checksum"], "seeded inputs differ from the ones the reference ran on"
    kw = {k: case[k] for k in ("ref_feature", "src_features", "ref_proj", "src_projs", "depth_min", "depth_max", "depth", "view_weights")}
    mod = _oracle_stage(golden_weights, spec["stage"])
    with torch.no_grad():
        torch.manual_seed(spec["seed"] + 1000)  # the reference drew its random hypotheses from this stream
        b = mod(**kw)
    assert len(b[0]) == len(gold["depths"])
    for x, y in zip(gold["depths"], b[0]):
        assert torch.equal(x, y)
    assert torch.equal(gold["score"], b[1]) and torch.equal(gold["view_weights"], b[2])


def test_warp_and_helpers_bit_identical():
    ref = torch.load(VECTORS, map_location="cpu")
    case = pm_cases.make_stage_inputs(pm_cases.STAGE_CASES["stage2_small"])
    B, C, H, W = case["ref_feature"].shape
    depth, offsets = pm_cases.warp_case_inputs(B, H, W)  # the first depth plane is behind the camera
    assert pm_cases.checksum({"depth": depth, **offsets}) == ref["checksum"], "seeded inputs differ from the ones the reference ran on"
    b = pm_oracle.homography_warp(case["src_features"][0], case["src_projs"][0], case["ref_proj"], depth)
    assert torch.equal(ref["warped"], b)
    assert float(b[:, :, 0].abs().max()) == 0.0
    # neighbour tables + grid
    for kind, count in (("propagation", 16), ("evaluation", 9)):
        g_or = pm_oracle.sampling_grid(pm_oracle.neighbour_table(kind, count, ref["dilation"]), offsets[kind], H, W)
        assert torch.equal(ref["grids"][kind], g_or)


def test_full_network_bit_identical(golden_weights, golden_net_case):
    mine = PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=pm_oracle.PatchMatchOracle)
    load_reference_state(mine, golden_weights)
    mine.eval()
    mine.stack_views = False  # the reference runs FeatureNet view by view
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    assert pm_cases.checksum(inp) == golden_net_case["checksum"]
    with torch.no_grad():
        torch.manual_seed(pm_cases.NET_CASE["seed"] + 1000)
        b = mine([i.clone() for i in inp["images"]], inp["intrinsics"].clone(), inp["extrinsics"].clone(), inp["depth_min"], inp["depth_max"])
    assert torch.equal(golden_net_case["depth"], b[0]) and torch.equal(golden_net_case["confidence"], b[1])
    assert set(golden_net_case["per_stage"]) == set(b[2])
    for s, ds in golden_net_case["per_stage"].items():
        for x, y in zip(ds, b[2][s]):
            assert torch.equal(x, y)
