"""The oracle against the committed golden fixtures (generated from the unmodified reference by
tests/golden/make_golden.py).  Needs nothing outside this repository.
Same torch build + CPU => the comparison is tight (1e-6 relative; it is bit-exact in the build box)."""
import pytest
import torch

from oracle import pm_oracle
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state
from tests import pm_cases

TOL = 1e-6


def _oracle_stage(weights, stage):
    mod = pm_oracle.PatchMatchOracle(**pm_cases.stage_ctor_kwargs(stage))
    mod.load_state_dict(pm_cases.stage_state(weights, stage), strict=True)
    return mod.eval()


def _run_stage(weights, spec):
    case = pm_cases.make_stage_inputs(spec)
    mod = _oracle_stage(weights, spec["stage"])
    if case["rand48"] is not None:
        mod.rand_source = lambda size, device: case["rand48"].to(device)
    kw = {k: case[k] for k in ("ref_feature", "src_features", "ref_proj", "src_projs", "depth_min", "depth_max", "depth", "view_weights")}
    with torch.no_grad():
        return case, mod(**kw)


@pytest.mark.parametrize("name", list(pm_cases.STAGE_CASES))
def test_oracle_matches_golden_stage(golden_weights, golden_stage_cases, name):
    gold = golden_stage_cases[name]
    case, out = _run_stage(golden_weights, pm_cases.STAGE_CASES[name])
    assert pm_cases.checksum(case) == gold["checksum"], "seeded inputs differ from the ones the fixture was made with"
    for x, y in zip(out[0], gold["depths"]):
        assert pm_cases.rel_l1(x, y) <= TOL
    assert pm_cases.rel_l1(out[1], gold["score"]) <= 1e-5
    assert pm_cases.rel_l1(out[2], gold["view_weights"]) <= TOL


def test_oracle_matches_golden_config1(golden_weights, golden_config1):
    case, out = _run_stage(golden_weights, pm_cases.CONFIG1)
    assert pm_cases.checksum(case) == golden_config1["checksum"]
    assert pm_cases.rel_l1(out[0][-1], golden_config1["depths"][-1]) <= TOL
    assert pm_cases.rel_l1(out[1], golden_config1["score"]) <= 1e-5


def test_oracle_matches_golden_network(golden_weights, golden_net_case):
    net = PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=pm_oracle.PatchMatchOracle)
    load_reference_state(net, golden_weights)
    net.eval()
    net.stack_views = False
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    assert pm_cases.checksum(inp) == golden_net_case["checksum"]
    net.patchmatch_3.rand_source = lambda size, device: inp["rand48"].to(device)
    with torch.no_grad():
        depth, conf, per_stage = net([i.clone() for i in inp["images"]], inp["intrinsics"].clone(), inp["extrinsics"].clone(), inp["depth_min"], inp["depth_max"])
    assert pm_cases.rel_l1(depth, golden_net_case["depth"]) <= TOL
    assert pm_cases.rel_l1(conf, golden_net_case["confidence"]) <= 1e-5
    for s, ds in golden_net_case["per_stage"].items():
        for x, y in zip(per_stage[s], ds):
            assert pm_cases.rel_l1(x, y) <= TOL
