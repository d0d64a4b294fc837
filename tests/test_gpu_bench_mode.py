"""Parity of the network in the configuration bench.py TIMES (VERDICT r1, weak #1), against the fp32 oracle (the
reference's op sequence in full fp32 on the same device, the stage-3 random draw shared through `rand_source`).

The timed configuration is: `cudnn.allow_tf32 = False` (bench.py's default since round 2) -> every convolution runs on the
native channels-last tensor-core kernel with the error-compensated 3xTF32 split (fp32-accurate), `cudnn.benchmark` on, the
forward replayed from the DepthEngine's CUDA graph.  torch's default flags (TF32 operands in the native and the cuDNN
convs) land outside north_star's 1e-3 relative L1 against the fp32 oracle (tests/analysis_tf32_modes.py shows that even
rounding only the WEIGHTS to TF32 costs more than that), so that mode is not the default; it is still measured here and
reported by bench.py as `value_tf32`, labelled as outside the bound.

Sizes: BASELINE config 2 (640x512, 1+4 views), config 3 (1600x1184, 1+4 views), config 4's per-GPU batch taken to 8
reference views on one GPU (640x512).  Observed values are printed as one JSON line per case (pytest -s shows them)."""
import json

import pytest
import torch

from oracle import pm_oracle
from patchmatchnet_b200 import PatchmatchNet, load_reference_state, ops, synthetic
from tests import pm_cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
NORTH_STAR_TOL = 1e-3


def _net(weights, cls=None):
    net = PatchmatchNet(**pm_cases.NET_KWARGS) if cls is None else PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=cls)
    load_reference_state(net, weights)
    return net.eval().to(DEV)


def _record(row):
    print(json.dumps(row))


@pytest.mark.parametrize("B,H,W,n_views,slots", [(1, 512, 640, 5, 3), (1, 1184, 1600, 5, 1), (8, 512, 640, 5, 1)],
                         ids=["cfg2_640x512", "cfg3_1600x1184", "batch8_640x512"])
def test_timed_configuration_matches_fp32_oracle(golden_weights, B, H, W, n_views, slots):
    from patchmatchnet_b200.engine import DepthEngine

    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark,
           torch.backends.cudnn.deterministic)
    inp = synthetic.make_inputs(B, n_views, H, W, seed=5)
    g = torch.Generator().manual_seed(1234)
    rand48 = torch.rand(B, 48, H // 8, W // 8, generator=g).to(DEV)
    draw = lambda size, device: rand48
    args = lambda: ([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                    inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
    try:
        # ---- the timed configuration: exactly what bench.py sets up ----
        torch.backends.cudnn.allow_tf32 = False         # bench.py default: fp32-accurate convolutions
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.benchmark = True           # bench.py / reference eval.py:301
        torch.backends.cudnn.deterministic = False
        assert ops.conv_precision() == 3, "native convs must run the 3xTF32 split in the timed mode"
        assert ops.conv_prefers_native(64, 64, 3), "every conv is native in the timed mode"
        mine = _net(golden_weights)
        mine.patchmatch_3.rand_source = draw
        eng = DepthEngine(mine, B, n_views, H, W, device=DEV, use_graph=True, n_slots=slots)
        d_timed, c_timed = eng.infer(inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])
        d_timed, c_timed = d_timed.clone(), c_timed.clone()
        d_again, _ = eng.infer(inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])
        assert eng.use_graph and eng._slots[0]["graph"] is not None, "the timed mode replays a CUDA graph"
        replay_drift = pm_cases.rel_l1(d_again, d_timed)
        with torch.no_grad():
            # ---- the fp32 oracle: reference op sequence, full fp32, same device, same random draw ----
            orc = _net(golden_weights, pm_oracle.PatchMatchOracle)
            orc.patchmatch_3.rand_source = draw
            d_orc, c_orc, _ = orc(*args())
        # ---- torch's default flags (TF32 operands), as round 1 timed it: measured, reported, NOT the timed mode ----
        torch.backends.cudnn.allow_tf32 = True
        mine_tf32 = _net(golden_weights)
        mine_tf32.patchmatch_3.rand_source = draw
        with torch.no_grad():
            d_tf32, _, _ = mine_tf32(*args())
        torch.cuda.synchronize()
    finally:
        (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark,
         torch.backends.cudnn.deterministic) = old
    err_timed = pm_cases.rel_l1(d_timed, d_orc)
    err_tf32 = pm_cases.rel_l1(d_tf32, d_orc)
    conf_mean = float((c_timed.cpu() - c_orc.cpu()).abs().mean())
    row = {"case": f"B{B} {W}x{H} 1+{n_views - 1} views", "timed_mode": "fp32-accurate convs (3xTF32), CUDA-graph replay",
           "timed_mode_rel_l1_vs_fp32_oracle": err_timed, "tf32_mode_rel_l1_vs_fp32_oracle": err_tf32,
           "graph_replay_drift": replay_drift, "confidence_mean_abs_diff": conf_mean, "bound": NORTH_STAR_TOL}
    print("bench-mode parity:", json.dumps(row))
    _record(row)
    assert torch.isfinite(d_timed).all() and torch.isfinite(d_tf32).all()
    assert replay_drift <= 1e-6, replay_drift
    assert err_timed <= NORTH_STAR_TOL, err_timed
    assert err_timed <= 2e-4, err_timed  # what the fp32 parity suite holds the network to
    assert err_tf32 <= 2e-2, err_tf32    # sanity only: this mode is documented as outside the 1e-3 bound


def test_eval_mode_with_grad_enabled_is_differentiable(golden_weights):
    """ADVICE r1 (medium): eval() with autograd on must not take the folded / native inference branches (constants built
    under no_grad, cudnn_convolution_relu has no derivative): every FeatureNet / Refinement parameter gets a gradient,
    as in the reference, which is fully differentiable in eval mode."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False  # both paths fp32-accurate, so that they can be compared at the end
    try:
        _eval_mode_grad_body(golden_weights)
    finally:
        torch.backends.cudnn.allow_tf32 = old


def _eval_mode_grad_body(golden_weights):
    net = _net(golden_weights)
    inp = synthetic.make_inputs(1, 3, 64, 80, seed=2)
    fixed = torch.rand(1, 48, 8, 10, device=DEV)
    net.patchmatch_3.rand_source = lambda size, device: fixed
    for p in net.parameters():
        p.grad = None
    with torch.enable_grad():
        depth, conf, per_stage = net([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                                     inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
        assert depth.requires_grad
        # the stages hand each other DETACHED depth maps (reference net.py:270): FeatureNet is reached through the per-stage
        # outputs, which is what the reference's loss sums over (net.py:321-342)
        loss = depth.mean() + sum(d.mean() for s in (3, 2, 1) for d in per_stage[s])
        loss.backward()
    missing = [n for n, p in net.named_parameters()
               if p.grad is None and (n.startswith("feature.") or n.startswith("upsample_net."))]
    assert not missing, missing
    with torch.no_grad():  # and the inference fast path still agrees with it
        d2, _, _ = net([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                       inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
    assert pm_cases.rel_l1(d2, depth) <= NORTH_STAR_TOL
