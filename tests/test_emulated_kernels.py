"""The CUDA kernels' own source, executed on the CPU by the lockstep warp emulator (tests/warp_emu.h), against the oracle.

pm_kernels.cu is compiled by g++ with -DPM_EMU (tests/emu_kernels.cpp); every CUDA thread of a block is a fiber, warp
collectives and barriers synchronise them.  This checks, without a GPU, what the GPU parity tests check on the box -- lane
mappings, the per-pixel layered cell numbering, shuffles, shared-memory plumbing, epilogues -- at small sizes, and for MORE
launch configurations (rows per warp pass, gather pipelining) than the GPU suite sweeps.  Numerics: the emulated build
computes in the same fp32 operation order except for FMA contraction and the fast reciprocal/exponential intrinsics, so the
GPU tests' tolerances apply unchanged.  TEST INFRASTRUCTURE: nothing here is on the product path."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from oracle import pm_oracle
from patchmatchnet_b200 import _native, synthetic
from tests import pm_cases

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="session")
def emu():
    srcs = [os.path.join(REPO, "tests", f) for f in ("emu_kernels.cpp", "emu_backward.cpp")]
    deps = srcs + [os.path.join(REPO, "tests", "warp_emu.h"), os.path.join(REPO, "include", "patchmatch_b200.h")]
    deps += [os.path.join(REPO, "patchmatchnet_b200", "csrc", f) for f in ("pm_kernels.cu", "pm_backward.cu", "pm_math.cuh", "pm_warpcorr4.cuh")]
    out = os.path.join(REPO, "tests", "_emu_kernels.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")  # vector_types.h only
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-I{cuda_inc}", "-o", out] + srcs, check=True, cwd=os.path.join(REPO, "tests"))
    lib = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.emu_warp_corr3.argtypes = [P] * 5 + [ctypes.POINTER(_native.MlpStruct), P, P] + [I] * 13
    lib.emu_warp_corr3.restype = I
    lib.emu_warp_corr4.argtypes = [P] * 5 + [ctypes.POINTER(_native.MlpStruct), P, P] + [I] * 15
    lib.emu_warp_corr4.restype = I
    lib.emu_adaptive_eval.argtypes = [P] * 5 + [I] + [P] * 5 + [I] * 6 + [ctypes.c_float, I, I, I]
    lib.emu_adaptive_eval.restype = I
    lib.emu_init_propagate.argtypes = [P, P, I, P, P, P, P, I, I, I, I, I, I, I, I, ctypes.c_float]
    lib.emu_init_propagate.restype = I
    lib.emu_offset_corr.argtypes = [P, P, I, ctypes.POINTER(_native.MlpStruct), P] + [I] * 7
    lib.emu_offset_corr.restype = I
    F32 = ctypes.c_float
    LL = ctypes.c_longlong
    lib.emu_relative_projection.argtypes = [P, LL, P, LL, I, I, P]
    lib.emu_pack_nhwc.argtypes = [P, I, I, I, I, I, P]
    lib.emu_photometric_confidence.argtypes = [P, P] + [I] * 6
    lib.emu_upsample2x_add_nhwc.argtypes = [P] * 4 + [I] * 4
    lib.emu_aggregate_views.argtypes = [P] * 3 + [I] * 6
    lib.emu_aggregate_views_score.argtypes = [P, P, ctypes.POINTER(_native.MlpStruct), P] + [I] * 7
    lib.emu_warp_corr_generic.argtypes = [P] * 6 + [I] * 9
    for fn in ("emu_relative_projection", "emu_pack_nhwc", "emu_photometric_confidence", "emu_upsample2x_add_nhwc", "emu_aggregate_views",
               "emu_aggregate_views_score", "emu_warp_corr_generic"):
        getattr(lib, fn).restype = I
    lib.emu_warp_corr_backward.argtypes = [P] * 8 + [I] * 9
    lib.emu_aggregate_views_backward.argtypes = [P] * 5 + [I] * 6
    lib.emu_offset_corr_backward.argtypes = [P] * 4 + [I] * 7
    lib.emu_init_propagate_backward.argtypes = [P] * 6 + [I] * 7 + [F32]
    lib.emu_adaptive_eval_backward.argtypes = [P] * 14 + [I] * 6 + [F32, I]
    for fn in ("emu_warp_corr_backward", "emu_aggregate_views_backward", "emu_offset_corr_backward", "emu_init_propagate_backward",
               "emu_adaptive_eval_backward"):
        getattr(lib, fn).restype = I
    return lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def _aligned(t):
    """contiguous float32 copy whose storage is 32-byte aligned (what the 256-bit gather loads require)"""
    buf = torch.empty(t.numel() + 8, dtype=torch.float32)
    shift = (-buf.data_ptr() // 4) % 8
    out = buf[shift:shift + t.numel()].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 32 == 0
    return out


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def maxabs(a, b):
    return float((a.double() - b.double()).abs().max())


def _warp_case(B, V, C, H, W, D, Hs=None, Ws=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    Hs, Ws = Hs or H, Ws or W
    ref = torch.randn(B, C, H, W, generator=g)
    srcs = [torch.randn(B, C, Hs, Ws, generator=g) for _ in range(V)]
    Kc, Ec = synthetic.make_cameras(B, V + 1, H * 8, W * 8)
    ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 3)
    depth = 350.0 + 700.0 * torch.rand(B, D, H, W, generator=g)
    depth = torch.sort(depth, dim=1)[0]
    depth[:, 0, : max(1, H // 4)] = -20.0  # behind the camera -> exactly 0
    vw = torch.rand(B, V, H, W, generator=g)
    return ref, srcs, ref_proj.contiguous(), [m.contiguous() for m in src_projs], depth, vw


def _rt(ref_proj, src_projs):
    """what pmb200_relative_projection computes: src . inverse(ref) in float64, [V,B,12] float32"""
    inv = torch.linalg.inv(ref_proj.double())
    rows = []
    for sp in src_projs:
        rel = sp.double() @ inv
        rows.append(torch.cat([rel[:, :3, :3].reshape(-1, 9), rel[:, :3, 3]], dim=1))
    return torch.stack(rows).float().contiguous()


def _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G):
    return torch.stack([pm_oracle.groupwise_correlation(pm_oracle.homography_warp(s, sp, ref_proj, depth), ref, G)
                        for s, sp in zip(srcs, src_projs)])


def _run_ka(emu, ref, srcs, rt, depth, G, epi, dc, pipe, vw=None, head=None, keep_sims=False, ostride=1):
    B, C, H, W = ref.shape
    V, D = len(srcs), depth.shape[1]
    Hs, Ws = srcs[0].shape[-2:]
    ref_n = _aligned(nhwc(ref))
    src_n = _aligned(torch.stack([nhwc(s) for s in srcs]))
    shape = {0: (V, B, G, D, H, W), 1: (B, G, D, H, W), 2: (B, D, H, W, ostride), 3: (B, V, H, W)}[epi]
    out = torch.zeros(shape) if epi == 3 else torch.full(shape, -77.0)
    sims = torch.full((V, B, G, D, H, W), -77.0) if keep_sims else None
    depth_c, vw_c = depth.contiguous(), None if vw is None else vw.contiguous()
    out_ptr = out.data_ptr() + 4 * (ostride - 1)  # ostride 2: the .y lane of an interleaved (xnorm, score) buffer
    rc = emu.emu_warp_corr3(_ptr(ref_n), _ptr(src_n), _ptr(rt), _ptr(depth_c), _ptr(vw_c), head, out_ptr, _ptr(sims), ostride,
                            V, B, C, G, H, W, Hs, Ws, D, epi, dc, pipe)
    assert rc == 0, rc
    return (out, sims) if keep_sims else out


KA_SHAPES = [
    (64, 8, 9, 13, 20, 1, 2),  # stage-3 shape class; D not a multiple of the rows per pass
    (32, 8, 10, 11, 16, 2, 2),  # stage 2, batch 2
    (16, 4, 7, 19, 8, 1, 3),  # stage 1: 16 pixels per warp, ragged pixel count
    (16, 4, 5, 6, 5, 1, 1),  # single view, odd hypothesis count
    (64, 8, 3, 3, 1, 1, 2),  # single hypothesis, tiny map
]
# Source-view counts the evaluation configurations run (DTU 5, ETH3D / Tanks and Temples 7, a 10-source pair.txt) and the
# limit PMB200_MAX_VIEWS = 16.  K-A4's producer gives lane v view v's footprint box, and its consumers read view v's
# weight from s_vw[v * PIX + pixel]; with 4 consumer warps (PIX = 32) V = 16 fills all 16 view-weight registers of a lane.
KA_VIEW_SHAPES = [
    (32, 8, 6, 9, 10, 1, 6),  # 6 views: a multiple of the 2- and 3-slot rings, so every item starts in the same slot
    (64, 8, 5, 7, 9, 1, 9),  # 9 views: more footprint boxes than a tile row has pixels (8), odd against the 2- and 4-slot rings
    (16, 4, 6, 11, 8, 1, 16),  # the view limit: every view-weight register of a lane carries a view
]
KA_SHAPES += KA_VIEW_SHAPES


def _configs(C):
    ppw = 32 // (C // 8)
    return [(dc, pipe) for dc in (4, 8, 16) for pipe in (0, 1) if (ppw * dc) % 32 == 0]


@pytest.mark.parametrize("C,G,H,W,D,B,V", KA_SHAPES)
def test_emulated_warp_corr_matches_oracle(emu, C, G, H, W, D, B, V):
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    rt = _rt(ref_proj, src_projs)
    scale = max(1.0, float(want.abs().max()))
    wsum = 1e-5 + vw.sum(1)
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    for dc, pipe in _configs(C):
        got = _run_ka(emu, ref, srcs, rt, depth, G, 0, dc, pipe)
        assert maxabs(got, want) <= 2e-5 * scale, (dc, pipe)
        assert float(got[:, :, :, 0, : max(1, H // 4)].abs().max()) == 0.0
        got_f = _run_ka(emu, ref, srcs, rt, depth, G, 1, dc, pipe, vw=vw)
        assert maxabs(got_f, want_f) <= 2e-5 * scale, (dc, pipe)


def test_emulated_warp_corr_source_map_of_other_size(emu):
    C, G, H, W, D, B, V = 32, 8, 12, 20, 8, 1, 2
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, Hs=9, Ws=14, seed=5)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    got = _run_ka(emu, ref, srcs, _rt(ref_proj, src_projs), depth, G, 0, 8, 1)
    assert maxabs(got, want) <= 5e-5 * max(1.0, float(want.abs().max()))


def _random_head(cls, G, seed):
    torch.manual_seed(seed)
    head = cls(G)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.running_mean.normal_(0, 0.3)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    return head.eval()


@pytest.mark.parametrize("C,G,H,W,D,B,V", KA_SHAPES[:4] + KA_VIEW_SHAPES)
def test_emulated_fused_heads_match_unfused(emu, C, G, H, W, D, B, V):
    from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet

    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D + 1)
    rt = _rt(ref_proj, src_projs)
    sims = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    wsum = 1e-5 + vw.sum(1)
    agg = (sims * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    with torch.no_grad():
        sim_head = _random_head(SimilarityNet, G, 1)
        want = sim_head(agg)
        pw = _random_head(PixelwiseNet, G, 2)
        want_vw = torch.cat([pw(sims[v]) for v in range(V)], dim=1)
    for dc, pipe in _configs(C):
        got = _run_ka(emu, ref, srcs, rt, depth, G, 2, dc, pipe, vw=vw, head=sim_head.folded())
        assert maxabs(got[..., 0], want) <= 2e-5 * max(1.0, float(want.abs().max())), (dc, pipe)
        got_vw, kept = _run_ka(emu, ref, srcs, rt, depth, G, 3, dc, pipe, head=pw.folded(), keep_sims=True)
        assert maxabs(got_vw, want_vw) <= 1e-5, (dc, pipe)
        assert maxabs(kept, sims) <= 2e-5 * max(1.0, float(sims.abs().max()))
    # the score epilogue writing the .y lane of an interleaved (xnorm, score) buffer
    dc, pipe = _configs(C)[0]
    xs = _run_ka(emu, ref, srcs, rt, depth, G, 2, dc, pipe, vw=vw, head=sim_head.folded(), ostride=2)
    assert bool((xs[..., 0] == -77.0).all()) and maxabs(xs[..., 1], want) <= 2e-5 * max(1.0, float(want.abs().max()))


# ---- K-A generation 4 (pm_warpcorr4.cuh): persistent producer / consumer pipeline over TMA-staged windows ----------------


def _run_ka4(emu, ref, srcs, rt, depth, G, epi, nw, cap, grid, stages=2, vw=None, head=None, keep_sims=False, ostride=1):
    B, C, H, W = ref.shape
    V, D = len(srcs), depth.shape[1]
    Hs, Ws = srcs[0].shape[-2:]
    ref_n = _aligned(nhwc(ref))
    src_n = _aligned(torch.stack([nhwc(s) for s in srcs]))
    shape = {0: (V, B, G, D, H, W), 1: (B, G, D, H, W), 2: (B, D, H, W, ostride), 3: (B, V, H, W)}[epi]
    out = torch.zeros(shape) if epi == 3 else torch.full(shape, -77.0)
    sims = torch.full((V, B, G, D, H, W), -77.0) if keep_sims else None
    depth_c, vw_c = depth.contiguous(), None if vw is None else vw.contiguous()
    out_ptr = out.data_ptr() + 4 * (ostride - 1)
    rc = emu.emu_warp_corr4(_ptr(ref_n), _ptr(src_n), _ptr(rt), _ptr(depth_c), _ptr(vw_c), head, out_ptr, _ptr(sims), ostride,
                            V, B, C, G, H, W, Hs, Ws, D, epi, nw, cap, grid, stages)
    assert rc == 0, rc
    return (out, sims) if keep_sims else out


# (consumer warps, texels per window slot, persistent CTAs, ring depth): a roomy slot with one CTA per item; a slot too small for most
# boxes (clipped windows -> part of the cells take the global path) with 3 CTAs walking all items through the rings; a
# slot of 16 texels (nearly everything from global memory) with a single CTA
KA4_CONFIGS = [(4, 512, 0, 2), (8, 512, 0, 4), (4, 48, 3, 3), (8, 40, 2, 2), (4, 16, 1, 4)]


@pytest.mark.parametrize("C,G,H,W,D,B,V", KA_SHAPES)
def test_emulated_warp_corr4_matches_oracle(emu, C, G, H, W, D, B, V):
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    rt = _rt(ref_proj, src_projs)
    scale = max(1.0, float(want.abs().max()))
    wsum = 1e-5 + vw.sum(1)
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    for nw, cap, grid, st in KA4_CONFIGS:
        got = _run_ka4(emu, ref, srcs, rt, depth, G, 0, nw, cap, grid, st)
        assert maxabs(got, want) <= 2e-5 * scale, (nw, cap, grid, st)
        assert float(got[:, :, :, 0, : max(1, H // 4)].abs().max()) == 0.0  # behind the camera: exactly 0
        got_f = _run_ka4(emu, ref, srcs, rt, depth, G, 1, nw, cap, grid, st, vw=vw)
        assert maxabs(got_f, want_f) <= 2e-5 * scale, (nw, cap, grid, st)


def test_emulated_warp_corr4_source_map_of_other_size(emu):
    C, G, H, W, D, B, V = 32, 8, 12, 20, 8, 1, 2
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, Hs=9, Ws=14, seed=5)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    for nw, cap, grid, st in KA4_CONFIGS[:3]:
        got = _run_ka4(emu, ref, srcs, _rt(ref_proj, src_projs), depth, G, 0, nw, cap, grid, st)
        assert maxabs(got, want) <= 5e-5 * max(1.0, float(want.abs().max()))


def test_emulated_warp_corr4_equals_generation_3(emu):
    """Same inputs through both generations: the per-view similarities agree to rounding (different summation order of the
    channel dot products), on a map large enough for full tiles, clustered hypotheses (long runs of one cell) and a view
    whose footprints leave the source map."""
    C, G, H, W, D, B, V = 32, 8, 21, 37, 16, 1, 3
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=3)
    depth = (600.0 + 4.0 * torch.arange(D).view(1, D, 1, 1) + 30.0 * torch.rand(B, 1, H, W)).expand(B, D, H, W).contiguous()
    rt = _rt(ref_proj, src_projs)
    g3 = _run_ka(emu, ref, srcs, rt, depth, G, 0, 8, 1)
    for nw, cap, grid, st in ((4, 256, 0, 2), (8, 64, 5, 3)):
        g4 = _run_ka4(emu, ref, srcs, rt, depth, G, 0, nw, cap, grid, st)
        assert maxabs(g4, g3) <= 1e-5 * max(1.0, float(g3.abs().max()))


@pytest.mark.parametrize("C,G,H,W,D,B,V", KA_SHAPES[:4] + KA_VIEW_SHAPES)
def test_emulated_warp_corr4_fused_heads_match_unfused(emu, C, G, H, W, D, B, V):
    from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet

    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D + 1)
    rt = _rt(ref_proj, src_projs)
    sims = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    wsum = 1e-5 + vw.sum(1)
    agg = (sims * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    with torch.no_grad():
        sim_head = _random_head(SimilarityNet, G, 1)
        want = sim_head(agg)
        pw = _random_head(PixelwiseNet, G, 2)
        want_vw = torch.cat([pw(sims[v]) for v in range(V)], dim=1)
    for nw, cap, grid, st in KA4_CONFIGS[:4]:
        got = _run_ka4(emu, ref, srcs, rt, depth, G, 2, nw, cap, grid, st, vw=vw, head=sim_head.folded())
        assert maxabs(got[..., 0], want) <= 2e-5 * max(1.0, float(want.abs().max())), (nw, cap, grid, st)
        got_vw, kept = _run_ka4(emu, ref, srcs, rt, depth, G, 3, nw, cap, grid, st, head=pw.folded(), keep_sims=True)
        assert maxabs(got_vw, want_vw) <= 1e-5, (nw, cap, grid, st)
        assert maxabs(kept, sims) <= 2e-5 * max(1.0, float(sims.abs().max()))
    nw, cap, grid, st = KA4_CONFIGS[2]
    xs = _run_ka4(emu, ref, srcs, rt, depth, G, 2, nw, cap, grid, st, vw=vw, head=sim_head.folded(), ostride=2)
    assert bool((xs[..., 0] == -77.0).all()) and maxabs(xs[..., 1], want) <= 2e-5 * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize("D,K,dil,H,W,B,inverse,TP,DY", [(16, 9, 4, 11, 13, 1, False, 32, 4), (8, 9, 6, 9, 14, 2, True, 16, 8),
                                                         (8, 17, 4, 12, 16, 1, False, 16, 16), (5, 9, 2, 7, 7, 1, True, 8, 32),
                                                         (40, 9, 2, 6, 9, 1, False, 32, 8)])
def test_emulated_adaptive_eval_matches_oracle(emu, D, K, dil, H, W, B, inverse, TP, DY):
    g = torch.Generator().manual_seed(D + K)
    dmin, dmax = torch.full((B,), 425.0), torch.full((B,), 935.0)
    scale = 0.0125
    depth = torch.sort(430.0 + 500.0 * torch.rand(B, D, H, W, generator=g), dim=1, descending=inverse)[0].contiguous()
    score0 = (torch.randn(B, D, H, W, generator=g) * 2.0).contiguous()
    off = (torch.randn(B, 2 * K, H, W, generator=g) * 1.5).contiguous()
    fw = (torch.rand(B, K, H, W, generator=g) + 0.05).contiguous()
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), off.view(B, 2 * K, H * W), H, W)
    w = pm_oracle.depth_similarity_weight(depth, dmin, dmax, grid, scale, K) * fw.unsqueeze(1)
    w = w / torch.sum(w, dim=2).unsqueeze(2)
    s = torch.sum(pm_oracle._border_sample(score0, grid).view(B, D, K, H, W) * w, dim=2)
    want_prob = torch.exp(F.log_softmax(s, dim=1))
    want_depth = pm_oracle._Evaluation.regress(depth, want_prob, inverse)
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    xnorm = ((1.0 / depth - inv_max) / (inv_min - inv_max)).contiguous()
    xs = torch.stack([xnorm, score0], dim=-1).contiguous()
    off_cl = off.permute(0, 2, 3, 1).contiguous()  # channels-last memory
    for sc, xn, inter, o, cl in ((score0, None, None, off, 0), (score0, xnorm, None, off_cl, 1), (None, None, xs, off, 0)):
        prob, dep = torch.full((B, D, H, W), -1.0), torch.full((B, H, W), -1.0)
        rc = emu.emu_adaptive_eval(_ptr(sc), _ptr(depth), _ptr(xn), _ptr(inter), _ptr(o), cl, _ptr(fw), _ptr(dmin), _ptr(dmax),
                                   _ptr(prob), _ptr(dep), B, D, H, W, K, dil, scale, 1 if inverse else 0, TP, DY)
        assert rc == 0
        assert maxabs(prob, want_prob) <= 5e-6
        assert pm_cases.rel_l1(dep, want_depth) <= 1e-6
        assert maxabs(prob.sum(1), torch.ones(B, H, W)) <= 1e-5

MODE_RANDOM, MODE_PERTURB, MODE_PASSTHROUGH = 0, 1, 2  # patchmatchnet_b200.ops.MODE_*


@pytest.mark.parametrize(
    "mode,Ns,Kp,dil,H,W,B",
    [
        ("random", 48, 16, 2, 9, 13, 1),  # 64 hypotheses: two per lane
        ("random", 48, 0, 2, 8, 10, 1),
        ("perturb", 16, 16, 2, 11, 9, 2),
        ("perturb", 8, 8, 4, 13, 17, 1),
        ("perturb", 8, 4, 4, 9, 11, 1),
        ("perturb", 8, 0, 6, 12, 15, 2),
        ("perturb", 3, 8, 2, 9, 10, 1),  # odd sample count
        ("perturb", 100, 16, 2, 6, 7, 1),  # > 64 hypotheses: generic path
        ("pass", 1, 8, 2, 9, 10, 1),
    ],
)
def test_emulated_init_propagate_matches_oracle(emu, mode, Ns, Kp, dil, H, W, B):
    g = torch.Generator().manual_seed(Ns + Kp + H)
    dmin = torch.full((B,), 425.0) + torch.arange(B) * 3.0
    dmax = torch.full((B,), 935.0) - torch.arange(B) * 4.0
    scale = 0.025
    if mode == "random":
        u = torch.rand(B, 48, H, W, generator=g)
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, 16, torch.empty(0), u.device, lambda size, device: u)
        seed, m = u, MODE_RANDOM
    else:
        depth = 400.0 + 560.0 * torch.rand(B, 1, H, W, generator=g)
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, Ns, depth, depth.device)
        seed, m = depth, (MODE_PERTURB if mode == "perturb" else MODE_PASSTHROUGH)
    off, want = None, init
    if Kp > 0:
        off = (torch.randn(B, 2 * Kp, H, W, generator=g) * 2.0).contiguous()
        grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("propagation", Kp, dil), off.view(B, 2 * Kp, H * W), H, W)
        want = pm_oracle.propagate(init, grid)
    D = Ns + Kp
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    want_x = (1.0 / want - inv_max) / (inv_min - inv_max)
    seed = seed.contiguous()
    for cl in (0, 1):
        o = off if (off is None or not cl) else off.permute(0, 2, 3, 1).contiguous()
        got = torch.full((B, D, H, W), -1.0)
        xs = torch.full((B, D, H, W, 2), -7.0)  # xnorm goes to the .x lane of the interleaved buffer
        rc = emu.emu_init_propagate(_ptr(seed), _ptr(o), cl, _ptr(dmin), _ptr(dmax), _ptr(got), _ptr(xs), 2, m, B, H, W, Ns, Kp, dil, scale)
        assert rc == 0
        assert got.shape == want.shape and pm_cases.rel_l1(got, want) <= 1e-6 and maxabs(got, want) <= 2e-3
        assert maxabs(xs[..., 0], want_x) <= 5e-6 and bool((xs[..., 1] == -7.0).all())
        if Kp > 0:
            assert bool((got[:, 1:] >= got[:, :-1]).all())  # sorted ascending


@pytest.mark.parametrize("C,G,K,dil,H,W,B", [(64, 8, 9, 2, 9, 13, 1), (32, 8, 9, 4, 11, 14, 2), (16, 4, 9, 6, 13, 19, 1), (16, 4, 17, 4, 12, 18, 1)])
def test_emulated_offset_corr_matches_oracle(emu, C, G, K, dil, H, W, B):
    from patchmatchnet_b200.patchmatch import FeatureWeightNet

    g = torch.Generator().manual_seed(K + C)
    ref = torch.randn(B, C, H, W, generator=g)
    off = (torch.randn(B, 2 * K, H, W, generator=g) * 2.5).contiguous()
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), off.view(B, 2 * K, H * W), H, W)
    want = pm_oracle._FeatureWeightHead(K, G).neighbour_correlation(ref, grid)  # [B,G,K,H,W]
    ref_n = _aligned(nhwc(ref))
    got = torch.full((B, G, K, H, W), -1.0)
    assert emu.emu_offset_corr(_ptr(ref_n), _ptr(off), 0, None, _ptr(got), B, C, G, H, W, K, dil) == 0
    assert maxabs(got, want) <= 2e-5 * max(1.0, float(want.abs().max()))
    got_cl = torch.full((B, G, K, H, W), -1.0)
    off_cl = off.permute(0, 2, 3, 1).contiguous()
    assert emu.emu_offset_corr(_ptr(ref_n), _ptr(off_cl), 1, None, _ptr(got_cl), B, C, G, H, W, K, dil) == 0
    assert torch.equal(got_cl, got)
    with torch.no_grad():
        fw = _random_head(lambda gg: FeatureWeightNet(K, gg), G, 3)
        want_fw = fw(want)
    got_fw = torch.full((B, K, H, W), -1.0)
    assert emu.emu_offset_corr(_ptr(ref_n), _ptr(off), 0, fw.folded(), _ptr(got_fw), B, C, G, H, W, K, dil) == 0
    assert maxabs(got_fw, want_fw) <= 1e-5


# ------------------------------------------------------------------------------------------------
# backward kernels (pm_backward.cu) against torch autograd on the oracle -- the CPU twin of tests/test_gpu_backward.py
# ------------------------------------------------------------------------------------------------


def close(got, want, tol=2e-5):
    got, want = got.detach().double(), want.detach().double()
    assert got.shape == want.shape, (got.shape, want.shape)
    scale = max(1e-12, float(want.abs().max()))
    err = float((got - want).abs().max())
    assert err <= tol * scale, f"max err {err:.3e} vs scale {scale:.3e}"


@pytest.mark.parametrize("C,G,H,W,D,B,V", [(64, 8, 7, 9, 6, 1, 2), (32, 8, 9, 10, 8, 2, 2), (16, 4, 9, 14, 5, 1, 3)])
def test_emulated_warp_corr_backward(emu, C, G, H, W, D, B, V):
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C + D)
    rt = _rt(ref_proj, src_projs)
    ref_n, src_n = _aligned(nhwc(ref)), _aligned(torch.stack([nhwc(s) for s in srcs]))
    depth_c, vw_c = depth.contiguous(), vw.contiguous()
    for weighted in (False, True):
        r = ref.clone().requires_grad_(True)
        ss = [s.clone().requires_grad_(True) for s in srcs]
        sims = torch.stack([pm_oracle.groupwise_correlation(pm_oracle.homography_warp(s, sp, ref_proj, depth), r, G) for s, sp in zip(ss, src_projs)])
        if weighted:  # view weights detached, as on every iteration that uses the fused average
            gw = torch.randn(B, G, D, H, W, generator=torch.Generator().manual_seed(2))
            wsum = 1e-5 + vw.sum(1)
            out = (sims * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
        else:
            gw = torch.randn(V, B, G, D, H, W, generator=torch.Generator().manual_seed(1))
            out = sims
        (out * gw).sum().backward()
        d_ref = _aligned(torch.full((B, H, W, C), -3.0))
        d_src = _aligned(torch.full((V, B, H, W, C), -3.0))
        rc = emu.emu_warp_corr_backward(_ptr(ref_n), _ptr(src_n), _ptr(rt), _ptr(depth_c), _ptr(vw_c) if weighted else None, _ptr(gw.contiguous()),
                                        _ptr(d_ref), _ptr(d_src), V, B, C, G, H, W, H, W, D)
        assert rc == 0
        close(d_ref.permute(0, 3, 1, 2), r.grad)
        for v in range(V):
            close(d_src[v].permute(0, 3, 1, 2), ss[v].grad)


def test_emulated_aggregate_views_backward(emu):
    g = torch.Generator().manual_seed(3)
    V, B, G, D, H, W = 3, 2, 8, 6, 5, 7
    sims = torch.randn(V, B, G, D, H, W, generator=g)
    vw = torch.rand(B, V, H, W, generator=g)
    gw = torch.randn(B, G, D, H, W, generator=g)
    s1, w1 = sims.clone().requires_grad_(True), vw.clone().requires_grad_(True)
    agg = (s1 * w1.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + w1.sum(1))[:, None, None]
    (agg * gw).sum().backward()
    d_s, d_w = torch.full_like(sims, -3.0), torch.full_like(vw, -3.0)
    assert emu.emu_aggregate_views_backward(_ptr(sims), _ptr(vw), _ptr(gw), _ptr(d_s), _ptr(d_w), V, B, G, D, H, W) == 0
    close(d_s, s1.grad)
    close(d_w, w1.grad)


@pytest.mark.parametrize("C,G,K,dil,H,W,B", [(64, 8, 9, 2, 9, 13, 1), (32, 8, 9, 4, 11, 14, 1), (16, 4, 17, 4, 12, 16, 1)])
def test_emulated_offset_corr_backward(emu, C, G, K, dil, H, W, B):
    g = torch.Generator().manual_seed(K + C)
    ref = torch.randn(B, C, H, W, generator=g)
    off = (torch.randn(B, 2 * K, H, W, generator=g) * 2.5).contiguous()
    gw = torch.randn(B, G, K, H, W, generator=g)
    o1 = off.clone().requires_grad_(True)
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), o1.view(B, 2 * K, H * W), H, W)
    corr = pm_oracle._FeatureWeightHead(K, G).neighbour_correlation(ref, grid)
    (corr * gw).sum().backward()
    d_off = torch.full_like(off, -3.0)
    assert emu.emu_offset_corr_backward(_ptr(_aligned(nhwc(ref))), _ptr(off), _ptr(gw), _ptr(d_off), B, C, G, H, W, K, dil) == 0
    close(d_off, o1.grad, 5e-5)


@pytest.mark.parametrize("mode,Ns,Kp,dil,H,W,B", [("random", 48, 16, 2, 9, 13, 1), ("perturb", 16, 16, 2, 9, 13, 1), ("perturb", 8, 8, 4, 11, 14, 2), ("perturb", 8, 4, 4, 7, 9, 1)])
def test_emulated_init_propagate_backward(emu, mode, Ns, Kp, dil, H, W, B):
    g = torch.Generator().manual_seed(Ns + Kp)
    dmin, dmax = torch.full((B,), 425.0), torch.full((B,), 935.0)
    scale = 0.025
    off = (torch.randn(B, 2 * Kp, H, W, generator=g) * 2.0).contiguous()
    gw = torch.randn(B, Ns + Kp, H, W, generator=g)
    o1 = off.clone().requires_grad_(True)
    if mode == "random":
        u = torch.rand(B, 48, H, W, generator=g)
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, 16, torch.empty(0), u.device, lambda size, device: u)
        seed, m = u, MODE_RANDOM
    else:
        depth = 430.0 + 500.0 * torch.rand(B, 1, H, W, generator=g)
        init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, Ns, depth, depth.device)
        seed, m = depth, MODE_PERTURB
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("propagation", Kp, dil), o1.view(B, 2 * Kp, H * W), H, W)
    (pm_oracle.propagate(init, grid) * gw).sum().backward()
    d_off = torch.full_like(off, -3.0)
    rc = emu.emu_init_propagate_backward(_ptr(seed.contiguous()), _ptr(off), _ptr(dmin), _ptr(dmax), _ptr(gw), _ptr(d_off), m, B, H, W, Ns, Kp, dil, scale)
    assert rc == 0
    close(d_off, o1.grad, 1e-4)


@pytest.mark.parametrize("D,K,dil,H,W,B,inverse", [(16, 9, 2, 9, 13, 1, False), (8, 9, 6, 11, 14, 1, True), (8, 17, 4, 10, 12, 1, False)])
def test_emulated_adaptive_eval_backward(emu, D, K, dil, H, W, B, inverse):
    g = torch.Generator().manual_seed(D + K)
    dmin, dmax = torch.full((B,), 425.0), torch.full((B,), 935.0)
    scale = 0.0125
    depth = torch.sort(430.0 + 500.0 * torch.rand(B, D, H, W, generator=g), dim=1, descending=inverse)[0].contiguous()
    score0 = (torch.randn(B, D, H, W, generator=g) * 2.0).contiguous()
    off = (torch.randn(B, 2 * K, H, W, generator=g) * 1.5).contiguous()
    fw = (torch.rand(B, K, H, W, generator=g) + 0.05).contiguous()
    gdepth = torch.randn(B, H, W, generator=g)
    gprob = torch.randn(B, D, H, W, generator=g)
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    xnorm = ((1.0 / depth - inv_max) / (inv_min - inv_max)).contiguous()
    for use_prob in (False, True):
        s1, d1, o1, f1 = [t.clone().requires_grad_(True) for t in (score0, depth, off, fw)]
        grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), o1.view(B, 2 * K, H * W), H, W)
        w = pm_oracle.depth_similarity_weight(d1.detach(), dmin, dmax, grid.detach(), scale, K) * f1.unsqueeze(1)
        w = w / torch.sum(w, dim=2).unsqueeze(2)
        s = torch.sum(pm_oracle._border_sample(s1, grid).view(B, D, K, H, W) * w, dim=2)
        prob = torch.exp(F.log_softmax(s, dim=1))
        out = pm_oracle._Evaluation.regress(d1, prob, inverse)
        ((out * gdepth).sum() + ((prob * gprob).sum() if use_prob else 0.0)).backward()
        d_s, d_d, d_o, d_f = [torch.full_like(t, -3.0) for t in (score0, depth, off, fw)]
        prob_c = prob.detach().contiguous()
        rc = emu.emu_adaptive_eval_backward(_ptr(score0), _ptr(depth), _ptr(xnorm), _ptr(off), _ptr(fw), _ptr(dmin), _ptr(dmax), _ptr(prob_c),
                                            _ptr(gdepth), _ptr(gprob) if use_prob else None, _ptr(d_s), _ptr(d_d), _ptr(d_o), _ptr(d_f),
                                            B, D, H, W, K, dil, scale, 1 if inverse else 0)
        assert rc == 0
        for got, want, tol in zip((d_s, d_d, d_o, d_f), (s1.grad, d1.grad, o1.grad, f1.grad), (5e-5, 5e-5, 2e-4, 1e-4)):
            close(got, want, tol)


# ------------------------------------------------------------------------------------------------
# helper kernels
# ------------------------------------------------------------------------------------------------


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    return arr


def test_emulated_relative_projection_matches_inverse(emu):
    Kc, Ec = synthetic.make_cameras(3, 5, 512, 640)
    ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 2)  # views unbound from [B,N,4,4]: batch stride 5*16
    rt = torch.full((len(src_projs), 3, 12), -1.0)
    assert emu.emu_relative_projection(_ptr(ref_proj), ref_proj.stride(0), _ptr_array(src_projs), src_projs[0].stride(0), len(src_projs), 3, _ptr(rt)) == 0
    want = _rt(ref_proj, src_projs)
    for v in range(len(src_projs)):
        assert maxabs(rt[v], want[v]) <= 1e-6 * float(want[v].abs().max())


def test_emulated_pack_nhwc(emu):
    maps = [torch.randn(2, 24, 7, 9) for _ in range(3)]
    out = torch.full((3, 2, 7, 9, 24), -1.0)
    assert emu.emu_pack_nhwc(_ptr_array(maps), 3, 2, 24, 7, 9, _ptr(out)) == 0
    for i, m in enumerate(maps):
        assert torch.equal(out[i], m.permute(0, 2, 3, 1))


def test_emulated_photometric_confidence(emu):
    g = torch.Generator().manual_seed(4)
    for (B, D, h, w, H0, W0) in [(2, 8, 16, 20, 32, 40), (1, 8, 9, 7, 17, 15), (1, 5, 6, 6, 6, 6)]:
        score = torch.softmax(torch.randn(B, D, h, w, generator=g) * 2.0, dim=1).contiguous()
        sum4 = 4 * F.avg_pool3d(F.pad(score.unsqueeze(1), pad=(0, 0, 0, 0, 1, 2)), (4, 1, 1), stride=1, padding=0).squeeze(1)
        idx = torch.sum(score * torch.arange(D, dtype=torch.float).view(1, D, 1, 1), dim=1).unsqueeze(1).long().clamp(0, D - 1)
        want = F.interpolate(torch.gather(sum4, 1, idx), size=[H0, W0], mode="nearest").squeeze(1)
        got = torch.full((B, H0, W0), -1.0)
        assert emu.emu_photometric_confidence(_ptr(score), _ptr(got), B, D, h, w, H0, W0) == 0
        bad = (got - want).abs() > 1e-5  # a pixel whose expectation sits on an integer may flip bins
        assert float(bad.float().mean()) <= 0.002


def test_emulated_upsample2x_add(emu):
    for (N, C, h, w) in [(2, 32, 7, 9), (1, 16, 1, 3)]:
        x = torch.randn(N, C, h, w)
        y = torch.randn(N, C, 2 * h, 2 * w)
        bias = torch.randn(C)
        want = F.interpolate(x, scale_factor=2.0, mode="bilinear", align_corners=False) + y + bias.view(1, C, 1, 1)
        out = torch.full((N, 2 * h, 2 * w, C), -1.0)
        assert emu.emu_upsample2x_add_nhwc(_ptr(_aligned(nhwc(x))), _ptr(_aligned(nhwc(y))), _ptr(_aligned(bias)), _ptr(out), N, h, w, C) == 0
        assert maxabs(out.permute(0, 3, 1, 2), want) <= 1e-5


def test_emulated_aggregate_views_and_score(emu):
    from patchmatchnet_b200.patchmatch import SimilarityNet

    g = torch.Generator().manual_seed(8)
    V, B, G, D, H, W = 3, 2, 8, 6, 5, 7
    sims = torch.randn(V, B, G, D, H, W, generator=g)
    vw = torch.rand(B, V, H, W, generator=g)
    want = (sims * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + vw.sum(1))[:, None, None]
    got = torch.full((B, G, D, H, W), -1.0)
    assert emu.emu_aggregate_views(_ptr(sims), _ptr(vw), _ptr(got), V, B, G, D, H, W) == 0
    assert maxabs(got, want) <= 2e-6 * float(want.abs().max())
    with torch.no_grad():
        head = _random_head(SimilarityNet, G, 1)
        want_s = head(want)
    xs = torch.full((B, D, H, W, 2), -7.0)
    assert emu.emu_aggregate_views_score(_ptr(sims), _ptr(vw), head.folded(), xs.data_ptr() + 4, 2, V, B, G, D, H, W) == 0
    assert bool((xs[..., 0] == -7.0).all()) and maxabs(xs[..., 1], want_s) <= 2e-5 * max(1.0, float(want_s.abs().max()))


@pytest.mark.parametrize("C,G", [(24, 3), (32, 4)])
def test_emulated_generic_warp_corr(emu, C, G):
    B, V, H, W, D = 1, 2, 10, 12, 7
    ref, srcs, ref_proj, src_projs, depth, vw = _warp_case(B, V, C, H, W, D, seed=C)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    rt = _rt(ref_proj, src_projs)
    ref_n, src_n = nhwc(ref), torch.stack([nhwc(s) for s in srcs]).contiguous()
    got = torch.full((V, B, G, D, H, W), -1.0)
    assert emu.emu_warp_corr_generic(_ptr(ref_n), _ptr(src_n), _ptr(rt), _ptr(depth.contiguous()), None, _ptr(got), V, B, C, G, H, W, H, W, D) == 0
    assert maxabs(got, want) <= 2e-5 * max(1.0, float(want.abs().max()))
    wsum = 1e-5 + vw.sum(1)
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / wsum[:, None, None]
    got_f = torch.full((B, G, D, H, W), -1.0)
    assert emu.emu_warp_corr_generic(_ptr(ref_n), _ptr(src_n), _ptr(rt), _ptr(depth.contiguous()), _ptr(vw.contiguous()), _ptr(got_f), V, B, C, G, H, W, H, W, D) == 0
    assert maxabs(got_f, want_f) <= 2e-5 * max(1.0, float(want.abs().max()))
