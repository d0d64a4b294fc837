"""Requests whose views differ in size, without a GPU: the oracles against what the unmodified reference computed on such
requests (tests/golden/multisize_case.pt, written by tests/golden/make_multisize_golden.py), the per-view instantiations of
K-A under the lockstep warp emulator (tests/emu_views.cpp) against the oracle, the ragged pack layout, the grouping of
reconstruct's requests into size signatures and the argument checks of the new entry points."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import geo_oracle as go
from oracle import pm_oracle
from patchmatchnet_b200 import _native, ops, synthetic
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state
from patchmatchnet_b200.reconstruct import group_requests, is_uniform
from tests import multisize_cases, pm_cases

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "multisize_case.pt")


@pytest.fixture(scope="module")
def golden_multisize():
    return torch.load(GOLDEN, map_location="cpu")


# ------------------------------------------------------------------------------------------------
# the oracles against the reference
# ------------------------------------------------------------------------------------------------
def test_network_oracle_reproduces_the_reference(golden_weights, golden_multisize):
    gold = golden_multisize["net"]
    mine = PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=pm_oracle.PatchMatchOracle)
    load_reference_state(mine, golden_weights)
    mine.eval()
    inp = multisize_cases.make_net_inputs()
    assert pm_cases.checksum(inp) == gold["checksum"], "seeded inputs differ from the ones the reference ran on"
    assert len({tuple(im.shape[-2:]) for im in inp["images"]}) == 4
    with torch.no_grad():
        torch.manual_seed(multisize_cases.NET_SEED + 1000)
        b = mine([i.clone() for i in inp["images"]], inp["intrinsics"].clone(), inp["extrinsics"].clone(), inp["depth_min"], inp["depth_max"])
    assert torch.equal(gold["depth"], b[0]) and torch.equal(gold["confidence"], b[1])
    assert set(gold["per_stage"]) == set(b[2])
    for s, ds in gold["per_stage"].items():
        for x, y in zip(ds, b[2][s]):
            assert torch.equal(x, y)


def test_geo_oracle_reproduces_the_reference(golden_multisize):
    gold = golden_multisize["geo"]
    sc = multisize_cases.make_geo_scene(seed=0)
    assert len({d.shape for d in sc["src_depths"]}) == 4
    for i, (d, k, e) in enumerate(zip(sc["src_depths"], sc["src_Ks"], sc["src_Es"])):
        m, rep = go.check_geometric_consistency(sc["ref_depth"], sc["ref_K"], sc["ref_E"], d, k, e, 1.0, 0.01)
        assert np.array_equal(m, gold["per_view_masks"][i].numpy())
        assert np.array_equal(rep, gold["per_view_depths"][i].numpy())
    photo, msum, final, avg = go.fuse_reference_view(sc["ref_depth"], sc["ref_K"], sc["ref_E"], sc["src_depths"], sc["src_Ks"],
                                                     sc["src_Es"], sc["confidence"])
    assert np.array_equal(photo, gold["photo_mask"].numpy()) and np.array_equal(msum, gold["geo_mask_sum"].numpy())
    assert np.array_equal(final, gold["final_mask"].numpy()) and np.array_equal(avg, gold["depth_est_averaged"].numpy())
    assert 0.05 < final.mean() < 0.95


# ------------------------------------------------------------------------------------------------
# K-A per-view instantiations under the warp emulator
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_views():
    src = os.path.join(REPO, "tests", "emu_views.cpp")
    deps = [src, os.path.join(REPO, "tests", "warp_emu.h"), os.path.join(REPO, "include", "patchmatch_b200.h")]
    deps += [os.path.join(REPO, "patchmatchnet_b200", "csrc", f) for f in ("pm_kernels.cu", "pm_math.cuh", "pm_warpcorr4.cuh")]
    out = os.path.join(REPO, "tests", "_emu_views.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")  # vector_types.h only
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-I{cuda_inc}", "-o", out, src], check=True,
                       cwd=os.path.join(REPO, "tests"))
    lib = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    PV = ctypes.POINTER(_native.ViewExtent)
    lib.emu_warp_corr3_views.argtypes = [P, P, PV] + [P] * 3 + [ctypes.POINTER(_native.MlpStruct), P, P] + [I] * 11
    lib.emu_warp_corr3_views.restype = I
    lib.emu_warp_corr_generic_views.argtypes = [P, P, PV] + [P] * 4 + [I] * 7
    lib.emu_warp_corr_generic_views.restype = I
    return lib


def _aligned(n):
    """zeroed float32 buffer of n floats whose storage is 32-byte aligned (what the 256-bit gather loads require)"""
    buf = torch.zeros(n + 8, dtype=torch.float32)
    shift = (-buf.data_ptr() // 4) % 8
    return buf[shift:shift + n]


def nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


def maxabs(a, b):
    return float((a.detach().double().cpu() - b.detach().double().cpu()).abs().max())


def _ragged(srcs, C):
    """host ViewPack of NCHW maps, laid out exactly as ops.pack_nhwc_views lays them out"""
    B = srcs[0].shape[0]
    shapes = [tuple(s.shape[-2:]) for s in srcs]
    offsets, total = ops.ViewPack.layout(shapes, B, C)
    data = _aligned(total)
    for s, o in zip(srcs, offsets):
        data[o:o + s.numel()] = nhwc(s).reshape(-1)
    return ops.ViewPack(data, offsets, [h for h, _ in shapes], [w for _, w in shapes], B, C)


def _sized_case(B, C, H, W, D, sizes, seed=0):
    """reference map [B,C,H,W], one source map per entry of `sizes`, cameras seeing a common scene: each source's intrinsics
    are the stage-3 intrinsics of a camera whose image has that source's size"""
    g = torch.Generator().manual_seed(seed)
    ref = torch.randn(B, C, H, W, generator=g)
    srcs = [torch.randn(B, C, h, w, generator=g) for h, w in sizes]
    Kc, Ec = synthetic.make_cameras(B, len(sizes) + 1, H * 8, W * 8)
    for i, (h, w) in enumerate(sizes):
        Kc[:, i + 1, 0, 2] = w * 4
        Kc[:, i + 1, 1, 2] = h * 4
    ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 3)
    depth = 350.0 + 700.0 * torch.rand(B, D, H, W, generator=g)
    depth = torch.sort(depth, dim=1)[0]
    depth[:, 0, : max(1, H // 4)] = -20.0  # behind the camera -> exactly 0
    vw = torch.rand(B, len(sizes), H, W, generator=g)
    return ref, srcs, ref_proj.contiguous(), [m.contiguous() for m in src_projs], depth, vw


def _rt(ref_proj, src_projs):
    inv = torch.linalg.inv(ref_proj.double())
    rows = []
    for sp in src_projs:
        rel = sp.double() @ inv
        rows.append(torch.cat([rel[:, :3, :3].reshape(-1, 9), rel[:, :3, 3]], dim=1))
    return torch.stack(rows).float().contiguous()


def _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G):
    return torch.stack([pm_oracle.groupwise_correlation(pm_oracle.homography_warp(s, sp, ref_proj, depth), ref, G)
                        for s, sp in zip(srcs, src_projs)])


# (C, G, H, W, D, B, source sizes): sizes from 1x1 up to larger than the reference, portrait and landscape
KA_VIEW_CASES = [
    (64, 8, 9, 13, 20, 1, [(9, 13), (13, 9), (1, 1), (15, 22)]),
    (32, 8, 10, 11, 16, 2, [(7, 12), (10, 11), (14, 6)]),
    (16, 4, 7, 19, 8, 1, [(19, 7), (1, 3), (7, 19), (11, 25), (2, 1)]),
]


def _configs(C):
    ppw = 32 // (C // 8)
    return [(dc, pipe) for dc in (4, 8, 16) for pipe in (0, 1) if (ppw * dc) % 32 == 0]


@pytest.mark.parametrize("C,G,H,W,D,B,sizes", KA_VIEW_CASES)
def test_emulated_views_kernel_matches_oracle(emu_views, C, G, H, W, D, B, sizes):
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, sizes, seed=C + D)
    V = len(sizes)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    scale = max(1.0, float(want.abs().max()))
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + vw.sum(1))[:, None, None]
    pack, rt = _ragged(srcs, C), _rt(ref_proj, src_projs)
    ref_n = _aligned(ref.numel()).view(B, H, W, C)
    ref_n.copy_(nhwc(ref))
    depth_c, vw_c = depth.contiguous(), vw.contiguous()
    for dc, pipe in _configs(C):
        got = torch.full((V, B, G, D, H, W), -77.0)
        assert emu_views.emu_warp_corr3_views(ref_n.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth_c.data_ptr(),
                                              None, None, got.data_ptr(), None, 1, V, B, C, G, H, W, D, 0, dc, pipe) == 0
        assert maxabs(got, want) <= 2e-5 * scale, (dc, pipe)
        for v, (h, w) in enumerate(sizes):  # behind the camera -> exactly 0 (a 1-pixel extent maps every point onto its pixel)
            if h > 1 and w > 1:
                assert float(got[v, :, :, 0, : max(1, H // 4)].abs().max()) == 0.0
        got_f = torch.full((B, G, D, H, W), -77.0)
        assert emu_views.emu_warp_corr3_views(ref_n.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth_c.data_ptr(),
                                              vw_c.data_ptr(), None, got_f.data_ptr(), None, 1, V, B, C, G, H, W, D, 1, dc, pipe) == 0
        assert maxabs(got_f, want_f) <= 2e-5 * scale, (dc, pipe)


@pytest.mark.parametrize("C,G", [(12, 3), (32, 8)])
def test_emulated_generic_views_kernel_matches_oracle(emu_views, C, G):
    B, H, W, D = 1, 6, 9, 5
    sizes = [(6, 9), (9, 6), (1, 1), (8, 12)]
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, sizes, seed=3)
    V = len(sizes)
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    scale = max(1.0, float(want.abs().max()))
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + vw.sum(1))[:, None, None]
    pack, rt = _ragged(srcs, C), _rt(ref_proj, src_projs)
    ref_n, depth_c, vw_c = nhwc(ref), depth.contiguous(), vw.contiguous()
    got = torch.full((V, B, G, D, H, W), -77.0)
    assert emu_views.emu_warp_corr_generic_views(ref_n.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth_c.data_ptr(),
                                                 None, got.data_ptr(), V, B, C, G, H, W, D) == 0
    assert maxabs(got, want) <= 2e-5 * scale
    got_f = torch.full((B, G, D, H, W), -77.0)
    assert emu_views.emu_warp_corr_generic_views(ref_n.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth_c.data_ptr(),
                                                 vw_c.data_ptr(), got_f.data_ptr(), V, B, C, G, H, W, D) == 0
    assert maxabs(got_f, want_f) <= 2e-5 * scale


# ------------------------------------------------------------------------------------------------
# ragged pack layout
# ------------------------------------------------------------------------------------------------
def test_view_pack_layout():
    shapes = [(1, 1), (64, 80), (80, 64), (7, 13), (3, 5)]
    for B, C in ((1, 64), (2, 32), (1, 16), (3, 12)):
        offsets, total = ops.ViewPack.layout(shapes, B, C)
        assert offsets[0] == 0
        ends = [o + B * h * w * C for o, (h, w) in zip(offsets, shapes)]
        for o, e, nxt in zip(offsets, ends, offsets[1:] + [total]):
            assert o % ops.ViewPack.ALIGN_FLOATS == 0 and o % 4 == 0  # 256-byte views: aligned 16- and 32-byte gathers
            assert e <= nxt < e + ops.ViewPack.ALIGN_FLOATS  # no overlap, no more padding than the alignment needs
        assert total % ops.ViewPack.ALIGN_FLOATS == 0
    pack = ops.ViewPack(torch.zeros(total), offsets, [h for h, _ in shapes], [w for _, w in shapes], 3, 12)
    assert [(e.offset, e.height, e.width) for e in pack.extents] == [(o, h, w) for o, (h, w) in zip(offsets, shapes)]
    assert pack.view(2).shape == (3, 80, 64, 12)


# ------------------------------------------------------------------------------------------------
# reconstruct: size signatures
# ------------------------------------------------------------------------------------------------
L, P, S = (1200, 1600), (1600, 1200), (600, 800)


def test_group_requests_with_duplicates_keeps_order():
    sigs = [(L, L, P), (L, L, L), (L, L, P), (P, L, L), (L, L, L), (L, L, P)]
    groups = group_requests(sigs)
    assert list(groups) == [(L, L, P), (L, L, L), (P, L, L)]
    assert groups[(L, L, P)] == [0, 2, 5] and groups[(L, L, L)] == [1, 4] and groups[(P, L, L)] == [3]
    assert not is_uniform((L, L, P)) and is_uniform((L, L, L)) and is_uniform((P,))


def test_group_requests_uniform_scan_is_one_group():
    sigs = [(L,) * 6] * 9
    assert group_requests(sigs) == {(L,) * 6: list(range(9))}


def test_group_requests_every_signature_different():
    sigs = [(L, P, S), (P, L, S), (S, L, P), (L, S, P), (L, L, S)]
    groups = group_requests(sigs)
    assert list(groups.values()) == [[0], [1], [2], [3], [4]]
    # a request's views are its signature, in request order: the same views in another order are another signature
    assert len(group_requests([(L, P), (P, L)])) == 2
    assert group_requests([]) == {}


# ------------------------------------------------------------------------------------------------
# argument checks of the new entry points (each returns PMB200_EINVAL before touching the GPU)
# ------------------------------------------------------------------------------------------------
def _have_library():
    try:
        _native.lib()
        return True
    except _native.NativeLibraryMissing:
        return False


BAD_EXTENTS = {
    "zero height": (0, 0, 8),
    "negative width": (0, 8, -1),
    "too many pixels for the tap key": (0, 1 << 15, 1 << 14),
    "misaligned offset": (6, 8, 8),
    "negative offset": (-4, 8, 8),
    "pack beyond 32-bit tap indices": ((1 << 33) - 64, 8, 8),
}


@pytest.mark.skipif(not _have_library(), reason="libpmb200.so is not built")
@pytest.mark.parametrize("bad", list(BAD_EXTENTS))
def test_views_entry_points_reject_malformed_extents(bad):
    lib = _native.lib()
    V, B, C, G, H, W, D = 2, 1, 32, 8, 8, 8, 4
    ext = (_native.ViewExtent * V)()
    ext[0].offset, ext[0].height, ext[0].width = 0, 8, 8
    ext[1].offset, ext[1].height, ext[1].width = BAD_EXTENTS[bad]
    fake = 1 << 20  # never dereferenced: the checks run first
    head = _native.MlpStruct()
    assert lib.pmb200_warp_corr_views(fake, fake, ext, fake, fake, None, fake, V, B, C, G, H, W, D, None) == -1
    assert lib.pmb200_warp_corr_score_views(fake, fake, ext, fake, fake, fake, head, fake, 1, V, B, C, G, H, W, D, None) == -1
    assert lib.pmb200_warp_corr_view_weights_views(fake, fake, ext, fake, fake, head, fake, None, V, B, C, G, H, W, D, None) == -1
    if bad in ("zero height", "negative width", "negative offset"):
        assert lib.pmb200_geometric_filter_views(fake, fake, fake, ext, fake, V, H, W, 1.0, 0.01, 0.8, 3, fake, fake, fake, fake, None) == -1


@pytest.mark.skipif(not _have_library(), reason="libpmb200.so is not built")
def test_views_entry_points_reject_bad_view_counts_and_null_extents():
    lib = _native.lib()
    fake = 1 << 20
    ext = (_native.ViewExtent * 65)()
    for e in ext:
        e.offset, e.height, e.width = 0, 4, 4
    head = _native.MlpStruct()
    for V in (0, 17):
        assert lib.pmb200_warp_corr_views(fake, fake, ext, fake, fake, None, fake, V, 1, 32, 8, 4, 4, 4, None) == -1
        assert lib.pmb200_warp_corr_score_views(fake, fake, ext, fake, fake, fake, head, fake, 1, V, 1, 32, 8, 4, 4, 4, None) == -1
        assert lib.pmb200_warp_corr_view_weights_views(fake, fake, ext, fake, fake, head, fake, None, V, 1, 32, 8, 4, 4, 4, None) == -1
    for V in (0, 65):
        assert lib.pmb200_geometric_filter_views(fake, fake, fake, ext, fake, V, 4, 4, 1.0, 0.01, 0.8, 3, fake, fake, fake, fake, None) == -1
    assert lib.pmb200_warp_corr_views(fake, fake, None, fake, fake, None, fake, 2, 1, 32, 8, 4, 4, 4, None) == -1
    assert lib.pmb200_geometric_filter_views(fake, fake, fake, None, fake, 2, 4, 4, 1.0, 0.01, 0.8, 3, fake, fake, fake, fake, None) == -1
    # the fast path's 256-bit loads need a 32-byte aligned pack
    assert lib.pmb200_warp_corr_views(fake, fake + 16, ext, fake, fake, None, fake, 2, 1, 32, 8, 4, 4, 4, None) == -1
