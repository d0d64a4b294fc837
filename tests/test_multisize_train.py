"""Training on views of different sizes, without a GPU: autograd through the oracle against what the unmodified reference
computed on such requests in train() mode (tests/golden/multisize_train_case.pt, written by
tests/golden/make_multisize_train_golden.py), the ragged-pack backward of K-A under the lockstep warp emulator
(tests/emu_views_backward.cpp) against oracle autograd, the argument checks of pmb200_warp_corr_views_backward, the
gradient layout of PackNHWCViews, the batch-size check of the training loader, --image-extension and convert_eth3d's bytes."""
import ctypes
import hashlib
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from oracle import pm_oracle
from patchmatchnet_b200 import _native, convert_eth3d, data_io, ops, train
from patchmatchnet_b200 import autograd as ag
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state, patchmatchnet_loss
from tests import multisize_train_cases, pm_cases
from tests.test_multisize import _aligned, _ragged, _rt, _sized_case, nhwc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(REPO, "tests", "golden", "multisize_train_case.pt")


@pytest.fixture(scope="module")
def golden_train():
    return torch.load(GOLDEN, map_location="cpu")


def oracle_train_step(weights, case):
    """The training step of the reference on this project's network shell with the CPU oracle stage -> (loss, per_stage,
    {name: grad or None})."""
    net = PatchmatchNet(**pm_cases.NET_KWARGS, patchmatch_cls=pm_oracle.PatchMatchOracle)
    load_reference_state(net, weights)
    net.train()
    net.patchmatch_3.rand_source = lambda size, device: case["rand48"].to(device)
    _, _, per_stage = net([im.clone() for im in case["images"]], case["intrinsics"].clone(), case["extrinsics"].clone(),
                          case["depth_min"], case["depth_max"])
    loss = patchmatchnet_loss(per_stage, case["gts"], case["masks"])
    loss.backward()
    return loss.detach(), per_stage, {k: (p.grad.clone() if p.grad is not None else None) for k, p in net.named_parameters()}


# ------------------------------------------------------------------------------------------------
# the oracle's training step against the reference
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2])
def test_oracle_training_step_reproduces_the_reference(golden_weights, golden_train, B):
    gold = golden_train[f"train_b{B}"]
    case = multisize_train_cases.make_case(B)
    assert pm_cases.checksum({k: case[k] for k in ("images", "intrinsics", "extrinsics", "depth_min", "depth_max", "rand48")}) == gold["checksum"]
    assert len({tuple(im.shape[-2:]) for im in case["images"]}) == 4
    loss, per_stage, grads = oracle_train_step(golden_weights, case)
    # the oracle stage runs the reference's op sequence: the forward and the loss are bit-identical.  Gradients are compared
    # within 1e-5 of each tensor's largest gradient, plus the half step of the fixture's 12-bit storage: FeatureNet's are float32
    # sums that autograd accumulates in another order on this shell than on the reference (1.6e-6 seen), and CPU convolution
    # backward kernels sum in a machine-dependent order (the reference's own gradients differ in the last bits between CPUs).
    assert torch.equal(loss, gold["loss"])
    assert set(per_stage) == set(gold["per_stage"])
    for s, ds in gold["per_stage"].items():
        for x, y in zip(ds, per_stage[s]):
            assert torch.equal(x, y.detach())
    want = multisize_train_cases.unpack_grads(gold["grads"])
    assert list(grads) == list(want)
    for k, w in want.items():
        assert (w is None) == (grads[k] is None), k
        if w is None:
            continue
        ref, scale = w
        bound = 1e-5 * scale + multisize_train_cases.half_step(scale)
        assert float((grads[k].double() - ref).abs().max()) <= bound, k


# ------------------------------------------------------------------------------------------------
# the ragged-pack backward under the warp emulator
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu_views_bwd():
    src = os.path.join(REPO, "tests", "emu_views_backward.cpp")
    deps = [src, os.path.join(REPO, "tests", "warp_emu.h"), os.path.join(REPO, "include", "patchmatch_b200.h")]
    deps += [os.path.join(REPO, "patchmatchnet_b200", "csrc", f) for f in ("pm_backward.cu", "pm_math.cuh")]
    out = os.path.join(REPO, "tests", "_emu_views_backward.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")  # vector_types.h only
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-I{cuda_inc}", "-o", out, src], check=True,
                       cwd=os.path.join(REPO, "tests"))
    lib = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.emu_warp_corr_views_backward.argtypes = [P, P, ctypes.POINTER(_native.ViewExtent)] + [P] * 6 + [I] * 7
    lib.emu_warp_corr_views_backward.restype = I
    return lib


def oracle_warp_corr_grads(ref, srcs, ref_proj, src_projs, depth, vw, G, weighted, seed):
    """torch autograd through the oracle's warp + group correlation (and the detached view-weighted average) ->
    (incoming gradient, d_ref [B,C,H,W], [d_src_v [B,C,H_v,W_v]])"""
    B, _, H, W = ref.shape
    V, D = len(srcs), depth.shape[1]
    r = ref.clone().requires_grad_(True)
    ss = [s.clone().requires_grad_(True) for s in srcs]
    sims = torch.stack([pm_oracle.groupwise_correlation(pm_oracle.homography_warp(s, sp, ref_proj, depth), r, G)
                        for s, sp in zip(ss, src_projs)])
    g = torch.Generator().manual_seed(seed)
    if weighted:  # view weights detached, as on every iteration that uses the fused average
        gw = torch.randn(B, G, D, H, W, generator=g)
        out = (sims * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + vw.sum(1))[:, None, None]
    else:
        gw = torch.randn(V, B, G, D, H, W, generator=g)
        out = sims
    (out * gw).sum().backward()
    return gw, r.grad, [s.grad for s in ss]


def close(got, want, tol=2e-5):
    got, want = got.detach().double(), want.detach().double()
    assert got.shape == want.shape, (got.shape, want.shape)
    scale = max(1e-12, float(want.abs().max()))
    err = float((got - want).abs().max())
    assert err <= tol * scale, f"max err {err:.3e} vs scale {scale:.3e}"


# (C, G, H, W, D, B, source sizes): every (C, G) class, sizes from 1x1 up to larger than the reference, portrait and
# landscape, B = 2
BWD_VIEW_CASES = [
    (64, 8, 9, 13, 6, 1, [(9, 13), (13, 9), (1, 1), (15, 22)]),
    (32, 8, 10, 11, 8, 2, [(7, 12), (10, 11), (14, 6)]),
    (16, 4, 7, 19, 5, 1, [(19, 7), (1, 3), (7, 19), (11, 25), (2, 1)]),
    (16, 4, 8, 10, 4, 2, [(5, 6), (12, 15)]),
]


@pytest.mark.parametrize("weighted", [False, True], ids=["sims", "weighted"])
@pytest.mark.parametrize("C,G,H,W,D,B,sizes", BWD_VIEW_CASES)
def test_emulated_views_backward_matches_oracle_autograd(emu_views_bwd, C, G, H, W, D, B, sizes, weighted):
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, sizes, seed=C + D + B)
    V = len(sizes)
    gw, want_ref, want_srcs = oracle_warp_corr_grads(ref, srcs, ref_proj, src_projs, depth, vw, G, weighted, seed=V + D)
    pack, rt = _ragged(srcs, C), _rt(ref_proj, src_projs)
    ref_n = _aligned(ref.numel()).view(B, H, W, C)
    ref_n.copy_(nhwc(ref))
    d_ref = _aligned(ref.numel()).fill_(-3.0)
    d_src = _aligned(pack.data.numel()).fill_(-3.0)
    end = max(o + B * h * w * C for o, (h, w) in zip(pack.offsets, sizes))
    rc = emu_views_bwd.emu_warp_corr_views_backward(
        ref_n.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth.contiguous().data_ptr(),
        vw.contiguous().data_ptr() if weighted else None, gw.contiguous().data_ptr(), d_ref.data_ptr(), d_src.data_ptr(),
        V, B, C, G, H, W, D)
    assert rc == 0
    close(d_ref.view(B, H, W, C).permute(0, 3, 1, 2), want_ref)
    got = ops.ViewPack(d_src, pack.offsets, pack.heights, pack.widths, B, C)
    for v in range(V):
        close(got.view(v).permute(0, 3, 1, 2), want_srcs[v])
    # the padding between views is zeroed with the pack; the tail after the last view is not the entry point's
    covered = torch.zeros(d_src.numel(), dtype=torch.bool)
    for o, (h, w) in zip(pack.offsets, sizes):
        covered[o:o + B * h * w * C] = True
    gap = ~covered[:end]
    if gap.any():  # C = 64 views are whole multiples of the alignment: no padding
        assert float(d_src[:end][gap].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------
# argument checks of pmb200_warp_corr_views_backward (PMB200_EINVAL / PMB200_EUNSUPPORTED before anything is written)
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
    "pack beyond 2^31 float4 elements": ((1 << 33) - 64, 8, 8),
}


def _host_outputs():
    """host buffers standing in for d_ref / d_src: a rejected call must leave them as they are"""
    return torch.full((64,), -5.0), torch.full((256,), -7.0)


@pytest.mark.skipif(not _have_library(), reason="libpmb200.so is not built")
@pytest.mark.parametrize("bad", list(BAD_EXTENTS))
def test_views_backward_rejects_malformed_extents(bad):
    lib = _native.lib()
    V, B, C, G, H, W, D = 2, 1, 32, 8, 8, 8, 4
    ext = (_native.ViewExtent * V)()
    ext[0].offset, ext[0].height, ext[0].width = 0, 8, 8
    ext[1].offset, ext[1].height, ext[1].width = BAD_EXTENTS[bad]
    fake = 1 << 20  # inputs: never dereferenced, the checks run first
    d_ref, d_src = _host_outputs()
    assert lib.pmb200_warp_corr_views_backward(fake, fake, ext, fake, fake, None, fake, d_ref.data_ptr(), d_src.data_ptr(),
                                               V, B, C, G, H, W, D, None) == -1
    assert b"warp_corr_views_backward" in _native.lib().pmb200_last_error()
    assert torch.equal(d_ref, _host_outputs()[0]) and torch.equal(d_src, _host_outputs()[1])


@pytest.mark.skipif(not _have_library(), reason="libpmb200.so is not built")
def test_views_backward_rejects_bad_view_counts_null_extents_and_other_classes():
    lib = _native.lib()
    fake = 1 << 20
    ext = (_native.ViewExtent * 17)()
    for e in ext:
        e.offset, e.height, e.width = 0, 4, 4
    d_ref, d_src = _host_outputs()
    call = lambda ext_, V, C=32, G=8: lib.pmb200_warp_corr_views_backward(
        fake, fake, ext_, fake, fake, None, fake, d_ref.data_ptr(), d_src.data_ptr(), V, 1, C, G, 4, 4, 4, None)
    assert call(ext, 0) == -1 and call(ext, 17) == -1
    assert call(None, 2) == -1
    assert call(ext, 2, C=12, G=3) == -2  # PMB200_EUNSUPPORTED, as the uniform backward
    assert torch.equal(d_ref, _host_outputs()[0]) and torch.equal(d_src, _host_outputs()[1])


# ------------------------------------------------------------------------------------------------
# PackNHWCViews: each map receives its slice of the flat gradient, re-viewed as NCHW
# ------------------------------------------------------------------------------------------------
def test_pack_nhwc_views_gradient_layout():
    B, C = 2, 12
    shapes = [(3, 5), (5, 3), (1, 1), (4, 7)]
    offsets, total = ops.ViewPack.layout(shapes, B, C)
    ctx = types.SimpleNamespace(slices=[(o, torch.Size((B, C, h, w))) for o, (h, w) in zip(offsets, shapes)])
    g = torch.arange(total, dtype=torch.float32)
    grads = ag.PackNHWCViews.backward(ctx, g)
    assert len(grads) == len(shapes)
    for (h, w), o, d in zip(shapes, offsets, grads):
        assert d.shape == (B, C, h, w)
        b, c, y, x = torch.meshgrid(*(torch.arange(n) for n in (B, C, h, w)), indexing="ij")
        assert torch.equal(d, g[o + ((b * h + y) * w + x) * C + c])


# ------------------------------------------------------------------------------------------------
# the training driver: batches whose samples disagree in size, --image-extension
# ------------------------------------------------------------------------------------------------
def _sample(sizes):
    return {"images": [np.zeros((3, h, w), np.float32) for h, w in sizes], "intrinsics": np.zeros((len(sizes), 3, 3), np.float32),
            "extrinsics": np.zeros((len(sizes), 4, 4), np.float32), "depth_min": 1.0, "depth_max": 2.0,
            "depth_gt": np.zeros((1,) + sizes[0], np.float32), "mask": np.zeros((1,) + sizes[0], bool), "filename": "x"}


def test_collate_names_the_sizes_of_a_mixed_batch():
    mixed = [(64, 80), (80, 64), (64, 80)]
    batch = train.collate([_sample(mixed), _sample(mixed)])  # samples agree view by view: one batch
    assert [tuple(im.shape) for im in batch["images"]] == [(2, 3, 64, 80), (2, 3, 80, 64), (2, 3, 64, 80)]
    with pytest.raises(RuntimeError, match=r"view 1: 80x64 and 64x80.*one sample per rank"):
        train.collate([_sample(mixed), _sample([(64, 80), (64, 80), (64, 80)])])
    with pytest.raises(RuntimeError, match=r"view 0: 64x80 and 48x80"):
        train.collate([_sample(mixed), _sample([(48, 80), (80, 64), (64, 80)])])
    assert train.collate([]) is None


def test_image_extension_option(tmp_path):
    assert train.parse_args([]).image_extension == ".jpg"
    assert train.parse_args(["--image-extension", ".png"]).image_extension == ".png"
    # convert_eth3d's output trains with --image-extension .png; its views differ in size
    raw, conv = tmp_path / "raw", tmp_path / "conv"
    conv.mkdir()
    scan_list = multisize_train_cases.write_raw_eth3d_tree(str(raw))
    convert_eth3d.convert(str(raw), str(conv), scan_list)
    ds = train.MVSDataset(str(conv), num_views=2, scan_list=scan_list, image_extension=".png")
    s = ds[0]
    assert {im.shape[1:] for im in s["images"]} == {(24, 32), (32, 24)}
    assert s["depth_gt"].shape[1:] == s["images"][0].shape[1:]
    with pytest.raises(FileNotFoundError):
        train.MVSDataset(str(conv), num_views=2, scan_list=scan_list)[0]  # the default .jpg is not there


# ------------------------------------------------------------------------------------------------
# convert_eth3d against the reference's convert_eth3d_dataset.py
# ------------------------------------------------------------------------------------------------
def test_convert_eth3d_writes_the_reference_bytes(tmp_path, golden_train):
    gold = golden_train["eth3d"]
    raw, conv = tmp_path / "raw", tmp_path / "conv"
    conv.mkdir()
    scan_list = multisize_train_cases.write_raw_eth3d_tree(str(raw))
    assert convert_eth3d.main(["--input-folder", str(raw), "--output-folder", str(conv), "--scan-list", scan_list]) == 0
    files = sorted(os.path.relpath(os.path.join(d, f), conv) for d, _, fs in os.walk(conv) for f in fs)
    assert files == gold["files"]
    for f, want in zip(files, gold["sha256"]):
        assert hashlib.sha256(open(os.path.join(conv, f), "rb").read()).hexdigest() == want, f


def test_convert_eth3d_messages(tmp_path):
    with pytest.raises(Exception, match="Invalid input folder"):
        convert_eth3d.main(["--input-folder", str(tmp_path / "x")])
    with pytest.raises(Exception, match="Invalid output folder"):
        convert_eth3d.main(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path / "x")])
    with pytest.raises(Exception, match="Invalid input scan list"):
        convert_eth3d.main(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path), "--scan-list", "nope.txt"])


def test_read_image_dictionary(tmp_path):
    p = tmp_path / "index2prefix.txt"
    p.write_text("3\n7 images/a_undistorted.png\n0 b.JPG \n12 c/d.png\nignored after the count\n")
    assert data_io.read_image_dictionary(str(p)) == {7: "images/a_undistorted.png", 0: "b.JPG", 12: "c/d.png"}
