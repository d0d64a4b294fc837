"""Training on views of different sizes on the GPU: pmb200_warp_corr_views_backward against oracle autograd and against the
uniform backward on uniform packs, a full PatchmatchNet train step on mixed-size requests against the reference's recorded
gradients (tests/golden/multisize_train_case.pt) and the oracle, the case of uniform sources of another size than the
reference, and `train` for two epochs on a mixed-size .png scene followed by `reconstruct` on its checkpoint."""
import os

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import _native, data_io, ops, reconstruct, synthetic, train
from patchmatchnet_b200 import autograd as ag
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state, patchmatchnet_loss
from tests import multisize_cases, multisize_train_cases, pm_cases, scene_cases
from tests.geo_cases import plane_depth
from tests.test_gpu_backward import compare_param_grads
from tests.test_multisize import _sized_case, nhwc
from tests.test_multisize_train import oracle_train_step, oracle_warp_corr_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multisize_train_case.pt")


@pytest.fixture(autouse=True)
def fp32_reference_ops():
    """The PyTorch convolutions the kernels are compared with run in full fp32 (no TF32 operands)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def close(got, want, tol=2e-5):
    got, want = got.detach().double().cpu(), want.detach().double().cpu()
    assert got.shape == want.shape, (got.shape, want.shape)
    scale = max(1e-12, float(want.abs().max()))
    err = float((got - want).abs().max())
    assert err <= tol * scale, f"max err {err:.3e} vs scale {scale:.3e}"


BWD_CASES = [  # (C, G, H, W, D, B, source sizes): the three (C, G) classes, sizes from 1x1 to larger than the reference
    (64, 8, 13, 21, 12, 1, [(13, 21), (21, 13), (1, 1), (30, 40)]),
    (32, 8, 19, 27, 16, 2, [(15, 30), (27, 19), (19, 27)]),
    (16, 4, 22, 35, 8, 1, [(35, 22), (2, 3), (22, 35), (40, 60), (11, 17)]),
]


@pytest.mark.parametrize("weighted", [False, True], ids=["sims", "weighted"])
@pytest.mark.parametrize("C,G,H,W,D,B,sizes", BWD_CASES)
def test_views_backward_matches_oracle_autograd(C, G, H, W, D, B, sizes, weighted):
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, sizes, seed=C + D + B)
    gw, want_ref, want_srcs = oracle_warp_corr_grads(ref, srcs, ref_proj, src_projs, depth, vw, G, weighted, seed=len(sizes) + D)
    pack = ops.pack_nhwc_views([s.to(DEV) for s in srcs])
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    d_ref, d_src = ag.warp_corr_views_backward(nhwc(ref.to(DEV)), pack, rt, depth.to(DEV).contiguous(),
                                               vw.to(DEV).contiguous() if weighted else None, gw.to(DEV).contiguous(), G)
    close(d_ref.permute(0, 3, 1, 2), want_ref)
    got = ops.ViewPack(d_src, pack.offsets, pack.heights, pack.widths, B, C)
    for v in range(len(sizes)):
        close(got.view(v).permute(0, 3, 1, 2), want_srcs[v])
    covered = torch.zeros(d_src.numel(), dtype=torch.bool, device=DEV)
    for v in range(len(sizes)):
        covered[pack.offsets[v]:pack.offsets[v] + got.view(v).numel()] = True
    if (~covered).any():  # the padding between views is zeroed, and so is the tail after the last view
        assert float(d_src[~covered].abs().max()) == 0.0


@pytest.mark.parametrize("weighted", [False, True], ids=["sims", "weighted"])
@pytest.mark.parametrize("C,G", [(64, 8), (32, 8), (16, 4)])
def test_views_backward_equals_the_uniform_backward_on_uniform_packs(C, G, weighted):
    B, H, W, D, Hs, Ws, V = 2, 24, 32, 8, 20, 28, 3
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, [(Hs, Ws)] * V, seed=C)
    gen = torch.Generator().manual_seed(9)
    gw = (torch.randn(B, G, D, H, W, generator=gen) if weighted else torch.randn(V, B, G, D, H, W, generator=gen)).to(DEV)
    ref_n = nhwc(ref.to(DEV))
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    depth, vw_d = depth.to(DEV).contiguous(), (vw.to(DEV).contiguous() if weighted else None)
    uni = ops.pack_nhwc([s.to(DEV) for s in srcs])
    d_ref_u, d_src_u = torch.empty_like(ref_n), torch.empty_like(uni)
    rc = _native.lib().pmb200_warp_corr_backward(ref_n.data_ptr(), uni.data_ptr(), rt.data_ptr(), depth.data_ptr(),
                                                 None if vw_d is None else vw_d.data_ptr(), gw.data_ptr(), d_ref_u.data_ptr(),
                                                 d_src_u.data_ptr(), V, B, C, G, H, W, Hs, Ws, D, None)
    _native.check(rc, "warp_corr_backward")
    pack = ops.pack_nhwc_views([s.to(DEV) for s in srcs])
    d_ref_v, d_src_v = ag.warp_corr_views_backward(ref_n, pack, rt, depth, vw_d, gw, G)
    torch.cuda.synchronize()
    assert torch.equal(d_ref_u, d_ref_v)  # owned by the pixel's lane group: plain stores in the same order
    got = ops.ViewPack(d_src_v, pack.offsets, pack.heights, pack.widths, B, C)
    for v in range(V):  # 128-bit atomics: equal up to the order in which the adds land
        close(got.view(v), d_src_u[v], tol=1e-6)


# ---- a full train step ----------------------------------------------------------------------------------------------------

def native_train_step(weights, case):
    net = PatchmatchNet(**pm_cases.NET_KWARGS)
    load_reference_state(net, weights)
    net = net.to(DEV).train()
    net.patchmatch_3.rand_source = lambda size, device: case["rand48"].to(device)
    _, _, per_stage = net([im.to(DEV) for im in case["images"]], case["intrinsics"].to(DEV), case["extrinsics"].to(DEV),
                          case["depth_min"].to(DEV), case["depth_max"].to(DEV))
    loss = patchmatchnet_loss(per_stage, [t.to(DEV) for t in case["gts"]], [m.to(DEV) for m in case["masks"]])
    loss.backward()
    return loss.item(), {k: (p.grad.detach().cpu() if p.grad is not None else None) for k, p in net.named_parameters()}


@pytest.mark.parametrize("B", [1, 2])
def test_network_training_step_on_mixed_sizes_matches_reference_and_oracle(golden_weights, B):
    """The thresholds of test_network_training_step_matches_oracle (tests/test_gpu_backward.py)."""
    gold = torch.load(GOLDEN, map_location="cpu")[f"train_b{B}"]
    case = multisize_train_cases.make_case(B)
    assert len({tuple(im.shape[-2:]) for im in case["images"][1:]}) == 4  # sources that differ from each other: ragged pack
    lm, gm = native_train_step(golden_weights, case)
    lo, _, go = oracle_train_step(golden_weights, case)
    # the reference's gradients as the fixture stores them: within 2^-12 of each tensor's largest gradient, far inside these bounds
    ref_grads = {k: (None if w is None else w[0].float()) for k, w in multisize_train_cases.unpack_grads(gold["grads"]).items()}
    for lw, gw in ((float(gold["loss"]), ref_grads), (float(lo), go)):
        assert abs(lm - lw) <= 2e-4 * abs(lw)
        compare_param_grads(gm, gw, rtol=2e-2, atol_of_global=2e-3)


def test_network_training_step_with_uniform_sources_of_another_size(golden_weights):
    """Reference 64x80, every source 80x64: a reference pack and a source pack on the uniform backward."""
    sizes = [(64, 80), (80, 64), (80, 64), (80, 64)]
    inp = multisize_cases.make_net_inputs(sizes=sizes, seed=77)
    g = torch.Generator().manual_seed(78)
    gts = [synthetic.DEPTH_MIN + 500.0 * torch.rand(1, 1, 64 >> l, 80 >> l, generator=g) for l in range(4)]
    masks = [torch.rand(1, 1, 64 >> l, 80 >> l, generator=g) > 0.2 for l in range(4)]
    case = dict(inp, gts=gts, masks=masks)
    lm, gm = native_train_step(golden_weights, case)
    lo, _, go = oracle_train_step(golden_weights, case)
    assert abs(lm - float(lo)) <= 2e-4 * abs(float(lo))
    compare_param_grads(gm, go, rtol=2e-2, atol_of_global=2e-3)


# ---- the command on a mixed-size .png scene -------------------------------------------------------------------------------

def _write_mixed_png_training_set(root, sizes):
    from PIL import Image

    H0, W0 = sizes[0]
    base = os.path.join(root, "scan1")
    for sub in ("cams", "depth_gt", "images"):
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    with open(os.path.join(base, "pair.txt"), "w") as f:
        f.write(scene_cases.pair_text(scene_cases.all_pairs(len(sizes), 2)))
    for v, ((K, E), (h, w)) in enumerate(zip(scene_cases.cameras(len(sizes), H0, W0), sizes)):
        K = K.copy()
        K[0, 2], K[1, 2] = w / 2 + 1.5 * v, h / 2
        with open(os.path.join(base, "cams", "%08d_cam.txt" % v), "w") as f:
            f.write(scene_cases.cam_text(K, E))
        depth = plane_depth(K, E, h, w, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float32)
        depth[: h // 8] = 0.0
        data_io.save_map(os.path.join(base, "depth_gt", "%08d.pfm" % v), depth)
        Image.fromarray(scene_cases.texture(K, E, h, w)).save(os.path.join(base, "images", "%08d.png" % v))
    for name in ("train.txt", "val.txt"):
        with open(os.path.join(root, name), "w") as f:
            f.write("scan1\n")


def test_train_two_epochs_on_a_mixed_size_png_scene_then_reconstruct(tmp_path):
    sizes = multisize_cases.mixed_sizes(4, 96, 128)  # view 1 portrait
    root, out = str(tmp_path / "data"), str(tmp_path / "run")
    _write_mixed_png_training_set(root, sizes)
    args = train.parse_args(["--input-folder", root, "--output-folder", out, "--train-list", os.path.join(root, "train.txt"),
                             "--test-list", os.path.join(root, "val.txt"), "--num-views", "2", "--batch-size", "1",
                             "--epochs", "2", "--summary-freq", "1", "--num-workers", "0", "--image-max-dim", "-1",
                             "--image-extension", ".png"])
    res = train.run(args)
    assert res["start_epoch"] == 0
    assert sorted(os.listdir(out)) == ["module_000000.pt", "module_000001.pt", "params_000000.ckpt", "params_000001.ckpt",
                                       "train_log.jsonl"]
    ck = torch.load(os.path.join(out, "params_000001.ckpt"), map_location="cpu")
    assert all(torch.isfinite(v).all() for v in ck["model"].values() if v.is_floating_point())
    # reconstruct reads the checkpoint (the scene's images as reconstruct reads them: .jpg)
    scene = str(tmp_path / "scene")
    multisize_cases.write_mixed_scene(scene, sizes, n_src=2)
    reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", scene, "--output-type", "depth", "--num-views", "2",
                                                    "--checkpoint-path", os.path.join(out, "params_000001.ckpt"),
                                                    "--output-folder", str(tmp_path / "rec")]), log=lambda *a: None)
    for v in range(len(sizes)):
        d = data_io.read_map(str(tmp_path / "rec" / "depth_est" / ("%08d.pfm" % v)))
        assert d.shape[:2] == sizes[v] and np.isfinite(d).all()
