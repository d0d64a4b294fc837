"""Views of different sizes on the GPU: the *_views entry points of K-A and pmb200_geometric_filter_views against the
oracles, their bit equality with the uniform entry points on uniform packs, the native network against the reference's
recorded outputs on a mixed-size request (tests/golden/multisize_case.pt), DepthEngine(view_sizes=...), reconstruct on a scene
that mixes orientations, and a two-camera COLMAP model through colmap_input -> reconstruct -> colmap_output."""
import os

import numpy as np
import pytest
import torch

from oracle import geo_oracle as go
from patchmatchnet_b200 import colmap_input as ci, colmap_output as cout, data_io, ops, reconstruct, synthetic
from patchmatchnet_b200.engine import DepthEngine
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state
from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet
from tests import colmap_cases as cc, multisize_cases, pm_cases, scene_cases
from tests.test_multisize import _oracle_sims, _sized_case, maxabs, nhwc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
NET_DEPTH_TOL = 2e-4  # tests/test_gpu_parity.py, test_network_matches_reference_golden


@pytest.fixture(autouse=True)
def fp32_reference_ops():
    """The PyTorch heads and convolutions the kernels are compared with run in full fp32 (no TF32 operands)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _random_head(cls, G, seed):
    torch.manual_seed(seed)
    head = cls(G)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm3d):  # non-trivial running statistics and affine terms
            m.running_mean.normal_(0, 0.3)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    return head.eval()


KA_CASES = [  # (C, G, H, W, D, B, source sizes): the three fast-path classes and the generic kernel
    (64, 8, 13, 21, 20, 1, [(13, 21), (21, 13), (1, 1), (30, 40)]),
    (32, 8, 19, 27, 16, 2, [(15, 30), (27, 19), (19, 27)]),
    (16, 4, 22, 35, 8, 1, [(35, 22), (2, 3), (22, 35), (40, 60), (11, 17)]),
    (12, 3, 9, 14, 6, 1, [(14, 9), (9, 14), (1, 2)]),
]


def _device_case(C, G, H, W, D, B, sizes, seed):
    ref, srcs, ref_proj, src_projs, depth, vw = _sized_case(B, C, H, W, D, sizes, seed=seed)
    rt = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs])
    want = _oracle_sims(ref, srcs, ref_proj, src_projs, depth, G)
    return ref, srcs, rt, depth, vw, want, ops.pack_nhwc_views([s.to(DEV) for s in srcs]), nhwc(ref.to(DEV))


@pytest.mark.parametrize("C,G,H,W,D,B,sizes", KA_CASES)
def test_warp_corr_views_matches_oracle(C, G, H, W, D, B, sizes):
    ref, srcs, rt, depth, vw, want, pack, ref_n = _device_case(C, G, H, W, D, B, sizes, seed=C + D)
    assert all(o % 4 == 0 for o in pack.offsets) and pack.data.data_ptr() % 32 == 0
    for v, s in enumerate(srcs):  # the pack holds each view channels-last at its own size
        assert torch.equal(pack.view(v).cpu(), nhwc(s))
    scale = max(1.0, float(want.abs().max()))
    got = ops.warp_corr(ref_n, pack, rt, depth.to(DEV), G)
    assert maxabs(got, want) <= 2e-5 * scale
    want_f = (want * vw.permute(1, 0, 2, 3)[:, :, None, None]).sum(0) / (1e-5 + vw.sum(1))[:, None, None]
    assert maxabs(ops.warp_corr(ref_n, pack, rt, depth.to(DEV), G, vw.to(DEV)), want_f) <= 2e-5 * scale
    if (C, G) not in ops.FUSED_HEAD_SHAPES:
        return
    # fused heads: the per-view form against the unfused per-view sims + the PyTorch heads
    sim_net, pw_net = _random_head(SimilarityNet, G, 5).to(DEV), _random_head(PixelwiseNet, G, 6).to(DEV)
    with torch.no_grad():
        score = ops.warp_corr_score(ref_n, pack, rt, depth.to(DEV), G, vw.to(DEV), sim_net.folded())
        want_score = sim_net(ops.warp_corr(ref_n, pack, rt, depth.to(DEV), G, vw.to(DEV)))
        assert maxabs(score, want_score) <= 2e-5 * max(1.0, float(want_score.abs().max()))
        w, sims = ops.warp_corr_view_weights(ref_n, pack, rt, depth.to(DEV), G, pw_net.folded(), keep_sims=True)
        assert torch.equal(sims, got)
        want_w = torch.stack([pw_net(got[v]).squeeze(1) for v in range(len(sizes))], 1)
        assert maxabs(w, want_w) <= 1e-5


@pytest.mark.parametrize("C,G", [(64, 8), (32, 8), (16, 4), (12, 3)])
def test_views_entry_points_on_a_uniform_pack_equal_the_uniform_ones(C, G):
    H, W, D, B, V = 13, 17, 12, 2, 3
    ref, srcs, rt, depth, vw, _, pack, ref_n = _device_case(C, G, H, W, D, B, [(11, 19)] * V, seed=3)
    stacked = torch.stack([nhwc(s.to(DEV)) for s in srcs])
    d, w = depth.to(DEV), vw.to(DEV)
    ops.set_tuning("ka_gen", 3)  # the per-view form runs generation 3; compare like with like
    try:
        assert torch.equal(ops.warp_corr(ref_n, pack, rt, d, G), ops.warp_corr(ref_n, stacked, rt, d, G))
        assert torch.equal(ops.warp_corr(ref_n, pack, rt, d, G, w), ops.warp_corr(ref_n, stacked, rt, d, G, w))
        if (C, G) in ops.FUSED_HEAD_SHAPES:
            sim_net, pw_net = _random_head(SimilarityNet, G, 5).to(DEV), _random_head(PixelwiseNet, G, 6).to(DEV)
            a = ops.warp_corr_score(ref_n, pack, rt, d, G, w, sim_net.folded())
            assert torch.equal(a, ops.warp_corr_score(ref_n, stacked, rt, d, G, w, sim_net.folded()))
            a = ops.warp_corr_view_weights(ref_n, pack, rt, d, G, pw_net.folded(), keep_sims=True)
            b = ops.warp_corr_view_weights(ref_n, stacked, rt, d, G, pw_net.folded(), keep_sims=True)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    finally:
        ops.set_tuning("reset")


def _geo_run(sc, srcs):
    cams = ops.compose_filter_cameras(sc["ref_K"], sc["ref_E"], list(sc["src_Ks"]), list(sc["src_Es"]))
    out = ops.geometric_filter(torch.from_numpy(sc["ref_depth"]).to(DEV), torch.from_numpy(sc["confidence"]).to(DEV), srcs, cams)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def _geo_compare(got, want):  # the tolerances of tests/test_geo.py
    photo, msum, final, avg = got
    wphoto, wsum, wfinal, wavg = want
    n = wsum.size
    assert np.array_equal(photo, wphoto)
    flipped = msum != wsum
    assert flipped.sum() <= max(1, int(1e-4 * n))
    assert (final != wfinal).sum() <= max(1, int(1e-4 * n))
    same = ~flipped
    assert avg.dtype == np.float64 and np.all(np.abs(avg[same] - wavg[same]) <= 1e-6 * np.abs(wavg[same]))


def test_geometric_filter_views_matches_the_reference_and_the_oracle():
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multisize_case.pt"))["geo"]
    sc = multisize_cases.make_geo_scene(seed=0)
    got = _geo_run(sc, [torch.from_numpy(d).to(DEV) for d in sc["src_depths"]])
    _geo_compare(got, [gold[k].numpy() for k in ("photo_mask", "geo_mask_sum", "final_mask", "depth_est_averaged")])
    want = go.fuse_reference_view(sc["ref_depth"], sc["ref_K"], sc["ref_E"], sc["src_depths"], sc["src_Ks"], sc["src_Es"], sc["confidence"])
    _geo_compare(got, want)
    # on maps of one size the per-view filter is the stacked one, bit for bit
    same = dict(sc, src_depths=[sc["src_depths"][0]] * 3, src_Ks=[sc["src_Ks"][0]] * 3, src_Es=[sc["src_Es"][0]] * 3)
    a = _geo_run(same, [torch.from_numpy(d).to(DEV) for d in same["src_depths"]])
    b = _geo_run(same, torch.from_numpy(np.stack(same["src_depths"])).to(DEV))
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def _net(weights):
    net = PatchmatchNet(**pm_cases.NET_KWARGS)
    load_reference_state(net, weights)
    return net.eval().to(DEV)


def test_network_matches_the_reference_on_a_mixed_size_request(golden_weights):
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multisize_case.pt"))["net"]
    net = _net(golden_weights)
    inp = multisize_cases.make_net_inputs()
    assert pm_cases.checksum(inp) == gold["checksum"]
    net.patchmatch_3.rand_source = lambda size, device: inp["rand48"].to(device)
    calls = {}
    real = ops.pack_nhwc_views
    ops.pack_nhwc_views = lambda maps: calls.setdefault("n", []).append(1) or real(maps)
    try:
        with torch.no_grad():
            depth, conf, per_stage = net([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV),
                                         inp["depth_min"].to(DEV), inp["depth_max"].to(DEV))
    finally:
        ops.pack_nhwc_views = real
    assert len(calls["n"]) == 3  # every stage took the ragged pack
    assert pm_cases.rel_l1(depth, gold["depth"]) <= NET_DEPTH_TOL
    for s, ds in gold["per_stage"].items():
        for x, y in zip(per_stage[s], ds):
            assert pm_cases.rel_l1(x, y) <= NET_DEPTH_TOL
    assert maxabs(conf, gold["confidence"]) <= 5e-2
    assert float((conf.cpu() - gold["confidence"]).abs().mean()) <= 1e-3


def test_depth_engine_with_view_sizes_replays_what_an_eager_forward_computes(golden_weights):
    sizes = [(96, 128), (128, 96), (96, 128), (64, 80)]
    inp = multisize_cases.make_net_inputs(sizes, seed=5)
    args = ([im.to(DEV) for im in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV), inp["depth_min"].to(DEV),
            inp["depth_max"].to(DEV))
    net = _net(golden_weights)
    fixed = torch.rand(1, 48, 12, 16, device=DEV)
    net.patchmatch_3.rand_source = lambda size, device: fixed  # pinned: graph and eager forwards see the same draw
    outs = {}
    for use_graph in (True, False):
        eng = DepthEngine(net, 1, len(sizes), 96, 128, n_slots=2, use_graph=use_graph, view_sizes=sizes)
        for k in range(2):
            eng.set_device_inputs(k, *args)
        runs = []
        for _ in range(2):
            d, c = eng.run_slot(1)
            runs.append((d.clone(), c.clone()))
        assert runs[0][0].shape == (1, 1, 96, 128) and runs[0][1].shape == (1, 96, 128)
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])  # reruns
        outs[use_graph] = runs[0]
        del eng
    assert torch.equal(outs[True][0], outs[False][0]) and torch.equal(outs[True][1], outs[False][1])
    net.patchmatch_3.rand_source = None
    # unpinned draws through the serving loop: two engines built alike give the same maps, request by request
    host = dict(images=[i.pin_memory() for i in inp["images"]], intrinsics=inp["intrinsics"].pin_memory(),
                extrinsics=inp["extrinsics"].pin_memory(), depth_min=inp["depth_min"].pin_memory(), depth_max=inp["depth_max"].pin_memory())
    runs = []
    for _ in range(2):
        eng = DepthEngine(net, 1, len(sizes), 96, 128, n_slots=2, seed=3, view_sizes=sizes)
        seen = {}
        h2d, _ = eng.infer_stream([host] * 5, on_result=lambda i, dd, cc: seen.__setitem__(i, (dd.clone(), cc.clone())))
        assert sorted(seen) == list(range(5)) and h2d >= sum(i.numel() * 4 for i in inp["images"])
        runs.append(seen)
        del eng
    for i in range(5):
        assert torch.equal(runs[0][i][0], runs[1][i][0]) and torch.equal(runs[0][i][1], runs[1][i][1]), i
    d, c = DepthEngine(net, 1, len(sizes), 96, 128, n_slots=1, view_sizes=sizes).infer(
        inp["images"], inp["intrinsics"], inp["extrinsics"], inp["depth_min"], inp["depth_max"])
    assert d.shape == (1, 1, 96, 128) and torch.isfinite(d).all() and c.shape == (1, 96, 128)


DTU_THRES = ["--geo-pixel-thres", "1", "--geo-depth-thres", "0.01", "--geo-mask-thres", "3", "--photo-thres", "0.8"]


def _run(*argv):
    return reconstruct.reconstruct(reconstruct.parse_args([str(a) for a in argv]), log=lambda *a: None)


def _files(out_dir, sub):
    d = os.path.join(out_dir, sub)
    return {n: open(os.path.join(d, n), "rb").read() for n in sorted(os.listdir(d))}


def test_reconstruct_a_scene_that_mixes_orientations(tmp_path):
    from PIL import Image

    sizes = multisize_cases.mixed_sizes(6, 128, 160)
    scene = str(tmp_path / "scene")
    multisize_cases.write_mixed_scene(scene, sizes, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *DTU_THRES]
    s1 = _run(*common, "--output-folder", tmp_path / "a", "--output-type", "both")
    s2 = _run(*common, "--output-folder", tmp_path / "b", "--output-type", "both")
    _run(*common, "--output-folder", tmp_path / "split", "--output-type", "depth")
    _run(*common, "--output-folder", tmp_path / "split", "--output-type", "fusion")
    assert s1["depth_maps"] == 6 and s1["points"] > 0 and s1["engines_built"] >= 2 and s1["engine_setup_seconds"] > 0
    for sub in ("depth_est", "confidence", "mask"):  # deterministic, and both == depth then fusion
        a = _files(str(tmp_path / "a"), sub)
        assert a == _files(str(tmp_path / "b"), sub) == _files(str(tmp_path / "split"), sub)
    ply = lambda d: open(os.path.join(d, "fused.ply"), "rb").read()
    assert ply(tmp_path / "a") == ply(tmp_path / "b") == ply(tmp_path / "split")
    read = lambda kind, v: data_io.read_map(str(tmp_path / "a" / kind / f"{v:08d}.pfm"))[..., 0]
    for v, hw in enumerate(sizes):
        assert read("depth_est", v).shape == hw and read("confidence", v).shape == hw
    # masks against the oracle, with test_fusion_matches_the_oracle's flip allowance
    pairs = data_io.read_pair_file(os.path.join(scene, "pair.txt"))

    def cam(v):
        img, oh, ow = data_io.read_image(os.path.join(scene, "images", f"{v:08d}.jpg"))
        k, e, _ = data_io.read_cam_file(os.path.join(scene, "cams", f"{v:08d}_cam.txt"))
        return data_io.scale_intrinsics(k, img.shape[:2], oh, ow), e

    mask = lambda v, k: np.array(Image.open(str(tmp_path / "a" / "mask" / f"{v:08d}_{k}.png"))) == 255
    flips_ok = lambda got, want: (got != want).sum() <= max(1, int(1e-4 * want.size))
    for ref, srcs in pairs:
        K, E = cam(ref)
        cams = [cam(s) for s in srcs]
        with np.errstate(divide="ignore", invalid="ignore"):
            photo, msum, final, _ = go.fuse_reference_view(read("depth_est", ref), K, E, [read("depth_est", s) for s in srcs],
                                                           [c[0] for c in cams], [c[1] for c in cams], read("confidence", ref),
                                                           1.0, 0.01, 0.8, 3)
        assert np.array_equal(mask(ref, "photo"), photo)
        assert flips_ok(mask(ref, "geo"), msum >= 3) and flips_ok(mask(ref, "final"), final)


def test_two_camera_colmap_model_through_the_chain(tmp_path):
    """Two COLMAP cameras of different resolution (a landscape and a portrait one) -> colmap_input -> reconstruct -> colmap_output."""
    from PIL import Image

    n_views = 5
    sizes = [(128, 160) if i % 2 == 0 else (160, 128) for i in range(n_views)]
    cams = []
    for i, ((K, E), (h, w)) in enumerate(zip(scene_cases.cameras(n_views, 128, 160), sizes)):
        K = K.copy()
        K[0, 2], K[1, 2] = w / 2, h / 2  # one camera per orientation: same intrinsics within a camera
        cams.append((K, E))
    rng = np.random.default_rng(4)
    k0, e0 = (c.astype(np.float64) for c in cams[0])
    depth0 = scene_cases.plane_depth(*cams[0], 128, 160, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float64)
    n_points = 3000
    u, v = rng.uniform(2, 157, n_points), rng.uniform(2, 125, n_points)
    d = depth0[v.astype(int), u.astype(int)]
    xyz = (np.linalg.inv(e0) @ np.vstack([np.linalg.inv(k0) @ np.stack([u, v, np.ones(n_points)]) * d, np.ones(n_points)]))[:3].T
    ids = np.arange(1, n_points + 1, dtype=np.uint64) * np.uint64(7)
    cameras = [(1, "PINHOLE", 160, 128, [cams[0][0][0, 0], cams[0][0][1, 1], 80.0, 64.0]),
               (2, "PINHOLE", 128, 160, [cams[1][0][0, 0], cams[1][0][1, 1], 64.0, 80.0])]
    images = []
    for i, ((k, e), (h, w)) in enumerate(zip(cams, sizes)):
        k, e = k.astype(np.float64), e.astype(np.float64)
        p = k @ (e[:3, :3] @ xyz.T + e[:3, 3:4])
        px, py = p[0] / p[2], p[1] / p[2]
        seen = np.nonzero((px >= 0) & (px < w) & (py >= 0) & (py < h))[0]
        images.append((i + 1, cc.rotation_to_quaternion(e[:3, :3]), e[:3, 3], 1 + i % 2, "view_%02d.png" % i, ids[seen].astype(np.int64)))
    model = {"cameras": cameras, "images": images, "point_ids": ids, "xyz": xyz, "rgb": np.zeros((n_points, 3), np.uint8),
             "error": np.zeros(n_points)}
    colmap = tmp_path / "colmap"
    cc.write_bin(str(colmap / "sparse"), model)
    (colmap / "images").mkdir()
    for i, ((k, e), (h, w)) in enumerate(zip(cams, sizes)):
        Image.fromarray(scene_cases.texture(k, e, h, w)).save(str(colmap / "images" / ("view_%02d.png" % i)))
    scene, results, ws = tmp_path / "scene", tmp_path / "results", tmp_path / "ws"
    for dd in (scene, ws):
        dd.mkdir()
    assert ci.main(["--input-folder", str(colmap), "--output-folder", str(scene), "--num-src-images", str(n_views - 1)]) == 0
    stats = _run("--input-folder", scene, "--output-folder", results, "--checkpoint-path", WEIGHTS, "--num-views", "2",
                 "--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05")
    assert stats["depth_maps"] == n_views and stats["points"] > 0
    assert os.path.getsize(results / "fused.ply") > 200
    assert cout.main(["--input-folder", str(scene), "--results-folder", str(results), "--output-folder", str(ws)]) == 0
    for i, hw in enumerate(sizes):
        got = data_io.read_map(str(ws / "stereo" / "depth_maps" / f"{i:08d}.jpg.geometric.bin"))
        assert got.shape[:2] == hw
