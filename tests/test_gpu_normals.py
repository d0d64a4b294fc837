"""Surface normals and oriented fusion on the GPU: pmb200_depth_normals against oracle/normals_oracle.py, the oriented fusion
against the plain one, and the --normals options of reconstruct and colmap_output end to end.

Normal tolerances (tests/normals_cases.check_against_oracle): zero / non-zero classification may differ on at most 1e-4 of
the pixels, since a threshold can be met within rounding (the kernel's float64 sums contract into fused multiply-adds and
its eigen solve is closed-form; the oracle's are not); where the oracle's eigen gap is at least 1e-3 lambda_max the angle
is <= 1e-5 rad, up to sign for a normal seen edge-on, whose orientation rounding decides; every non-zero normal has unit
length to 1e-6 and faces the camera."""
import os

import numpy as np
import pytest
import torch

from oracle import normals_oracle as no
from patchmatchnet_b200 import colmap_input as ci, colmap_output as cout, data_io, ops, reconstruct
from tests import colmap_cases as cc, multisize_cases, normals_cases as nc, scene_cases

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
THRES = ["--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]


def _gpu(depth, K, **kw):
    return ops.estimate_normals(torch.from_numpy(np.asarray(depth, dtype=np.float32)).to(DEV), K, **kw).cpu().numpy()


def _check(depth, K, **kw):
    depth = np.asarray(depth, dtype=np.float32)
    got = _gpu(depth, K, **kw)
    nc.check_against_oracle(got, depth, K, **kw)
    return got


@pytest.mark.parametrize("name", ["fronto", "tilted", "step", "holes", "noisy"])
def test_kernel_matches_the_oracle_on_analytic_maps(name):
    H, W = 45, 67
    c = {"fronto": nc.fronto, "tilted": nc.tilted, "step": nc.step, "holes": lambda h, w: nc.holes(h, w)[0],
         "noisy": nc.noisy}[name](H, W)
    got = _check(c["depth"], c["K"])
    nonzero = (got != 0).any(-1)
    assert nonzero.mean() > 0.85
    if name != "noisy":
        assert nc.angle(got[nonzero].astype(np.float64), c["want"][nonzero]).max() < 1e-3


def test_kernel_zero_cases():
    c = nc.tilted(21, 30)
    strip = np.where(np.arange(21)[:, None] == 10, c["depth"], np.nan)
    assert (_gpu(strip, c["K"]) == 0).all()  # collinear inliers
    assert (_gpu(c["depth"], c["K"], min_inliers=50) == 0).all()  # a 7 x 7 window holds at most 49
    depth = np.full((21, 30), 1000.0)
    depth[10, 10] = 500.0
    got = _gpu(depth, c["K"])
    assert (got[10, 10] == 0).all() and (got[0, 0] != 0).any()
    assert (_gpu(np.zeros((21, 30)), c["K"]) == 0).all()


@pytest.mark.parametrize("H,W", [(1, 1), (7, 5), (1, 40), (33, 1), (9, 33), (37, 53), (61, 83), (1200, 1600)])
def test_kernel_sizes(H, W):
    c = nc.noisy(H, W, seed=H + W) if min(H, W) > 1 else nc.tilted(H, W)
    kw = {} if min(H, W) > 1 else {"min_inliers": 2}
    got = _check(c["depth"], c["K"], **kw)
    if min(H, W) > 1 and H * W > 35:
        assert (got != 0).any(-1).mean() > 0.5


@pytest.mark.parametrize("radius", [1, 2, 3, 4, 5, 6, 7])
def test_kernel_every_radius(radius):
    c = nc.noisy(70, 101, seed=radius)
    for thres, m in ((0.01, 6), (0.002, 3)):
        _check(c["depth"], c["K"], radius=radius, depth_thres=thres, min_inliers=m)
    with pytest.raises(RuntimeError, match="radius"):
        _gpu(c["depth"], c["K"], radius=radius + 7)


@pytest.fixture(scope="module")
def uniform_runs(tmp_path_factory):
    """The seeded plane scene (tests/scene_cases) reconstructed with and without --normals."""
    root = tmp_path_factory.mktemp("normals_scene")
    scene = str(root / "scene")
    scene_cases.write_scene(scene, 6, 128, 160, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *THRES]
    for name, extra in (("plain", []), ("normals", ["--normals"])):
        reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(root / name)] + extra), log=lambda *a: None)
    return scene, root


def test_kernel_on_a_network_depth_map_and_run_to_run(uniform_runs):
    scene, root = uniform_runs
    depth = data_io.read_map(str(root / "plain" / "depth_est" / "00000000.pfm"))[..., 0]
    _, oh, ow = data_io.read_image(os.path.join(scene, "images", "00000000.jpg"))
    k, _, _ = data_io.read_cam_file(os.path.join(scene, "cams", "00000000_cam.txt"))
    K = data_io.scale_intrinsics(k, depth.shape, oh, ow)
    frac = (_check(depth, K) != 0).any(-1).mean()
    assert frac > 0.5, frac
    for kw in ({}, {"radius": 5, "depth_thres": 0.005}, {"radius": 1, "min_inliers": 3}):
        got = _check(depth, K, **kw)
        again = _gpu(depth, K, **kw)
        assert got.tobytes() == again.tobytes()


def _ply(path):
    raw = open(path, "rb").read()
    head, _, body = raw.partition(b"end_header\n")
    return head.decode().split("\n"), body


def _files(d):
    out = {}
    for sub, _, names in os.walk(d):
        for n in names:
            out[os.path.relpath(os.path.join(sub, n), d)] = open(os.path.join(sub, n), "rb").read()
    return out


def _check_oriented_run(plain_dir, normals_dir):
    a, b = _files(plain_dir), _files(normals_dir)
    assert sorted(a) == sorted(b) and "fused.ply" in a
    for name in a:
        if name != "fused.ply":
            assert a[name] == b[name], name
    head_p, body_p = _ply(os.path.join(plain_dir, "fused.ply"))
    head_n, body_n = _ply(os.path.join(normals_dir, "fused.ply"))
    props = [line.split()[-1] for line in head_n if line.startswith("property")]
    assert props == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    assert [line for line in head_n if "element" in line] == [line for line in head_p if "element" in line]
    plain = np.frombuffer(body_p, dtype=np.uint8).reshape(-1, 15)
    rec = np.frombuffer(body_n, dtype=np.uint8).reshape(-1, 27)
    assert len(rec) == len(plain) > 0
    assert np.array_equal(np.concatenate([rec[:, :12], rec[:, 24:]], 1), plain)  # positions and colours
    _, nrm, _ = no.split_oriented(rec)
    nz = (nrm != 0).any(-1)
    assert nz.mean() > 0.5 and np.abs(np.linalg.norm(nrm[nz].astype(np.float64), axis=-1) - 1).max() < 1e-5


def test_reconstruct_normals_changes_only_fused_ply(uniform_runs):
    _, root = uniform_runs
    _check_oriented_run(str(root / "plain"), str(root / "normals"))


def test_reconstruct_normals_with_portrait_views(tmp_path):
    scene = str(tmp_path / "scene")
    multisize_cases.write_mixed_scene(scene, multisize_cases.mixed_sizes(5, 96, 128), n_src=4)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "2", *THRES]
    for name, extra in (("plain", []), ("normals", ["--normals"])):
        reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / name)] + extra),
                                log=lambda *a: None)
    _check_oriented_run(str(tmp_path / "plain"), str(tmp_path / "normals"))
    # the fusion-only form reads depth_est from disk and gives the same files
    before = _files(str(tmp_path / "normals"))
    reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / "normals"), "--output-type", "fusion",
                                                             "--normals"]), log=lambda *a: None)
    assert _files(str(tmp_path / "normals")) == before


def test_oriented_fusion_equals_the_plain_fusion():
    rng = np.random.default_rng(11)
    H, W = 301, 257  # not a multiple of the 256-pixel block
    mask = torch.from_numpy(rng.random((H, W)) < 0.4).to(DEV)
    avg = torch.from_numpy(rng.uniform(400, 900, (H, W))).to(DEV)
    img = torch.from_numpy(rng.random((H, W, 3), dtype=np.float32)).to(DEV)
    c = nc.noisy(H, W, seed=3)
    c["depth"][::7, ::5] = 0.0  # pixels without a normal
    normals = ops.estimate_normals(torch.from_numpy(c["depth"]).to(DEV), c["K"])
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    E[:3, 3] = [5.0, 20.0, -7.0]
    cam = ops.compose_fusion_camera(c["K"], E)
    plain = ops.fuse_points(mask, avg, img, cam).cpu().numpy()
    rec = ops.fuse_points(mask, avg, img, cam, normals).cpu().numpy()
    assert rec.shape == (len(plain), 27) and len(plain) == int(mask.sum())
    assert np.array_equal(np.concatenate([rec[:, :12], rec[:, 24:]], 1), plain)
    _, nrm, _ = no.split_oriented(rec)
    want = no.world_normals(normals.cpu().numpy()[mask.cpu().numpy()], E)
    np.testing.assert_allclose(nrm, want, rtol=0, atol=2e-7)
    zero = (want == 0).all(-1)
    assert zero.any() and (nrm[zero] == 0).all() and not np.signbit(nrm[zero]).any()
    with pytest.raises(RuntimeError, match="normals"):
        ops.fuse_points(mask, avg, img, cam, normals[1:])


def test_colmap_output_writes_normal_maps(tmp_path):
    from PIL import Image

    from tests.test_gpu_colmap import _plane_model

    n_views, (H, W) = 5, (128, 160)
    model, cams = _plane_model(n_views, H, W, 3000, seed=4)
    colmap = tmp_path / "colmap"
    cc.write_bin(str(colmap / "sparse"), model)
    (colmap / "images").mkdir()
    for i, (k, e) in enumerate(cams):
        Image.fromarray(scene_cases.texture(k, e, H, W)).save(str(colmap / "images" / ("view_%02d.png" % i)))
    scene, results, plain, ws = (tmp_path / n for n in ("scene", "results", "plain", "ws"))
    for d in (scene, plain, ws):
        d.mkdir()
    assert ci.main(["--input-folder", str(colmap), "--output-folder", str(scene), "--num-src-images", str(n_views - 2)]) == 0
    reconstruct.reconstruct(reconstruct.parse_args([
        "--input-folder", str(scene), "--output-folder", str(results), "--checkpoint-path", WEIGHTS, "--num-views", "2",
        "--image-max-dim", "80", *THRES]), log=lambda *a: None)
    assert cout.main(["--input-folder", str(scene), "--results-folder", str(results), "--output-folder", str(plain)]) == 0
    assert cout.main(["--input-folder", str(scene), "--results-folder", str(results), "--output-folder", str(ws), "--normals"]) == 0
    a, b = _files(str(plain)), _files(str(ws))
    maps = sorted(n for n in b if n.startswith(os.path.join("stereo", "normal_maps")))
    assert maps == [os.path.join("stereo", "normal_maps", f"{i:08d}.jpg.geometric.bin") for i in range(n_views)]
    assert {n: v for n, v in b.items() if n not in maps} == a
    for i in range(n_views):
        depth = data_io.read_map(str(results / "depth_est" / f"{i:08d}.pfm"))[..., 0]
        assert depth.shape == (64, 80)  # --image-max-dim 80 on 128 x 160 images
        k, _, _ = data_io.read_cam_file(str(scene / "cams" / f"{i:08d}_cam.txt"))
        want = ops.estimate_normals(torch.from_numpy(depth).to(DEV), data_io.scale_intrinsics(k, depth.shape, H, W)).cpu().numpy()
        path = str(ws / "stereo" / "normal_maps" / f"{i:08d}.jpg.geometric.bin")
        assert open(path, "rb").read().startswith(b"80&64&3&")  # W&H&C& at the depth map's size
        got = data_io.read_map(path)
        assert got.shape == (64, 80, 3) and np.array_equal(got, want)
        assert (got != 0).any(-1).mean() > 0.3
