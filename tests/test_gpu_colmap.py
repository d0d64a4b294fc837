"""COLMAP interop on the GPU: view scores and depth ranges (csrc/pm_colmap.cu through ops) against the CPU oracle,
oracle/colmap_oracle.py; the colmap_input command against the reference's recorded files (tests/golden/colmap_io.npz); and the
chain COLMAP model -> colmap_input -> reconstruct -> colmap_output.

Scores agree with the oracle to 1e-11 relative and depth ranges to 1e-12: the GPU's acos / exp and numpy's libm and BLAS dot
differ in the last bits only.  Models are generated from seeds (tests/colmap_cases.py)."""
import os

import numpy as np
import pytest

from oracle import colmap_oracle as co
from patchmatchnet_b200 import colmap_input as ci, colmap_output as cout, data_io, reconstruct
from tests import colmap_cases as cc, scene_cases
from tests.test_colmap import colmap_folder, golden, want_text  # noqa: F401  (golden is a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")


def _obs(sm):
    return [sm.obs_points[sm.obs_offsets[i]:sm.obs_offsets[i + 1]] for i in range(len(sm.obs_offsets) - 1)]


def _gpu(sm, theta0=5.0, sigma1=1.0, sigma2=10.0):
    s, r = ci.gpu_scores_and_ranges(sm, theta0, sigma1, sigma2, DEV)
    return s.cpu().numpy(), r.cpu().numpy()


def _check_against_oracle(sm, **kw):
    got_s, got_r = _gpu(sm, **kw)
    want_s = co.view_scores(sm.centers, _obs(sm), sm.xyz, **kw)
    want_r = np.array(co.depth_ranges(sm.extrinsics, _obs(sm), sm.xyz))
    assert (got_s == got_s.T).all() and (np.diag(got_s) == 0).all()
    assert ((got_s == 0) == (want_s == 0)).all()
    np.testing.assert_allclose(got_s, want_s, rtol=1e-11, atol=0)
    np.testing.assert_allclose(got_r, want_r, rtol=1e-12, atol=0)
    return got_s


def _model_dir(tmp_path, m, name="m"):
    d = str(tmp_path / name)
    cc.write_bin(d, m)
    return d


def test_fixture_scores_and_ranges_match_the_oracle(golden, tmp_path):
    root = colmap_folder(golden, str(tmp_path))
    sm = ci.prepare(*ci.read_model(os.path.join(root, "sparse")))
    _check_against_oracle(sm)
    _check_against_oracle(sm, theta0=3.0, sigma1=2.0, sigma2=7.5)


def test_60_image_model_matches_the_oracle_and_is_deterministic(tmp_path):
    m = cc.make_model(60, 60, 18000, track=5, n_invalid=7, id_base=2 ** 40, arc=2.0)
    iid, q, t, cid, name, obs = m["images"][10]
    m["images"][10] = (iid, q, t, cid, name, np.concatenate([obs, obs[obs != -1][:25]]))  # duplicates in one image
    sm = ci.prepare(*ci.read_model(_model_dir(tmp_path, m)))
    assert 1400 < sm.obs_points.size / 60 < 1600
    first = _check_against_oracle(sm)
    again, _ = _gpu(sm)
    assert first.tobytes() == again.tobytes()


def test_duplicates_collinear_and_coincident_points():
    # centres (0,0,-5), (1,0,-5), (2.5,0,-5) on a line; point 0 on that line beyond them (the cosine rounds to 1 or above),
    # point 1 on camera 0's centre (contributes 0 to pairs with camera 0), point 2 off the line, listed twice in images 0 and 1
    e = np.stack([np.eye(4)] * 3)
    e[:, 0, 3] = [0.0, -1.0, -2.5]
    e[:, 2, 3] = 5.0
    sm = ci.SceneModel(intrinsics=[np.eye(3)] * 3, extrinsics=e, centers=np.stack([ci.camera_center(x) for x in e]),
                       xyz=np.array([[7.3, 0.0, -5.0], [0.0, 0.0, -5.0], [1.0, 3.0, 0.5]]),
                       obs_offsets=np.array([0, 4, 8, 10], dtype=np.int32),
                       obs_points=np.array([2, 0, 1, 2, 0, 2, 2, 1, 0, 1], dtype=np.int32))
    got = _check_against_oracle(sm)
    assert np.isfinite(got).all() and got[0, 1] > 0 and got[0, 2] > 0


def test_pairs_without_shared_points_tie_in_descending_order(tmp_path):
    m = cc.make_model(5, 9, 400, track=2, arc=6.0)  # short tracks: most pairs share nothing
    sm = ci.prepare(*ci.read_model(_model_dir(tmp_path, m)))
    scores = _check_against_oracle(sm)
    for i, row in enumerate(ci.select_views(scores, -1)):
        zeros = [k for k, s in row if s == 0]
        assert len(zeros) >= 2 and zeros == sorted(zeros, reverse=True) and i in zeros


def test_command_writes_the_references_files(golden, tmp_path):
    root = colmap_folder(golden, str(tmp_path / "in"))
    out = str(tmp_path / "out")
    os.makedirs(out)
    assert ci.main(["--input-folder", root, "--output-folder", out]) == 0
    for i in range(12):
        with open(os.path.join(out, "cams", f"{i:08d}_cam.txt"), "rb") as f:
            assert f.read() == want_text(golden, f"input.cams/{i:08d}_cam.txt"), i
        name = f"img_{i:04d}.png"
        assert open(os.path.join(out, "images", f"{i:08d}.jpg"), "rb").read() == golden["file.images/" + name].tobytes()
    with open(os.path.join(out, "pair.txt"), "rb") as f:
        assert f.read() == want_text(golden, "input.pair.txt")


def _plane_model(n_views, H, W, n_points, seed):
    """A COLMAP model of scene_cases' plane scene: its cameras, and plane points seen from view 0, observed by every view they
    project into."""
    cams = scene_cases.cameras(n_views, H, W)
    rng = np.random.default_rng(seed)
    k0, e0 = (c.astype(np.float64) for c in cams[0])
    depth0 = scene_cases.plane_depth(*cams[0], H, W, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float64)
    u, v = rng.uniform(2, W - 3, n_points), rng.uniform(2, H - 3, n_points)
    d = depth0[v.astype(int), u.astype(int)]
    cam = np.linalg.inv(k0) @ np.stack([u, v, np.ones(n_points)]) * d
    xyz = (np.linalg.inv(e0) @ np.vstack([cam, np.ones(n_points)]))[:3].T
    ids = np.arange(1, n_points + 1, dtype=np.uint64) * np.uint64(7)
    cameras, images = [], []
    for i, (k, e) in enumerate(cams):
        k, e = k.astype(np.float64), e.astype(np.float64)
        cameras.append((i + 1, "PINHOLE", W, H, [k[0, 0], k[1, 1], k[0, 2], k[1, 2]]))
        p = k @ (e[:3, :3] @ xyz.T + e[:3, 3:4])
        px, py = p[0] / p[2], p[1] / p[2]
        seen = np.nonzero((px >= 0) & (px < W) & (py >= 0) & (py < H))[0]
        images.append((i + 1, cc.rotation_to_quaternion(e[:3, :3]), e[:3, 3], i + 1, "view_%02d.png" % i, ids[seen].astype(np.int64)))
    return {"cameras": cameras, "images": images, "point_ids": ids, "xyz": xyz, "rgb": np.zeros((n_points, 3), np.uint8),
            "error": np.zeros(n_points)}, cams


def test_chain_colmap_model_to_reconstruct_to_colmap_workspace(tmp_path):
    from PIL import Image

    n_views, (H, W) = 6, (128, 160)
    model, cams = _plane_model(n_views, H, W, 3000, seed=4)
    colmap = tmp_path / "colmap"
    cc.write_bin(str(colmap / "sparse"), model)
    (colmap / "images").mkdir()
    for i, (k, e) in enumerate(cams):
        Image.fromarray(scene_cases.texture(k, e, H, W)).save(str(colmap / "images" / ("view_%02d.png" % i)))
    scene, results, ws = tmp_path / "scene", tmp_path / "results", tmp_path / "ws"
    for d in (scene, ws):
        d.mkdir()
    assert ci.main(["--input-folder", str(colmap), "--output-folder", str(scene), "--num-src-images", str(n_views - 2)]) == 0
    for i, (k, e) in enumerate(cams):
        depth = scene_cases.plane_depth(k, e, H, W, scene_cases.PLANE_N, scene_cases.PLANE_D0)
        _, _, rng = data_io.read_cam_file(str(scene / "cams" / f"{i:08d}_cam.txt"))
        assert depth.min() - 1 <= rng[0] < depth[H // 2, W // 2] < rng[1] <= depth.max() + 1, (i, rng, depth.min(), depth.max())
    pairs = data_io.read_pair_file(str(scene / "pair.txt"))
    assert [r for r, _ in pairs] == list(range(n_views)) and all(r not in s and len(s) == n_views - 2 for r, s in pairs)
    stats = reconstruct.reconstruct(reconstruct.parse_args([
        "--input-folder", str(scene), "--output-folder", str(results), "--checkpoint-path", WEIGHTS, "--num-views", "2",
        "--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]), log=lambda *a: None)
    assert stats["depth_maps"] == n_views and stats["points"] > 0
    assert os.path.getsize(results / "fused.ply") > 200
    assert cout.main(["--input-folder", str(scene), "--results-folder", str(results), "--output-folder", str(ws)]) == 0
    for i in range(n_views):
        for kind, sub in (("depth_est", "depth_maps"), ("confidence", "confidence_maps")):
            got = data_io.read_map(str(ws / "stereo" / sub / f"{i:08d}.jpg.geometric.bin"))
            want = data_io.read_map(str(results / kind / f"{i:08d}.pfm"))
            assert got.shape == want.shape and (got == want).all()
    fusion = (ws / "stereo" / "fusion.cfg").read_text().split("\n")
    assert fusion[0].split(",")[0] == "00000000.jpg" and len(fusion[0].split(",")) == n_views - 1
