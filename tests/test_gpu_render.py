"""The renderer on the GPU: ops.render_points and ops.render_mesh bit-identical to tests/render_oracle.py (RGB and depth), reruns,
empty inputs and clouds above 2^24 points; agreement with the analytic TSDF sphere and with a view's own fused points; and
the render command end to end after reconstruct --mesh."""
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

from patchmatchnet_b200 import data_io, ops, reconstruct, render
from tests import mesh_cases as mc
from tests import render_cases as rc
from tests import render_oracle as ro
from tests import scene_cases
from tests.geo_cases import plane_depth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")


def _d(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _same(got, want):
    g_rgb, g_depth = (t.cpu().numpy() for t in got)
    w_rgb, w_depth = want
    assert g_rgb.shape == w_rgb.shape and g_depth.shape == w_depth.shape
    bad = np.argwhere((g_rgb != w_rgb).any(-1) | (g_depth.view(np.uint32) != w_depth.view(np.uint32)))
    assert bad.size == 0, (len(bad), bad[:5], g_rgb[tuple(bad[0])], w_rgb[tuple(bad[0])], g_depth[tuple(bad[0])], w_depth[tuple(bad[0])])


@pytest.fixture(scope="module")
def cloud():
    return rc.cloud(1_200_000, seed=3)


@pytest.mark.parametrize("point_size,shade", [(1, False), (1, True), (3, True), (7, False)])
def test_render_points_equals_the_oracle(cloud, point_size, shade):
    xyz, rgb, nrm = cloud
    P = rc.pinhole()
    got = ops.render_points(_d(xyz), _d(rgb), _d(nrm), P, rc.W, rc.H, 0.5, point_size=point_size, shade=shade, background=(10, 20, 30))
    want = ro.render_points(xyz, rgb, nrm, P, rc.W, rc.H, 0.5, point_size=point_size, shade=shade, background=(10, 20, 30))
    assert (want[1] > 0).mean() > 0.5
    _same(got, want)
    again = ops.render_points(_d(xyz), _d(rgb), _d(nrm), P, rc.W, rc.H, 0.5, point_size=point_size, shade=shade, background=(10, 20, 30))
    for a, b in zip(got, again):
        assert torch.equal(a, b)


def test_render_points_without_colours_from_a_rotated_camera(cloud):
    xyz, _, nrm = cloud
    E = mc.look_at(np.array([0.5, -0.3, -1.0]), np.array([0.0, 0.0, 4.0])).astype(np.float64)
    P = rc.pinhole(E=E)
    _same(ops.render_points(_d(xyz), None, _d(nrm), P, 257, 131, 0.1, point_size=5, shade=True),
          ro.render_points(xyz, None, nrm, P, 257, 131, 0.1, point_size=5, shade=True))


@pytest.mark.parametrize("shade", [False, True])
def test_render_mesh_equals_the_oracle(shade):
    xyz, rgb, faces = rc.mesh(seed=1)
    P = rc.pinhole()
    t = ro.setup(ro.project_vertices(*ro.camera(P)[:1], xyz, rc.W, rc.H, 0.05), faces, rc.W, rc.H)
    bw = t["x1"] - t["x0"] + 1
    assert (t["ok"] & (bw > 16)).sum() > 10 and (t["ok"] & (bw <= 16)).sum() > 100  # both raster paths carry faces
    got = ops.render_mesh(_d(xyz), _d(rgb), _d(faces), P, rc.W, rc.H, 0.05, shade=shade)
    want = ro.render_mesh(xyz, rgb, faces, P, rc.W, rc.H, 0.05, shade=shade)
    assert (want[1] > 0).all()  # the far quad fills the frame
    _same(got, want)
    again = ops.render_mesh(_d(xyz), _d(rgb), _d(faces), P, rc.W, rc.H, 0.05, shade=shade)
    for a, b in zip(got, again):
        assert torch.equal(a, b)
    # without colours, from a camera close to the grid (most faces take the large-triangle path)
    E = mc.look_at(np.array([0.1, 0.05, 1.2]), np.array([0.0, 0.0, 3.0])).astype(np.float64)
    P = rc.pinhole(E=E, w=401, h=333)
    _same(ops.render_mesh(_d(xyz), None, _d(faces), P, 401, 333, 0.05, shade=shade),
          ro.render_mesh(xyz, None, faces, P, 401, 333, 0.05, shade=shade))


def test_empty_inputs_give_the_background():
    P = rc.pinhole()
    e3 = torch.empty((0, 3), dtype=torch.float32, device=DEV)
    rgb, depth = ops.render_points(e3, None, None, P, 7, 5, 0.1, background=(1, 2, 3))
    assert (rgb.cpu().numpy() == [1, 2, 3]).all() and (depth == 0).all()
    rgb, depth = ops.render_mesh(e3, None, torch.empty((0, 3), dtype=torch.int32, device=DEV), P, 7, 5, 0.1, background=(1, 2, 3))
    assert (rgb.cpu().numpy() == [1, 2, 3]).all() and (depth == 0).all()
    with pytest.raises(ValueError):
        ops.render_mesh(_d(np.zeros((3, 3), np.float32)), None, _d(np.array([[0, 1, 3]], np.int32)), P, 7, 5, 0.1)
    with pytest.raises(ValueError):
        ops.render_points(e3, None, None, P, 7, 5, 0.1, point_size=4)


def test_cloud_above_2_24_points():
    n = (1 << 24) + 300_000
    rng = np.random.default_rng(5)
    xyz = np.stack([rng.uniform(-1, 1, n), rng.uniform(-0.75, 0.75, n), rng.uniform(4.0, 6.0, n)], 1).astype(np.float32)
    xyz[1 << 24:, 2] = 2.0  # the last points are the nearest: the winners carry indices above 2^24
    xyz[1 << 24:, :2] *= 0.5
    rgb = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    P = rc.pinhole(f=100.0, w=200, h=150)
    got = ops.render_points(_d(xyz), _d(rgb), None, P, 200, 150, 0.1)
    want = ro.render_points(xyz, rgb, None, P, 200, 150, 0.1)
    _same(got, want)
    assert (want[1] == 2.0).sum() > 1000


def test_tsdf_sphere_depth_within_one_voxel():
    """The TSDF mesh of the analytic sphere, rendered from each scene camera: its depth is within one voxel of the analytic
    depth on every pixel where both are valid, away from the silhouette (2 pixels), where a ray grazes the surface."""
    sc = mc.sphere_scene()
    s = 0.05
    verts, faces = ops.tsdf_mesh(_d(sc["seeds"]), [_d(d) for d in sc["depths"]], [_d(i) for i in sc["images"]], sc["Ks"], sc["Es"], s)
    xyz = verts[:, :12].contiguous().view(torch.float32).view(-1, 3)
    col = verts[:, 12:].contiguous()
    for K, E, want in zip(sc["Ks"], sc["Es"], sc["depths"]):
        h, w = want.shape
        P = K.astype(np.float64) @ E.astype(np.float64)[:3]
        _, depth = ops.render_mesh(xyz, col, faces, P, w, h, 0.01, shade=True)
        got = depth.cpu().numpy()
        valid = want > 0
        interior = valid.copy()
        for dy in range(-2, 3):
            for dx in range(-2, 3):
                interior &= np.roll(np.roll(valid, dy, 0), dx, 1)
        both = interior & (got > 0)
        assert both.sum() > 0.9 * interior.sum()
        assert np.abs(got[both] - want[both]).max() <= s, np.abs(got[both] - want[both]).max()


def test_fused_points_cover_exactly_the_final_mask():
    H, W = 96, 128
    cams = scene_cases.cameras(3, H, W)
    K, E = cams[2]
    rng = np.random.default_rng(4)
    depth = plane_depth(K, E, H, W, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float64)
    final = rng.random((H, W)) < 0.6
    img = rng.random((H, W, 3)).astype(np.float32)
    body = ops.fuse_points(_d(final), _d(depth), _d(img), ops.compose_fusion_camera(K, E))
    xyz = body[:, :12].contiguous().view(torch.float32).view(-1, 3)
    P = K.astype(np.float64) @ E.astype(np.float64)[:3]
    _, got = ops.render_points(xyz, body[:, 12:].contiguous(), None, P, W, H, 1.0)
    got = got.cpu().numpy()
    assert ((got > 0) == final).all()
    rel = np.abs(got[final] - depth[final]) / depth[final]
    assert rel.max() <= 1e-5, rel.max()


def _png(path):
    return np.array(Image.open(path))


def test_render_command_after_reconstruct_mesh(tmp_path):
    scene, out = str(tmp_path / "scene"), str(tmp_path / "out")
    sc = scene_cases.write_scene(scene, 6, 96, 128, n_src=5)
    scene_cases.write_fusion_maps(out, sc["cams"], 96, 128, seed=3)
    reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", scene, "--output-folder", out, "--checkpoint-path", WEIGHTS,
                                                    "--output-type", "fusion", "--geo-mask-thres", "2", "--mesh", "--mesh-voxel-size",
                                                    "5"]), log=lambda *a: None)
    K = np.array([[300.0, 0, 159.5], [0, 300.0, 99.5], [0, 0, 1]])
    Ev = np.eye(4)
    Ev[:3, 3] = [0.0, 0.0, 50.0]
    vp = str(tmp_path / "vp.json")
    with open(vp, "w") as f:
        json.dump({"class_name": "PinholeCameraParameters", "extrinsic": Ev.ravel(order="F").tolist(),
                   "intrinsic": {"width": 320, "height": 200, "intrinsic_matrix": K.ravel(order="F").tolist()}}, f)
    for name in ("fused.ply", "mesh.ply"):
        dst = str(tmp_path / ("r_" + name))
        ply = os.path.join(out, name)
        stats = render.render(render.parse_args(["--ply", ply, "--input-folder", scene, "--views", "0", "3", "--orbit", "4",
                                                 "--viewpoint", vp, "--depth", "--shade", "--width", "160", "--height", "120",
                                                 "--output-folder", dst]), log=lambda *a: None)
        assert stats["frames"] == 7 and stats["render_seconds"] > 0 and stats["upload_seconds"] >= 0
        want = {"view_00000000", "view_00000003", "viewpoint"} | {"orbit_%04d" % k for k in range(4)}
        assert set(os.listdir(dst)) == {s + e for s in want for e in (".png", ".pfm")}
        xyz, rgb, nrm, faces = data_io.read_ply(ply)
        assert (faces is not None) == (name == "mesh.ply")
        d_xyz = _d(xyz)
        box = render.percentile_box(d_xyz)
        for stem, P, w, h in render.frames(render.parse_args(["--ply", ply, "--input-folder", scene, "--views", "0", "3", "--orbit",
                                                              "4", "--viewpoint", vp, "--width", "160", "--height", "120"]), box):
            png, pfm = _png(os.path.join(dst, stem + ".png")), data_io.read_map(os.path.join(dst, stem + ".pfm"))
            assert png.shape == (h, w, 3) and pfm.shape[:2] == (h, w)
            near = 1e-3 * np.linalg.norm(render.camera_centre(P) - (box[0] + box[1]) / 2)
            if faces is not None:
                img, depth = ops.render_mesh(d_xyz, _d(rgb), _d(faces), P, w, h, near, shade=True)
            else:
                img, depth = ops.render_points(d_xyz, _d(rgb), _d(nrm), P, w, h, near, shade=True)
            assert (png == img.cpu().numpy()).all() and (pfm[..., 0] == depth.cpu().numpy()).all()
            assert (depth > 0).any(), stem
        assert _png(os.path.join(dst, "view_00000000.png")).shape == (96, 128, 3)
