"""The TSDF mesher on the GPU: allocation, integration and extraction against oracle/mesh_oracle.py, ops.tsdf_mesh end to end
on the analytic sphere (closed, outward, bit-identical reruns, views of mixed sizes, 300+ views), and reconstruct --mesh.

Integration tolerances: a weight may differ where a voxel projects onto a pixel-rounding tie (at most 1e-5 of the voxels);
where the weights agree tsdf is within 1e-5 and colour within 1."""
import os

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from patchmatchnet_b200 import data_io, ops, reconstruct
from tests import mesh_cases as mc, scene_cases

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
THRES = ["--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]


def _dev(sc):
    return ([torch.from_numpy(d).to(DEV) for d in sc["depths"]], [torch.from_numpy(i).to(DEV) for i in sc["images"]],
            torch.from_numpy(sc["seeds"]).to(DEV))


def _keys(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module")
def sphere():
    sc = mc.sphere_scene()
    return sc, 0.05


def test_allocation_equals_the_oracle(sphere):
    sc, s = sphere
    for trunc in (1, 3, 4):
        got = _keys(ops.tsdf_allocate(torch.from_numpy(sc["seeds"]).to(DEV), s, trunc))
        assert np.array_equal(got, mo.allocate(sc["seeds"], s, trunc))


def test_allocation_with_a_far_outlier_stays_proportional():
    rng = np.random.default_rng(4)
    pts = rng.normal(size=(5000, 3)).astype(np.float32) * 0.2
    far = np.concatenate([pts, np.array([[4000.0, -2500.0, 9000.0], [-70000.0, 3.0, 1.0]], np.float32)])
    s = 0.01
    base = _keys(ops.tsdf_allocate(torch.from_numpy(pts).to(DEV), s, 3))
    got = _keys(ops.tsdf_allocate(torch.from_numpy(far).to(DEV), s, 3))
    assert np.array_equal(got, mo.allocate(far, s, 3))
    assert len(base) < len(got) <= len(base) + 16
    with pytest.raises(ValueError, match="does not fit"):
        ops.tsdf_allocate(torch.tensor([[1e6, 0.0, 0.0]], device=DEV), s, 3)
    with pytest.raises(ValueError, match="does not fit"):
        ops.tsdf_allocate(torch.tensor([[float("nan"), 0.0, 0.0]], device=DEV), s, 3)
    assert ops.tsdf_allocate(torch.zeros((0, 3), device=DEV), s, 3).shape == (0,)


def _check_volume(got, want):
    tsdf, weight, colour = (t.cpu().numpy() for t in got)
    wt, ww, wc = want
    same = weight == ww
    assert (~same).mean() <= 1e-5, (~same).sum()
    assert np.abs(tsdf[same] - wt[same]).max() <= 1e-5
    assert np.abs(colour[same, :3].astype(int) - wc[same].astype(int)).max() <= 1
    assert (colour[:, 3] == 0).all()
    return same


def test_integration_equals_the_oracle(sphere):
    sc, s = sphere
    depths, images, seeds = _dev(sc)
    keys = ops.tsdf_allocate(seeds, s, 3)
    got = ops.tsdf_integrate(keys, depths, images, sc["Ks"], sc["Es"], s, 3)
    want = mo.integrate(_keys(keys), s, 3, sc["depths"], sc["images"], sc["Ks"], sc["Es"])
    _check_volume(got, want)
    assert (want[1] > 0).mean() > 0.1


def test_extraction_equals_the_oracle_on_the_gpu_grid(sphere):
    sc, s = sphere
    depths, images, seeds = _dev(sc)
    for min_weight in (1, 3):
        keys = ops.tsdf_allocate(seeds, s, 3)
        vol = ops.tsdf_integrate(keys, depths, images, sc["Ks"], sc["Es"], s, 3)
        verts, faces = ops.tsdf_extract(keys, *vol, s, min_weight)
        pos, col, wf = mo.marching_cubes(_keys(keys), s, *(t.cpu().numpy() for t in vol), min_weight=min_weight)
        v = verts.cpu().numpy()
        assert v.shape == (len(pos), 15)
        gp = v[:, :12].copy().view(np.float32)
        assert np.abs(gp - pos).max() <= 1e-6 * max(1.0, np.abs(pos).max())
        assert np.array_equal(v[:, 12:], col)
        assert np.array_equal(faces.cpu().numpy(), wf)


def _check_sphere(verts, faces, s):
    v = verts.cpu().numpy()
    pos = v[:, :12].copy().view(np.float32)
    f = faces.cpu().numpy()
    mc.check_closed_manifold(f, len(pos))
    n = mc.face_normals(pos, f)
    c = pos[f].astype(np.float64).mean(1) - mc.SPHERE_CENTRE
    assert ((n * c).sum(1) > 0).all()
    radial = np.linalg.norm(pos.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS
    assert np.abs(radial).max() < 0.5 * s


def test_sphere_end_to_end_and_bit_identical_reruns(sphere):
    sc, s = sphere
    depths, images, seeds = _dev(sc)
    a = ops.tsdf_mesh(seeds, depths, images, sc["Ks"], sc["Es"], s)
    b = ops.tsdf_mesh(seeds, depths, images, sc["Ks"], sc["Es"], s)
    _check_sphere(*a, s)
    assert a[0].cpu().numpy().tobytes() == b[0].cpu().numpy().tobytes()
    assert a[1].cpu().numpy().tobytes() == b[1].cpu().numpy().tobytes()


def test_sphere_with_views_of_mixed_sizes():
    sc = mc.sphere_scene(n_views=15, sizes=[(120, 160), (160, 120), (97, 133)])
    s = 0.05
    depths, images, seeds = _dev(sc)
    _check_sphere(*ops.tsdf_mesh(seeds, depths, images, sc["Ks"], sc["Es"], s), s)
    keys = ops.tsdf_allocate(seeds, s, 3)
    _check_volume(ops.tsdf_integrate(keys, depths, images, sc["Ks"], sc["Es"], s, 3),
                  mo.integrate(_keys(keys), s, 3, sc["depths"], sc["images"], sc["Ks"], sc["Es"]))


def test_sphere_with_300_views():
    sc = mc.sphere_scene(n_views=317, H=36, W=48, f=50.0)
    s = 0.08
    depths, images, seeds = _dev(sc)
    keys = ops.tsdf_allocate(seeds, s, 3)
    _check_volume(ops.tsdf_integrate(keys, depths, images, sc["Ks"], sc["Es"], s, 3),
                  mo.integrate(_keys(keys), s, 3, sc["depths"], sc["images"], sc["Ks"], sc["Es"]))
    _check_sphere(*ops.tsdf_mesh(seeds, depths, images, sc["Ks"], sc["Es"], s), s)


def test_tsdf_mesh_memory_error_names_the_blocks(sphere):
    sc, _ = sphere
    depths, images, seeds = _dev(sc)
    big = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (1000000, 3)).astype(np.float32)).to(DEV) * 1000
    with pytest.raises(ValueError, match="blocks.*larger voxel size"):
        ops.tsdf_mesh(big, depths, images, sc["Ks"], sc["Es"], 0.01)


# ---- reconstruct --mesh -----------------------------------------------------------------------------------------------------

def _files(d):
    out = {}
    for sub, _, names in os.walk(d):
        for n in names:
            out[os.path.relpath(os.path.join(sub, n), d)] = open(os.path.join(sub, n), "rb").read()
    return out


def test_reconstruct_mesh_on_the_plane_scene(tmp_path):
    scene = str(tmp_path / "scene")
    scene_cases.write_scene(scene, 6, 128, 160, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *THRES]
    run = lambda out, *extra: reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / out), *extra]),
                                                      log=lambda *a: None)
    run("plain")
    stats = run("mesh", "--mesh")
    plain, mesh = _files(str(tmp_path / "plain")), _files(str(tmp_path / "mesh"))
    assert sorted(mesh) == sorted(list(plain) + ["mesh.ply"])
    for name in plain:
        assert mesh[name] == plain[name], name
    assert stats["mesh_faces"] > 1000 and stats["mesh_vertices"] > 500 and stats["mesh_seconds"] > 0
    pts = data_io.read_ply_points(str(tmp_path / "mesh" / "mesh.ply"))
    assert len(pts) == stats["mesh_vertices"]
    # the network's maps of this small scene are noisy: the mesh must be no farther from the plane than the fused points
    near, fused = mc.plane_distance(pts), mc.plane_distance(data_io.read_ply_points(str(tmp_path / "mesh" / "fused.ply")))
    assert np.median(near) <= np.median(fused) + 6.0, (np.median(near), np.median(fused))
    # the fusion-only form reads the maps from disk and gives the same mesh.ply
    before = _files(str(tmp_path / "mesh"))
    run("mesh", "--mesh", "--output-type", "fusion")
    assert _files(str(tmp_path / "mesh")) == before


def test_reconstruct_mesh_from_analytic_plane_maps(tmp_path):
    """--output-type fusion over the plane's analytic maps (tests/scene_cases.write_fusion_maps: exact depth, corrupted in
    blocks by 0.5-5 %, 0.05 noise): the mesh lies on the plane."""
    scene, out = str(tmp_path / "scene"), str(tmp_path / "out")
    sc = scene_cases.write_scene(scene, 6, 96, 128, n_src=5)
    scene_cases.write_fusion_maps(out, sc["cams"], 96, 128, seed=3)
    s = 5.0
    stats = reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", scene, "--output-folder", out, "--checkpoint-path",
                                                            WEIGHTS, "--output-type", "fusion", "--geo-mask-thres", "2", "--mesh",
                                                            "--mesh-voxel-size", str(s)]), log=lambda *a: None)
    dist = mc.plane_distance(data_io.read_ply_points(os.path.join(out, "mesh.ply")))
    assert stats["mesh_faces"] > 500
    assert np.median(dist) < 0.25 * s and np.percentile(dist, 99) < 1.0 * s, (np.median(dist) / s, np.percentile(dist, 99) / s)
