"""The Poisson mesher on the GPU: node by node against the float64 oracle (oracle/poisson_oracle.py) at depths 5 and 6, the
geometry of spheres and an open hemisphere, dropped points and reruns, a 10M-point cloud at depth 10 checked at sampled nodes
and by a float64 residual, and reconstruct --poisson on the plane scene."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo, poisson_oracle as po
from patchmatchnet_b200 import data_io, ops, poisson, reconstruct
from tests import mesh_cases as mc, scene_cases
from tests.test_gpu_mesh import THRES, WEIGHTS, _files
from tests.test_poisson import sphere_cloud

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-5


def hemisphere_cloud(n: int = 20000):
    xyz, nrm = sphere_cloud(n)
    keep = nrm[:, 2] > -0.2
    return xyz[keep], nrm[keep]


def colours_of(xyz):
    return np.clip(np.rint(255 * mc.colour_of(xyz.astype(np.float64))), 0, 255).astype(np.uint8)


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


CASES = {"sphere": lambda: sphere_cloud(), "hemisphere": lambda: hemisphere_cloud()}


@pytest.mark.parametrize("depth", [5, 6])
@pytest.mark.parametrize("case", sorted(CASES))
def test_matches_the_oracle_node_by_node(case, depth):
    xyz, nrm = CASES[case]()
    rgb = colours_of(xyz)
    ref = po.poisson(xyz, nrm, rgb, depth=depth, exact=depth == 5)
    fields, st = ops.poisson_fields(_t(xyz), _t(nrm), depth=depth, tol=TOL)
    assert st["N"] == ref["N"] and st["h"] == ref["h"] and st["I0"] == tuple(int(v) for v in ref["I0"])
    assert st["kept"] == int(ref["inside"].sum()) and st["converged"]
    rho, b, chi = (fields[k].cpu().numpy() for k in ("rho", "b", "chi"))
    w = fields["w"].cpu().numpy()
    assert np.abs(rho - ref["rho"]).max() <= 1e-5 * np.abs(ref["rho"]).max()
    assert np.allclose(w, ref["w"], rtol=1e-5, atol=0)
    assert np.abs(b - ref["b"]).max() <= 1e-5 * np.abs(ref["b"]).max()
    assert po.relative_residual(b, chi) <= 2 * TOL
    assert np.abs(chi - ref["chi"]).max() < 1e-3
    assert abs(st["iso"] - ref["iso"]) < 1e-5
    # the mesh: marching cubes of the GPU's own band field, and the nearest point's colours
    verts, faces, st2 = ops.poisson_mesh(_t(xyz), _t(nrm), _t(rgb), depth=depth, tol=TOL)
    assert st2 == st
    keys = mo.allocate(xyz[ref["inside"]], st["h"], 2)
    tsdf, weight = po.band_field(keys, np.array(st["I0"]), st["N"], chi, st["iso"])
    pos, _, want_faces = mo.marching_cubes(keys, st["h"], tsdf, weight, np.zeros((len(tsdf), 3), np.uint8))
    v = verts.cpu().numpy()
    assert np.array_equal(v[:, :12].copy().view(np.float32), pos)
    assert np.array_equal(faces.cpu().numpy(), want_faces)
    assert np.array_equal(v[:, 12:], po.nearest_colours(pos, xyz[ref["inside"]], rgb[ref["inside"]]))


@pytest.mark.parametrize("nonuniform", [False, True], ids=["uniform", "nonuniform"])
def test_sphere_is_closed_and_outward(nonuniform):
    xyz, nrm = sphere_cloud(200000, nonuniform)
    verts, faces, st = ops.poisson_mesh(_t(xyz), _t(nrm), depth=7)
    pos = verts.cpu().numpy().view(np.float32).reshape(-1, 3)
    f = faces.cpu().numpy()
    mc.check_closed_manifold(f, len(pos))
    n = mc.face_normals(pos, f)
    assert ((n * (pos[f].astype(np.float64).mean(1) - mc.SPHERE_CENTRE)).sum(1) > 0).all()
    radial = np.linalg.norm(pos.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS
    assert np.abs(radial).max() < 0.4 * st["h"], np.abs(radial).max() / st["h"]
    assert st["converged"] and verts.shape[1] == 12


def test_hemisphere_stays_in_the_band():
    from scipy.spatial import cKDTree

    xyz, nrm = hemisphere_cloud(100000)
    band = 2
    verts, faces, st = ops.poisson_mesh(_t(xyz), _t(nrm), depth=7, band=band)
    pos = verts.cpu().numpy().view(np.float32).reshape(-1, 3)
    assert len(faces) > 1000
    d, _ = cKDTree(xyz.astype(np.float64)).query(pos.astype(np.float64))
    # the band is whole 8^3-voxel blocks: a meshed voxel lies within band + 8 voxels of a point per axis, a vertex one more
    assert d.max() <= (band + 9) * math.sqrt(3) * st["h"], d.max() / st["h"]


def test_dropped_points_change_nothing_and_reruns_are_identical():
    xyz, nrm = sphere_cloud(30000)
    rgb = colours_of(xyz)
    a = ops.poisson_mesh(_t(xyz), _t(nrm), _t(rgb), depth=6)
    bad_xyz = np.concatenate([xyz, xyz[:3], [[np.nan, 0, 0]]]).astype(np.float32)
    bad_nrm = np.concatenate([nrm, np.zeros((3, 3)), [[0, 0, 1]]]).astype(np.float32)
    bad_rgb = np.concatenate([rgb, np.full((4, 3), 7, np.uint8)])
    # the dropped rows interleaved with the kept ones, which keep their order
    idx = np.concatenate([np.arange(len(xyz))[:, None], np.full((len(xyz), 1), -1)], 1).ravel()
    idx[1::2][:4] = np.arange(len(xyz), len(xyz) + 4)
    idx = idx[idx >= 0]
    b = ops.poisson_mesh(_t(bad_xyz[idx]), _t(bad_nrm[idx]), _t(bad_rgb[idx]), depth=6)
    assert b[2]["dropped"] == 4 and b[2]["kept"] == len(xyz)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = ops.poisson_mesh(_t(xyz), _t(nrm), _t(rgb), depth=6)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1]) and a[2] == c[2]


def test_no_kept_point_raises():
    with pytest.raises(ValueError, match="no point is kept"):
        ops.poisson_mesh(_t(np.zeros((4, 3), np.float32)), _t(np.zeros((4, 3), np.float32)))


def _relative_residual_torch(b: torch.Tensor, chi: torch.Tensor, slab: int = 32) -> float:
    """||b - A chi|| / ||b|| in float64, slab by slab, from shifted copies of chi (independent of the native stencil)."""
    N = chi.shape[0] - 1
    rr, bb = 0.0, float((b.double() ** 2).sum())
    for z0 in range(1, N, slab):
        z1 = min(z0 + slab, N)
        c = chi[z0 - 1 : z1 + 1].double()
        acc = torch.zeros((z1 - z0, N - 1, N - 1), dtype=torch.float64, device=chi.device)
        for dz in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    nz = (dx != 0) + (dy != 0) + (dz != 0)
                    wgt = [8.0 / 3.0, 0.0, -1.0 / 6.0, -1.0 / 12.0][nz]
                    if wgt:
                        acc += wgt * c[1 + dz : 1 + dz + z1 - z0, 1 + dy : N + dy, 1 + dx : N + dx]
        r = b[z0:z1, 1:N, 1:N].double() - acc
        rr += float((r * r).sum())
    return math.sqrt(rr / bb)


def test_depth_10_at_scale():
    n, depth = 10_000_000, 10
    need = ops.poisson_mesh_bytes(depth, n) + (1025 ** 3) * 16 + n * 8
    free = torch.cuda.mem_get_info(DEV)[0]
    if need > free:
        pytest.skip(f"depth 10 with {n} points needs {need / 2 ** 30:.1f} GiB, {free / 2 ** 30:.1f} GiB free on this shared card")
    d = mc.fibonacci(n)
    xyz = _t((mc.SPHERE_CENTRE + d).astype(np.float32))
    nrm = _t(d.astype(np.float32))
    fields, st = ops.poisson_fields(xyz, nrm, depth=depth, tol=TOL)
    assert st["N"] == 1024 and st["kept"] == n
    print("depth 10:", st)
    assert _relative_residual_torch(fields["b"], fields["chi"]) <= 2 * TOL
    # rho and b at 10k sampled nodes with rho > 0, from the points around them in float64
    h, I0 = st["h"], torch.tensor(st["I0"], dtype=torch.float64, device=DEV)
    u = xyz.double() / h - 0.5 - I0
    base = u.floor().clamp(0, 1023).long()
    f = u - base
    rho = fields["rho"].reshape(-1)
    g = torch.Generator(device="cpu").manual_seed(0)
    occupied = torch.nonzero(rho > 0).squeeze(1)
    sample = occupied[torch.randperm(len(occupied), generator=g)[:10000].to(DEV)].sort().values
    want_rho = torch.zeros(len(sample), dtype=torch.float64, device=DEV)
    rho_p = torch.zeros(n, dtype=torch.float64, device=DEV)
    corners = []
    for k in range(8):
        c = torch.tensor([k & 1, (k >> 1) & 1, k >> 2], device=DEV)
        wt = torch.where(c.bool(), f, 1 - f).prod(1)
        node = (base[:, 0] + c[0]) + 1025 * ((base[:, 1] + c[1]) + 1025 * (base[:, 2] + c[2]))
        corners.append((c, wt, node))
        rho_p += wt * rho[node]
        pos = torch.searchsorted(sample, node).clamp(max=len(sample) - 1)
        hit = sample[pos] == node
        want_rho.index_add_(0, pos[hit], wt[hit])
    assert (rho[sample] - want_rho).abs().max() <= 1e-5 * want_rho.abs().max()
    w = 1 / rho_p
    assert torch.allclose(fields["w"], w, rtol=1e-5, atol=0)
    unit = nrm.double() / nrm.double().norm(dim=1, keepdim=True)
    want_b = torch.zeros(len(sample), dtype=torch.float64, device=DEV)
    for c, wt, node in corners:
        sgn = torch.where(c.bool(), 1.0, -1.0).double()
        wa = torch.where(c.bool(), f, 1 - f)
        grad = torch.stack([sgn[0] * wa[:, 1] * wa[:, 2], wa[:, 0] * sgn[1] * wa[:, 2], wa[:, 0] * wa[:, 1] * sgn[2]], 1)
        val = w * (unit * grad).sum(1)
        pos = torch.searchsorted(sample, node).clamp(max=len(sample) - 1)
        hit = sample[pos] == node
        want_b.index_add_(0, pos[hit], val[hit])
    zyx = torch.stack([sample // (1025 * 1025), (sample // 1025) % 1025, sample % 1025], 1)
    interior = ((zyx > 0) & (zyx < 1024)).all(1)
    got_b = fields["b"].reshape(-1)[sample].double()
    assert (got_b - torch.where(interior, want_b, 0.0)).abs().max() <= 1e-5 * want_b.abs().max()
    del fields, u, base, f, rho_p, corners, w, unit
    torch.cuda.empty_cache()
    verts, faces, st2 = ops.poisson_mesh(xyz, nrm, depth=depth, tol=TOL)
    pos = verts.cpu().numpy().view(np.float32).reshape(-1, 3)
    radial = np.linalg.norm(pos.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - 1.0
    assert np.abs(radial).max() < 0.5 * st["h"], np.abs(radial).max() / st["h"]  # measured on an H100: 0.43 h
    assert len(faces) > 1_000_000


def test_reconstruct_poisson_on_the_plane_scene(tmp_path):
    scene = str(tmp_path / "scene")
    scene_cases.write_scene(scene, 6, 128, 160, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *THRES, "--normals"]
    run = lambda out, *extra: reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / out), *extra]),
                                                      log=lambda *a: None)
    plain_stats = run("plain")
    stats = run("poisson", "--poisson", "--poisson-depth", "7")
    assert not any(k.startswith("poisson") for k in plain_stats)
    plain, mesh = _files(str(tmp_path / "plain")), _files(str(tmp_path / "poisson"))
    assert sorted(mesh) == sorted(list(plain) + ["mesh_poisson.ply"])
    for name in plain:
        assert mesh[name] == plain[name], name
    assert stats["poisson_faces"] > 1000 and stats["poisson_vertices"] > 500 and stats["poisson_cycles"] > 0
    path = str(tmp_path / "poisson" / "mesh_poisson.ply")
    near = mc.plane_distance(data_io.read_ply_points(path))
    fused = mc.plane_distance(data_io.read_ply_points(str(tmp_path / "poisson" / "fused.ply")))
    assert np.median(near) <= np.median(fused) + 6.0, (np.median(near), np.median(fused))
    out = str(tmp_path / "standalone.ply")
    poisson.main(["--ply", str(tmp_path / "poisson" / "fused.ply"), "--output", out, "--depth", "7"])
    assert open(out, "rb").read() == open(path, "rb").read()
