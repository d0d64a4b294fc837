"""The mesh texturer on the GPU against oracle/texture_oracle.py, bit for bit (labels, charts, placements, texture coordinate
bits and page bytes): the TSDF sphere raw and simplified, the plane, and views of different sizes; the round trip through
the textured renderer; edge cases; bit-identical reruns; reconstruct --mesh-texture and the texture command end to end;
and the tnt and eth3d scene-size rows simplified to 1 % against texture_mesh_bytes."""
import os

import numpy as np
import pytest
import torch

from oracle import texture_oracle as to
from patchmatchnet_b200 import data_io, ops, reconstruct, texture
from tests import mesh_cases as mc, render_oracle as ro, scene_cases
from tests.test_gpu_mesh_at_scene_sizes import build_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
THRES = ["--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _tsdf(scene, s, share=None):
    verts, faces = ops.tsdf_mesh(_d(scene["seeds"]), [_d(x) for x in scene["depths"]], [_d(x) for x in scene["images"]],
                                 scene["Ks"], scene["Es"], s)
    xyz, rgb = verts[:, :12].contiguous().view(torch.float32), verts[:, 12:].contiguous()
    if share is not None:
        body, faces, _ = ops.simplify_mesh(xyz, rgb, faces, int(faces.shape[0] * share))
        xyz, rgb = body[:, :12].contiguous().view(torch.float32), body[:, 12:].contiguous()
    return xyz, rgb, faces


def _gpu(xyz, rgb, faces, images, Ks, Es):
    uv, page, pages, stats = ops.texture_mesh(xyz, rgb, faces, [_d(i) for i in images], Ks, Es)
    return uv.cpu().numpy(), page.cpu().numpy(), pages.cpu().numpy(), stats


def _same(xyz, rgb, faces, images, Ks, Es):
    got = _gpu(xyz, rgb, faces, images, Ks, Es)
    want = to.texture(xyz.cpu().numpy(), None if rgb is None else rgb.cpu().numpy(), faces.cpu().numpy(), images, Ks, Es)
    label, table, _, _ = ops.texture_labels(xyz, faces, [_d(i) for i in images], Ks, Es)
    assert np.array_equal(label.cpu().numpy(), want["label"])
    assert np.array_equal(table.cpu().numpy(), want["table"])
    assert np.array_equal(got[0].view(np.uint32), want["uv"].view(np.uint32))
    assert np.array_equal(got[1], want["page"])
    assert got[2].shape == want["pages"].shape and np.array_equal(got[2], want["pages"])
    st = got[3]
    assert st["charts"] == len(want["table"]) and st["untextured_faces"] == int((want["label"] < 0).sum())
    print(f"[texture] {faces.shape[0]} faces: {st}")
    return got, want


@pytest.fixture(scope="module")
def sphere():
    return mc.sphere_scene()


@pytest.mark.parametrize("share", [None, 0.1, 0.02])
def test_sphere_equals_the_oracle(sphere, share):
    xyz, rgb, faces = _tsdf(sphere, 0.05, share)
    got, want = _same(xyz, rgb, faces, sphere["images"], sphere["Ks"], sphere["Es"])
    assert (want["label"] >= 0).mean() > 0.9


def test_plane_equals_the_oracle():
    scn = mc.plane_scene()
    xyz, rgb, faces = _tsdf(scn, 8.0)
    _same(xyz, rgb, faces, scn["images"], scn["Ks"], scn["Es"])


def test_views_of_different_sizes_equal_the_oracle():
    scn = mc.sphere_scene(n_views=8, sizes=[(120, 160), (160, 120), (90, 200)])
    xyz, rgb, faces = _tsdf(scn, 0.05, 0.1)
    _same(xyz, rgb, faces, scn["images"], scn["Ks"], scn["Es"])


def test_reruns_are_bit_identical(sphere):
    xyz, rgb, faces = _tsdf(sphere, 0.05, 0.1)
    a = _gpu(xyz, rgb, faces, sphere["images"], sphere["Ks"], sphere["Es"])
    b = _gpu(xyz, rgb, faces, sphere["images"], sphere["Ks"], sphere["Es"])
    for x, y in zip(a[:3], b[:3]):
        assert np.array_equal(x, y)


def test_round_trip_reproduces_the_input_pixels(sphere):
    """Rendering the textured mesh from a texturing view reproduces that view's pixels wherever the front face carries the
    view's label (the images are not resized, so every texel is an input byte).  A pixel may differ only where the float32
    interpolation of the texture coordinate lands on the other side of a texel boundary.  Observed on an H100: 0 of 60 905
    pixels differ; up to 0.1 % is allowed."""
    xyz, rgb, faces = _tsdf(sphere, 0.05, 0.1)
    images = [np.rint(im * 255).astype(np.float32) / np.float32(255) for im in sphere["images"]]
    uv, page, pages, _ = ops.texture_mesh(xyz, rgb, faces, [_d(i) for i in images], sphere["Ks"], sphere["Es"])
    label = ops.texture_labels(xyz, faces, [_d(i) for i in images], sphere["Ks"], sphere["Es"])[0].cpu().numpy()
    vws = to.views(sphere["Ks"], sphere["Es"], [im.shape[1:] for im in images], to.box_centre(xyz.cpu().numpy()))
    checked = differ = 0
    for v, (P, C, near, W, H) in enumerate(vws):
        img, _ = ops.render_mesh_textured(xyz, faces, uv, page, pages, P, W, H, near)
        P32, _ = ro.camera(P)
        zbuf, _ = ro.mesh_zbuffer(ro.project_vertices(P32, xyz.cpu().numpy(), W, H, np.float32(near)), faces.cpu().numpy(), W, H)
        hit = zbuf != ro.EMPTY
        win = np.full(zbuf.shape, -1)
        win[hit] = (zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        mine = hit & (label[np.maximum(win, 0)] == v)
        want = np.rint(images[v] * np.float32(255)).astype(np.uint8).transpose(1, 2, 0)
        diff = (img.cpu().numpy() != want).any(2) & mine
        checked += int(mine.sum())
        differ += int(diff.sum())
    print(f"[round trip] {differ} of {checked} pixels differ")
    assert checked > 10000
    assert differ <= 1e-3 * checked


def test_edge_cases():
    scn = mc.sphere_scene(n_views=3)
    xyz, rgb, faces = _tsdf(scn, 0.1)
    imgs = [_d(i) for i in scn["images"]]
    # empty mesh
    uv, page, pages, st = ops.texture_mesh(xyz, rgb, faces[:0], imgs, scn["Ks"], scn["Es"])
    assert uv.shape == (0, 3, 2) and page.shape == (0,) and st["charts"] == 0
    # seen by no view: the cameras turned away; every face untextured, with its vertices' mean colour
    away = [np.diag([1, 1, -1, 1]).astype(np.float32) @ E for E in scn["Es"]]
    got, want = _same(xyz, rgb, faces, scn["images"], scn["Ks"], away)
    assert (want["label"] < 0).all() and got[3]["charts"] == 0
    f = faces.cpu().numpy()
    c = rgb.cpu().numpy().astype(np.float64)[f]
    mean = np.rint(((c[:, 0] + c[:, 1]) + c[:, 2]) / 3.0).astype(np.uint8)
    S = got[2].shape[1]
    tx = np.floor(got[0][:, 0, 0] * S).astype(int)
    ty = np.floor((1 - got[0][:, 0, 1]) * S).astype(int)
    assert np.array_equal(got[2][got[1], ty, tx], mean)
    # a view that sees nothing next to ones that do, and a face outside every image
    Ks, Es = list(scn["Ks"]) + [scn["Ks"][0]], list(scn["Es"]) + [away[0]]
    far = torch.tensor([[50.0, 50.0, 50.0], [51.0, 50.0, 50.0], [50.0, 51.0, 50.0]], device=DEV)
    xyz2 = torch.cat([xyz, far])
    faces2 = torch.cat([faces, torch.arange(xyz.shape[0], xyz.shape[0] + 3, dtype=torch.int32, device=DEV)[None]])
    rgb2 = torch.cat([rgb, torch.full((3, 3), 7, dtype=torch.uint8, device=DEV)])
    got, want = _same(xyz2, rgb2, faces2, list(scn["images"]) + [scn["images"][0]], Ks, Es)
    assert want["label"][-1] == -1 and not (want["label"] == 3).any()
    assert got[2][got[1][-1], int(np.floor((1 - got[0][-1, 0, 1]) * S)), int(np.floor(got[0][-1, 0, 0] * S))].tolist() == [7, 7, 7]


def test_quality_against_vertex_colours():
    """A finely tessellated plane with a checkerboard rendered from 6 views; its 2 % simplification textured from those
    renders and vertex-coloured, both rendered from held-out viewpoints and compared with the fine mesh's renders.  Measured
    mean absolute errors on an H100: 2.80 textured, 36.46 with vertex colours; the textured error must stay below a quarter
    of the vertex-coloured one."""
    n = 200
    g = np.stack(np.meshgrid(np.linspace(-1, 1, n + 1), np.linspace(-1, 1, n + 1)), -1).reshape(-1, 2)
    xyz = np.concatenate([g, np.full((len(g), 1), 4.0)], 1).astype(np.float32)
    i = np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]
    i = i.ravel()
    faces = np.concatenate([np.stack([i, i + n + 2, i + 1], 1), np.stack([i, i + n + 1, i + n + 2], 1)]).astype(np.int32)
    cen = xyz[faces].mean(1)
    check = ((np.floor(cen[:, 0] * 8) + np.floor(cen[:, 1] * 8)) % 2).astype(bool)
    # the checkerboard per face: split the vertices so each face carries its own colour
    fx = xyz[faces].reshape(-1, 3)
    fc = np.repeat(np.where(check[:, None], [[230, 40, 40]], [[30, 60, 200]]).astype(np.uint8), 3, 0)
    ff = np.arange(len(fx), dtype=np.int32).reshape(-1, 3)
    W = H = 256

    def cam(ex, ey):
        E = mc.look_at(np.array([ex, ey, 0.0]), np.array([0.0, 0.0, 4.0]))
        K = np.array([[300, 0, 127.5], [0, 300, 127.5], [0, 0, 1]], np.float32)
        return K, E

    train = [cam(x, y) for x, y in ((0, 0), (0.8, 0), (-0.8, 0), (0, 0.8), (0, -0.8), (0.6, 0.6))]
    test = [cam(x, y) for x, y in ((0.4, -0.3), (-0.5, 0.5), (0.2, 0.6))]

    def shot(K, E, X, C, F):
        P = K.astype(np.float64) @ E.astype(np.float64)[:3, :4]
        img, _ = ops.render_mesh(_d(X), _d(C), _d(F), P, W, H, 0.01)
        return img.cpu().numpy()

    images = [(shot(K, E, fx, fc, ff).transpose(2, 0, 1) / np.float32(255)).astype(np.float32) for K, E in train]
    xyz_d = _d(xyz)
    body, sfaces, _ = ops.simplify_mesh(xyz_d, _d(np.zeros((len(xyz), 3), np.uint8)), _d(faces), len(faces) // 50)
    sx = body[:, :12].contiguous().view(torch.float32)
    # vertex colours of the simplified mesh: the fine render's colour at each vertex in the frontal view
    K0, E0 = train[0]
    P0 = K0.astype(np.float64) @ E0.astype(np.float64)[:3, :4]
    u, v, _ = to.project64(P0, sx.cpu().numpy().astype(np.float64))
    front = images[0].transpose(1, 2, 0)
    vcol = np.rint(front[np.clip(np.rint(v).astype(int), 0, H - 1), np.clip(np.rint(u).astype(int), 0, W - 1)] * 255).astype(np.uint8)
    uv, page, pages, _ = ops.texture_mesh(sx, None, sfaces, [_d(i) for i in images], [k for k, _ in train], [e for _, e in train])
    err_tex, err_vc = [], []
    for K, E in test:
        P = K.astype(np.float64) @ E.astype(np.float64)[:3, :4]
        ref = shot(K, E, fx, fc, ff).astype(np.float64)
        tex, _ = ops.render_mesh_textured(sx, sfaces, uv, page, pages, P, W, H, 0.01)
        vc, _ = ops.render_mesh(sx, _d(vcol), sfaces, P, W, H, 0.01)
        err_tex.append(np.abs(tex.cpu().numpy() - ref).mean())
        err_vc.append(np.abs(vc.cpu().numpy() - ref).mean())
    print(f"[quality] mean absolute error: textured {np.mean(err_tex):.2f}, vertex colours {np.mean(err_vc):.2f}")
    assert np.mean(err_tex) < 0.25 * np.mean(err_vc)


# ---- end to end ---------------------------------------------------------------------------------------------------------------

def _files(d):
    out = {}
    for sub, _, names in os.walk(d):
        for n in names:
            out[os.path.relpath(os.path.join(sub, n), d)] = open(os.path.join(sub, n), "rb").read()
    return out


def test_reconstruct_mesh_texture_and_the_command(tmp_path):
    scene = str(tmp_path / "scene")
    scene_cases.write_scene(scene, 6, 128, 160, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *THRES, "--mesh"]
    run = lambda out, *extra: reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / out), *extra]),
                                                      log=lambda *a: None)
    plain_stats = run("plain", "--mesh-target-faces", "2000")
    stats = run("tex", "--mesh-target-faces", "2000", "--mesh-texture")
    plain, tex = _files(str(tmp_path / "plain")), _files(str(tmp_path / "tex"))
    new = sorted(set(tex) - set(plain))
    assert "mesh_textured.obj" in new and "mesh_textured.mtl" in new and "mesh_textured_00.png" in new
    assert all(n.startswith("mesh_textured") for n in new)
    for name in plain:
        assert tex[name] == plain[name], name
    assert not any(k.startswith("texture") for k in plain_stats)
    assert stats["texture_pages"] >= 1 and stats["texture_seconds"] > 0
    refs = [ref for ref, _ in data_io.read_pair_file(os.path.join(scene, "pair.txt"))]
    out = str(tmp_path / "cli")
    os.makedirs(out)
    texture.main(["--ply", str(tmp_path / "tex" / "mesh_simplified.ply"), "--input-folder", scene, "--views", *map(str, refs),
                  "--output", os.path.join(out, "mesh_textured")])
    cli = _files(out)
    assert sorted(cli) == new
    for name in new:
        assert cli[name] == tex[name], name


# ---- at scene sizes -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tnt", "eth3d"])
def test_scene_size_row_at_one_percent(name):
    row = build_scene(name, DEV)
    verts, faces = ops.tsdf_mesh(row["seeds"], row["depths"], row["images"], row["Ks"], row["Es"], row["s"])
    xyz, rgb = verts[:, :12].contiguous().view(torch.float32), verts[:, 12:].contiguous()
    body, sfaces, _ = ops.simplify_mesh(xyz, rgb, faces, faces.shape[0] // 100)
    del verts, faces, xyz, rgb
    images, Ks, Es = row["images"], row["Ks"], row["Es"]
    del row
    sx, srgb = body[:, :12].contiguous().view(torch.float32), body[:, 12:].contiguous()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    uv, page, pages, st = ops.texture_mesh(sx, srgb, sfaces, images, Ks, Es)
    torch.cuda.synchronize()
    used = torch.cuda.max_memory_allocated() - base
    budget = ops.texture_mesh_bytes(sx.shape[0], sfaces.shape[0], [tuple(i.shape[1:]) for i in images]) + \
        (st["pages"] - 1) * st["page_side"] ** 2 * 3
    print(f"[{name} 1 %] {sfaces.shape[0]} faces, {len(images)} views: {st}; peak {used / 2 ** 20:.1f} MiB of {budget / 2 ** 20:.1f} MiB")
    assert used <= budget
    assert st["textured_faces"] > 0.8 * sfaces.shape[0]
