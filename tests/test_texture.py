"""The mesh texturer without a GPU: a hand-worked case through oracle/texture_oracle.py (candidates with an occluder, labels,
the chart rectangle, texture coordinates and texels), the host build of pm_texture_math.cuh (tests/host_texture.cpp)
against the oracle bit for bit, the shelf packer through the C ABI, the OBJ writer and reader, and the commands' argument
checks."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import texture_oracle as to
from patchmatchnet_b200 import data_io, ops, reconstruct, texture

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


def _cam(f, cx, cy, centre):
    K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float32)
    E = np.eye(4, dtype=np.float32)
    E[:3, 3] = -np.asarray(centre, np.float32)
    return K, E


def hand_case():
    """A quad at z = 5 (faces 0 and 1, wound towards the cameras) and an occluder (face 2) at z = 2.5 that hides part of
    face 1 from camera 1 (at x = 3) but lies beside the quad for camera 0 (at the origin); 64 x 64 images, f = 20."""
    xyz = np.array([[-1, -1, 5], [1, -1, 5], [1, 1, 5], [-1, 1, 5],
                    [1, 0.1, 2.5], [1.5, 0.5, 2.5], [1, 0.5, 2.5]], np.float32)
    faces = np.array([[0, 2, 1], [0, 3, 2], [4, 5, 6]], np.int64)
    cams = [_cam(20.0, 31.5, 31.5, (0, 0, 0)), _cam(20.0, 31.5, 31.5, (3, 0, 0))]
    rng = np.random.default_rng(5)
    images = [(rng.integers(0, 256, (3, 64, 64)) / 255.0).astype(np.float32) for _ in cams]
    return xyz, faces, images, [c[0] for c in cams], [c[1] for c in cams]


def test_hand_worked_case():
    xyz, faces, images, Ks, Es = hand_case()
    vws = to.views(Ks, Es, [(64, 64)] * 2, to.box_centre(xyz))
    cand = []
    for v in vws:
        vis, cov = to.visibility(xyz, faces, v)
        cand.append(to.candidates(xyz, faces, v, vis, cov))
        if v is vws[1]:
            assert vis[1] >= 1 and 10 * vis[1] < 9 * cov[1]  # the occluder hides more than 10 % of face 1 from camera 1
            assert vis[0] == cov[0] > 0
    assert cand[0][:2].tolist() == [True, True] and cand[1][:2].tolist() == [True, False]
    out = to.texture(xyz, None, faces, images, Ks, Es)
    # face 1 has camera 0 alone; face 0 ties or nearly ties and its neighbour's label decides: camera 0
    assert out["label"][:2].tolist() == [0, 0]
    assert out["chart"][:2].tolist() == [0, 0]
    row = out["table"][0]
    # the quad projects to u, v in [27.5, 35.5] in camera 0: the rectangle is floor - 2 .. ceil + 2
    assert row.tolist() == [0, 0, 25, 25, 14, 14]
    pg, ox, oy = out["places"][0]
    S = out["S"]
    assert S == 4096
    # corner 0 of face 0 is vertex 0 at (27.5, 27.5)
    a = 27.5 - 25 + ox
    b = 27.5 - 25 + oy
    assert out["uv"][0, 0].tolist() == [np.float32((a + 0.5) / S), np.float32(1 - (b + 0.5) / S)]
    want = np.rint(np.float32(255) * images[0][:, 25:39, 25:39]).astype(np.uint8).transpose(1, 2, 0)
    assert np.array_equal(out["pages"][pg, oy:oy + 14, ox:ox + 14], want)
    assert out["pages"].sum() > 0


# ---- the host build of pm_texture_math.cuh ------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hosttex(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hosttex") / "_hosttex.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_texture.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.ht_faces.argtypes = [P, P, ctypes.c_double, ctypes.c_int, ctypes.c_int, P, ctypes.c_int, P, P]
    lib.ht_scores.argtypes = [P, P, P, ctypes.c_int, P]
    lib.ht_uvs.argtypes = [P, P, ctypes.c_int, ctypes.c_int, P, P]
    return lib


def test_host_faces_equal_the_oracle(hosttex):
    rng = np.random.default_rng(11)
    for trial in range(6):
        W, H = int(rng.integers(50, 400)), int(rng.integers(50, 400))
        centre = rng.normal(size=3) * 0.3
        K = np.array([[rng.uniform(30, 150), 0, W / 2], [0, rng.uniform(30, 150), H / 2], [0, 0, 1]], np.float32)
        E = np.eye(4, dtype=np.float32)
        E[:3, 3] = -centre.astype(np.float32)
        (Pm, C, near, _, _), = to.views([K], [E], [(H, W)], np.zeros(3))
        n = 2000
        x = (rng.normal(size=(n, 3, 3)) + np.array([0, 0, 6])).astype(np.float32)
        q = np.zeros((n, 9))
        cand = np.zeros(n, np.int32)
        hosttex.ht_faces(np.ascontiguousarray(Pm).ctypes.data, np.ascontiguousarray(C).ctypes.data, near, W, H, x.ctypes.data, n,
                         q.ctypes.data, cand.ctypes.data)
        u, v, z = to.project64(Pm, x.astype(np.float64))
        assert np.array_equal(q.reshape(n, 3, 3)[..., 0].view(np.uint64), u.view(np.uint64))
        assert np.array_equal(q.reshape(n, 3, 3)[..., 1].view(np.uint64), v.view(np.uint64))
        assert np.array_equal(q.reshape(n, 3, 3)[..., 2].view(np.uint64), z.view(np.uint64))
        ones = np.ones(n, np.int64)
        # candidates() indexes xyz by faces: the corners become their own vertices
        want = to.candidates(x.reshape(-1, 3), np.arange(3 * n).reshape(n, 3), (Pm, C, near, W, H), ones, ones)
        assert np.array_equal(cand.astype(bool), want)
        assert 0 < cand.sum() < n


def test_host_scores_and_coordinates_equal_the_oracle(hosttex):
    rng = np.random.default_rng(12)
    n = 5000
    d = rng.integers(1, 5000, n).astype(np.int32)
    m = (d + rng.integers(0, 5000, n)).astype(np.int32)
    same = rng.integers(0, 9, n).astype(np.int32)
    out = np.zeros(n)
    hosttex.ht_scores(d.ctypes.data, m.ctypes.data, same.ctypes.data, n, out.ctypes.data)
    want = d.astype(np.float64) / m.astype(np.float64) + to.LAMBDA * same.astype(np.float64)
    assert np.array_equal(out.view(np.uint64), want.view(np.uint64))
    S = 8192
    uvin = rng.uniform(0, 2000, (n, 2))
    frame = np.stack([np.floor(uvin[:, 0]) - rng.integers(2, 40, n), np.floor(uvin[:, 1]) - rng.integers(2, 40, n),
                      rng.integers(0, S - 64, n), rng.integers(0, S - 64, n)], 1).astype(np.int32)
    uv = np.zeros((n, 2), np.float32)
    cell = np.zeros((n, 2), np.float32)
    hosttex.ht_uvs(uvin.ctypes.data, frame.ctypes.data, n, S, uv.ctypes.data, cell.ctypes.data)
    f = frame.astype(np.float64)
    a, b = (uvin[:, 0] - f[:, 0]) + f[:, 2], (uvin[:, 1] - f[:, 1]) + f[:, 3]
    assert np.array_equal(uv[:, 0], ((a + 0.5) / S).astype(np.float32))
    assert np.array_equal(uv[:, 1], (1.0 - (b + 0.5) / S).astype(np.float32))
    assert np.array_equal(cell[:, 0], ((f[:, 2] + 2) / S).astype(np.float32))
    assert np.array_equal(cell[:, 1], (1.0 - (f[:, 3] + 2) / S).astype(np.float32))


# ---- the packer -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1, 2])
def test_packer_places_without_overlap_inside_the_page(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 3000))
    big = 9000 if seed == 2 else 1500
    sizes = np.stack([rng.integers(1, big, n), rng.integers(1, big, n)], 1)
    cells = int(rng.integers(0, 500))
    places, S, pages = ops.texture_pack(sizes, cells)
    again = ops.texture_pack(sizes, cells)
    assert np.array_equal(places, again[0]) and (S, pages) == again[1:]
    want_places, want_S, want_pages = to.pack(sizes, cells)
    assert np.array_equal(places, want_places) and (S, pages) == (want_S, want_pages)
    assert S >= sizes.max() and S in (4096, 8192, 16384)
    allsz = np.concatenate([sizes, np.full((cells, 2), 4)])
    assert (places[:, 1] >= 0).all() and (places[:, 1] + allsz[:, 0] <= S).all()
    assert (places[:, 2] >= 0).all() and (places[:, 2] + allsz[:, 1] <= S).all()
    for p in range(pages):
        sel = np.flatnonzero(places[:, 0] == p)
        x0, y0 = places[sel, 1], places[sel, 2]
        x1, y1 = x0 + allsz[sel, 0], y0 + allsz[sel, 1]
        order = np.argsort(x0)
        for i in range(len(sel)):  # rectangles that overlap in x must be disjoint in y
            j = order[np.searchsorted(x0[order], x1[i]):]
            k = np.setdiff1d(np.arange(len(sel)), np.concatenate([j, [i]]))
            k = k[x1[k] > x0[i]]
            assert not ((y0[k] < y1[i]) & (y0[i] < y1[k])).any()


def test_packer_rejects_a_side_above_16384():
    with pytest.raises(ValueError, match="16384"):
        ops.texture_pack([[16385, 4]], 0)


# ---- OBJ ------------------------------------------------------------------------------------------------------------------

def test_obj_round_trip(tmp_path):
    rng = np.random.default_rng(3)
    xyz = rng.normal(size=(40, 3)).astype(np.float32)
    faces = rng.integers(0, 40, (60, 3)).astype(np.int32)
    uv = rng.uniform(0, 1, (60, 3, 2)).astype(np.float32)
    page = rng.integers(0, 3, 60).astype(np.int32)
    pages = rng.integers(0, 256, (3, 16, 16, 3)).astype(np.uint8)
    stem = str(tmp_path / "m")
    data_io.save_obj(stem, xyz, faces, uv, page, pages)
    assert sorted(os.listdir(tmp_path)) == ["m.mtl", "m.obj", "m_00.png", "m_01.png", "m_02.png"]
    x, f, u, p, pg = data_io.read_obj(stem + ".obj")
    order = np.argsort(page, kind="stable")  # grouped by page, original order within a page
    assert np.array_equal(x, xyz) and np.array_equal(f, faces[order]) and np.array_equal(u, uv[order])
    assert np.array_equal(p, page[order]) and np.array_equal(pg, pages)
    bad = tmp_path / "bad.obj"
    bad.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")
    with pytest.raises(ValueError, match="subset"):
        data_io.read_obj(str(bad))
    bad.write_text("v 0 0 0\nvn 0 0 1\n")
    with pytest.raises(ValueError, match="subset"):
        data_io.read_obj(str(bad))


# ---- commands -------------------------------------------------------------------------------------------------------------

def test_texture_command_checks(tmp_path):
    from tests import scene_cases

    scene = tmp_path / "scene"
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    mesh = str(tmp_path / "m.ply")
    data_io.save_ply(mesh, torch.zeros((3, 15), dtype=torch.uint8), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    out = str(tmp_path / "o" / "tex")
    with pytest.raises(ValueError, match="does not exist"):
        texture.main(["--ply", mesh, "--input-folder", str(scene), "--output", out])
    os.makedirs(tmp_path / "o")
    with pytest.raises(ValueError, match="no such file"):
        texture.main(["--ply", str(tmp_path / "missing.ply"), "--input-folder", str(scene), "--output", out])
    with pytest.raises(ValueError, match="view 99"):
        texture.main(["--ply", mesh, "--input-folder", str(scene), "--output", out, "--views", "0", "99"])
    assert texture.check_args(texture.build_parser().parse_args(["--ply", mesh, "--input-folder", str(scene), "--output", out])) == [0, 1, 2]
    assert os.listdir(tmp_path / "o") == []


def test_reconstruct_texture_option(tmp_path):
    from tests import scene_cases

    assert "mesh_texture" not in vars(reconstruct.parse_args([]))
    assert reconstruct.mesh_options(reconstruct.parse_args(["--mesh", "--mesh-texture"])).mesh_texture
    scene, out = tmp_path / "scene", tmp_path / "out"
    out.mkdir()
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"")
    base = ["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt), "--output-type", "fusion"]
    with pytest.raises(ValueError, match="--mesh-texture needs --mesh"):
        reconstruct.main(base + ["--mesh-texture"])
    assert os.listdir(out) == []


def test_texture_mesh_rejects_bad_arguments_before_any_launch():
    xyz = torch.zeros((3, 3))
    with pytest.raises(ValueError, match="CUDA"):
        ops.texture_mesh(xyz, None, torch.zeros((1, 3), dtype=torch.int32), [torch.zeros((3, 4, 4))], [np.eye(3)], [np.eye(4)])
