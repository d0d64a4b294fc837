"""The surface sampler on the GPU against oracle/sample_oracle.py, bit for bit: random meshes, TSDF meshes of the sphere scene
and their 1 % simplifications, a face with more than 10^7 samples, degenerate, repeated-index and non-finite faces,
unreferenced vertices and empty meshes; reruns; the exact count of a triangle with more than 2^31 samples and the refusal to
allocate its output; the scene-size dtu / tnt / eth3d rows simplified to 1 % at each scorer's spacing.  End to end, the three
evaluations' --surface on triangulations of their synthetic scenes, against the oracle scorers on oracle samples."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import dtu_oracle as do, mesh_oracle as mo, sample_oracle as so
from patchmatchnet_b200 import data_io, dtu_eval, eth3d_eval, ops, tnt_eval
from tests import dtu_cases, eth3d_cases as ec, mesh_cases as mc, tnt_cases
from tests import tnt_oracle as to

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gpu(xyz, faces, s, rgb=None):
    x = torch.from_numpy(np.ascontiguousarray(xyz, np.float32)).to(DEV)
    f = torch.from_numpy(np.ascontiguousarray(faces, np.int32).reshape(-1, 3)).to(DEV)
    c = None if rgb is None else torch.from_numpy(np.ascontiguousarray(rgb, np.uint8)).to(DEV)
    p, col = ops.sample_mesh(x, f, s, c)
    assert ops.sample_mesh_count(x, f, s) == p.shape[0]
    return p.cpu().numpy(), None if col is None else col.cpu().numpy()


def _same(got, want):
    gp, gc = got
    wp, wc = want
    assert gp.shape == wp.shape
    assert np.array_equal(gp.view(np.uint64), wp.view(np.uint64)), int((gp != wp).any(1).sum())
    if wc is not None:
        assert np.array_equal(gc, wc)


def _random_mesh(seed, nv=400, nf=900):
    rng = np.random.RandomState(seed)
    xyz = (rng.normal(size=(nv, 3)) * [1.0, 3.0, 0.2]).astype(np.float32)
    faces = rng.randint(0, nv - 20, (nf, 3)).astype(np.int32)  # the last 20 vertices are unreferenced
    faces[:20, 1] = faces[:20, 0]                                  # repeated indices: segments
    faces[20:25] = faces[20:25, :1]                                # points
    xyz[faces[30, 2]] = [np.nan, 0, 0]                             # non-finite corners
    xyz[faces[31, 0], 2] = np.inf
    return xyz, rng.randint(0, 256, (nv, 3)).astype(np.uint8), faces


@pytest.mark.parametrize("seed,s", [(0, 0.05), (1, 0.2), (2, 1.0), (3, 100.0)])
def test_random_meshes_bit_for_bit(seed, s):
    xyz, rgb, faces = _random_mesh(seed)
    want = so.sample(xyz, faces, s, rgb)
    got = _gpu(xyz, faces, s, rgb)
    _same(got, want)
    _same(_gpu(xyz, faces, s, rgb), got)  # reruns give the same bits
    p, c = _gpu(xyz, faces, s)
    assert c is None and np.array_equal(p.view(np.uint64), want[0].view(np.uint64))


def test_empty_meshes_and_unreferenced_vertices():
    xyz = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    p, c = _gpu(xyz, np.zeros((0, 3), np.int32), 0.1, np.zeros((3, 3), np.uint8))
    assert p.shape == (0, 3) and c.shape == (0, 3)
    p, _ = _gpu(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32), 0.1)
    assert p.shape == (0, 3)
    _same(_gpu(xyz, np.int32([[1, 1, 1]]), 0.1), (xyz[[1]].astype(np.float64), None))


@pytest.fixture(scope="module")
def sphere_meshes():
    scn = mc.sphere_scene()
    pos, col, faces, _, _ = mo.mesh(scn["seeds"], scn["depths"], scn["images"], scn["Ks"], scn["Es"], 0.05)
    x = torch.from_numpy(pos).to(DEV)
    body, f, _ = ops.simplify_mesh(x, torch.from_numpy(col).to(DEV), torch.from_numpy(faces.astype(np.int32)).to(DEV),
                                   max(len(faces) // 100, 4))
    b = body.cpu().numpy()
    small = (b[:, :12].copy().view(np.float32).reshape(-1, 3), b[:, 12:].copy(), f.cpu().numpy())
    return {"tsdf": (pos, col, faces.astype(np.int32)), "simplified": small}


@pytest.mark.parametrize("which,s", [("tsdf", 0.05), ("tsdf", 0.01), ("simplified", 0.05), ("simplified", 0.004)])
def test_sphere_meshes_bit_for_bit(sphere_meshes, which, s):
    xyz, rgb, faces = sphere_meshes[which]
    _same(_gpu(xyz, faces, s, rgb), so.sample(xyz, faces, s, rgb))
    if which == "tsdf" and s == 0.05:  # a marching-cubes triangle lies in one cube: edges <= 0.05 sqrt(3) sample to the vertices
        assert (so.lattice_sizes(xyz, faces, 0.09) == 1).all()
        p, _ = _gpu(xyz, faces, 0.09)
        assert np.array_equal(p, xyz.astype(np.float64))


def test_one_face_with_more_than_1e7_samples():
    xyz = np.float32([[0.1, -0.3, 2.0], [1.3, 0.2, 2.5], [-0.4, 1.1, 1.7]])
    rgb = np.uint8([[0, 10, 255], [255, 128, 3], [7, 200, 90]])
    faces = np.int32([[0, 1, 2]])
    s = 1.6e-4
    n = so.lattice_sizes(xyz, faces, s)
    assert so.face_samples(n)[0] > 10 ** 7
    _same(_gpu(xyz, faces, s, rgb), so.sample(xyz, faces, s, rgb))


def test_count_above_2_31_and_refusal_before_allocation():
    xyz = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    faces = np.int32([[0, 1, 2]])
    s = float(np.sqrt(2.0)) / 99999.5  # n = 100000: about 5e9 samples, 135 GB with colours
    n = int(so.lattice_sizes(xyz, faces, s)[0])
    want = 3 + (n + 1) * (n + 2) // 2 - 3
    assert want > 2 ** 31 and 27 * want > 80 * 2 ** 30
    x, f = torch.from_numpy(xyz).to(DEV), torch.from_numpy(faces).to(DEV)
    assert ops.sample_mesh_count(x, f, s) == want
    before = torch.cuda.memory_allocated(DEV)
    with pytest.raises(ValueError, match=f"{want} samples.*larger spacing"):
        ops.sample_mesh(x, f, s, torch.zeros((3, 3), dtype=torch.uint8, device=DEV))
    assert torch.cuda.memory_allocated(DEV) == before
    with pytest.raises(ValueError, match="face 0 .*larger spacing"):  # n >= 2^31
        ops.sample_mesh_count(x, f, 1e-12)


def test_argument_checks():
    x = torch.zeros((3, 3), dtype=torch.float32, device=DEV)
    f = torch.tensor([[0, 1, 3]], dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="outside"):
        ops.sample_mesh(x, f, 0.1)
    for bad in (0.0, -1.0, math.nan, math.inf, True):
        with pytest.raises(ValueError, match="spacing"):
            ops.sample_mesh(x, f[:, [0, 1, 2]] * 0, bad)


# ---- the scene-size rows ---------------------------------------------------------------------------------------------------

ROW_SPACING = {"dtu": 0.2, "tnt": 0.01 / 4, "eth3d": 0.005}


@pytest.mark.parametrize("name", ["dtu", "tnt", "eth3d"])
def test_scene_size_rows_simplified(name):
    from tests import test_gpu_mesh_at_scene_sizes as ms

    sc = ms.build_scene(name, DEV)
    verts, faces = ops.tsdf_mesh(sc["seeds"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], sc["s"], ms.TRUNC, 1)
    del sc
    xyz = verts[:, :12].contiguous().view(torch.float32).view(-1, 3)
    body, f, _ = ops.simplify_mesh(xyz, verts[:, 12:].contiguous(), faces, faces.shape[0] // 100)
    del verts, faces, xyz
    x = body[:, :12].contiguous().view(torch.float32).view(-1, 3)
    rgb = body[:, 12:].contiguous()
    s = ROW_SPACING[name]
    p, c = ops.sample_mesh(x, f, s, rgb)
    xh, fh, ch = x.cpu().numpy(), f.cpu().numpy(), rgb.cpu().numpy()
    nv, cnt = so.counts(xh, fh, s)
    assert p.shape[0] == nv + int(cnt.sum()) > 10 * fh.shape[0]
    rows = np.random.RandomState(5).randint(0, p.shape[0], 200000)
    rows[:1000] = np.arange(1000)
    rows[1000:2000] = p.shape[0] - 1 - np.arange(1000)
    want = so.sample_at(xh, fh, s, rows, ch)
    idx = torch.from_numpy(rows).to(DEV)
    _same((p[idx].cpu().numpy(), c[idx].cpu().numpy()), want)


# ---- the evaluations, end to end ---------------------------------------------------------------------------------------------

def _grid(fx, lo, hi, step):
    """A height field z = fx(x, y) triangulated on a grid of `step` over [lo, hi]^2: float32 [nv,3], int32 [nf,3]."""
    t = np.arange(lo, hi + step / 2, step)
    x, y = np.meshgrid(t, t, indexing="ij")
    xyz = np.stack([x.ravel(), y.ravel(), fx(x.ravel(), y.ravel())], 1)
    m = len(t)
    v = np.arange(m * m).reshape(m, m)
    a, b, c, d = v[:-1, :-1].ravel(), v[1:, :-1].ravel(), v[:-1, 1:].ravel(), v[1:, 1:].ravel()
    return xyz, np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)]).astype(np.int32)


def _save_mesh(path, xyz, faces):
    xyz = np.ascontiguousarray(xyz, np.float32)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    data_io.save_ply(path, torch.from_numpy(xyz).view(torch.uint8).view(-1, 12), torch.from_numpy(faces))


def _strip(lines):  # drop the wall-clock time of each line
    return [l.rsplit("  (", 1)[0] if l.startswith("scan") or ": precision" in l else l for l in lines]


def test_dtu_fine_and_coarse_height_fields(tmp_path, capsys):
    root, outputs = str(tmp_path / "MVS Data"), str(tmp_path / "outputs")
    c = dtu_cases.write_mvs_tree(root, outputs, [1], n_stl=20000, n_data=20000, side=40.0)[1]
    fx = lambda x, y: dtu_cases.height(x, y) + 600.0
    fine = _grid(fx, -20.0, 20.0, 0.1)
    assert (so.lattice_sizes(fine[0].astype(np.float32), fine[1], 0.2) == 1).all()  # every edge <= 0.2 mm
    coarse = _grid(fx, -20.0, 20.0, 4.0)
    _save_mesh(os.path.join(outputs, "scan1", "fine.ply"), *fine)
    _save_mesh(os.path.join(outputs, "scan1", "coarse.ply"), *coarse)

    def run(name, surface):
        out = str(tmp_path / f"{name}{int(surface)}.json")
        capsys.readouterr()
        assert dtu_eval.main(["--data-path", root, "--outputs", outputs, "--scans", "1", "--json", out, "--device", DEV,
                              "--ply-template", "{outputs}/scan{scan}/" + name + ".ply"] + (["--surface"] if surface else [])) == 0
        return json.load(open(out)), capsys.readouterr().out.splitlines()

    (a, la), (b, lb) = run("fine", False), run("fine", True)
    assert _strip(la) == _strip(lb)
    ra, rb = a["scans"][0], b["scans"][0]
    assert "surface" not in ra and set(rb) - set(ra) == {"surface"}
    assert rb["surface"] == {"spacing": 0.2, "n_faces": len(fine[1]), "n_samples": len(fine[0])}
    assert {k: v for k, v in ra.items() if k != "seconds"} == {k: v for k, v in rb.items() if k not in ("seconds", "surface")}
    assert a["final"] == b["final"]

    (v, _), (s, _), (fused, _) = run("coarse", False), run("coarse", True), run("fused", False)
    rv, rs, rf = v["scans"][0], s["scans"][0], fused["scans"][0]
    pts, _ = so.sample(coarse[0].astype(np.float32), coarse[1], 0.2)
    want = do.evaluate_scan(pts, c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"], dtu_eval.visiting_order(len(pts), 0))
    for k in want:
        assert rs[k] == (want[k] if k.endswith("count") or k.startswith("n_") else pytest.approx(want[k], rel=1e-9)), k
    assert rs["surface"]["n_samples"] == len(pts)
    assert rs["comp_mean"] < 2 * rf["comp_mean"] and rv["comp_mean"] > 5 * rs["comp_mean"]


def test_tnt_fine_and_coarse_height_fields(tmp_path, capsys):
    root = str(tmp_path)
    c = tnt_cases.write_tree(root, ["Alpha"], n_gt=30000, n_rec=25000)["Alpha"]
    to_rec = lambda p: tnt_cases.apply(np.linalg.inv(c["S"]), p)

    def mesh(step):
        xyz, faces = _grid(lambda x, y: 0.25 * np.sin(2.0 * x) * np.cos(1.5 * y) + 0.1 * x * y, -1.0, 1.0, step)
        return to_rec(xyz + tnt_cases.OFFSET).astype(np.float32), faces

    fine, coarse = mesh(0.0025), mesh(0.2)
    _save_mesh(os.path.join(root, "outputs", "Alpha", "fine.ply"), *fine)
    _save_mesh(os.path.join(root, "outputs", "Alpha", "coarse.ply"), *coarse)

    def run(name, surface):
        out = str(tmp_path / f"{name}{int(surface)}.json")
        capsys.readouterr()
        assert tnt_eval.main(["--gt-path", os.path.join(root, "gt"), "--outputs", os.path.join(root, "outputs"),
                              "--input", os.path.join(root, "scenes"), "--scenes", "Alpha", "--tau", "0.02", "--json", out,
                              "--ply-template", "{outputs}/{scene}/" + name + ".ply", "--device", DEV]
                             + (["--surface"] if surface else [])) == 0
        return json.load(open(out))["scenes"][0], capsys.readouterr().out.splitlines()

    (a, la), (b, lb) = run("fine", False), run("fine", True)
    s = b["surface"]["spacing"]
    assert s == pytest.approx(0.005 / 1.7, rel=1e-4)
    assert (so.lattice_sizes(fine[0], fine[1], s) == 1).all()
    assert _strip(la) == _strip(lb) and "surface" not in a
    assert {k: v for k, v in a.items() if k != "seconds"} == {k: v for k, v in b.items() if k not in ("seconds", "surface")}

    (v, _), (r, _) = run("coarse", False), run("coarse", True)
    pts, _ = so.sample(coarse[0], coarse[1], r["surface"]["spacing"])
    want = to.evaluate_scene(pts, c["gt"], c["crop"], np.asarray(r["init_transformation"]), 0.02)
    for k in ("n_source_scored", "n_gt_scored", "precision_count", "recall_count"):
        assert r[k] == want[k], k
    for k in ("precision", "recall", "fscore"):
        assert r[k] == pytest.approx(want[k], rel=1e-12), k
    assert r["recall"] > 0.7 and v["recall"] < 0.1


def _room_mesh():
    (x0, y0, z0), (x1, y1, z1) = ec.ROOM
    (a0, b0, _), (a1, b1, _) = ec.PILLAR
    box = lambda lo, hi: np.array([[lo[0], lo[1], lo[2]], [hi[0], lo[1], lo[2]], [hi[0], hi[1], lo[2]], [lo[0], hi[1], lo[2]],
                                   [lo[0], lo[1], hi[2]], [hi[0], lo[1], hi[2]], [hi[0], hi[1], hi[2]], [lo[0], hi[1], hi[2]]])
    xyz = np.concatenate([box((x0, y0, z0), (x1, y1, z1)), box((a0, b0, z0), (a1, b1, z1))]).astype(np.float32)
    quads = [[0, 1, 2, 3], [4, 5, 6, 7], [0, 1, 5, 4], [1, 2, 6, 5], [2, 3, 7, 6], [3, 0, 4, 7]]
    tri = [[q[0], q[1], q[2]] for q in quads] + [[q[0], q[2], q[3]] for q in quads]
    pillar = [[a + 8 for a in t] for t in tri[2:6] + tri[8:12]]  # its four sides
    return xyz, np.int32(tri + pillar)


def test_eth3d_room_with_two_triangles_per_wall(tmp_path, capsys):
    ec.write_tree(str(tmp_path), ["room"], n_az=120, n_el=50, n_surface=2000, n_outliers=40, n_hidden=20)
    _save_mesh(str(tmp_path / "outputs" / "room" / "mesh.ply"), *_room_mesh())
    res = {}
    for surface in (False, True):
        out = str(tmp_path / f"r{int(surface)}.json")
        assert eth3d_eval.main(["--gt-path", str(tmp_path / "gt"), "--outputs", str(tmp_path / "outputs"), "--json", out,
                                "--ply-template", "{outputs}/{scene}/mesh.ply", "--device", DEV]
                               + (["--surface"] if surface else [])) == 0
        res[surface] = json.load(open(out))["scenes"][0]
    assert "surface" not in res[False] and res[True]["surface"]["spacing"] == 0.005
    assert res[True]["surface"]["n_samples"] == so.counts(*_room_mesh(), 0.005)[0] + int(so.counts(*_room_mesh(), 0.005)[1].sum())
    for t in res[True]["tolerances"]:  # the scans are sparse, so accuracy is not the point here
        assert t["completeness"] > 0.99, t
    assert res[False]["tolerances"][0]["completeness"] < 0.01
