"""The mesh simplifier on the CPU: the oracle (oracle/simplify_oracle.py) on a bordered tilted grid, on the analytic sphere of
test_mesh.py and on hard inputs; round independence (a round's collapses applied one at a time in random orders give the
vectorised round's result); component removal; the kernels' per-edge functions (pm_simplify_math.cuh, built for the host from
tests/host_simplify.cpp) against the oracle bit for bit; argument checks of the C ABI, ops.simplify_mesh, save_ply's
x/y/z-only layout, the simplify command and reconstruct's options.

Bound fixed by running the oracle on the sphere (voxel 0.05): the radial vertex error is at most 0.2 at 10 % and 0.35 at
2 % of the faces; 0.25 and 0.45 are allowed."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo, simplify_oracle as so
from patchmatchnet_b200 import _native, data_io, ops, reconstruct, simplify
from tests import mesh_cases as mc, simplify_cases as sc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


def _p(a):
    return a.ctypes.data_as(P)


@pytest.fixture(scope="module")
def hostsimp(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostsimp") / "_hostsimp.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_simplify.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hs_edges.argtypes = [P] * 5 + [ctypes.c_int] + [P] * 5
    lib.hs_faces.argtypes = [P] * 4 + [ctypes.c_int] + [P] * 3
    return lib


@pytest.fixture(scope="module")
def sphere():
    scn = mc.sphere_scene()
    pos, col, faces, _, _ = mo.mesh(scn["seeds"], scn["depths"], scn["images"], scn["Ks"], scn["Es"], 0.05)
    return pos, col, faces


# ---- the oracle ---------------------------------------------------------------------------------------------------------------

def test_grid_keeps_its_plane_and_corners():
    xyz, faces, corners = sc.grid(20)
    extent = np.ptp(xyz.astype(np.float64), 0).max()
    assert sc.grid_plane_distance(xyz).max() == 0  # the input lies exactly on the plane
    # float64 positions between rounds, before the output rounding
    pos, col, q, f, topo = so.prepare(xyz, None, faces)
    rounds = 0
    while len(f) > 8:
        res = so.round_step(pos, col, q, f, 8, topo)
        assert res is not None
        pos, col, q, f, _, _ = res
        topo, rounds = None, rounds + 1
        assert sc.grid_plane_distance(pos[np.unique(f)]).max() <= 1e-9 * extent
    p, c, fo, r = so.simplify(xyz, None, faces, 8)
    assert r == rounds and len(fo) <= 8
    sc.check_invariants(p, fo)
    # the output: float32 rounding moves a coordinate up to 2^-20 (half a float32 ulp below 16) off the plane
    assert sc.grid_plane_distance(p).max() <= 1e-9 * extent + 2.0 ** -20 * 1.5
    for v in corners:
        assert (p == xyz[v]).all(1).any(), v


@pytest.mark.parametrize("share,bound", [(0.1, 0.25), (0.02, 0.45)])
def test_sphere_stays_a_closed_manifold(sphere, share, bound):
    pos, col, faces = sphere
    target = int(len(faces) * share)
    p, c, f, rounds = so.simplify(pos, col, faces, target)
    assert len(f) <= target
    sc.check_invariants(p, f)
    mc.check_closed_manifold(f.astype(np.int64), len(p))
    radial = np.linalg.norm(p.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS
    assert np.abs(radial).max() < bound


def _bordered(sphere):
    pos, col, faces = sphere
    cen = pos[faces].astype(np.float64).mean(1) - mc.SPHERE_CENTRE
    return pos, col, faces[cen[:, 2] < 0.6]


def _still_selectable(pos, col, q, faces, a, b, want_cost_bits):
    """Every selected edge not yet applied is still an edge, still valid, and has the cost it had when the round selected
    it: an earlier collapse of the round changed nothing it reads."""
    topo = so.Topology(faces, len(pos))
    key = so.evaluate(pos, q, topo)
    eid = topo.edge_id(a, b)
    assert (eid >= 0).all()
    k = key[eid]
    assert (k != so.NONE).all()
    assert np.array_equal(k >> np.uint64(32), want_cost_bits)


@pytest.mark.parametrize("which", ["sphere", "bordered"])
def test_round_independence(sphere, which):
    """The executable form of the selection argument: a round's collapses, applied one at a time in three random orders,
    give the vectorised round's result bit for bit; no mesh edge joins the endpoints of two selected edges; and at points
    along each sequence every selected edge not yet applied is still valid with its cost unchanged."""
    xyz, rgb, faces = sphere if which == "sphere" else _bordered(sphere)
    pos, col, q, f, topo = so.prepare(xyz, rgb, faces)
    rng = np.random.default_rng(5)
    for r in range(4):
        key = so.evaluate(pos, q, topo)
        npos, ncol, nq, nf, sel, topo = so.round_step(pos, col, q, f, 0, topo)
        a, b = topo.a[sel], topo.b[sel]
        assert len(sel) > 10
        owner = np.full(len(pos), -1)
        owner[a], owner[b] = np.arange(len(sel)), np.arange(len(sel))
        oa, ob = owner[topo.a], owner[topo.b]
        assert not ((oa >= 0) & (ob >= 0) & (oa != ob)).any(), "two selected edges are adjacent"
        cost_bits = key[sel] >> np.uint64(32)
        for _ in range(3):
            order = rng.permutation(len(sel))
            checks = set(np.linspace(0, len(sel) - 1, 6).astype(int).tolist())
            spos, scol, sq, sf = pos, col, q, f
            for n, i in enumerate(order):
                if n in checks:
                    rest = order[n:]
                    _still_selectable(spos, scol, sq, sf, a[rest], b[rest], cost_bits[rest])
                spos, scol, sq, sf = so.apply(spos, scol, sq, sf, a[i:i + 1], b[i:i + 1])
            assert np.array_equal(sf, nf)
            assert np.array_equal(spos.view(np.uint64), npos.view(np.uint64))
            assert np.array_equal(scol, ncol) and np.array_equal(sq.view(np.uint64), nq.view(np.uint64))
        pos, col, q, f, topo = npos, ncol, nq, nf, so.Topology(nf, len(npos))


@pytest.mark.parametrize("case", ["tetrahedron", "strip", "fan", "non_manifold", "slivers"])
@pytest.mark.parametrize("target", [0, 3])
def test_hard_inputs_keep_the_invariants(case, target):
    xyz, faces = getattr(sc, case)()
    p, c, f, rounds = so.simplify(xyz, None, faces, target)
    sc.check_invariants(p, f)
    if case == "slivers":  # zero-area faces neither stall the rounds nor survive as a flip
        assert sc.zero_area(xyz, faces).sum() == 6
        assert rounds > 0 and len(f) <= max(target, 8)
    if case == "tetrahedron":
        assert len(f) == 4 and rounds == 0
        mc.check_closed_manifold(f.astype(np.int64), len(p))


def test_empty_mesh_and_zero_target():
    p, c, f, r = so.simplify(np.zeros((0, 3), np.float32), None, np.zeros((0, 3), np.int32), 0)
    assert len(p) == 0 and len(f) == 0 and r == 0
    xyz, faces, _ = sc.grid(6)
    p, c, f, r = so.simplify(xyz, None, faces, 0)
    sc.check_invariants(p, f)
    assert len(f) < 10


@pytest.mark.parametrize("F", [0, 5, 50])
def test_component_removal(sphere, F):
    pos, col, faces = sphere
    xyz, ff, first = sc.floaters(pos, faces)
    lab = so.component_labels(ff.astype(np.int64), len(xyz))
    # labels are the smallest vertex index of each component
    assert set(np.unique(lab)) == {int(ff[:len(faces)].min())} | set(first)
    kept = so.remove_small_components(ff.astype(np.int64), len(xyz), F)
    sizes = {1: first[0], 4: first[1], 40: first[2]}
    for n, v in sizes.items():
        assert ((kept == v).any()) == (n >= F), (n, F)
    assert len(kept) - sum(n for n in sizes if n >= F) == len(faces)


# ---- the host build of pm_simplify_math.cuh against the oracle ------------------------------------------------------------------

def _random_quadrics(rng, n, xa, xb):
    """Sums of face and border planes around the edges, some rank-deficient (planar, one plane), some zero."""
    q = np.zeros((n, 10))
    for k in range(4):
        p = (xa * 0.5 + xb * 0.5) + rng.normal(size=(n, 3)) * 0.1  # planes through a point near the edge: solvable
        x = np.stack([p, p + rng.normal(size=(n, 3)), p + rng.normal(size=(n, 3))], 1)
        if k >= 2:
            x[::3, 2] = x[::3, 0] * 0.5 + x[::3, 1] * 0.5  # degenerate: collinear
        t, ok = so.face_terms(x[:, 0], x[:, 1], x[:, 2])
        use = ok & (rng.random(n) < 0.8)
        q = np.where(use[:, None], q + t, q)
        t, ok = so.border_terms(xa, xb, x[:, 0], x[:, 1], x[:, 2])
        use = ok & (rng.random(n) < 0.3)
        q = np.where(use[:, None], q + t, q)
    q[: n // 10] = 0.0
    near = slice(n // 10, n // 5)  # near-singular: one plane plus a whisper of another
    q[near] = so.face_terms(xa[near], xb[near], xa[near] + np.array([0.0, 0.0, 1.0]))[0]
    q[near] += 1e-12 * so.face_terms(xa[near], xb[near], xa[near] + np.array([1.0, 0.3, 0.0]))[0]
    return q


def test_host_edges_equal_the_oracle(hostsimp):
    rng = np.random.default_rng(11)
    n = 4000
    xa = rng.normal(size=(n, 3)) * 3
    xb = xa + rng.normal(size=(n, 3)) * 0.5
    xb[-20:] = xa[-20:]  # zero-length edges
    q = _random_quadrics(rng, n, xa, xb)
    ca, cb = rng.integers(0, 256, (n, 3)).astype(np.uint8), rng.integers(0, 256, (n, 3)).astype(np.uint8)
    v, solved, colour = np.zeros((n, 3)), np.zeros(n, np.int32), np.zeros((n, 3), np.uint8)
    cost, key = np.zeros(n), np.zeros(n, np.uint64)
    hostsimp.hs_edges(_p(q), _p(xa), _p(xb), _p(ca), _p(cb), n, _p(v), _p(solved), _p(colour), _p(cost), _p(key))
    wv, wsolved = so.placement(q, xa, xb)
    assert np.array_equal(v.view(np.uint64), wv.view(np.uint64))
    assert np.array_equal(solved.astype(bool), wsolved)
    assert 0.2 < wsolved.mean() < 0.95
    assert np.array_equal(colour, so.placement_colour(xa, xb, wv, ca, cb))
    assert np.array_equal(cost.view(np.uint64), so.quadric_cost(q, wv).view(np.uint64))
    assert np.array_equal(key, so.edge_key(so.quadric_cost(q, wv), np.arange(n)))


def test_host_faces_equal_the_oracle(hostsimp):
    rng = np.random.default_rng(12)
    n = 3000
    x = rng.normal(size=(n, 3, 3))
    x[: n // 10, 2] = x[: n // 10, 0]  # zero-area faces
    x[n // 10: n // 5, 2] = x[n // 10: n // 5, 0] * 0.25 + x[n // 10: n // 5, 1] * 0.75  # collinear
    edge = np.stack([x[:, 0], x[:, 1]], 1)
    slot = rng.integers(0, 3, n).astype(np.int32)
    v = x[np.arange(n), slot] + rng.normal(size=(n, 3)) * 2
    qf, qb, keeps = np.zeros((n, 10)), np.zeros((n, 10)), np.zeros(n, np.int32)
    hostsimp.hs_faces(_p(np.ascontiguousarray(x)), _p(np.ascontiguousarray(edge)), _p(slot), _p(v), n, _p(qf), _p(qb), _p(keeps))
    t, ok = so.face_terms(x[:, 0], x[:, 1], x[:, 2])
    assert np.array_equal(qf.view(np.uint64), np.where(ok[:, None], 0.0 + t, 0.0).view(np.uint64))
    t, ok = so.border_terms(x[:, 0], x[:, 1], x[:, 0], x[:, 1], x[:, 2])
    assert np.array_equal(qb.view(np.uint64), np.where(ok[:, None], 0.0 + t, 0.0).view(np.uint64))
    want = so.keeps_orientation(x[:, 0], x[:, 1], x[:, 2], slot, v)
    assert np.array_equal(keeps.astype(bool), want) and 0.2 < want.mean() < 0.95


# ---- argument checks ----------------------------------------------------------------------------------------------------------

def _rejects(rc):
    assert rc == -1, rc
    return _native.lib().pmb200_last_error().decode()


def test_abi_rejects_bad_arguments():
    lib = _native.lib()
    d = ctypes.c_void_p(16)
    counts = (ctypes.c_int64 * 3)()
    assert "null" in _rejects(lib.pmb200_simplify_mesh(None, None, 4, d, 2, 0, 0, counts, d, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_simplify_mesh(d, None, 4, None, 2, 0, 0, counts, d, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_simplify_mesh(d, None, 4, d, 2, 0, 0, None, d, 1 << 20, None))
    assert "2^31" in _rejects(lib.pmb200_simplify_mesh(d, None, -1, d, 2, 0, 0, counts, d, 1 << 20, None))
    assert "2^29" in _rejects(lib.pmb200_simplify_mesh(d, None, 4, d, 1 << 29, 0, 0, counts, d, 1 << 40, None))
    assert ">= 0" in _rejects(lib.pmb200_simplify_mesh(d, None, 4, d, 2, -1, 0, counts, d, 1 << 20, None))
    assert ">= 0" in _rejects(lib.pmb200_simplify_mesh(d, None, 4, d, 2, 0, -3, counts, d, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_simplify_mesh_write(4, 2, 1, None, None, d, d, 1 << 20, None))
    assert "n_faces_out" in _rejects(lib.pmb200_simplify_mesh_write(4, 2, 3, d, None, d, d, 1 << 20, None))
    assert lib.pmb200_simplify_mesh_workspace_bytes(-1, 0) == -1


def test_simplify_mesh_rejects_bad_arguments_before_any_launch():
    xyz, faces = torch.zeros((4, 3)), torch.zeros((2, 3), dtype=torch.int32)
    with pytest.raises(ValueError, match="CUDA"):
        ops.simplify_mesh(xyz, None, faces, 1)
    meta = torch.zeros((4, 3), device="meta")
    with pytest.raises(ValueError):
        ops.simplify_mesh(meta, None, faces, 1)


def test_simplify_mesh_checks_on_a_fake_device(monkeypatch):
    """The checks after the device test, with a wrapper that accepts CPU tensors: nothing reaches the library."""
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "_native", None)  # any library call would raise
    xyz, faces = torch.zeros((4, 3)), torch.tensor([[0, 1, 2], [1, 2, 3]], dtype=torch.int32)
    for kw, what in (({"target_faces": -1}, "target_faces"), ({"target_faces": 1.5}, "target_faces"),
                     ({"target_faces": 1, "min_component_faces": -2}, "min_component_faces")):
        with pytest.raises(ValueError, match=what):
            ops.simplify_mesh(xyz, None, faces, **kw)
    with pytest.raises(ValueError, match="outside"):
        ops.simplify_mesh(xyz, None, faces + 2, 1)
    with pytest.raises(ValueError, match="int32"):
        ops.simplify_mesh(xyz, None, faces.long(), 1)
    with pytest.raises(ValueError, match="rgb"):
        ops.simplify_mesh(xyz, torch.zeros((3, 3), dtype=torch.uint8), faces, 1)


def test_save_ply_xyz_only_layout(tmp_path):
    rng = np.random.default_rng(0)
    xyz = rng.normal(size=(5, 3)).astype(np.float32)
    body = torch.from_numpy(xyz.view(np.uint8).reshape(5, 12).copy())
    faces = torch.tensor([[0, 1, 2], [2, 3, 4]], dtype=torch.int32)
    path = str(tmp_path / "m.ply")
    data_io.save_ply(path, body, faces)
    raw = open(path, "rb").read()
    head, _, rest = raw.partition(b"end_header\n")
    assert head.decode() == ("ply\nformat binary_little_endian 1.0\nelement vertex 5\nproperty float x\nproperty float y\n"
                             "property float z\nelement face 2\nproperty list uchar int vertex_indices\n")
    assert rest[:60] == xyz.tobytes()
    p, c, n, f = data_io.read_ply(path)
    assert np.array_equal(p, xyz) and c is None and np.array_equal(f, faces.numpy())


def test_simplify_command_checks(tmp_path):
    pts = str(tmp_path / "pts.ply")
    data_io.save_ply(pts, torch.zeros((3, 15), dtype=torch.uint8))
    with pytest.raises(ValueError, match="no faces"):
        simplify.main(["--ply", pts, "--output", str(tmp_path / "o.ply"), "--target-faces", "1"])
    with pytest.raises(ValueError):
        simplify.main(["--ply", pts, "--output", str(tmp_path / "o.ply"), "--target-faces", "-1"])
    assert not os.path.exists(tmp_path / "o.ply")


def test_reconstruct_simplify_options(tmp_path, monkeypatch):
    a = reconstruct.parse_args([])
    assert not any(k.startswith("mesh") for k in vars(a))
    m = reconstruct.mesh_options(reconstruct.parse_args(["--mesh", "--mesh-target-faces", "100", "--mesh-min-component-faces", "5"]))
    assert (m.mesh_target_faces, m.mesh_min_component_faces) == (100, 5)
    from tests import scene_cases

    scene, out = tmp_path / "scene", tmp_path / "out"
    out.mkdir()
    scn = scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    scene_cases.write_fusion_maps(str(out), scn["cams"], 24, 32, seed=1)
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"")
    base = ["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt), "--output-type", "fusion"]
    before = sorted(os.listdir(out))
    for bad in (["--mesh-target-faces", "10"], ["--mesh", "--mesh-target-faces", "-1"], ["--mesh", "--mesh-min-component-faces", "3"],
                ["--mesh", "--mesh-target-faces", "10", "--mesh-min-component-faces", "-1"]):
        with pytest.raises(ValueError, match="mesh-"):
            reconstruct.main(base + bad)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        reconstruct.main(base + ["--mesh", "--mesh-target-faces", "10"])
    assert sorted(os.listdir(out)) == before
