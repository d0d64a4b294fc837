"""The surface sampler on the CPU: the kernels' own functions (pm_sample_math.cuh, built for the host from
tests/host_sample.cpp) against oracle/sample_oracle.py bit for bit; the count formula and the lattice order; the covering
guarantee and that every sample lies on its face; the vertex-set identity for meshes whose edges are at most the spacing;
argument checks of ops and of the evaluations' --surface flags; the sample command's PLY round trip."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import sample_oracle as so
from patchmatchnet_b200 import data_io, dtu_eval, eth3d_eval, ops, sample, tnt_eval

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


def _p(a):
    return None if a is None else a.ctypes.data_as(P)


@pytest.fixture(scope="module")
def hostsample(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostsample") / "_hostsample.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_sample.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hs_sizes.argtypes = [P, ctypes.c_longlong, ctypes.c_double, P, P]
    lib.hs_points.argtypes = [P, P, P, P, ctypes.c_longlong, P, P, P, P]
    return lib


def random_mesh(seed, nv=60, nf=120, scale=1.0):
    rng = np.random.RandomState(seed)
    xyz = (rng.normal(size=(nv, 3)) * scale).astype(np.float32)
    faces = rng.randint(0, nv, (nf, 3)).astype(np.int32)
    rgb = rng.randint(0, 256, (nv, 3)).astype(np.uint8)
    return xyz, rgb, faces


def grid_mesh(m, step, z=0.0):
    """An m x m vertex grid of spacing `step`, two triangles per cell."""
    x, y = np.meshgrid(np.arange(m) * step, np.arange(m) * step, indexing="ij")
    xyz = np.stack([x.ravel(), y.ravel(), np.full(m * m, z)], 1).astype(np.float32)
    v = np.arange(m * m).reshape(m, m)
    a, b, c, d = v[:-1, :-1].ravel(), v[1:, :-1].ravel(), v[:-1, 1:].ravel(), v[1:, 1:].ravel()
    return xyz, np.concatenate([np.stack([a, b, d], 1), np.stack([a, d, c], 1)]).astype(np.int32)


# ---- the host build against the oracle ----------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(4))
def test_host_sizes_equal_the_oracle(hostsample, seed):
    xyz, _, faces = random_mesh(seed)
    xyz[3] = np.nan
    xyz[5, 1] = np.inf
    s = [0.05, 0.3, 1.7, 1e-12][seed]
    x = np.ascontiguousarray(xyz[faces].reshape(-1, 9))
    n, cnt = np.zeros(len(faces), np.int64), np.zeros(len(faces), np.int64)
    hostsample.hs_sizes(_p(x), len(faces), s, _p(n), _p(cnt))
    assert np.array_equal(n, so.lattice_sizes(xyz, faces, s))
    assert np.array_equal(cnt, np.where(n >= so.MAX_LATTICE, 0, so.face_samples(n)))
    if seed == 3:
        assert (n == so.MAX_LATTICE).any()


@pytest.mark.parametrize("seed", range(3))
def test_host_points_and_colours_equal_the_oracle(hostsample, seed):
    rng = np.random.RandomState(10 + seed)
    m = 4000
    xyz = (rng.normal(size=(m, 9)) * [1, 10, 100, 1e3, 1e-3, 1, 7, 0.1, 3]).astype(np.float32)
    col = rng.randint(0, 256, (m, 9)).astype(np.uint8)
    n = np.concatenate([rng.randint(2, 40, m // 2), rng.randint(2, 2 ** 31, m - m // 2)]).astype(np.int64)
    k = (rng.uniform(size=m) * so.face_samples(n)).astype(np.int64)
    k[:10] = 0
    k[10:20] = so.face_samples(n[10:20]) - 1
    ij, nb = np.zeros((m, 2), np.int64), np.zeros(m, np.int64)
    p, rgb = np.zeros((m, 3)), np.zeros((m, 3), np.uint8)
    hostsample.hs_points(_p(xyz), _p(col), _p(n), _p(k), m, _p(ij), _p(nb), _p(p), _p(rgb))
    i, j = so.lattice_points(n, k)
    assert np.array_equal(ij, np.stack([i, j], 1))
    assert np.array_equal(nb, n)
    faces = np.arange(3 * m).reshape(m, 3)
    P_, C_ = so.points_at(xyz.reshape(-1, 3), col.reshape(-1, 3), faces, n, np.arange(m), i, j)
    assert np.array_equal(p.view(np.uint64), P_.view(np.uint64))
    assert np.array_equal(rgb, C_)


# ---- the definition ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 2, 3, 4, 7, 16, 33])
def test_lattice_order_and_count(n):
    want = [(i, j) for i in range(n + 1) for j in range(n - i + 1) if (i, j) not in ((0, 0), (n, 0), (0, n))]
    assert len(want) == so.face_samples(n) == max((n + 1) * (n + 2) // 2 - 3, 0)
    i, j = so.lattice_points(np.full(len(want), n), np.arange(len(want)))
    assert list(zip(i.tolist(), j.tolist())) == want


def test_lattice_inversion_at_the_largest_n():
    n = np.int64(2 ** 31 - 1)
    c = int(so.face_samples(n))
    k = np.array([0, 1, n - 2, n - 1, n, c // 2, c - 3, c - 2, c - 1], np.int64)
    i, j = so.lattice_points(n, k)
    N = (int(n) + 1) * (int(n) + 2) // 2
    for kk, ii, jj in zip(k.tolist(), i.tolist(), j.tolist()):  # python integers: exact
        p = kk + 1 if kk < n - 1 else kk + 2
        assert ii * (int(n) + 1) - ii * (ii - 1) // 2 + jj == p and 0 <= jj <= n - ii and p < N - 1


def test_count_formula_on_random_meshes():
    for seed in range(3):
        xyz, rgb, faces = random_mesh(seed)
        s = 0.2
        P_, C_ = so.sample(xyz, faces, s, rgb)
        nv, c = so.counts(xyz, faces, s)
        n = so.lattice_sizes(xyz, faces, s)
        assert len(P_) == len(C_) == nv + int(((n + 1) * (n + 2) // 2 - 3)[n > 1].sum())


@pytest.mark.parametrize("seed", range(3))
def test_covering_guarantee(seed):
    xyz, _, faces = random_mesh(seed, nv=30, nf=40)
    s = [0.1, 0.37, 2.5][seed]
    P_, _ = so.sample(xyz, faces, s)
    tree = cKDTree(P_)
    rng = np.random.RandomState(seed)
    w = rng.dirichlet(np.ones(3), (len(faces), 200))
    X = xyz.astype(np.float64)[faces]  # [nf,3,3]
    q = np.einsum("fkc,fqk->fqc", X, w).reshape(-1, 3)
    d, _ = tree.query(q)
    assert d.max() <= s * (1 + 1e-12), d.max()
    # the corners of the lattice's sub-triangles are the samples: the covering radius is reached only in the limit
    assert d.max() > 0.2 * min(s, np.ptp(xyz, 0).max())


def test_every_sample_lies_on_its_face():
    xyz, rgb, faces = random_mesh(5, nv=20, nf=30)
    s = 0.15
    n = so.lattice_sizes(xyz, faces, s)
    c = so.face_samples(n)
    P_, C_ = so.sample(xyz, faces, s, rgb)
    nv = len(so.referenced_vertices(xyz, faces))
    X = xyz.astype(np.float64)
    off = nv
    for f in range(len(faces)):
        if not c[f]:
            continue
        pts = P_[off:off + c[f]]
        A, B, C = X[faces[f]]
        M = np.stack([B - A, C - A], 1)
        uv, *_ = np.linalg.lstsq(M, (pts - A).T, rcond=None)
        scale = np.abs(X[faces[f]]).max() + 1
        assert np.abs(M @ uv - (pts - A).T).max() <= 1e-12 * scale
        if abs(np.linalg.det(M.T @ M)) > 1e-6:
            assert uv.min() >= -1e-9 and uv.sum(0).max() <= 1 + 1e-9
        col = C_[off:off + c[f]].astype(int)
        lo, hi = rgb[faces[f]].min(0).astype(int), rgb[faces[f]].max(0).astype(int)
        assert (col >= lo).all() and (col <= hi).all()
        off += c[f]


def test_meshes_with_short_edges_sample_to_their_referenced_vertices():
    xyz, faces = grid_mesh(12, 0.25)
    xyz = np.concatenate([xyz, np.float32([[9, 9, 9], [np.nan, 0, 0]])])  # unreferenced, and a non-finite unreferenced vertex
    diag = float(np.sqrt(np.float64(0.25) ** 2 * 2))
    for s in (diag, diag * 1.5, 100.0):
        P_, _ = so.sample(xyz, faces, s)
        assert np.array_equal(P_, xyz[:144].astype(np.float64))
    P_, _ = so.sample(xyz, faces, diag * (1 - 1e-9))  # just below: n = 2, the three edge midpoints of every face
    assert len(P_) == 144 + 3 * len(faces)


def test_degenerate_repeated_and_non_finite_faces():
    xyz = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [np.nan, 0, 0], [2, 2, 2]])
    faces = np.int32([[0, 0, 0], [0, 1, 1], [0, 1, 3], [1, 2, 4]])
    s = 0.5
    n = so.lattice_sizes(xyz, faces, s)
    assert n.tolist() == [1, 2, 0, int(math.ceil(np.sqrt(np.float64(8)) / 0.5))]
    P_, _ = so.sample(xyz, faces, s)
    assert np.array_equal(P_[:4], xyz[[0, 1, 2, 4]].astype(np.float64))  # vertex 3 is referenced but not finite
    seg = P_[4:4 + 3]  # the segment face 0-1-1 (n = 2): its lattice points lie on the segment
    assert np.array_equal(seg[:, 1:], np.zeros((3, 2))) and (seg[:, 0] >= 0).all() and (seg[:, 0] <= 1).all()


def test_shared_edges_appear_once_per_face():
    xyz, faces = grid_mesh(2, 1.0)  # two triangles sharing the diagonal
    P_, _ = so.sample(xyz, faces, 0.5)  # n = 3 on both (diagonal sqrt 2)
    u, cnt = np.unique(P_, axis=0, return_counts=True)
    assert cnt.max() >= 2  # midpoints of the diagonal, once per face


# ---- argument checks ----------------------------------------------------------------------------------------------------------

def test_ops_reject_cpu_tensors_and_bad_arguments():
    xyz, faces = grid_mesh(3, 1.0)
    with pytest.raises(ValueError, match="CUDA float32"):
        ops.sample_mesh(torch.from_numpy(xyz), torch.from_numpy(faces), 0.5)
    with pytest.raises(ValueError, match="CUDA float32"):
        ops.sample_mesh_count(torch.from_numpy(xyz), torch.from_numpy(faces), 0.5)


@pytest.mark.parametrize("bad", [["--surface-spacing", "0.1"], ["--surface", "--surface-spacing", "-1"],
                                 ["--surface", "--surface-spacing", "nan"], ["--surface", "--surface-spacing", "0"]])
def test_scorer_surface_flags_are_checked_before_any_work(tmp_path, bad):
    with pytest.raises(ValueError, match="surface"):
        dtu_eval.main(["--data-path", str(tmp_path / "missing"), "--scans", "1"] + bad)
    with pytest.raises(ValueError, match="surface"):
        tnt_eval.main(["--gt-path", str(tmp_path / "missing"), "--scenes", "Barn"] + bad)
    (tmp_path / "gt" / "s" / "dslr_scan_eval").mkdir(parents=True)
    (tmp_path / "gt" / "s" / eth3d_eval.MLP).write_text("<MeshLabProject/>")
    args = eth3d_eval.build_parser().parse_args(["--gt-path", str(tmp_path / "gt")] + bad)
    with pytest.raises(ValueError, match="surface"):
        eth3d_eval.check_args(args)


def test_tnt_default_spacing_is_a_quarter_tau_in_the_reconstruction_frame():
    from tests import tnt_cases as tc

    s = tc.similarity(1.7, [0.3, -0.5, 0.8], 0.6, [-3.0, 2.0, 0.5])
    assert tnt_eval.surface_spacing(0.02, s) == pytest.approx(0.005 / 1.7, rel=1e-12)
    with pytest.raises(ValueError, match="similarity"):
        tnt_eval.surface_spacing(0.02, np.diag([1.0, 1.0, -1.0, 1.0]))


def test_read_mesh_and_files_without_faces(tmp_path):
    xyz, faces = grid_mesh(3, 1.0)
    rgb = np.arange(27, dtype=np.uint8).reshape(9, 3)
    body = torch.cat([torch.from_numpy(xyz).view(torch.uint8).view(-1, 12), torch.from_numpy(rgb)], 1)
    data_io.save_ply(str(tmp_path / "m.ply"), body, torch.from_numpy(faces))
    data_io.save_ply(str(tmp_path / "p.ply"), body)
    x, c, f = sample.read_mesh(str(tmp_path / "m.ply"))
    assert np.array_equal(x, xyz) and np.array_equal(c, rgb) and np.array_equal(f, faces)
    with pytest.raises(ValueError, match="p.ply"):
        sample.read_mesh(str(tmp_path / "p.ply"))
    with pytest.raises(ValueError, match="p.ply"):
        sample.main(["--ply", str(tmp_path / "p.ply"), "--spacing", "0.5", "--output", str(tmp_path / "o.ply")])
    with pytest.raises(ValueError, match="--spacing"):
        sample.main(["--ply", str(tmp_path / "m.ply"), "--spacing", "-2", "--output", str(tmp_path / "o.ply")])


def test_sample_command_ply_round_trip(tmp_path, monkeypatch):
    """The command's file, with the oracle standing in for the GPU: read back through read_ply."""
    xyz, rgb, faces = random_mesh(3, nv=10, nf=8)
    body = torch.cat([torch.from_numpy(xyz).view(torch.uint8).view(-1, 12), torch.from_numpy(rgb)], 1)
    data_io.save_ply(str(tmp_path / "m.ply"), body, torch.from_numpy(faces))

    def fake(x, f, s, c=None):
        p, col = so.sample(x.numpy(), f.numpy(), s, None if c is None else c.numpy())
        return torch.from_numpy(p), None if col is None else torch.from_numpy(col)

    monkeypatch.setattr(sample.ops, "sample_mesh", fake)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    stats = sample.main(["--ply", str(tmp_path / "m.ply"), "--spacing", "0.3", "--output", str(tmp_path / "s.ply")], device="cpu")
    x, c, nrm, f = data_io.read_ply(str(tmp_path / "s.ply"))
    p, col = so.sample(xyz, faces, 0.3, rgb)
    assert f is None and nrm is None and stats["samples"] == len(p)
    assert np.array_equal(x, p.astype(np.float32)) and np.array_equal(c, col)
