"""The Poisson mesher on the CPU: the oracle (oracle/poisson_oracle.py) on spheres, its operators against the stated stencil,
the kernels' per-element formulas (pm_poisson_math.cuh, built for the host from tests/host_poisson.cpp) against the oracle,
the argument checks of the C ABI, ops.poisson_mesh and the poisson command, and the --poisson options of reconstruct."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import poisson_oracle as po
from patchmatchnet_b200 import _native, data_io, ops, poisson, reconstruct
from tests import mesh_cases as mc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


def sphere_cloud(n: int = 20000, nonuniform: bool = False):
    """Points on the mesh_cases sphere with exact outward normals; non-uniform: the upper half 10x denser."""
    d = mc.fibonacci(5 * n if nonuniform else n)
    if nonuniform:
        d = d[(d[:, 2] > 0) | (np.arange(len(d)) % 10 == 0)]
    return (mc.SPHERE_CENTRE + mc.SPHERE_RADIUS * d).astype(np.float32), d.astype(np.float32)


@pytest.fixture(scope="module")
def hostpoisson(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostpoisson") / "_hostpoisson.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_poisson.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hp_keep.argtypes = [P, P, P]
    lib.hp_quantile.restype = ctypes.c_double
    lib.hp_quantile.argtypes = [P, ctypes.c_longlong, ctypes.c_double]
    lib.hp_place.argtypes = [P, P, ctypes.c_int, ctypes.c_double, P, P]
    lib.hp_grid_coord.restype = ctypes.c_double
    lib.hp_grid_coord.argtypes = [ctypes.c_float, ctypes.c_double, ctypes.c_longlong]
    lib.hp_cell.argtypes = [ctypes.c_double, ctypes.c_int]
    lib.hp_corners.argtypes = [P, P, P]
    lib.hp_stencil.restype = ctypes.c_double
    lib.hp_stencil.argtypes = [ctypes.c_int] * 3
    return lib


def _p(a):
    return a.ctypes.data_as(P)


# ---- the oracle's operators ----------------------------------------------------------------------------------------------

def test_kronecker_matrix_is_the_27_point_stencil():
    n = 7
    A = po.kron_matrix(n).toarray()
    c = (3 * n * n + 3 * n + 3)  # interior node (3, 3, 3)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nz = (dx != 0) + (dy != 0) + (dz != 0)
                want = [8 / 3, 0.0, -1 / 6, -1 / 12][nz]
                assert abs(A[c, c + dx + n * dy + n * n * dz] - want) < 1e-15
    assert abs(A[c].sum()) < 1e-14 and np.count_nonzero(np.abs(A[c]) > 1e-15) == 21
    # apply_A agrees with the matrix on a random field
    rng = np.random.default_rng(0)
    chi = np.zeros((n + 2,) * 3)
    chi[1:-1, 1:-1, 1:-1] = rng.standard_normal((n, n, n))
    assert np.allclose(po.apply_A(chi)[1:-1, 1:-1, 1:-1].ravel(), A @ chi[1:-1, 1:-1, 1:-1].ravel(), atol=1e-12)


def test_galerkin_coarse_operator_is_twice_the_stencil_at_depth_5():
    nc = 15  # depth 5: 31 fine interior nodes per axis, 15 coarse
    P_ = po.prolongation(nc)
    lhs = (P_.T @ po.kron_matrix(2 * nc + 1) @ P_).tocsr()
    assert abs(lhs - 2 * po.kron_matrix(nc)).max() < 1e-12


# ---- the oracle on spheres ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("nonuniform", [False, True], ids=["uniform", "nonuniform"])
def test_oracle_sphere_is_a_closed_outward_manifold(nonuniform):
    xyz, nrm = sphere_cloud(nonuniform=nonuniform)
    r = po.poisson(xyz, nrm, depth=5)
    pos, faces, h = r["pos"], r["faces"], r["h"]
    mc.check_closed_manifold(faces, len(pos))
    n = mc.face_normals(pos, faces)
    c = pos[faces].astype(np.float64).mean(1) - mc.SPHERE_CENTRE
    assert ((n * c).sum(1) > 0).all()
    radial = np.linalg.norm(pos.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS
    assert np.abs(radial).max() < 0.4 * h, np.abs(radial).max() / h  # the oracle's own error: 0.33 h (uniform)
    assert -0.9 < r["iso"] < -0.5


# ---- the host build against the oracle ------------------------------------------------------------------------------------

def test_host_keep_and_normalise(hostpoisson):
    xyz = np.array([[0, 0, 0], [np.nan, 0, 0], [0, 0, 0], [0, 0, 0], [1, 2, 3], [0, 0, 0]], np.float32)
    nrm = np.array([[3, 4, 0], [1, 0, 0], [0, 0, 0], [np.inf, 0, 0], [1e-30, 0, 0], [1e30, 1e30, 1e30]], np.float32)
    m, unit = po.keep(xyz, nrm)
    for i in range(len(xyz)):
        out = np.zeros(3)
        assert hostpoisson.hp_keep(_p(xyz[i].copy()), _p(nrm[i].copy()), _p(out)) == int(m[i])
        if m[i]:
            assert np.array_equal(out, unit[i])
    assert m.tolist() == [True, False, False, False, True, True]


def test_host_quantiles_and_placement(hostpoisson):
    rng = np.random.default_rng(1)
    for m in (1, 2, 7, 1000):
        v = np.sort(rng.standard_normal(m).astype(np.float32).astype(np.float64))
        for q in (0.0, 0.01, 0.25, 0.4999, 0.99, 1.0):
            assert hostpoisson.hp_quantile(_p(v), m, q) == po.quantile(v, q)
    for depth in (5, 8, 10):
        for _ in range(20):
            pts = (rng.standard_normal((50, 3)) * rng.uniform(0.01, 100) + rng.uniform(-1000, 1000, 3)).astype(np.float32)
            q = float(rng.choice([0.0, 0.05]))
            N, h, I0, lo, hi = po.place(pts, depth, 1.1, q)
            hh, ii = ctypes.c_double(), np.zeros(3, np.int64)
            assert hostpoisson.hp_place(_p(lo), _p(hi), depth, 1.1, ctypes.byref(hh), _p(ii)) == 1
            assert hh.value == h and np.array_equal(ii, I0)
            u = po.grid_coords(pts, h, I0)
            for i in range(5):
                for a in range(3):
                    assert hostpoisson.hp_grid_coord(float(pts[i, a]), h, int(I0[a])) == u[i, a]
                    assert hostpoisson.hp_cell(u[i, a], N) == po.cells(u[i:i + 1], N)[0][0, a]
    zero = np.zeros(3)
    assert hostpoisson.hp_place(_p(zero), _p(zero), 5, 1.1, ctypes.byref(ctypes.c_double()), _p(np.zeros(3, np.int64))) == 0


def test_host_hat_weights_gradients_and_stencil(hostpoisson):
    rng = np.random.default_rng(2)
    f = np.concatenate([rng.uniform(0, 1, (50, 3)), [[0, 0, 0], [1, 1, 1], [0.5, 0, 1]]])
    base = np.zeros((len(f), 3), np.int64)
    for i in range(len(f)):
        w, g = np.zeros(8), np.zeros((8, 3))
        hostpoisson.hp_corners(_p(f[i].copy()), _p(w), _p(g))
        for k in range(8):
            _, wt, gr = po._corner(base[i:i + 1], f[i:i + 1], k)
            assert w[k] == wt[0] and np.array_equal(g[k], gr[0])
        assert abs(w.sum() - 1) < 1e-15 and np.abs(g.sum(0)).max() < 1e-15
    A = po.kron_matrix(3).toarray()
    for dz in (-2, -1, 0, 1, 2):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                want = A[13, 13 + dx + 3 * dy + 9 * dz] if abs(dz) <= 1 else 0.0
                assert abs(hostpoisson.hp_stencil(dx, dy, dz) - want) < 1e-15


# ---- argument checks ------------------------------------------------------------------------------------------------------

def _rejects(rc):
    assert rc == -1
    return _native.lib().pmb200_last_error().decode()


def test_abi_rejects_bad_arguments():
    lib = _native.lib()
    d = ctypes.c_void_p(16)
    g = _native.PoissonGrid()
    for depth in (4, 11):
        assert "depth" in _rejects(lib.pmb200_poisson_workspace_bytes(depth, 10))
        assert "depth" in _rejects(lib.pmb200_poisson_setup(d, d, None, 10, depth, 1.1, 0.0, ctypes.byref(g), d, 1 << 40, None))
    assert "2^28" in _rejects(lib.pmb200_poisson_workspace_bytes(5, 1 << 28))
    for scale in (0.99, float("nan"), float("inf")):
        assert "scale" in _rejects(lib.pmb200_poisson_setup(d, d, None, 10, 5, scale, 0.0, ctypes.byref(g), d, 1 << 40, None))
    for q in (-0.1, 0.5, float("nan")):
        assert "bbox_quantile" in _rejects(lib.pmb200_poisson_setup(d, d, None, 10, 5, 1.1, q, ctypes.byref(g), d, 1 << 40, None))
    assert "null" in _rejects(lib.pmb200_poisson_setup(None, d, None, 10, 5, 1.1, 0.0, ctypes.byref(g), d, 1 << 40, None))
    # a grid setup did not return is rejected by every later call
    r = _native.PoissonResult()
    assert "grid" in _rejects(lib.pmb200_poisson_density(ctypes.byref(g), None, None, d, 1 << 40, None))
    assert "grid" in _rejects(lib.pmb200_poisson_rhs(ctypes.byref(g), None, d, 1 << 40, None))
    assert "grid" in _rejects(lib.pmb200_poisson_solve(ctypes.byref(g), 1e-5, 50, ctypes.byref(r), None, d, 1 << 40, None))
    assert "grid" in _rejects(lib.pmb200_poisson_band(ctypes.byref(g), 0.0, d, 1, d, d, d, 1 << 40, None))
    assert "grid" in _rejects(lib.pmb200_poisson_colours(ctypes.byref(g), d, 1, d, 1 << 40, None))


def test_poisson_mesh_rejects_bad_arguments_before_any_launch():
    pts, nrm = torch.zeros((4, 3)), torch.ones((4, 3))
    for kw, what in (({"depth": 4}, "depth"), ({"depth": 11}, "depth"), ({"depth": 9.0}, "depth"), ({"scale": 0.5}, "scale"),
                     ({"scale": float("nan")}, "scale"), ({"band": 0}, "band"), ({"band": 5}, "band"),
                     ({"bbox_quantile": 0.5}, "bbox_quantile"), ({"bbox_quantile": -0.1}, "bbox_quantile"), ({"tol": -1.0}, "tol"),
                     ({"max_cycles": -1}, "max_cycles")):
        with pytest.raises(ValueError, match=what):
            ops.poisson_mesh(pts, nrm, **kw)
    with pytest.raises(ValueError, match="CUDA"):
        ops.poisson_mesh(pts, nrm)
    for depth, n in ((4, 10), (5, -1), (5, 1 << 28), (True, 10)):
        with pytest.raises(ValueError):
            ops.poisson_mesh_bytes(depth, n)


def test_poisson_command_rejects_a_ply_without_normals(tmp_path):
    body = torch.zeros((5, 15), dtype=torch.uint8)
    path = str(tmp_path / "plain.ply")
    data_io.save_ply(path, body)
    with pytest.raises(ValueError, match="no normals"):
        poisson.main(["--ply", path, "--output", str(tmp_path / "out.ply")])
    with pytest.raises(ValueError, match="depth"):
        poisson.main(["--ply", path, "--output", str(tmp_path / "out.ply"), "--depth", "12"])
    assert not os.path.exists(tmp_path / "out.ply")


# ---- reconstruct --poisson -------------------------------------------------------------------------------------------------

def test_reconstruct_poisson_option_defaults():
    a = reconstruct.parse_args([])
    assert not any(k.startswith("poisson") for k in vars(a))  # a run without the options has the namespace it always had
    p = reconstruct.poisson_options(a)
    assert (p.poisson, p.poisson_depth) == (False, 9)
    b = reconstruct.poisson_options(reconstruct.parse_args(["--normals", "--poisson", "--poisson-depth", "7"]))
    assert (b.poisson, b.poisson_depth) == (True, 7)


def test_reconstruct_poisson_without_normals_raises_and_writes_nothing(tmp_path):
    from tests import scene_cases

    scene, out = tmp_path / "scene", tmp_path / "out"
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"")
    base = ["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt)]
    for extra, what in ((["--poisson"], "--normals"), (["--normals", "--poisson", "--output-type", "depth"], "fusion"),
                        (["--normals", "--poisson", "--poisson-depth", "4"], "5..10"), (["--normals", "--poisson-depth", "6"], "--poisson")):
        with pytest.raises(ValueError, match=what):
            reconstruct.reconstruct(reconstruct.parse_args(base + extra))
    assert not out.exists()
