"""The TSDF mesher on the CPU: the oracle (oracle/mesh_oracle.py) on analytic scenes, the triangle table's invariants, the
kernels' per-voxel functions (pm_mesh_math.cuh, built for the host from tests/host_mesh.cpp) against the oracle, the C ABI's
argument checks, mesh.ply, and the --mesh options of reconstruct.

Bounds fixed by running the oracle on these scenes: the sphere's radial vertex error is at most 0.45 voxel (0.5 allowed),
the plane's vertex distance at most 0.07 voxel (0.1 allowed)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import mesh_oracle as mo
from patchmatchnet_b200 import _native, data_io, reconstruct
from tests import mesh_cases as mc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def hostmesh(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostmesh") / "_hostmesh.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_mesh.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hm_seed_range.argtypes = [ctypes.c_float, ctypes.c_double, ctypes.c_double, P, P]
    lib.hm_block_key.restype = ctypes.c_ulonglong
    lib.hm_block_key.argtypes = [ctypes.c_longlong] * 3
    lib.hm_integrate.argtypes = [P, ctypes.c_int, ctypes.c_double, ctypes.c_double, P, P, P, ctypes.c_int, P, P, P, P, P, P, P]
    lib.hm_cube_index.argtypes = [P]
    lib.hm_edge_vertex.argtypes = [P, P, ctypes.c_float, ctypes.c_float, P, P, P, P]
    lib.hm_table.argtypes = [P]
    return lib


@pytest.fixture(scope="module")
def sphere():
    sc = mc.sphere_scene()
    s = 0.05
    return sc, s, mo.mesh(sc["seeds"], sc["depths"], sc["images"], sc["Ks"], sc["Es"], s)


def _p(a):
    return a.ctypes.data_as(P)


# ---- oracle on analytic scenes -------------------------------------------------------------------------------------------

def test_oracle_sphere_is_a_closed_outward_manifold(sphere):
    sc, s, (pos, col, faces, keys, vol) = sphere
    mc.check_closed_manifold(faces, len(pos))
    n = mc.face_normals(pos, faces)
    c = pos[faces].astype(np.float64).mean(1) - mc.SPHERE_CENTRE
    assert ((n * c).sum(1) > 0).all()
    radial = np.linalg.norm(pos.astype(np.float64) - mc.SPHERE_CENTRE, axis=1) - mc.SPHERE_RADIUS
    assert np.abs(radial).max() < 0.5 * s
    # colours follow the surface colour
    want = mc.colour_of(pos.astype(np.float64)) * 255
    assert np.abs(col.astype(np.float64) - want).mean() < 8


def test_oracle_tilted_plane():
    pl = mc.plane_scene()
    s = 8.0
    pos, col, faces, keys, vol = mo.mesh(pl["seeds"], pl["depths"], pl["images"], pl["Ks"], pl["Es"], s)
    assert len(faces) > 1000
    assert mc.plane_distance(pos).max() < 0.1 * s
    assert len(np.unique(faces)) == len(pos)


def test_oracle_allocation_of_a_far_outlier():
    pts = np.array([[0.1, 0.2, 0.3], [0.11, 0.2, 0.3], [5000.0, -3000.0, 7000.0]], np.float32)
    keys = mo.allocate(pts, 0.01, 3)
    assert 2 <= len(keys) <= 16
    assert np.all(keys[1:] > keys[:-1])
    with pytest.raises(ValueError):
        mo.allocate(np.array([[1e9, 0, 0]], np.float32), 0.01, 3)


# ---- the triangle table ---------------------------------------------------------------------------------------------------

def test_table_vertices_lie_on_sign_change_edges():
    tab = mo.read_table()
    assert (tab[0] == -1).all() and (tab[255] == -1).all()
    for case in range(256):
        row = [int(e) for e in tab[case] if e >= 0]
        assert len(row) % 3 == 0 and (tab[case, len(row):] == -1).all()
        neg = [(case >> c) & 1 for c in range(8)]
        for e in row:
            a = tuple(mo.EDGE_OFFSET[e])
            b = tuple(mo.EDGE_OFFSET[e] + mo.UNIT[mo.EDGE_AXIS[e]])
            ca = [tuple(c) for c in mo.CORNERS].index(a)
            cb = [tuple(c) for c in mo.CORNERS].index(b)
            assert neg[ca] != neg[cb], (case, e)
        if 0 < case < 255:
            assert row, case


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_table_is_crack_free_on_random_fields(seed):
    """Every voxel of 2 x 2 x 2 blocks valid with random signs: each directed edge is used once, and an edge without its
    reverse lies on an outer face of the grid."""
    rng = np.random.default_rng(seed)
    keys = np.sort(mo.block_key(np.array([[i, j, k] for i in (0, 1) for j in (0, 1) for k in (0, 1)])))
    G = len(keys) * 512
    tsdf = rng.uniform(-1, 1, G).astype(np.float32)
    if seed % 2:
        tsdf = np.where(np.abs(tsdf) < 0.05, 0.0, tsdf).astype(np.float32)  # exact zeros count as positive
    pos, col, faces = mo.marching_cubes(keys, 1.0, tsdf, np.ones(G, np.float32), np.zeros((G, 3), np.uint8))
    assert len(faces) > 1000
    f = faces.astype(np.int64)
    n = len(pos)
    directed = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    keys_d = directed[:, 0] * n + directed[:, 1]
    assert len(np.unique(keys_d)) == len(keys_d)
    lone = ~np.isin(directed[:, 1] * n + directed[:, 0], keys_d)
    p = pos.astype(np.float64)
    lo, hi = 0.5, 15.5  # voxel centres of the outer layers
    a, b = p[directed[lone, 0]], p[directed[lone, 1]]
    on_face = ((np.isclose(a, lo) & np.isclose(b, lo)) | (np.isclose(a, hi) & np.isclose(b, hi))).any(1)
    assert on_face.all()
    assert lone.sum() < len(directed) / 4


# ---- host build of pm_mesh_math.cuh against the oracle --------------------------------------------------------------------

def test_host_table_equals_the_parsed_table(hostmesh):
    out = np.zeros((256, 16), np.int8)
    hostmesh.hm_table(_p(out))
    assert np.array_equal(out, mo.read_table())
    for e in range(12):
        assert hostmesh.hm_edge_offset(e) == int(mo.EDGE_OFFSET[e] @ [1, 2, 4]) and hostmesh.hm_edge_axis(e) == mo.EDGE_AXIS[e]
    for c in range(8):
        assert hostmesh.hm_corner_offset(c) == int(mo.CORNERS[c] @ [1, 2, 4])


def test_host_integration_matches_the_oracle(hostmesh, sphere):
    sc, s, (pos, col, faces, keys, vol) = sphere
    coords = mo.voxel_coords(keys).astype(np.int32)
    V = len(sc["depths"])
    K = np.stack([k.astype(np.float64) for k in sc["Ks"]])
    Rt = np.stack([e.astype(np.float64)[:3] for e in sc["Es"]])
    hw = np.array([d.shape for d in sc["depths"]], np.int32)
    dflat = np.concatenate([d.ravel() for d in sc["depths"]]).astype(np.float32)
    iflat = np.concatenate([i.ravel() for i in sc["images"]]).astype(np.float32)
    doff = np.cumsum([0] + [d.size for d in sc["depths"]])[:-1].astype(np.int64)
    ioff = np.cumsum([0] + [i.size for i in sc["images"]])[:-1].astype(np.int64)
    n = len(coords)
    tsdf, weight, rgb = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 3), np.uint8)
    hostmesh.hm_integrate(_p(coords), n, s, 3 * s, _p(K), _p(Rt), _p(hw), V, _p(dflat), _p(doff), _p(iflat), _p(ioff), _p(tsdf),
                          _p(weight), _p(rgb))
    assert np.array_equal(weight, vol[1]) and np.array_equal(tsdf, vol[0]) and np.array_equal(rgb, vol[2])
    assert (weight > 0).mean() > 0.1


def test_host_cube_index_and_edge_vertex(hostmesh):
    rng = np.random.default_rng(3)
    for _ in range(200):
        t = rng.uniform(-1, 1, 8).astype(np.float32)
        assert hostmesh.hm_cube_index(_p(t)) == int(((t < 0) * (1 << np.arange(8))).sum())
    for _ in range(200):
        xa = rng.uniform(-5, 5, 3)
        xb = xa + np.eye(3)[rng.integers(3)] * 0.37
        ta, tb = np.float32(rng.uniform(-1, 0)), np.float32(rng.uniform(1e-3, 1))
        ca, cb = rng.integers(0, 256, 3).astype(np.uint8), rng.integers(0, 256, 3).astype(np.uint8)
        pos, rgb = np.zeros(3, np.float32), np.zeros(3, np.uint8)
        hostmesh.hm_edge_vertex(_p(xa), _p(xb), float(ta), float(tb), _p(ca), _p(cb), _p(pos), _p(rgb))
        t = np.float64(ta) / (np.float64(ta) - np.float64(tb))
        assert np.array_equal(pos, (xa + t * (xb - xa)).astype(np.float32))
        assert np.array_equal(rgb, np.clip(np.rint(ca + t * (cb.astype(np.float64) - ca)), 0, 255).astype(np.uint8))


def test_host_seed_range_and_keys(hostmesh):
    lo, hi = ctypes.c_int(), ctypes.c_int()
    assert hostmesh.hm_seed_range(0.123, 0.01, 0.03, ctypes.byref(lo), ctypes.byref(hi)) == 1
    assert (lo.value, hi.value) == (int(np.floor((np.float64(np.float32(0.123)) - 0.03) / 0.01)),
                                    int(np.floor((np.float64(np.float32(0.123)) + 0.03) / 0.01)))
    assert hostmesh.hm_seed_range(1e6, 0.01, 0.03, ctypes.byref(lo), ctypes.byref(hi)) == 0
    assert hostmesh.hm_seed_range(float("nan"), 0.01, 0.03, ctypes.byref(lo), ctypes.byref(hi)) == 0
    b = np.array([[-3, 7, 1 << 19], [0, 0, 0], [-(1 << 20), (1 << 20) - 1, 5]])
    for row in b:
        assert hostmesh.hm_block_key(*[int(v) for v in row]) == int(mo.block_key(row))
        assert np.array_equal(mo.key_blocks(mo.block_key(row)[None])[0], row)


# ---- C ABI argument checks (no device needed: each is rejected before any launch) -----------------------------------------

def _rejects(rc):
    assert rc == -1, rc
    return _native.lib().pmb200_last_error().decode()


def test_abi_rejects_bad_arguments():
    lib = _native.lib()
    dummy = ctypes.c_void_p(16)
    nb = ctypes.c_int64(0)
    for trunc in (0, 5):
        assert "trunc" in _rejects(lib.pmb200_tsdf_alloc(dummy, 4, 0.1, trunc, ctypes.byref(nb), dummy, 1 << 20, None))
        assert "trunc" in _rejects(lib.pmb200_tsdf_integrate(dummy, 1, 0.1, trunc, dummy, 1, dummy, dummy, dummy, dummy, dummy, dummy,
                                                             1 << 20, None))
    for s in (0.0, -1.0, float("nan"), float("inf")):
        assert "voxel_size" in _rejects(lib.pmb200_tsdf_alloc(dummy, 4, s, 3, ctypes.byref(nb), dummy, 1 << 20, None))
        assert "voxel_size" in _rejects(lib.pmb200_tsdf_mesh_write(dummy, 1, s, dummy, dummy, dummy, 1, dummy, dummy, dummy, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_tsdf_alloc(None, 4, 0.1, 3, ctypes.byref(nb), dummy, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_tsdf_alloc(dummy, 4, 0.1, 3, None, dummy, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_tsdf_integrate(None, 1, 0.1, 3, dummy, 1, dummy, dummy, dummy, dummy, dummy, dummy, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_tsdf_mesh_count(dummy, 1, dummy, None, 1, dummy, dummy, 1 << 20, None))
    assert "null" in _rejects(lib.pmb200_tsdf_mesh_write(dummy, 1, 0.1, dummy, dummy, None, 1, dummy, dummy, dummy, 1 << 20, None))
    assert "n_views" in _rejects(lib.pmb200_tsdf_integrate(dummy, 1, 0.1, 3, dummy, 0, dummy, dummy, dummy, dummy, dummy, dummy, 1 << 20, None))
    assert lib.pmb200_tsdf_integrate_workspace_bytes(0) == -1
    assert "n_blocks" in _rejects(lib.pmb200_tsdf_integrate(dummy, 0, 0.1, 3, dummy, 1, dummy, dummy, dummy, dummy, dummy, dummy, 1 << 20, None))
    assert "n_blocks" in _rejects(lib.pmb200_tsdf_mesh_count(dummy, 1 << 22, dummy, dummy, 1, dummy, dummy, 1 << 20, None))
    assert lib.pmb200_tsdf_mesh_workspace_bytes(1 << 22) == -1 and lib.pmb200_tsdf_alloc_workspace_bytes(1 << 28) == -1
    assert "min_weight" in _rejects(lib.pmb200_tsdf_mesh_count(dummy, 1, dummy, dummy, 0, dummy, dummy, 1 << 20, None))
    assert "2^28" in _rejects(lib.pmb200_tsdf_alloc(dummy, 1 << 28, 0.1, 3, ctypes.byref(nb), dummy, 1 << 40, None))
    bad = (_native.TsdfView * 1)()
    bad[0].height, bad[0].width = 0, 10
    assert "H, W" in _rejects(lib.pmb200_tsdf_integrate(dummy, 1, 0.1, 3, ctypes.addressof(bad), 1, dummy, dummy, dummy, dummy, dummy,
                                                        dummy, 1 << 20, None))


def test_tsdf_mesh_rejects_bad_arguments_before_any_launch():
    from patchmatchnet_b200 import ops

    pts = torch.zeros((4, 3))
    d, img, K, E = torch.zeros((8, 8)), torch.zeros((3, 8, 8)), np.eye(3), np.eye(4)
    for kw, what in (({"voxel_size": 0.0}, "voxel_size"), ({"voxel_size": float("nan")}, "voxel_size"), ({"trunc": 5}, "trunc"),
                     ({"trunc": 0}, "trunc"), ({"min_weight": 0}, "min_weight")):
        args = {"voxel_size": 0.1, **kw}
        with pytest.raises(ValueError, match=what):
            ops.tsdf_mesh(pts, [d], [img], [K], [E], **args)
    with pytest.raises(ValueError, match="one depth"):
        ops.tsdf_mesh(pts, [], [], [], [], 0.1)
    with pytest.raises(ValueError, match="CUDA"):
        ops.tsdf_mesh(pts, [d], [img], [K], [E], 0.1)  # CPU maps: there is no CPU path


# ---- mesh.ply ---------------------------------------------------------------------------------------------------------------

def _mesh_body(n=5, nf=3, seed=0):
    rng = np.random.default_rng(seed)
    xyz = rng.normal(size=(n, 3)).astype(np.float32)
    rec = np.concatenate([xyz.view(np.uint8).reshape(n, 12), rng.integers(0, 256, (n, 3)).astype(np.uint8)], 1)
    faces = rng.integers(0, n, (nf, 3)).astype(np.int32)
    return xyz, torch.from_numpy(rec), torch.from_numpy(faces)


def test_save_ply_with_faces(tmp_path):
    xyz, body, faces = _mesh_body()
    plain, mesh = str(tmp_path / "plain.ply"), str(tmp_path / "mesh.ply")
    data_io.save_ply(plain, body)
    data_io.save_ply(mesh, body, faces)
    raw = open(mesh, "rb").read()
    head, _, rest = raw.partition(b"end_header\n")
    assert head.decode() == ("ply\nformat binary_little_endian 1.0\nelement vertex 5\nproperty float x\nproperty float y\n"
                             "property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nelement face 3\n"
                             "property list uchar int vertex_indices\n")
    assert rest[:75] == body.numpy().tobytes()
    want = b"".join(b"\x03" + f.astype("<i4").tobytes() for f in faces.numpy())
    assert rest[75:] == want and len(rest) == 75 + 3 * 13
    # without faces the file is the plain one, byte for byte
    assert open(plain, "rb").read() == raw[: raw.index(b"element face")] + b"end_header\n" + rest[:75]
    with pytest.raises(ValueError):
        data_io.save_ply(mesh, body, faces + 5)
    with pytest.raises(ValueError):
        data_io.save_ply(mesh, body, faces.to(torch.int64))


def test_read_ply_points_reads_a_mesh(tmp_path):
    xyz, body, faces = _mesh_body(n=40, nf=60, seed=2)
    path = str(tmp_path / "scan1" / "mesh.ply")
    os.makedirs(os.path.dirname(path))
    data_io.save_ply(path, body, faces)
    assert np.array_equal(data_io.read_ply_points(path), xyz.astype(np.float64))


# ---- reconstruct --mesh ---------------------------------------------------------------------------------------------------

def test_reconstruct_mesh_option_defaults():
    a = reconstruct.parse_args([])
    assert not any(k.startswith("mesh") for k in vars(a))  # a run without the options has the namespace it always had
    m = reconstruct.mesh_options(a)
    assert (m.mesh, m.mesh_voxel_size, m.mesh_trunc, m.mesh_min_weight) == (False, None, 3, 1)
    b = reconstruct.mesh_options(reconstruct.parse_args(["--mesh", "--mesh-voxel-size", "0.5", "--mesh-trunc", "2",
                                                         "--mesh-min-weight", "3"]))
    assert (b.mesh, b.mesh_voxel_size, b.mesh_trunc, b.mesh_min_weight) == (True, 0.5, 2, 3)
    assert reconstruct.mesh_options(reconstruct.parse_args(["--mesh"])).mesh_trunc == 3


def test_default_mesh_voxel_size():
    d = [torch.tensor([[0.0, 100.0], [200.0, 300.0]]), torch.tensor([[50.0, 0.0], [0.0, 0.0]]), torch.zeros((2, 2))]
    Ks = [np.diag([100.0, 100.0, 1.0]), np.diag([10.0, 10.0, 1.0]), np.diag([1.0, 1.0, 1.0])]
    # per view median valid depth / fx: 200 / 100 = 2 and 50 / 10 = 5; the empty view is skipped
    assert reconstruct.default_mesh_voxel_size(d, Ks) == 2.0 * 3.5


def test_reconstruct_mesh_without_cuda_writes_nothing(tmp_path, monkeypatch):
    from tests import scene_cases

    scene, out = tmp_path / "scene", tmp_path / "out"
    out.mkdir()
    sc = scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    scene_cases.write_fusion_maps(str(out), sc["cams"], 24, 32, seed=1)
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"")
    before = sorted(os.listdir(out))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        reconstruct.main(["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt),
                          "--output-type", "fusion", "--mesh"])
    assert sorted(os.listdir(out)) == before
    for bad in (["--mesh-trunc", "5"], ["--mesh-min-weight", "0"], ["--mesh-voxel-size", "-1"], ["--output-type", "depth"]):
        with pytest.raises(ValueError):
            reconstruct.main(["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt), "--mesh", *bad])
    assert sorted(os.listdir(out)) == before
