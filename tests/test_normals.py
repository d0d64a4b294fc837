"""Surface normals and oriented fusion output on the CPU: the oracle (oracle/normals_oracle.py) pinned on analytic depth
maps; the kernels' per-pixel functions (pm_geo_math.cuh, built for the host from tests/host_normals.cpp) against it; the C
ABI's argument checks; the oriented fused.ply; and the --normals options of reconstruct and colmap_output."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import normals_oracle as no
from patchmatchnet_b200 import _native, colmap_output, data_io, ops, reconstruct
from tests import normals_cases as nc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


@pytest.fixture(scope="module")
def hostnormals(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostnormals") / "_hostnormals.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_normals.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hn_depth_normals.argtypes = [P, ctypes.c_int, ctypes.c_int, P, ctypes.c_int, ctypes.c_double, ctypes.c_int, P]
    lib.hn_fuse_points_oriented.argtypes = [P] * 5 + [ctypes.c_int] * 2 + [P]
    return lib


def _host(lib, depth, K, radius=3, depth_thres=0.01, min_inliers=6):
    d = np.ascontiguousarray(depth, dtype=np.float32)
    H, W = d.shape
    kinv = np.ascontiguousarray(no.kinv64(K))
    out = np.empty((H, W, 3), dtype=np.float32)
    lib.hn_depth_normals(d.ctypes.data, H, W, kinv.ctypes.data, radius, depth_thres, min_inliers, out.ctypes.data)
    return out


# ---- the oracle on analytic maps (float64 depths: the plane is exact to rounding) ----

def test_oracle_fronto_parallel_plane():
    c = nc.fronto(24, 31)
    got, gap = no.estimate_normals(c["depth"], c["K"])
    assert np.abs(got - [0.0, 0.0, -1.0]).max() <= 1e-12 and (gap > 0.1).all()


@pytest.mark.parametrize("radius", [1, 3, 7])
def test_oracle_tilted_plane(radius):
    c = nc.tilted(29, 40)
    got, _ = no.estimate_normals(c["depth"], c["K"], radius=radius, min_inliers=4)  # a corner has 4 at radius 1
    assert (got != 0).any(-1).all() and nc.angle(got, c["want"]).max() <= 1e-9
    p = c["depth"][..., None] * no.rays(c["K"], 29, 40)
    assert (np.einsum("hwi,hwi->hw", got, p) < 0).all()  # faces the camera


def test_oracle_depth_step_keeps_each_side():
    c = nc.step(30, 40)
    got, _ = no.estimate_normals(c["depth"], c["K"])
    assert (got != 0).any(-1).all() and nc.angle(got, c["want"]).max() <= 1e-9  # including the columns next to the edge
    assert nc.angle(c["want"][:, 19], c["want"][:, 20]).min() > 0.2


def test_oracle_invalid_depths_give_zero():
    c, bad = nc.holes(32, 45)
    got, _ = no.estimate_normals(c["depth"], c["K"])
    assert (got[bad] == 0).all() and (got[~bad] != 0).any(-1).all()
    assert nc.angle(got[~bad], c["want"][~bad]).max() <= 1e-9


def test_oracle_too_few_inliers_give_zero():
    c = nc.tilted(20, 20)
    assert (no.estimate_normals(c["depth"], c["K"], radius=3, min_inliers=50)[0] == 0).all()  # at most 49 in the window
    depth = np.full((20, 20), 1000.0)
    depth[10, 10] = 500.0  # alone at its depth
    got, _ = no.estimate_normals(depth, c["K"])
    assert (got[10, 10] == 0).all() and (got[0, 0] != 0).any()


def test_oracle_collinear_inliers_give_zero():
    c = nc.tilted(21, 30)
    depth = np.full((21, 30), np.nan)
    depth[10] = c["depth"][10]  # a one-pixel-wide strip
    assert (no.estimate_normals(depth, c["K"])[0] == 0).all()
    depth[11] = c["depth"][11]  # two rows span the plane again
    got, _ = no.estimate_normals(depth, c["K"])
    assert (got[10:12, 1:-1] != 0).any(-1).all() and nc.angle(got[10:12, 1:-1], c["want"][10:12, 1:-1]).max() <= 1e-8


def test_oracle_oriented_records_layout():
    pos = np.array([[1.5, -2.0, 3.25]], dtype=np.float32)
    nrm = np.array([[0.0, 0.6, -0.8]], dtype=np.float32)
    col = np.array([[1, 2, 255]], dtype=np.uint8)
    rec = no.oriented_records(pos, nrm, col)
    assert rec.shape == (1, 27) and rec.tobytes() == pos.tobytes() + nrm.tobytes() + col.tobytes()
    assert all(np.array_equal(a, b) for a, b in zip(no.split_oriented(rec), (pos, nrm, col)))


def test_oracle_world_normals():
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]  # world -> camera: 90 degrees about z
    got = no.world_normals(np.array([[1.0, 0.0, 0.0], [0.0, 0.0, 0.0]]), E)
    assert np.array_equal(got, np.array([[0, -1, 0], [0, 0, 0]], dtype=np.float32))
    assert not np.signbit(got[1]).any()  # a zero normal stays +0


# ---- the kernels' per-pixel functions, built for the host ----

def _cases():
    out = {"fronto": nc.fronto(17, 23), "tilted": nc.tilted(29, 40), "step": nc.step(30, 41), "holes": nc.holes(33, 45)[0],
           "noisy": nc.noisy(61, 83)}
    strip = nc.tilted(21, 30)
    strip["depth"] = np.where(np.arange(21)[:, None] == 10, strip["depth"], np.nan)
    out["strip"] = strip
    return out


@pytest.mark.parametrize("name", ["fronto", "tilted", "step", "holes", "noisy", "strip"])
def test_host_pixel_function_matches_the_oracle(hostnormals, name):
    c = _cases()[name]
    depth = np.asarray(c["depth"], dtype=np.float32)
    got = _host(hostnormals, depth, c["K"])
    nc.check_against_oracle(got, depth, c["K"], angle_tol=1e-6)
    if name == "strip":
        assert (got == 0).all()
    elif name != "noisy":
        assert nc.angle(got[(got != 0).any(-1)].astype(np.float64), c["want"][(got != 0).any(-1)]).max() < 1e-3


@pytest.mark.parametrize("radius", [1, 2, 5, 7])
def test_host_pixel_function_radii_and_thresholds(hostnormals, radius):
    c = nc.noisy(37, 53, seed=radius)
    for thres, m in ((0.01, 6), (0.002, 3), (0.05, 20)):
        got = _host(hostnormals, c["depth"], c["K"], radius, thres, m)
        nc.check_against_oracle(got, c["depth"], c["K"], angle_tol=1e-6, radius=radius, depth_thres=thres, min_inliers=m)


def test_host_too_few_inliers(hostnormals):
    c = nc.tilted(20, 20)
    assert (_host(hostnormals, c["depth"], c["K"], 3, 0.01, 50) == 0).all()
    assert (_host(hostnormals, c["depth"], c["K"], 1, 0.01, 10) == 0).all()


def test_host_oriented_fusion_matches_the_oracle(hostnormals):
    rng = np.random.default_rng(5)
    H, W = 9, 13
    mask = (rng.random((H, W)) < 0.6).astype(np.uint8)
    avg = rng.uniform(400, 900, (H, W))
    img = rng.random((H, W, 3), dtype=np.float32)
    normals = rng.normal(size=(H, W, 3)).astype(np.float32)
    normals /= np.linalg.norm(normals, axis=-1, keepdims=True)
    normals[0, :] = 0.0
    mask[0, :3] = 1
    K = nc.intrinsics(H, W)
    E = np.eye(4, dtype=np.float32)
    E[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    E[:3, 3] = [10.0, -4.0, 30.0]
    cam = ops.compose_fusion_camera(K, E).numpy()
    body = np.zeros((H * W, 27), dtype=np.uint8)
    n = hostnormals.hn_fuse_points_oriented(mask.ctypes.data, avg.ctypes.data, img.ctypes.data, normals.ctypes.data,
                                            cam.ctypes.data, H, W, body.ctypes.data)
    assert n == mask.sum()
    pos, nrm, col = no.split_oriented(body[:n])
    sel = mask.astype(bool)
    want = no.world_normals(normals[sel], E)
    np.testing.assert_allclose(nrm, want, rtol=0, atol=2e-7)
    assert (nrm[:3] == 0).all() and not np.signbit(nrm[:3]).any()
    # positions and colours: the plain fusion's per-pixel function
    from oracle import geo_oracle as go

    want_v, want_c = go.fuse_points(sel, avg, img, K, E)
    assert np.array_equal(col, want_c)
    np.testing.assert_allclose(pos, want_v, rtol=1e-6)


# ---- C ABI argument checks: rejected before any launch (no GPU here) ----

def test_depth_normals_rejects_bad_arguments_without_gpu():
    lib = _native.lib()
    one = ctypes.c_void_p(16)
    kinv = (ctypes.c_double * 9)(*np.eye(3).ravel())
    fn = lib.pmb200_depth_normals
    assert fn(None, kinv, 4, 4, 3, 0.01, 6, one, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert fn(one, None, 4, 4, 3, 0.01, 6, one, None) == -1
    assert fn(one, kinv, 4, 4, 3, 0.01, 6, None, None) == -1
    for H, W in ((0, 4), (4, 0), (-1, 4), (1 << 16, 1 << 15)):
        assert fn(one, kinv, H, W, 3, 0.01, 6, one, None) == -1
        assert b"bad size" in lib.pmb200_last_error()
    for r in (0, -1, 8, 100):
        assert fn(one, kinv, 4, 4, r, 0.01, 6, one, None) == -1
        assert b"radius" in lib.pmb200_last_error()
    for t, m in ((-0.1, 6), (float("nan"), 6), (0.01, 0)):
        assert fn(one, kinv, 4, 4, 3, t, m, one, None) == -1
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.estimate_normals(torch.ones(4, 4), np.eye(3, dtype=np.float32))


def test_fuse_points_oriented_rejects_bad_arguments_without_gpu():
    lib = _native.lib()
    one = ctypes.c_void_p(16)
    fn = lib.pmb200_fuse_points_oriented
    for i in range(5):
        ptrs = [one] * 5
        ptrs[i] = None
        assert fn(*ptrs, 4, 4, one, one, one, None) == -1
        assert b"null pointer" in lib.pmb200_last_error()
    assert fn(one, one, one, one, one, 4, 4, one, None, one, None) == -1
    for H, W in ((0, 4), (4, -2), (1 << 16, 1 << 15)):
        assert fn(one, one, one, one, one, H, W, one, one, one, None) == -1
        assert b"bad size" in lib.pmb200_last_error()


# ---- the oriented fused.ply ----

def test_save_ply_oriented_header_and_bytes(tmp_path):
    rng = np.random.default_rng(2)
    pos = rng.normal(size=(5, 3)).astype(np.float32)
    nrm = rng.normal(size=(5, 3)).astype(np.float32)
    col = rng.integers(0, 256, (5, 3), dtype=np.uint8)
    rec = no.oriented_records(pos, nrm, col)
    path = str(tmp_path / "o.ply")
    data_io.save_ply(path, [torch.from_numpy(rec[:2]), torch.from_numpy(rec[2:])])
    want_head = (b"ply\nformat binary_little_endian 1.0\nelement vertex 5\nproperty float x\nproperty float y\n"
                 b"property float z\nproperty float nx\nproperty float ny\nproperty float nz\nproperty uchar red\n"
                 b"property uchar green\nproperty uchar blue\nend_header\n")
    assert open(path, "rb").read() == want_head + rec.tobytes()
    assert np.array_equal(data_io.read_ply_points(path), pos.astype(np.float64))  # the normals are skipped
    with pytest.raises(ValueError, match="one size"):
        data_io.save_ply(path, [torch.from_numpy(rec), torch.zeros((1, 15), dtype=torch.uint8)])
    with pytest.raises(ValueError):
        data_io.save_ply(path, torch.zeros((1, 20), dtype=torch.uint8))


def test_save_ply_plain_records_unchanged(tmp_path):
    body = torch.arange(30, dtype=torch.uint8).reshape(2, 15)
    path = str(tmp_path / "p.ply")
    data_io.save_ply(path, body)
    head = (b"ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\n"
            b"property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    assert open(path, "rb").read() == head + body.numpy().tobytes()


# ---- the commands' options ----

RECONSTRUCT_DEFAULTS = {
    "input_folder": None, "output_folder": "", "checkpoint_path": None, "file_format": ".pfm", "input_type": "params",
    "output_type": "both", "num_views": 20, "image_max_dim": -1, "scan_list": "", "patchmatch_interval_scale": [0.005, 0.0125, 0.025],
    "patchmatch_range": [6, 4, 2], "patchmatch_iteration": [1, 2, 2], "patchmatch_num_sample": [8, 8, 16],
    "propagate_neighbors": [0, 8, 16], "evaluate_neighbors": [9, 9, 9], "geo_pixel_thres": 1.0, "geo_depth_thres": 0.01,
    "geo_mask_thres": 5, "photo_thres": 0.5, "seed": 0, "tf32": False,
}


def test_reconstruct_normals_option():
    args = vars(reconstruct.parse_args([]))
    assert args.pop("normals") is False
    assert args == RECONSTRUCT_DEFAULTS
    assert reconstruct.parse_args(["--normals"]).normals is True


def test_colmap_output_normals_option():
    args = vars(colmap_output.parse_args([]))
    assert args.pop("normals") is False
    assert args == {"input_folder": None, "results_folder": "", "output_folder": ""}
    assert colmap_output.parse_args(["--normals"]).normals is True


def test_colmap_output_normals_without_cuda_writes_nothing(tmp_path, monkeypatch):
    from tests import scene_cases

    scene, out = tmp_path / "scene", tmp_path / "ws"
    out.mkdir()
    sc = scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    scene_cases.write_fusion_maps(str(scene), sc["cams"], 24, 32, seed=1)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        colmap_output.main(["--input-folder", str(scene), "--output-folder", str(out), "--normals"])
    assert os.listdir(out) == []
