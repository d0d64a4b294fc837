"""DTU evaluation without a GPU: the CPU oracle (oracle/dtu_oracle.py), the PLY point reader, the ground-truth loader and the
argument checks of the point-cloud C ABI.

The oracle cannot be pinned to MATLAB (neither MATLAB nor the DTU data is available), so it is pinned here by small cases
whose answers are worked out by hand in the test: a chain of points exactly dst apart, duplicates at distance 0, points on
and around MaxDistCP's block boundaries, coordinates that land exactly on .5 before MATLAB's round, an empty side (NaN) and
an even-count median."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import dtu_oracle as do
from patchmatchnet_b200 import _native, data_io, dtu_eval
from tests import dtu_cases


# ---- thinning ---------------------------------------------------------------------------------------------------------------

def _line(xs):
    return np.array([[x, 0.0, 0.0] for x in xs])


def test_thin_chain_exactly_dst_apart_is_inclusive():
    pts = _line([0.0, 0.25, 0.5, 0.75, 1.0])  # exact binary fractions: neighbours are exactly dst = 0.25 apart
    # in order: 0 kept, removes 1 (at exactly dst); 2 kept, removes 3; 4 kept
    assert do.thin(pts, [0, 1, 2, 3, 4], 0.25).tolist() == [True, False, True, False, True]
    # 1 first removes 0 and 2; 0 and 2 are gone; 3 is still in (removed points remove nothing) and removes 4
    assert do.thin(pts, [1, 0, 2, 3, 4], 0.25).tolist() == [False, True, False, True, False]
    # just beyond dst nothing is removed
    assert do.thin(_line([0.0, 0.25 + 2 ** -40]), [0, 1], 0.25).tolist() == [True, True]


def test_thin_duplicates():
    pts = np.array([[1.0, 2.0, 3.0]] * 3 + [[1.3, 2.0, 3.0]])
    # the first visited copy survives, the other copies are at distance 0; the point 0.3 away is beyond dst = 0.25
    assert do.thin(pts, [2, 0, 1, 3], 0.25).tolist() == [False, False, True, True]
    assert do.thin(pts, [3, 1, 0, 2], 0.25).tolist() == [False, True, False, True]


# ---- MaxDistCP ----------------------------------------------------------------------------------------------------------------

BLOCK_BB = np.array([[0.0, 0.0, 0.0], [200.0, 200.0, 200.0]])  # floor(200 / 60) = 3: blocks [0,60) [60,120) [120,180) [180,240)
BLOCK_TO = np.array([[10.0, 10.0, 10.0]])
BLOCK_FROM = np.array([
    [60.0, 10.0, 10.0],   # on the boundary: block 1, widened [0,180) holds the to point -> 50
    [120.0, 10.0, 10.0],  # block 2, widened [60,240) is empty -> 60
    [119.0, 10.0, 10.0],  # block 1 -> 109: the script keeps values above 60 (the GPU caps them)
    [-0.5, 10.0, 10.0],   # below the first block: in no block -> 60 although the to point is 10.5 away
    [190.0, 10.0, 10.0],  # block 3, widened [120,300) is empty -> 60
    [240.0, 10.0, 10.0],  # 240 is the (exclusive) high end of block 3 and there is no block 4 -> 60
])
BLOCK_WANT = [50.0, 60.0, 109.0, 60.0, 60.0, 60.0]


def test_max_dist_cp_blocks():
    assert do.max_dist_cp(BLOCK_TO, BLOCK_FROM, BLOCK_BB, 60.0).tolist() == BLOCK_WANT


def test_max_dist_cp_is_the_nearest_distance_below_the_cap():
    rng = np.random.RandomState(3)
    to = rng.uniform(0, 150, (400, 3))
    frm = rng.uniform(-20, 170, (300, 3))
    got = do.max_dist_cp(to, frm, np.array([[0, 0, 0], [150, 150, 150.0]]), 60.0)
    want = np.sqrt(((frm[:, None, :] - to[None]) ** 2).sum(-1)).min(1)
    inside = ((frm >= 0) & (frm < 180)).all(1)
    np.testing.assert_allclose(got[inside], want[inside], rtol=1e-12)
    assert (got[~inside] == 60.0).all()


# ---- mask, plane, statistics --------------------------------------------------------------------------------------------------

def test_mask_uses_matlab_round_half_away_from_zero():
    mask = np.zeros((3, 1, 1), dtype=bool)
    mask[0, 0, 0] = True   # voxel 1
    mask[2, 0, 0] = True   # voxel 3
    bb = np.array([[0.0, 0.0, 0.0], [3.0, 1.0, 1.0]])
    q = np.array([
        [1.5, 0.0, 0.0],   # 1.5 / 1 + 1 = 2.5 -> 3 (rint would give 2, which is false)
        [-0.5, 0.0, 0.0],  # 0.5 -> 1 (rint would give 0, outside)
        [0.4, 0.0, 0.0],   # 1.4 -> 1
        [0.6, 0.0, 0.0],   # 1.6 -> 2: false
        [-1.5, 0.0, 0.0],  # -0.5 -> -1: outside
        [2.5, 0.0, 0.0],   # 3.5 -> 4: outside
    ])
    want = [True, True, True, False, False, False]
    assert do.data_in_mask(q, mask, bb, 1.0).tolist() == want
    got = dtu_eval.data_in_mask(torch.as_tensor(q), torch.as_tensor(mask), torch.as_tensor(bb[0]), 1.0)
    assert got.tolist() == want
    assert dtu_eval.matlab_round(torch.tensor([2.5, -2.5, 0.5, -0.5, 0.49999999999999994, 1.4], dtype=torch.float64)).tolist() == [3, -3, 1, -1, 0, 1]


def test_plane_is_strict():
    q = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 2.0], [0.0, 0.0, 3.0]])
    p = np.array([0.0, 0.0, 1.0, -2.0])
    assert do.stl_above_plane(q, p).tolist() == [False, False, True]
    assert dtu_eval.above_plane(torch.as_tensor(q), torch.as_tensor(p)).tolist() == [False, False, True]


def test_stats_even_median_empty_and_single():
    s = do.side_stats(np.array([4.0, 1.0, 3.0, 2.0]))
    assert s == {"count": 4, "mean": 2.5, "median": 2.5, "var": pytest.approx(5.0 / 3.0, rel=1e-15)}
    e = do.side_stats(np.array([]))
    assert e["count"] == 0 and all(math.isnan(e[k]) for k in ("mean", "median", "var"))
    assert do.side_stats(np.array([7.0])) == {"count": 1, "mean": 7.0, "median": 7.0, "var": 0.0}
    for d in ([4.0, 1.0, 3.0, 2.0], [], [7.0], [5.0, 1.0, 2.0]):
        got, want = dtu_eval.side_stats(torch.tensor(d, dtype=torch.float64)), do.side_stats(np.array(d))
        assert got.keys() == want.keys()
        for k in got:
            assert (math.isnan(got[k]) and math.isnan(want[k])) or got[k] == pytest.approx(want[k], rel=1e-15)


def test_oracle_scan_with_an_empty_side_gives_nan():
    # every data point is more than 20 mm from the only STL point -> accuracy has no values
    data = np.array([[50.0, 50.0, 50.0], [90.0, 50.0, 50.0]])
    stl = np.array([[10.0, 10.0, 10.0]])
    mask = np.ones((200, 200, 200), dtype=bool)
    r = do.evaluate_scan(data, stl, mask, np.array([[0, 0, 0], [199.0, 199, 199]]), 1.0, [0, 0, 1.0, 0], [0, 1])
    assert r["n_thinned"] == 2 and r["acc_count"] == 0 and math.isnan(r["acc_mean"]) and math.isnan(r["acc_median"])
    assert r["comp_count"] == 0 and math.isnan(r["comp_mean"])  # 69.3 and 80+ mm: both beyond 20


def test_visiting_order_is_seeded():
    a, b = dtu_eval.visiting_order(1000, 5), dtu_eval.visiting_order(1000, 5)
    assert (a == b).all() and sorted(a.tolist()) == list(range(1000))
    assert not (a == dtu_eval.visiting_order(1000, 6)).all()


def test_summary_is_the_mean_of_the_per_scan_means():
    s = dtu_eval.summarize([{"acc_mean": 0.3, "comp_mean": 0.2}, {"acc_mean": 0.5, "comp_mean": 0.4}])
    assert s["acc"] == pytest.approx(0.4) and s["comp"] == pytest.approx(0.3) and s["overall"] == pytest.approx(0.35)


# ---- PLY reader -----------------------------------------------------------------------------------------------------------------

def test_read_ply_round_trip_through_save_ply(tmp_path):
    rng = np.random.RandomState(0)
    xyz = rng.uniform(-500, 500, (257, 3)).astype(np.float32)
    rgb = rng.randint(0, 256, (257, 3)).astype(np.uint8)
    body = np.concatenate([xyz.view(np.uint8).reshape(257, 12), rgb], axis=1)
    path = str(tmp_path / "fused.ply")
    data_io.save_ply(path, torch.from_numpy(body))
    got = data_io.read_ply_points(path)
    assert got.dtype == np.float64 and got.shape == (257, 3)
    assert (got == xyz.astype(np.float64)).all()


def test_read_ply_extra_and_reordered_properties(tmp_path):
    n = 50
    rng = np.random.RandomState(1)
    props = [("nx", "<f4"), ("red", "u1"), ("z", "<f8"), ("alpha", "u1"), ("y", "<f4"), ("quality", "<i4"), ("x", "<f4")]
    rec = np.zeros(n, dtype=props)
    for k, _ in props:
        rec[k] = rng.uniform(0, 100, n).astype(rec[k].dtype)
    names = {"<f4": "float", "u1": "uchar", "<f8": "double", "<i4": "int"}
    header = "ply\nformat binary_little_endian 1.0\ncomment made by a test\nelement vertex %d\n" % n
    header += "".join(f"property {names[t]} {k}\n" for k, t in props)
    header += "element face 0\nproperty list uchar int vertex_indices\nend_header\n"
    path = tmp_path / "extra.ply"
    path.write_bytes(header.encode() + rec.tobytes())
    got = data_io.read_ply_points(str(path))
    want = np.stack([rec["x"].astype(np.float64), rec["y"].astype(np.float64), rec["z"]], axis=1)
    assert (got == want).all()


def test_read_ply_ascii(tmp_path):
    path = tmp_path / "a.ply"
    path.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty uchar red\nproperty float y\nproperty float x\n"
                    "property float z\nend_header\n1 2.5 -1 0.125\n2 0 0 0\n3 1e3 7 -8\n")
    assert data_io.read_ply_points(str(path)).tolist() == [[-1.0, 2.5, 0.125], [0.0, 0.0, 0.0], [7.0, 1000.0, -8.0]]


def test_read_ply_rejects_big_endian_and_junk(tmp_path):
    path = tmp_path / "be.ply"
    path.write_bytes(b"ply\nformat binary_big_endian 1.0\nelement vertex 1\nproperty float x\nproperty float y\n"
                     b"property float z\nend_header\n" + np.zeros(3, ">f4").tobytes())
    with pytest.raises(ValueError, match="binary_big_endian"):
        data_io.read_ply_points(str(path))
    junk = tmp_path / "junk.ply"
    junk.write_bytes(b"not a ply\n")
    with pytest.raises(ValueError, match="not a PLY"):
        data_io.read_ply_points(str(junk))
    noz = tmp_path / "noz.ply"
    noz.write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nend_header\n1 2\n")
    with pytest.raises(ValueError, match="lacks x, y or z"):
        data_io.read_ply_points(str(noz))


# ---- ground truth loader --------------------------------------------------------------------------------------------------------

def test_load_scan_truth_from_savemat_files(tmp_path):
    root, outputs = str(tmp_path / "MVS Data"), str(tmp_path / "outputs")
    cases = dtu_cases.write_mvs_tree(root, outputs, [4], n_stl=500, n_data=600)
    truth = dtu_eval.load_scan_truth(root, 4)
    c = cases[4]
    assert (truth["stl_points"] == c["stl"]).all()
    assert truth["obs_mask"].dtype == bool and (truth["obs_mask"] == c["obs_mask"]).all()
    assert truth["bb"].shape == (2, 3) and (truth["bb"] == c["bb"]).all()
    assert isinstance(truth["res"], float) and truth["res"] == c["res"]
    assert truth["plane"].shape == (4,) and (truth["plane"] == c["plane"]).all()
    assert (data_io.read_ply_points(os.path.join(outputs, "scan4", "fused.ply")) == c["data"]).all()


# ---- C ABI argument checks (no CUDA call is made) -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    _native.build_library()
    return _native.lib()


def test_point_cloud_abi_rejects_bad_arguments(lib):
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    bb = (ctypes.c_double * 6)(0, 0, 0, 1, 1, 1)
    assert lib.pmb200_thin_points(None, one, 10, 0.2, one, one, one, 1 << 20, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_thin_points(one, one, 10, 0.2, one, None, one, 1 << 20, None) == -1
    assert lib.pmb200_thin_points(one, one, -1, 0.2, one, one, one, 1 << 20, None) == -1
    assert lib.pmb200_thin_points(one, one, 10, 0.0, one, one, one, 1 << 20, None) == -1
    assert b"dst" in lib.pmb200_last_error()
    assert lib.pmb200_thin_points(one, one, 10, float("nan"), one, one, one, 1 << 20, None) == -1
    assert lib.pmb200_nearest_distance(None, 10, one, 10, bb, 60.0, 1.0, one, one, 1 << 20, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_nearest_distance(one, 10, one, 10, None, 60.0, 1.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_nearest_distance(one, 10, one, 10, bb, 60.0, 1.0, None, one, 1 << 20, None) == -1
    assert lib.pmb200_nearest_distance(one, 10, one, 10, bb, -1.0, 1.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_nearest_distance(one, 10, one, 10, bb, 60.0, 0.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_nearest_distance(one, 10, one, 10, bb, 60.0, 0.2, one, one, 1 << 20, None) == -1  # < 60 / 256
    assert lib.pmb200_nearest_distance(one, -5, one, 10, bb, 60.0, 1.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_thin_points_workspace_bytes(-1) == -1
    assert lib.pmb200_nearest_distance_workspace_bytes(1 << 31) == -1
