"""Tanks and Temples evaluation without a GPU: the file readers, the CPU oracle (tests/tnt_oracle.py) on hand cases, the
host-side pieces of patchmatchnet_b200/tnt_eval.py (Umeyama, RANSAC, histogram edges, F-score rule) and the argument checks
of the new point-cloud C ABI calls."""
import ctypes
import json
import math

import numpy as np
import pytest

from patchmatchnet_b200 import _native, ops, tnt_eval
from tests import tnt_cases
from tests import tnt_oracle as to


# ---- readers --------------------------------------------------------------------------------------------------------------

def test_readers_on_a_written_tree(tmp_path):
    cases = tnt_cases.write_tree(str(tmp_path), ["Synth"], n_gt=2000, n_rec=1500)
    c = cases["Synth"]
    truth = tnt_eval.load_scene_truth(str(tmp_path / "gt"), "Synth")
    assert (truth["points"] == c["gt"]).all()
    assert truth["crop"]["orthogonal_axis"] == 2 and truth["crop"]["axis_min"] == c["crop"]["axis_min"]
    assert (truth["crop"]["polygon"] == c["crop"]["polygon"]).all()
    assert (truth["trans"] == c["trans"]).all()
    assert truth["log"].shape == (40, 4, 4) and (truth["log"] == c["log"]).all()
    centres = tnt_eval.camera_centres(str(tmp_path / "scenes" / "Synth"))
    want = tnt_cases.apply(np.linalg.inv(c["S"]), tnt_cases.apply(c["trans"], c["log"][:, :3, 3]))
    np.testing.assert_allclose(centres, want, atol=1e-4)  # the cam files hold float32 extrinsics


def test_crop_json_axes_and_rejection(tmp_path):
    p = tmp_path / "c.json"
    for name, axis in (("X", 0), ("y", 1), ("Z", 2)):
        p.write_text(json.dumps({"axis_min": -1, "axis_max": 2.5, "bounding_polygon": [[0, 0, 0], [1, 0, 0], [1, 1, 0]],
                                 "orthogonal_axis": name}))
        c = tnt_eval.read_crop_json(str(p))
        assert c["orthogonal_axis"] == axis and c["axis_min"] == -1.0 and c["axis_max"] == 2.5 and c["polygon"].shape == (3, 3)
    p.write_text(json.dumps({"axis_min": 0, "axis_max": 1, "bounding_polygon": [], "orthogonal_axis": "W"}))
    with pytest.raises(ValueError, match="X, Y or Z"):
        tnt_eval.read_crop_json(str(p))


def test_log_and_trans_readers(tmp_path):
    log = tmp_path / "a.log"
    log.write_text("0 0 0\n1 0 0 2\n0 1 0 3\n0 0 1 4\n0 0 0 1\n\n1 1 0\n2 0 0 5\n0 2 0 6\n0 0 2 7\n0 0 0 1\n")
    m = tnt_eval.read_log(str(log))
    assert m.shape == (2, 4, 4) and m[0, :3, 3].tolist() == [2, 3, 4] and m[1, 0, 0] == 2.0
    log.write_text("0 0 0\n1 0 0 2\n")
    with pytest.raises(ValueError, match="5 lines per frame"):
        tnt_eval.read_log(str(log))
    tr = tmp_path / "t.txt"
    tr.write_text("1 0 0 0.5\n0 1 0 0\n0 0 1 0\n0 0 0 1\n")
    assert tnt_eval.read_trans(str(tr))[0, 3] == 0.5
    tr.write_text("1 0 0\n0 1 0\n")
    with pytest.raises(ValueError, match="4 x 4"):
        tnt_eval.read_trans(str(tr))


# ---- crop rule ----------------------------------------------------------------------------------------------------------------

SQUARE = {"orthogonal_axis": 2, "axis_min": -1.0, "axis_max": 1.0,
          "polygon": np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [2.0, 2.0, 0.0], [0.0, 2.0, 0.0]])}
HAND_POINTS = np.array([
    [1.0, 1.0, 0.0],    # interior
    [0.0, 0.0, 0.0],    # vertex (0,0): v = 0 is not > v of the edges meeting there -> no crossing -> out
    [2.0, 2.0, 0.0],    # vertex (2,2): the left edge crosses at u = 0 < 2 and the right one at u = 2 (not < 2) -> in
    [0.0, 2.0, 0.0],    # vertex (0,2): crossings at u = 0 (not < 0) and 2 -> out
    [1.0, 0.0, 0.0],    # bottom edge (horizontal): v = 0 crosses nothing -> out
    [1.0, 2.0, 0.0],    # top edge (horizontal): v = 2 crosses the sides at 0 (< 1) and 2 -> in
    [0.0, 1.0, 0.0],    # left edge: crossing at 0 is not < 0 -> out
    [2.0, 1.0, 0.0],    # right edge: 0 < 2 counts, 2 does not -> in
    [1.0, 1.0, 1.0],    # on axis_max: inclusive -> in
    [1.0, 1.0, -1.0],   # on axis_min -> in
    [1.0, 1.0, 1.0 + 2 ** -40],  # just above axis_max -> out
    [3.0, 1.0, 0.0],    # right of the square: two crossings -> out
])
HAND_WANT = [True, False, True, False, False, True, False, True, True, True, False, False]


def test_crop_hand_cases_on_the_oracle():
    assert to.crop(HAND_POINTS, SQUARE).tolist() == HAND_WANT
    # the same points with Y orthogonal: (u, v) = (x, z)
    yv = dict(SQUARE, orthogonal_axis=1, polygon=SQUARE["polygon"][:, [0, 2, 1]])
    assert to.crop(HAND_POINTS[:, [0, 2, 1]], yv).tolist() == HAND_WANT


# ---- voxel and uniform down-sampling ----------------------------------------------------------------------------------------

def test_voxel_means_and_origin_rule():
    # min bound (0,0,0), s = 1: origin -0.5, so x in [-0.5, 0.5) is voxel 0 and [0.5, 1.5) voxel 1
    p = np.array([[0.0, 0, 0], [0.4, 0, 0], [0.5, 0, 0], [1.4, 0, 0], [0.2, 0.6, 0], [0.1, 0, 0]])
    got = to.voxel_downsample(p, 1.0)
    want = [[(0.0 + 0.4 + 0.1) / 3, 0, 0], [0.2, 0.6, 0], [(0.5 + 1.4) / 2, 0, 0]]  # voxels (0,0,0), (0,1,0), (1,0,0)
    np.testing.assert_allclose(got, want, rtol=1e-15)
    # the origin follows the cloud's own min bound: shifting every point by 0.3 shifts the means, not the grouping
    np.testing.assert_allclose(to.voxel_downsample(p + 0.3, 1.0), np.asarray(want) + 0.3, rtol=1e-14)
    assert to.voxel_downsample(np.zeros((0, 3)), 1.0).shape == (0, 3)


def test_uniform_downsample_rule():
    import torch

    p = np.arange(30).reshape(10, 3)
    assert to.uniform_downsample(p, 10) is p  # n <= max: unchanged
    assert to.uniform_downsample(p, 4)[:, 0].tolist() == [0, 6, 12, 18, 24]  # k = round(2.5) = 2 (half to even)
    assert to.uniform_downsample(p, 3)[:, 0].tolist() == [0, 9, 18, 27]      # k = round(3.33) = 3
    assert to.uniform_downsample(p, 2)[:, 0].tolist() == [0, 15]           # k = round(5) = 5: rows 0, 5
    for m in (2, 3, 4, 10):
        assert tnt_eval.uniform_downsample(torch.as_tensor(p), m).tolist() == to.uniform_downsample(p, m).tolist()


# ---- Umeyama, ICP, RANSAC ---------------------------------------------------------------------------------------------------

def test_umeyama_recovers_a_known_similarity():
    rng = np.random.RandomState(0)
    src = rng.uniform(-5, 5, (50, 3)) + [40.0, -20.0, 7.0]
    s = tnt_cases.similarity(2.3, [1, 2, 3], 1.1, [5.0, -7.0, 0.25])
    dst = tnt_cases.apply(s, src)
    np.testing.assert_allclose(to.umeyama(src, dst), s, atol=1e-12, rtol=0)
    np.testing.assert_allclose(tnt_eval.umeyama(src, dst), s, atol=1e-12, rtol=0)
    # the moments path of ops.icp, relative to an origin near the points
    o = src.mean(0) + 0.5
    p, q = src - o, dst - o
    m = np.concatenate([[len(p), 0.0], p.sum(0), q.sum(0), (q[:, :, None] * p[:, None, :]).sum(0).reshape(9), [(p * p).sum()]])
    rel = ops.umeyama_from_moments(m)
    world = np.eye(4)
    world[:3, :3] = rel[:3, :3]
    world[:3, 3] = rel[:3, 3] + o - rel[:3, :3] @ o
    np.testing.assert_allclose(world, s, atol=1e-11, rtol=0)
    assert (ops.umeyama_from_moments(np.zeros(18)) == np.eye(4)).all()


def test_umeyama_reflection_gives_a_rotation():
    rng = np.random.RandomState(1)
    src = rng.uniform(-1, 1, (30, 3))
    dst = src * [1.0, 1.0, -1.0] * 1.5  # a reflection: the best proper similarity flips the smallest singular direction
    for u in (to.umeyama(src, dst), tnt_eval.umeyama(src, dst)):
        r = u[:3, :3] / np.cbrt(np.linalg.det(u[:3, :3]))
        assert np.linalg.det(u[:3, :3]) > 0
        np.testing.assert_allclose(r @ r.T, np.eye(3), atol=1e-12)
    np.testing.assert_allclose(to.umeyama(src, dst), tnt_eval.umeyama(src, dst), atol=1e-12)


def test_oracle_icp_converges_and_stops():
    rng = np.random.RandomState(2)
    tgt = tnt_cases.surface(rng, 3000)
    shift = np.eye(4)
    shift[:3, 3] = tnt_cases.OFFSET
    s = shift @ tnt_cases.similarity(1.01, [0, 0, 1], 0.02, [0.01, -0.02, 0.005]) @ np.linalg.inv(shift)  # about the surface
    src = tnt_cases.apply(np.linalg.inv(s), tgt[:2000])
    r = to.icp(src, tgt, 0.2, max_iteration=50)
    np.testing.assert_allclose(r["transformation"], s, atol=1e-6)
    assert r["fitness"] == 1.0 and r["iterations"] < 50 and r["inlier_rmse"] < 1e-6
    one = to.icp(src, tgt, 0.2, max_iteration=1)
    assert one["iterations"] == 1 and len(one["history"]) == 2
    none = to.icp(src + 100.0, tgt, 0.2, max_iteration=5)  # no correspondences: identity updates, converged at once
    assert none["fitness"] == 0.0 and none["iterations"] == 1 and (none["transformation"] == np.eye(4)).all()


def test_oracle_correspondence_tie_goes_to_the_smallest_index():
    tgt = np.array([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [5.0, 0, 0]])
    idx, d2 = to.correspondences(np.array([[0.0, 0, 0], [4.5, 0, 0], [9.0, 0, 0]]), tgt, 1.0)
    assert idx.tolist() == [0, 3, -1] and d2[0] == 1.0 and d2[1] == 0.25


def test_ransac_is_seeded_and_matches_the_loop():
    c = tnt_cases.make_scene(3, n_gt=10, n_rec=10)
    src = tnt_cases.apply(np.linalg.inv(c["S"]), tnt_cases.apply(c["trans"], c["log"][:, :3, 3]))
    tgt = tnt_cases.apply(c["trans"], c["log"][:, :3, 3])
    tgt = tgt + np.random.RandomState(5).normal(0, 0.01, tgt.shape)  # noisy centres: RMSE ties are not roundoff
    src[:5] += 3.0  # five outlier cameras
    a = tnt_eval.trajectory_alignment(src, tgt, seed=4, iterations=3000, chunk=700)
    b = tnt_eval.trajectory_alignment(src, tgt, seed=4, iterations=3000, chunk=3000)
    assert a["best_sample"] == b["best_sample"] and (a["transformation"] == b["transformation"]).all()
    assert a["inliers"] == len(src) - 5
    np.testing.assert_allclose(a["transformation"], c["S"], atol=0.05)
    samples = tnt_eval.ransac_samples(len(src), 3000, 4)
    assert all(len(set(r)) == 6 for r in samples.tolist()) and samples.min() >= 0 and samples.max() < len(src)
    want, best = to.ransac(src, tgt, samples)
    assert best[2] == a["best_sample"] and best[0] == a["inliers"]
    np.testing.assert_allclose(a["transformation"], want, atol=1e-12)
    with pytest.raises(ValueError, match="--init trans"):
        tnt_eval.trajectory_alignment(src, tgt[:-1])


# ---- scoring rules ----------------------------------------------------------------------------------------------------------

def test_fscore_edge_cases_on_the_oracle():
    cv = dict(SQUARE)
    gt = np.array([[1.0, 1.0, 0.0], [1.5, 1.0, 0.0]])
    far = np.array([[1.0, 1.9, 0.0]])
    r = to.score(far, gt, cv, np.eye(4), 0.01)  # nothing within tau: P + R = 0
    assert r["precision"] == 0 and r["recall"] == 0 and r["fscore"] == 0
    r = to.score(np.zeros((0, 3)), gt, cv, np.eye(4), 0.01)  # empty reconstruction
    assert r["n_source_scored"] == 0 and r["fscore"] == 0
    r = to.score(gt[:1], gt, cv, np.eye(4), 0.01)
    assert r["precision"] == 1.0 and r["recall"] == 0.5 and r["fscore"] == pytest.approx(2 / 3, rel=1e-15)


def test_histogram_edges_follow_numpy():
    import torch

    for tau in (0.003, 0.01, 0.025):
        edges = tnt_eval.histogram_edges(tau, "cpu")
        assert (edges.numpy() == np.arange(0, 5 * tau, tau / 100)).all()
        d = np.concatenate([np.random.RandomState(0).uniform(0, 6 * tau, 2000), edges.numpy()[[0, 7, -1]], [5 * tau]])
        got = tnt_eval.cumulative_histogram(torch.as_tensor(d), edges)
        want = np.cumsum(np.histogram(d, np.arange(0, 5 * tau, tau / 100))[0]) / len(d)
        assert (got == want).all()


def test_known_tau_table_and_cpu_refusal():
    assert tnt_eval.SCENE_TAU["Ignatius"] == 0.003 and tnt_eval.SCENE_TAU["Church"] == 0.025 and len(tnt_eval.SCENE_TAU) == 7
    with pytest.raises(RuntimeError, match="CUDA"):
        tnt_eval.evaluate_scene(np.zeros((1, 3)), np.zeros((1, 3)), SQUARE, np.eye(4), 0.01, device="cpu")


# ---- C ABI argument checks (no CUDA call is made) -------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    _native.build_library()
    return _native.lib()


def test_tnt_abi_rejects_bad_arguments(lib):
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    eye = (ctypes.c_double * 16)(*np.eye(4).reshape(16).tolist())
    bad = (ctypes.c_double * 16)(*(np.eye(4).reshape(16).tolist()[:15] + [2.0]))
    nan = (ctypes.c_double * 16)(*([float("nan")] + np.eye(4).reshape(16).tolist()[1:]))
    poly = (ctypes.c_double * (3 * 200))()
    o3 = (ctypes.c_double * 3)(0, 0, 0)
    assert lib.pmb200_crop_polygon(None, 10, eye, 2, 0.0, 1.0, poly, 4, one, one, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_crop_polygon(one, 10, eye, 3, 0.0, 1.0, poly, 4, one, one, None) == -1
    assert b"orthogonal_axis" in lib.pmb200_last_error()
    assert lib.pmb200_crop_polygon(one, 10, eye, 2, 0.0, 1.0, poly, 129, one, one, None) == -1
    assert b"128" in lib.pmb200_last_error()
    assert lib.pmb200_crop_polygon(one, 10, bad, 2, 0.0, 1.0, poly, 4, one, one, None) == -1
    assert b"last row" in lib.pmb200_last_error()
    assert lib.pmb200_crop_polygon(one, 10, nan, 2, 0.0, 1.0, poly, 4, one, one, None) == -1
    assert lib.pmb200_crop_polygon(one, -1, eye, 2, 0.0, 1.0, poly, 4, one, one, None) == -1
    bounds = (ctypes.c_double * 6)(0, 0, 0, 1, 1, 1)
    assert lib.pmb200_voxel_downsample(one, 10, bounds, 0.0, one, one, one, 1 << 20, None) == -1
    assert b"voxel_size" in lib.pmb200_last_error()
    assert lib.pmb200_voxel_downsample(one, 10, bounds, 1e-12, one, one, one, 1 << 20, None) == -1
    assert b"int32" in lib.pmb200_last_error()
    flipped = (ctypes.c_double * 6)(0, 0, 0, 1, -1, 1)
    assert lib.pmb200_voxel_downsample(one, 10, flipped, 0.1, one, one, one, 1 << 20, None) == -1
    assert b"bounds" in lib.pmb200_last_error()
    assert lib.pmb200_voxel_downsample(one, 10, bounds, 0.1, one, None, one, 1 << 20, None) == -1
    assert lib.pmb200_voxel_downsample_workspace_bytes(-1) == -1
    assert lib.pmb200_icp_target(None, 10, 1.0, one, 1 << 20, None) == -1
    assert lib.pmb200_icp_target(one, 10, 0.0, one, 1 << 20, None) == -1
    assert b"cell" in lib.pmb200_last_error()
    assert lib.pmb200_icp_target_workspace_bytes(1 << 31) == -1
    assert lib.pmb200_icp_query(one, 10, eye, o3, 1.0, one, 10, 1.0, None, None, one, 1 << 20, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_icp_query(one, 10, eye, o3, 1.0, one, 10, 1.0 / 512, None, one, one, 1 << 20, None) == -1
    assert b"max_dist / 256" in lib.pmb200_last_error()
    assert lib.pmb200_icp_query(one, 10, bad, o3, 1.0, one, 10, 1.0, None, one, one, 1 << 20, None) == -1
    assert b"last row" in lib.pmb200_last_error()
    inf3 = (ctypes.c_double * 3)(0, math.inf, 0)
    assert lib.pmb200_icp_query(one, 10, eye, inf3, 1.0, one, 10, 1.0, None, one, one, 1 << 20, None) == -1
    assert b"origin" in lib.pmb200_last_error()
    assert lib.pmb200_icp_query(one, 10, eye, o3, 1.0, one, 10, 1.0, None, one, one, 8, None) == -1
    assert b"workspace" in lib.pmb200_last_error()
    assert lib.pmb200_icp_query_workspace_bytes(-3) == -1
