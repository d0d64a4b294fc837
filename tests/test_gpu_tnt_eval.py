"""Tanks and Temples evaluation on the GPU (csrc/pm_cloud.cu through ops / tnt_eval) against the CPU oracle,
tests/tnt_oracle.py.

Crop masks and transformed points must be the oracle's bits; down-sampled voxel sets the oracle's, with means within 1e-12
relative; correspondences the oracle's indices (ties included); ICP the oracle's iteration and correspondence counts with
the transformation within 1e-9 per element; evaluate_scene the oracle's counts, hence its precision, recall and F-score."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import ops, tnt_eval
from tests import tnt_cases
from tests import tnt_oracle as to
from tests.test_tnt_eval import HAND_POINTS, HAND_WANT, SQUARE

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _d(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=DEV)


def _gpu_crop(points, cv, t=None):
    out, keep = ops.crop_points(_d(points), cv["orthogonal_axis"], cv["axis_min"], cv["axis_max"], cv["polygon"], t)
    return out.cpu().numpy(), keep.cpu().numpy()


def test_crop_hand_cases_on_gpu():
    for axis, perm in ((2, [0, 1, 2]), (1, [0, 2, 1]), (0, [1, 2, 0])):
        # (u, v) = (x, y) for Z, (x, z) for Y, (y, z) for X: move the hand case's columns there
        pts = np.zeros_like(HAND_POINTS)
        poly = np.zeros_like(SQUARE["polygon"])
        pts[:, perm] = HAND_POINTS
        poly[:, perm] = SQUARE["polygon"]
        cv = dict(SQUARE, orthogonal_axis=axis, polygon=poly)
        out, keep = _gpu_crop(pts, cv)
        assert keep.astype(bool).tolist() == HAND_WANT, axis
        assert (out == pts).all()


def test_crop_matches_the_oracle_bit_for_bit():
    rng = np.random.RandomState(4)
    cv = tnt_cases.crop_volume()
    pts = tnt_cases.OFFSET + rng.uniform(-1.2, 1.2, (200000, 3))
    pts[:1000, :2] = cv["polygon"][rng.randint(0, 6, 1000), :2]  # on the vertices
    t = tnt_cases.similarity(1.0003, [1, 1, 0], 1e-4, [1e-3, 0, -2e-3])
    out, keep = _gpu_crop(pts, cv, t)
    moved = to.transform(pts, t)
    assert (out == moved).all()
    want = to.crop(moved, cv)
    assert (keep.astype(bool) == want).all(), (keep.astype(bool) != want).sum()
    assert 0 < want.sum() < len(pts)


def _voxel_clouds():
    rng = np.random.RandomState(5)
    surf = tnt_cases.surface(rng, 120000)
    dup = np.concatenate([surf[:5000]] * 3)
    far = np.concatenate([rng.uniform(0, 1, (3000, 3)), rng.uniform(0, 1, (3000, 3)) + 4.0e5])  # 2^39 voxels: split key
    return [("surface", surf, 0.01), ("duplicates", dup, 0.02), ("split_key", far, 1e-3)]


@pytest.mark.parametrize("idx", range(3), ids=["surface", "duplicates", "split_key"])
def test_voxel_downsample_matches_the_oracle(idx):
    name, pts, s = _voxel_clouds()[idx]
    want = to.voxel_downsample(pts, s)
    got = ops.voxel_downsample(_d(pts), s).cpu().numpy()
    assert got.shape == want.shape, name
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    again = ops.voxel_downsample(_d(pts), s).cpu().numpy()
    assert (again == got).all()


def test_correspondences_match_the_oracle():
    rng = np.random.RandomState(6)
    tgt = tnt_cases.surface(rng, 40000)
    src = tnt_cases.surface(rng, 30000) + rng.normal(0, 0.01, (30000, 3))
    for r, cell in ((0.05, None), (0.4, None), (0.05, 0.05 / 256)):
        res = ops.icp(_d(src), _d(tgt), r, max_iteration=0, cell=cell, return_correspondences=True)
        got = res["correspondence_set"].cpu().numpy()
        want, d2 = to.correspondences(src, tgt, r)
        assert (got == want).all(), (r, cell, (got != want).sum())
        ok = want >= 0
        assert res["history"][0][0] == ok.sum() and res["history"][0][1] == pytest.approx(d2[ok].sum(), rel=1e-12)
        assert res["iterations"] == 0


def test_correspondence_ties_go_to_the_smallest_index():
    g = np.arange(-3, 4, dtype=np.float64)
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    perm = np.random.RandomState(7).permutation(len(lattice))
    tgt = lattice[perm]
    src = np.array([[0.5, 0.0, 0.0], [0.5, 0.5, 0.0], [0.5, 0.5, 0.5], [2.5, -1.5, 0.0], [0.0, 0.0, 0.0], [9.0, 9.0, 9.0]])
    res = ops.icp(_d(src), _d(tgt), 1.0, max_iteration=0, return_correspondences=True)
    got = res["correspondence_set"].cpu().numpy()
    want, _ = to.correspondences(src, tgt, 1.0)
    assert got.tolist() == want.tolist()
    # every tied candidate is at the same distance, and the pick is the smallest index among them
    for i in range(4):
        d = np.linalg.norm(tgt - src[i], axis=1)
        assert want[i] == np.nonzero(d == d.min())[0].min() and (d == d.min()).sum() >= 2
    assert want[5] == -1


def _down_scene(seed=100):
    c = tnt_cases.make_scene(seed)
    s = tnt_cases.apply(c["S"], c["rec"])
    s[:, :2] += 0.01  # start ICP away from the injected similarity
    s = to.voxel_downsample(s[to.crop(s, c["crop"])], c["tau"])
    g = to.voxel_downsample(c["gt"][to.crop(c["gt"], c["crop"])], c["tau"])
    return c, s, g


def test_icp_matches_the_oracle():
    c, s, g = _down_scene()
    r = 20 * c["tau"]
    want = to.icp(s, g, r, max_iteration=20)
    got = ops.icp(_d(s), _d(g), r, max_iteration=20)
    assert got["iterations"] == want["iterations"] and 1 < got["iterations"]
    assert [h[0] for h in got["history"]] == [h[0] for h in want["history"]]
    np.testing.assert_allclose([h[1] for h in got["history"]], [h[1] for h in want["history"]], rtol=1e-9)
    np.testing.assert_allclose(got["transformation"], want["transformation"], atol=1e-9, rtol=0)
    assert got["fitness"] == want["fitness"] and got["inlier_rmse"] == pytest.approx(want["inlier_rmse"], rel=1e-9)
    again = ops.icp(_d(s), _d(g), r, max_iteration=20)
    assert (again["transformation"] == got["transformation"]).all() and again["history"] == got["history"]


def _check_scene(got, want):
    for k in ("n_source_scored", "n_gt_scored", "precision_count", "recall_count"):
        assert got[k] == want[k], k
    assert got["precision"] == want["precision"] and got["recall"] == want["recall"] and got["fscore"] == want["fscore"]
    assert (np.asarray(got["cum_precision"]) == want["cum_precision"]).all()
    assert (np.asarray(got["cum_recall"]) == want["cum_recall"]).all()
    for a, b in zip(got["rounds"], want["rounds"]):
        assert (a["n_source"], a["n_target"], a["iterations"], a["correspondences"]) == \
               (b["n_source"], b["n_target"], b["iterations"], b["correspondences"])
        np.testing.assert_allclose(a["transformation"], b["transformation"], atol=1e-9, rtol=0)
    np.testing.assert_allclose(got["transformation"], want["transformation"], atol=1e-9, rtol=0)


def test_evaluate_scene_matches_the_oracle_and_recovers_the_similarity():
    c = tnt_cases.make_scene(101, n_gt=40000, n_rec=30000)
    tgt = tnt_cases.apply(c["trans"], c["log"][:, :3, 3])
    centres = tnt_cases.apply(np.linalg.inv(c["S"]), tgt)
    init = tnt_eval.trajectory_alignment(centres, tgt, seed=0, iterations=2000)["transformation"]
    np.testing.assert_allclose(init, c["S"], atol=1e-9)
    got = tnt_eval.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"], device=DEV)
    want = to.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"])
    _check_scene(got, want)
    moved = np.linalg.norm(tnt_cases.apply(np.asarray(got["transformation"]), c["rec"]) - tnt_cases.apply(c["S"], c["rec"]), axis=1)
    assert moved.mean() < c["tau"] / 2 and moved.max() < c["tau"]
    assert 0.5 < got["precision"] <= 1 and 0.5 < got["recall"] < 1  # the missed strip costs recall
    again = tnt_eval.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"], device=DEV)
    assert again == got


def test_clouds_above_2_24_points():
    """Index widths: 2^24 + 2^20 points.  Voxels: a lattice where each voxel holds exactly 4 points, so the count and every
    mean are known; crop and correspondences: a sampled subset against the oracle."""
    n_cells = (2 ** 24 + 2 ** 20) // 4
    side = int(np.ceil(n_cells ** (1 / 3)))
    k = np.arange(n_cells, dtype=np.int64)
    cell = np.stack([k % side, (k // side) % side, k // (side * side)], 1).astype(np.float64)
    offs = np.array([[0.1, 0.1, 0.1], [0.3, 0.2, 0.1], [0.1, 0.4, 0.3], [0.2, 0.1, 0.35]])
    pts = (cell[:, None, :] + 0.5 + offs[None]).reshape(-1, 3) + 100.0  # min bound 100.6: origin 100.1, cells stay aligned
    n = pts.shape[0]
    assert n > 2 ** 24
    dp = _d(pts)
    down = ops.voxel_downsample(dp, 1.0)
    assert down.shape[0] == n_cells
    pick = np.random.RandomState(8).randint(0, n_cells, 2000)
    want = cell[pick] + 0.5 + offs.mean(0) + 100.0
    got = down.cpu().numpy()
    order = np.lexsort((cell[:, 2], cell[:, 1], cell[:, 0]))  # ascending (x, y, z) voxel order
    np.testing.assert_allclose(got[np.argsort(order)][pick], want, rtol=1e-12)
    cv = {"orthogonal_axis": 2, "axis_min": 100.0, "axis_max": 100.0 + side / 2,
          "polygon": np.array([[99.0, 99.0, 0], [100.0 + side, 99.0, 0], [99.0, 100.0 + side, 0]])}
    _, keep = ops.crop_points(dp, cv["orthogonal_axis"], cv["axis_min"], cv["axis_max"], cv["polygon"])
    keep = keep.cpu().numpy()
    sub = np.random.RandomState(9).randint(0, n, 20000)
    assert (keep[sub] == to.crop(pts[sub], cv)).all() and 0 < keep.sum() < n
    tgt = pts[::64] + 0.01
    res = ops.icp(dp, _d(tgt), 0.5, max_iteration=0, return_correspondences=True)
    corr = res["correspondence_set"].cpu().numpy()
    assert res["history"][0][0] == (corr >= 0).sum()
    want_idx, _ = to.correspondences(pts[sub], tgt, 0.5)
    assert (corr[sub] == want_idx).all()


def test_command_line_on_a_synthetic_tree(tmp_path):
    root = str(tmp_path)
    cases = tnt_cases.write_tree(root, ["Alpha"], n_gt=30000, n_rec=25000)
    out = str(tmp_path / "tnt.json")
    env = dict(os.environ, PYTHONPATH=REPO + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run([sys.executable, "-m", "patchmatchnet_b200.tnt_eval", "--gt-path", os.path.join(root, "gt"),
                          "--outputs", os.path.join(root, "outputs"), "--input", os.path.join(root, "scenes"),
                          "--scenes", "Alpha", "--tau", "0.02", "--seed", "3", "--json", out], cwd=root, env=env,
                         capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout + res.stderr
    line = res.stdout.strip().splitlines()[0]
    assert line.startswith("Alpha: precision ")
    r = json.load(open(out))["scenes"][0]
    c = cases["Alpha"]
    assert r["alignment"]["inliers"] == 40
    np.testing.assert_allclose(r["init_transformation"], c["S"], atol=1e-4)  # from the float32 cam files
    want = to.evaluate_scene(c["rec"], c["gt"], c["crop"], np.asarray(r["init_transformation"]), 0.02)
    _check_scene(r, want)
    assert f"f-score {want['fscore']:.4f}" in line
    assert r["n_source_cropped"] >= r["n_source_scored"] > 0 and r["n_gt_cropped"] >= r["n_gt_scored"] > 0
    bad = subprocess.run([sys.executable, "-m", "patchmatchnet_b200.tnt_eval", "--gt-path", os.path.join(root, "gt"),
                          "--scenes", "Alpha"], cwd=root, env=env, capture_output=True, text=True, timeout=300)
    assert bad.returncode != 0 and "--tau" in bad.stderr
