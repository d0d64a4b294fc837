"""DTU evaluation on the GPU (csrc/pm_cloud.cu through ops / dtu_eval) against the CPU oracle, oracle/dtu_oracle.py.

Fixtures are generated from seeds in this file.  Thinning must give the oracle's keep mask bit for bit for the same visiting
order; distances must agree to 1e-12 relative wherever the oracle's value is below 60 mm and be exactly 60 elsewhere
(MaxDistCP keeps values above 60 that the GPU caps, and points outside its blocks get 60); per-scan statistics agree to 1e-9."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import dtu_oracle as do
from patchmatchnet_b200 import dtu_eval, ops
from tests import dtu_cases
from tests.test_dtu_eval import BLOCK_BB, BLOCK_FROM, BLOCK_TO, _clouds

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu_thin(points, order, dst):
    rank = np.empty(len(order), dtype=np.int32)
    rank[np.asarray(order, dtype=np.int64)] = np.arange(len(order), dtype=np.int32)
    keep = ops.thin_points(torch.as_tensor(points, device=DEV), torch.as_tensor(rank, device=DEV), dst)
    return keep.cpu().numpy()


@pytest.mark.parametrize("idx", range(4), ids=["uniform", "clustered", "duplicates", "lattice"])
def test_thinning_matches_the_sequential_oracle_bit_for_bit(idx):
    name, pts, dst = _clouds()[idx]
    order = dtu_eval.visiting_order(pts.shape[0], 7 + idx)
    want = do.thin(pts, order, dst)
    got = _gpu_thin(pts, order, dst)
    assert got.dtype == bool and (got == want).all(), f"{name}: {(got != want).sum()} of {pts.shape[0]} differ"
    assert 0 < want.sum() < pts.shape[0]


def test_thinning_hand_cases_on_gpu():
    pts = np.array([[0.0, 0, 0], [0.25, 0, 0], [0.5, 0, 0], [0.75, 0, 0], [1.0, 0, 0]])
    assert _gpu_thin(pts, [1, 0, 2, 3, 4], 0.25).tolist() == [False, True, False, True, False]
    dup = np.array([[1.0, 2.0, 3.0]] * 3 + [[1.3, 2.0, 3.0]])
    assert _gpu_thin(dup, [2, 0, 1, 3], 0.25).tolist() == [False, False, True, True]
    assert _gpu_thin(np.zeros((0, 3)), [], 0.2).tolist() == []


def _check_distances(got, want):
    below = want < 60.0
    np.testing.assert_allclose(got[below], want[below], rtol=1e-12, atol=0)
    assert (got[~below] == 60.0).all()


def test_block_hand_case_on_gpu():
    got = ops.nearest_distance(torch.as_tensor(BLOCK_TO, device=DEV), torch.as_tensor(BLOCK_FROM, device=DEV), BLOCK_BB, 60.0)
    assert got.cpu().tolist() == [50.0, 60.0, 60.0, 60.0, 60.0, 60.0]


@pytest.mark.parametrize("cell", [None, 0.25, 7.0])
def test_distances_match_the_block_oracle(cell):
    """Both directions of a synthetic scan; cell = None is the default search cell, 0.25 mm (the smallest allowed) sends most
    queries on to the coarse level, 7 mm puts hundreds of points in a fine cell.  The result must not depend on it."""
    c = dtu_cases.make_scan(5, n_stl=30000, n_data=30000, outlier_frac=0.05)
    stl, data, bb = c["stl"], c["data"], c["bb"]
    for to, frm in ((stl, data), (data, stl)):
        got = ops.nearest_distance(torch.as_tensor(to, device=DEV), torch.as_tensor(frm, device=DEV), bb, 60.0, cell=cell)
        _check_distances(got.cpu().numpy(), do.max_dist_cp(to, frm, bb, 60.0))


def test_far_outliers_and_empty_to_cloud():
    rng = np.random.RandomState(2)
    to = rng.uniform(0, 20, (2000, 3))
    frm = np.concatenate([rng.uniform(0, 20, (500, 3)), rng.uniform(-500, 500, (500, 3)), [[1e7, 0, 0], [np.inf, 0, 0]]])
    bb = np.array([[-500.0, -500, -500], [500.0, 500, 500]])
    got = ops.nearest_distance(torch.as_tensor(to, device=DEV), torch.as_tensor(frm, device=DEV), bb, 60.0, cell=0.25)
    _check_distances(got.cpu().numpy(), do.max_dist_cp(to, frm, bb, 60.0))
    empty = ops.nearest_distance(torch.zeros((0, 3), dtype=torch.float64, device=DEV), torch.as_tensor(frm, device=DEV), bb)
    assert (empty.cpu().numpy() == 60.0).all()
    none = ops.nearest_distance(torch.as_tensor(to, device=DEV), torch.zeros((0, 3), dtype=torch.float64, device=DEV), bb)
    assert none.shape == (0,)


def _scan_case():
    return dtu_cases.make_scan(21, n_stl=40000, n_data=60000)


def test_evaluate_scan_matches_the_oracle():
    c = _scan_case()
    got = dtu_eval.evaluate_scan(c["data"], c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"], seed=3, device=DEV)
    order = dtu_eval.visiting_order(c["data"].shape[0], 3)
    want = do.evaluate_scan(c["data"], c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"], order)
    assert got.keys() == want.keys()
    for k in want:
        if k.endswith("count") or k.startswith("n_"):
            assert got[k] == want[k], k
        else:
            assert got[k] == pytest.approx(want[k], rel=1e-9), k
    assert 0 < got["n_thinned"] < got["n_data"] and got["acc_count"] > 0 and got["comp_count"] > 0


def test_same_seed_same_result():
    c = _scan_case()
    args = (c["data"], c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"])
    a = dtu_eval.evaluate_scan(*args, seed=9, device=DEV)
    b = dtu_eval.evaluate_scan(*args, seed=9, device=DEV)
    assert a == b
    other = dtu_eval.evaluate_scan(*args, seed=10, device=DEV)
    assert other["n_thinned"] != a["n_thinned"] or other["acc_mean"] != a["acc_mean"]


def test_command_line_on_a_synthetic_tree(tmp_path):
    root, outputs, out = str(tmp_path / "MVS Data"), str(tmp_path / "outputs"), str(tmp_path / "dtu.json")
    scans = [1, 4]
    cases = dtu_cases.write_mvs_tree(root, outputs, scans, n_stl=15000, n_data=20000)
    env = dict(os.environ, PYTHONPATH=REPO + os.pathsep + os.environ.get("PYTHONPATH", ""))
    res = subprocess.run([sys.executable, "-m", "patchmatchnet_b200.dtu_eval", "--data-path", root, "--outputs", outputs,
                          "--scans", *map(str, scans), "--seed", "2", "--json", out], cwd=str(tmp_path), env=env,
                         capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = res.stdout.strip().splitlines()
    assert lines[0].startswith("scan1: ") and lines[1].startswith("scan4: ")
    assert lines[-1].startswith("final evaluation result on 2 scans: acc.: ")
    result = json.load(open(out))
    per = {r["scan"]: r for r in result["scans"]}
    want = {}
    for s in scans:
        c = cases[s]
        want[s] = do.evaluate_scan(c["data"], c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"],
                                   dtu_eval.visiting_order(c["data"].shape[0], 2))
        for k in ("n_thinned", "acc_count", "comp_count"):
            assert per[s][k] == want[s][k]
        for k in ("acc_mean", "acc_median", "acc_var", "comp_mean", "comp_median", "comp_var"):
            assert per[s][k] == pytest.approx(want[s][k], rel=1e-9)
        assert f"acc. mean/median {want[s]['acc_mean']:.6f}/{want[s]['acc_median']:.6f}" in lines[scans.index(s)]
    acc = np.mean([want[s]["acc_mean"] for s in scans])
    comp = np.mean([want[s]["comp_mean"] for s in scans])
    assert result["final"]["overall"] == pytest.approx((acc + comp) / 2, rel=1e-9)
    assert f"acc.: {acc:.6f}, comp.: {comp:.6f}, overall: {(acc + comp) / 2:.6f}" in lines[-1]
    assert not math.isnan(result["final"]["overall"])
