"""ETH3D evaluation on the GPU (csrc/pm_scan.cu through ops / eth3d_eval) against the CPU oracle, tests/eth3d_oracle.py.

beam_observed must equal the oracle's brute force bit for bit (room queries, queries jittered around the cone's boundary, the
azimuth seam and the poles of the index, queries within r0 of a scanner, an empty scan); voxel_score's counts must be exact
and its sums within 1e-12 relative; evaluate_scene must reproduce the oracle's counts and scores at all six tolerances, bit
for bit on a rerun; the command's JSON must be evaluate_scene's; clouds above 2^24 points must complete with their designed
counts; colmap_input --sparse-folder must write what the same model under sparse/ gives."""
import json
import math
import os
import shutil

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import colmap_input as ci
from patchmatchnet_b200 import data_io, eth3d_eval, ops
from tests import colmap_cases as cc
from tests import eth3d_cases as ec
from tests import eth3d_oracle as eo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
R0, T = 0.001125, math.tan(math.radians(0.011))


def _d(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=DEV)


def _scene_scans(c):
    """GPU-transformed scene-frame scans (ops.crop_points' transform) and the oracle's, which must be the same bits."""
    out = []
    for s in c["scans"]:
        moved, _ = ops.crop_points(_d(s["points"]), 2, -math.inf, math.inf, np.zeros((0, 3)), s["matrix"])
        want = eo.transform(s["points"], s["matrix"])
        assert (moved.cpu().numpy() == want).all()
        out.append((want, s["matrix"][:3, 3].copy()))
    return out


def _check_beams(queries, scan, origin, r0=R0, t=T):
    got = ops.beam_observed(_d(queries), _d(scan), origin, r0, t).cpu().numpy().astype(bool)
    want = eo.beam_observed(queries, scan, origin, r0, t)
    assert (got == want).all(), f"{(got != want).sum()} of {len(want)} queries differ"
    return want


def _boundary_queries(rng, scan, origin, k, r0=R0, t=T):
    """Queries within +-1e-9 r of the free beam's boundary of random scan points: on the cone's side, near p (t' = a.a) and
    near the scanner (t' = 0)."""
    p = scan[rng.randint(scan.shape[0], size=k)] - origin
    r = np.linalg.norm(p, axis=1, keepdims=True)
    ah = p / r
    u = np.cross(ah, rng.normal(size=(k, 3)))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    jit = rng.uniform(-1e-9, 1e-9, (k, 1)) * r
    lam = rng.uniform(0.0, 1.0, (k, 1)) * r
    side = lam * ah + (r0 + lam * t + jit) * u
    near_p = (r + jit) * ah + rng.uniform(0, 0.5, (k, 1)) * (r0 + r * t) * u
    near_o = jit * ah + rng.uniform(0, 0.5, (k, 1)) * r0 * u
    return origin + np.concatenate([side, near_p, near_o])


def test_beam_observed_on_the_room_and_its_boundaries():
    c = ec.make_scene(11, n_az=160, n_el=70, n_surface=1500, n_outliers=150, n_hidden=60)
    rng = np.random.RandomState(12)
    total = 0
    for scan, origin in _scene_scans(c):
        want = _check_beams(c["rec"], scan, origin)
        total += want.sum()
        b = _boundary_queries(rng, scan, origin, 1500)
        want = _check_beams(b, scan, origin)
        assert 0.2 < want.mean() < 0.8  # both sides of the boundaries are present
    assert total > 0


def test_beam_observed_at_the_seam_and_the_poles():
    rng = np.random.RandomState(13)
    origin = np.array([0.3, -0.2, 0.1])
    dirs = []
    for az in (math.pi, -math.pi, math.pi - 1e-12):  # the azimuth seam: atan2 gives +pi or -pi on either side
        el = rng.uniform(-1.2, 1.2, 400)
        a = az + rng.uniform(-3e-3, 3e-3, 400)
        dirs.append(np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], 1))
    for pole in (1.0, -1.0):  # the poles: every azimuth meets there
        v = np.stack([rng.uniform(-3e-3, 3e-3, 600), rng.uniform(-3e-3, 3e-3, 600), np.full(600, pole)], 1)
        dirs.append(v / np.linalg.norm(v, axis=1, keepdims=True))
    d = np.concatenate(dirs)
    scan = origin + d * rng.uniform(2, 6, (d.shape[0], 1))
    scan[:40] = scan[:40] * [1, 0, 1] + [0, origin[1], 0]  # exactly on the seam's half-plane y = o_y, x < o_x
    b = _boundary_queries(rng, scan, origin, 1000)
    jittered = origin + (scan[rng.randint(scan.shape[0], size=3000)] - origin) * rng.uniform(0.01, 1.0, (3000, 1)) + \
        rng.normal(0, 2e-3, (3000, 3))
    want = _check_beams(np.concatenate([b, jittered]), scan, origin)
    assert 0.1 < want.mean() < 0.9
    for r0, t in ((0.05, 0.02), (0.0, 0.0)):  # a wide beam that spans many bins, and a zero-width one
        _check_beams(jittered, scan, origin, r0, t)


def test_beam_observed_near_the_scanner_and_on_an_empty_scan():
    c = ec.make_scene(14, n_az=120, n_el=50, n_surface=10, n_outliers=0, n_hidden=0)
    scan, origin = _scene_scans(c)[0]
    rng = np.random.RandomState(15)
    v = rng.normal(size=(2000, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    q = origin + v * rng.uniform(0, 1.0, (2000, 1)) * R0
    q[:5] = origin  # b = 0: in no beam
    want = _check_beams(q, scan, origin)
    assert want.mean() > 0.5 and not want[:5].any()
    out = torch.ones(2000, dtype=torch.uint8, device=DEV)
    out[::2] = 0
    before = out.clone()
    ops.beam_observed(_d(q), _d(np.zeros((0, 3))), origin, R0, T, out)
    assert torch.equal(out, before)
    # the mask: masked-out queries keep their value, the others are ORed
    mask = torch.zeros(2000, dtype=torch.bool, device=DEV)
    mask[:1000] = True
    out = torch.zeros(2000, dtype=torch.uint8, device=DEV)
    ops.beam_observed(_d(q), _d(scan), origin, R0, T, out, mask)
    got = out.cpu().numpy().astype(bool)
    assert (got[:1000] == want[:1000]).all() and not got[1000:].any()


def test_voxel_score_matches_the_oracle():
    rng = np.random.RandomState(16)
    n = 300000
    pts = rng.uniform(-3, 5, (n, 3))
    pts[:1000] = np.floor(pts[:1000] / 0.05) * 0.05  # on voxel faces
    d = rng.exponential(0.05, n)
    obs = rng.rand(n) < 0.4
    for tau in eo.TOLERANCES:
        for o in (obs, None):
            got = ops.voxel_score(_d(pts), _d(d), tau, torch.as_tensor(o, device=DEV) if o is not None else None)
            want = eo.voxel_score(pts, d, tau, o)
            assert (got["good"], got["bad"], got["excluded"], got["voxels"]) == want[:4], tau
            assert abs(got["fraction_sum"] - want[4]) <= 1e-12 * abs(want[4]), tau
            again = ops.voxel_score(_d(pts), _d(d), tau, torch.as_tensor(o, device=DEV) if o is not None else None)
            assert again == got
    empty = ops.voxel_score(_d(np.zeros((0, 3))), _d(np.zeros(0)), 0.1)
    assert empty == {"good": 0, "bad": 0, "excluded": 0, "voxels": 0, "fraction_sum": 0.0}
    with pytest.raises(RuntimeError, match="outside"):
        ops.voxel_score(_d([[0.0, 0.0, 2e6 * 0.01]]), _d([0.0]), 0.01)


def _scans(c):
    return [{"matrix": s["matrix"], "points": s["points"]} for s in c["scans"]]


def test_evaluate_scene_matches_the_oracle_and_reruns_bit_for_bit():
    c = ec.make_scene(17, n_az=200, n_el=80, n_surface=8000, n_outliers=150, n_hidden=60)
    want, _, _, _ = eo.evaluate(c["rec"], _scans(c))
    got = eth3d_eval.evaluate_scene(c["rec"], _scans(c), device=DEV)
    again = eth3d_eval.evaluate_scene(c["rec"], _scans(c), device=DEV)
    assert got == again
    assert len(got["tolerances"]) == 6
    for g, w in zip(got["tolerances"], want):
        for k in ("accurate", "inaccurate", "unobserved", "covered", "gt_points", "accuracy_voxels", "completeness_voxels"):
            assert g[k] == w[k], (g["tolerance"], k)
        for k in ("accuracy", "completeness", "f1"):
            assert abs(g[k] - w[k]) <= 1e-12, (g["tolerance"], k)
    last = got["tolerances"][-1]
    assert (last["inaccurate"], last["unobserved"]) == (150, 180)


def test_cli_json_equals_evaluate_scene_and_writes_clouds(tmp_path):
    cases = ec.write_tree(str(tmp_path), ["alpha", "beta"], n_az=120, n_el=50, n_surface=2000, n_outliers=40, n_hidden=20)
    out = str(tmp_path / "r.json")
    assert eth3d_eval.main(["--gt-path", str(tmp_path / "gt"), "--outputs", str(tmp_path / "outputs"), "--json", out,
                            "--accuracy-cloud", str(tmp_path / "clouds" / "{scene}_acc.ply"),
                            "--completeness-cloud", str(tmp_path / "clouds" / "{scene}_comp.ply"), "--device", DEV]) == 0
    with open(out) as f:
        j = json.load(f)
    assert [s["scene"] for s in j["scenes"]] == ["alpha", "beta"]
    for s in j["scenes"]:
        truth = eth3d_eval.load_scene_truth(str(tmp_path / "gt"), s["scene"])
        rec = data_io.read_ply_points(str(tmp_path / "outputs" / s["scene"] / "fused.ply"))
        want = json.loads(json.dumps(eth3d_eval.evaluate_scene(rec, truth["scans"], device=DEV)))
        assert {k: v for k, v in s.items() if k not in ("scene", "seconds")} == want
        acc = data_io.read_ply_points(str(tmp_path / "clouds" / f"{s['scene']}_acc.ply"))
        assert acc.shape == rec.shape and (acc == rec.astype(np.float32)).all()
        body = open(tmp_path / "clouds" / f"{s['scene']}_acc.ply", "rb").read().split(b"end_header\n", 1)[1]
        rgb = np.frombuffer(body, np.uint8).reshape(-1, 15)[:, 12:]
        t = s["tolerances"][1]  # the cloud tolerance 0.02 is the second default
        assert t["tolerance"] == 0.02
        assert (rgb == ec_colour(eth3d_eval.GREEN)).all(1).sum() == t["accurate"]
        assert (rgb == ec_colour(eth3d_eval.RED)).all(1).sum() == t["inaccurate"]
        assert (rgb == ec_colour(eth3d_eval.BLUE)).all(1).sum() == t["unobserved"]
        comp = open(tmp_path / "clouds" / f"{s['scene']}_comp.ply", "rb").read().split(b"end_header\n", 1)[1]
        rgb = np.frombuffer(comp, np.uint8).reshape(-1, 15)[:, 12:]
        assert (rgb == ec_colour(eth3d_eval.GREEN)).all(1).sum() == t["covered"] and rgb.shape[0] == t["gt_points"]
    for i, m in enumerate(j["mean"]):
        assert m["f1"] == pytest.approx(np.mean([s["tolerances"][i]["f1"] for s in j["scenes"]]), abs=0)
    assert len(cases) == 2


def ec_colour(c):
    return np.array(c, np.uint8)


def test_clouds_above_2_24_points():
    side = 4100  # 16.81 M points > 2^24 on the plane z = 2, seen by one scanner at the origin
    g = (np.arange(side) - side / 2) * 1e-3
    x, y = np.meshgrid(g, g, indexing="ij")
    plane = np.stack([x.ravel(), y.ravel(), np.full(side * side, 2.0)], 1)
    assert plane.shape[0] > 2 ** 24
    k = 1000
    rng = np.random.RandomState(18)
    pick = plane[rng.randint(plane.shape[0], size=k)]
    outliers = pick * 0.5  # halfway along a beam, 1 m from the plane
    hidden = pick * 1.5  # 1 m behind the plane
    rec = np.concatenate([plane, outliers, hidden])
    scans = [{"matrix": np.eye(4), "points": plane}]
    r = eth3d_eval.evaluate_scene(rec, scans, (0.01, 0.5), device=DEV)
    for t in r["tolerances"]:
        assert (t["accurate"], t["inaccurate"], t["unobserved"]) == (plane.shape[0], k, k)
        assert t["covered"] == t["gt_points"] == plane.shape[0]
        assert t["completeness"] == 1.0
    q = _d(rec)
    obs = ops.beam_observed(q, _d(plane), [0, 0, 0], R0, T, mask=torch.arange(rec.shape[0], device=DEV) >= plane.shape[0])
    o = obs.cpu().numpy().astype(bool)
    assert not o[:plane.shape[0]].any() and o[plane.shape[0]:plane.shape[0] + k].all() and not o[plane.shape[0] + k:].any()


def test_evaluate_scene_memory_estimate_refuses_what_does_not_fit(monkeypatch):
    monkeypatch.setattr(eth3d_eval, "_free_bytes", lambda dev: 1000)
    c = ec.make_scene(19, n_az=20, n_el=10, n_surface=50, n_outliers=5, n_hidden=2)
    with pytest.raises(ValueError, match="GiB of device memory"):
        eth3d_eval.evaluate_scene(c["rec"], _scans(c), device=DEV)


def test_colmap_input_sparse_folder_matches_sparse(tmp_path):
    m = cc.make_model(21, 6, 300, track=4)
    m["images"] = [(iid, q, t, cid, "dslr_images_undistorted/" + name.replace(".png", ".JPG"), obs)
                   for iid, q, t, cid, name, obs in m["images"]]
    eth, plain = str(tmp_path / "eth"), str(tmp_path / "plain")
    cc.write_txt(os.path.join(eth, "dslr_calibration_undistorted"), m)
    cc.write_txt(os.path.join(plain, "sparse"), m)
    from PIL import Image

    rng = np.random.default_rng(0)
    for root in (eth, plain):
        os.makedirs(os.path.join(root, "images", "dslr_images_undistorted"), exist_ok=True)
    for im in m["images"]:
        arr = rng.integers(0, 256, (48, 64, 3)).astype(np.uint8)
        for root in (eth, plain):
            Image.fromarray(arr).save(os.path.join(root, "images", im[4]), format="JPEG")
    assert ci.main(["--input-folder", eth, "--sparse-folder", "dslr_calibration_undistorted"]) == 0  # in place
    assert ci.main(["--input-folder", plain]) == 0
    for name in ["pair.txt"] + [f"cams/{i:08d}_cam.txt" for i in range(6)] + [f"images/{i:08d}.jpg" for i in range(6)]:
        a, b = os.path.join(eth, name), os.path.join(plain, name)
        assert not os.path.islink(a)
        assert open(a, "rb").read() == open(b, "rb").read(), name
    shutil.rmtree(eth)
