"""ETH3D evaluation without a GPU: the .mlp reader, the CPU oracle (tests/eth3d_oracle.py) on hand cases and on the synthetic
room of tests/eth3d_cases.py, and the command's argument checks."""
import math

import numpy as np
import pytest

from patchmatchnet_b200 import eth3d_eval
from tests import eth3d_cases as ec
from tests import eth3d_oracle as eo

R0, T = 0.001125, math.tan(math.radians(0.011))


# ---- .mlp reader ------------------------------------------------------------------------------------------------------------

def test_read_mlp_relative_paths_and_matrix_whitespace(tmp_path):
    m1 = np.arange(16, dtype=np.float64).reshape(4, 4) / 7
    m1[3] = [0, 0, 0, 1]
    text = ("<!DOCTYPE MeshLabDocument>\n<MeshLabProject>\n <MeshGroup>\n"
            '  <MLMesh label="a" filename="sub/a.ply">\n   <MLMatrix44>\n'
            + "\n".join("\t".join(f"{v:.17g}" for v in row) + "  " for row in m1) + "\n</MLMatrix44>\n  </MLMesh>\n"
            '  <MLMesh label="b" filename="../b.ply"><MLMatrix44>1 0 0 2 0 1 0 3 0 0 1 4 0 0 0 1</MLMatrix44></MLMesh>\n'
            " </MeshGroup>\n</MeshLabProject>\n")
    p = tmp_path / "scene" / "project.mlp"
    p.parent.mkdir()
    p.write_text(text)
    scans = eth3d_eval.read_mlp(str(p))
    assert [s["filename"] for s in scans] == [str(p.parent / "sub/a.ply"), str(p.parent / "../b.ply")]
    assert (scans[0]["matrix"] == m1).all()
    assert scans[1]["matrix"][:3, 3].tolist() == [2.0, 3.0, 4.0]


@pytest.mark.parametrize("body, match", [
    ("<MeshLabProject><MeshGroup>", "well-formed"),
    ("<MeshLabProject><MeshGroup></MeshGroup></MeshLabProject>", "no MLMesh"),
    ('<MeshLabProject><MLMesh label="a"><MLMatrix44>1 0 0 0 0 1 0 0 0 0 1 0 0 0 0 1</MLMatrix44></MLMesh></MeshLabProject>',
     "no filename"),
    ('<MeshLabProject><MLMesh filename="a.ply"></MLMesh></MeshLabProject>', "no MLMatrix44"),
    ('<MeshLabProject><MLMesh filename="a.ply"><MLMatrix44>1 0 0 0 0 1 0 0 0 0 1 0</MLMatrix44></MLMesh></MeshLabProject>',
     "16 numbers"),
    ('<MeshLabProject><MLMesh filename="a.ply"><MLMatrix44>1 0 0 0 0 1 0 0 0 0 1 0 0 0 x 1</MLMatrix44></MLMesh></MeshLabProject>',
     "not a number"),
    ('<MeshLabProject><MLMesh filename="a.ply"><MLMatrix44>1 0 0 0 0 1 0 0 0 0 1 0 0 0 0.5 1</MLMatrix44></MLMesh></MeshLabProject>',
     "0 0 0 1"),
    ('<MeshLabProject><MLMesh filename="a.ply"><MLMatrix44>1 0 0 nan 0 1 0 0 0 0 1 0 0 0 0 1</MLMatrix44></MLMesh></MeshLabProject>',
     "finite"),
])
def test_read_mlp_rejects_malformed_projects(tmp_path, body, match):
    p = tmp_path / "bad.mlp"
    p.write_text(body)
    with pytest.raises(ValueError, match=match) as e:
        eth3d_eval.read_mlp(str(p))
    assert str(p) in str(e.value)


def test_load_scene_truth_reads_binary_and_ascii_scans(tmp_path):
    cases = ec.write_tree(str(tmp_path), ["room"], n_az=40, n_el=20, n_surface=200, n_outliers=10, n_hidden=5)
    truth = eth3d_eval.load_scene_truth(str(tmp_path / "gt"), "room")
    want = cases["room"]["scans"]
    assert len(truth["scans"]) == len(want) == 3
    for got, w in zip(truth["scans"], want):
        assert (got["points"] == w["points"]).all()  # double properties and %.17g text round-trip exactly
        assert (got["matrix"] == w["matrix"]).all() and (got["origin"] == w["origin"]).all()
    assert eth3d_eval.find_scenes(str(tmp_path / "gt")) == ["room"]


# ---- beam predicate on hand cases ---------------------------------------------------------------------------------------------

def _one(p, q, o=(0.0, 0.0, 0.0), r0=R0, t=T):
    return bool(eo.beam_observed(np.array([q], np.float64), np.array([p], np.float64), o, r0, t)[0])


def test_beam_hand_cases():
    o = np.array([1.0, -2.0, 0.5])
    p = o + [10.0, 0.0, 0.0]
    for lam in (0.5, 2.0, 9.0):
        radius = R0 + lam * T  # the cone's radius at distance lam along the beam
        assert _one(p, o + [lam, radius - 1e-6, 0.0], o)
        assert not _one(p, o + [lam, radius + 1e-6, 0.0], o)
        assert _one(p, o + [lam, 0.0, -(radius - 1e-6)], o)
        assert not _one(p, o + [lam, 0.0, -(radius + 1e-6)], o)
    assert not _one(p, o + [10.0 + 1e-6, 0.0, 0.0], o)  # behind p
    assert not _one(p, o + [10.0, 0.0, 0.0], o)  # p itself: t' = a.a
    assert not _one(p, o + [-1.0, 0.0, 0.0], o)  # t' < 0
    assert not _one(p, o, o)  # b = 0: t' = 0
    assert not _one(o, o + [1.0, 0.0, 0.0], o)  # a = 0 is never a beam
    assert _one(p, o + [1e-4, 5e-4, 0.0], o)  # within r0 of the scanner
    assert _one(p, o + [1.0, 0.0, 0.0], o, r0=0.0, t=0.0)  # a zero-width beam still holds its own axis


def test_beam_oracle_is_brute_force_over_scans():
    rng = np.random.RandomState(1)
    scan = rng.normal(size=(50, 3)) * 3
    q = rng.normal(size=(40, 3))
    got = eo.beam_observed(q, scan, [0, 0, 0], 0.05, 0.01, chunk=7)
    want = np.array([any(_one(p, qq, r0=0.05, t=0.01) for p in scan) for qq in q])
    assert (got == want).all() and 0 < got.sum() < len(q)
    assert not eo.beam_observed(q, np.zeros((0, 3)), [0, 0, 0], R0, T).any()


# ---- voxel scores --------------------------------------------------------------------------------------------------------------

def test_voxel_score_hand_case():
    tau = 0.5
    pts = np.array([[0.1, 0.1, 0.1], [0.2, 0.3, 0.4], [0.4, 0.1, 0.2],  # voxel (0,0,0): good, bad, excluded
                    [-0.1, 0.2, 0.2],                                    # voxel (-1,0,0): bad
                    [1.0, 1.0, 1.0], [1.2, 1.4, 1.1],                    # voxel (2,2,2): good, good
                    [0.5, 0.0, 0.0]])                                    # voxel (1,0,0): excluded only
    d = np.array([0.5, 0.6, 0.7, 0.9, 0.0, 0.1, 2.0])
    obs = np.array([0, 1, 0, 1, 0, 0, 0], bool)
    good, bad, excl, voxels, s = eo.voxel_score(pts, d, tau, obs)
    assert (good, bad, excl, voxels) == (3, 2, 2, 3)
    assert s == 0.5 + 0.0 + 1.0
    good, bad, excl, voxels, s = eo.voxel_score(pts, d, tau)  # completeness: every point counts
    assert (good, bad, excl, voxels) == (3, 4, 0, 4) and s == 1 / 3 + 0.0 + 1.0 + 0.0


# ---- the room, with the oracle ----------------------------------------------------------------------------------------------

def _room(**kw):
    c = ec.make_scene(7, n_az=90, n_el=40, **kw)
    return c, [{"matrix": s["matrix"], "points": s["points"]} for s in c["scans"]]


def test_oracle_zero_noise_samples_are_accurate():
    c, scans = _room(n_surface=1500, noise=0.0, n_outliers=0, n_hidden=0)
    res, d_acc, _, _ = eo.evaluate(c["rec"], scans)
    assert d_acc.max() < 1e-6
    for r in res:
        assert r["accuracy"] == 1.0 and r["inaccurate"] == 0 and r["unobserved"] == 0
        assert 0 < r["completeness"] <= 1.0


def test_oracle_gives_the_designed_classes():
    c, scans = _room(n_surface=1500, noise=0.002, n_outliers=60, n_hidden=30)
    res, d_acc, d_comp, observed = eo.evaluate(c["rec"], scans)
    lab = c["labels"]
    assert (d_acc[lab > 0] > 0.5).all()
    assert observed[lab == 1].all()
    assert not observed[lab >= 2].any()
    for r in res:
        assert r["inaccurate"] >= 60 and r["unobserved"] >= 90
    last = res[-1]  # tau = 0.5: every surface sample is accurate, so the designed points are the only other classes
    assert (last["accurate"], last["inaccurate"], last["unobserved"]) == (1500, 60, 90)
    assert 0 < last["accuracy"] < 1 and last["covered"] <= last["gt_points"]


# ---- command-line checks ---------------------------------------------------------------------------------------------------

def test_cli_argument_errors_without_a_gpu(tmp_path):
    ec.write_tree(str(tmp_path), ["room"], n_az=20, n_el=10, n_surface=50, n_outliers=5, n_hidden=2)
    gt = str(tmp_path / "gt")
    with pytest.raises(SystemExit):
        eth3d_eval.main(["--gt-path", gt, "--tolerances", "0.01,abc"])
    with pytest.raises(SystemExit):
        eth3d_eval.main(["--gt-path", gt, "--tolerances", "0.01,-0.02"])
    with pytest.raises(ValueError, match="not a folder"):
        eth3d_eval.main(["--gt-path", str(tmp_path / "missing")])
    with pytest.raises(ValueError, match="beam-start-radius"):
        eth3d_eval.main(["--gt-path", gt, "--beam-start-radius", "-1"])
    with pytest.raises(ValueError, match="halfangle"):
        eth3d_eval.main(["--gt-path", gt, "--beam-divergence-halfangle-deg", "90"])
    with pytest.raises(ValueError, match="cloud-tolerance"):
        eth3d_eval.main(["--gt-path", gt, "--cloud-tolerance", "0"])
    with pytest.raises(ValueError, match="does not exist"):
        eth3d_eval.main(["--gt-path", gt, "--scenes", "room", "nowhere"])
    with pytest.raises(ValueError, match="no scene"):
        eth3d_eval.main(["--gt-path", str(tmp_path / "outputs")])
    args = eth3d_eval.build_parser().parse_args(["--gt-path", gt])
    assert eth3d_eval.check_args(args) == ["room"]
    assert args.tolerances == list(eth3d_eval.TOLERANCES) and args.cloud_tolerance == 0.02
