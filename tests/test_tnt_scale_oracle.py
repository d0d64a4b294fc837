"""The vectorised Tanks and Temples oracle (tests/tnt_oracle.py, the *_v forms) against the literal one, without a GPU.

The scene-size GPU tests (tests/test_gpu_tnt_eval_at_scene_sizes.py) compare the kernels with the *_v forms, because the
literal forms loop in Python over every point and voxel.  Here the two are shown equal bit for bit (points, means, sums) and
index for index (masks, correspondences) on the small cases of tests/test_tnt_eval.py and test_gpu_tnt_eval.py, and on
adversarial rows: points on polygon vertices and horizontal edges, on axis_min / axis_max, for every orthogonal axis; exact
distance ties on an integer lattice; duplicate points; empty clouds."""
import numpy as np
import pytest

from tests import tnt_cases
from tests import tnt_oracle as to
from tests.test_tnt_eval import HAND_POINTS, HAND_WANT, SQUARE

AXIS_PERM = ((2, [0, 1, 2]), (1, [0, 2, 1]), (0, [1, 2, 0]))  # orthogonal axis, where (u, v, w) of the Z case go


def _moved(points, polygon, perm):
    p, q = np.zeros_like(points), np.zeros_like(polygon)
    p[:, perm], q[:, perm] = points, polygon
    return p, q


# ---- crop -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("axis,perm", AXIS_PERM, ids=["Z", "Y", "X"])
def test_crop_v_on_the_hand_cases(axis, perm):
    pts, poly = _moved(HAND_POINTS, SQUARE["polygon"], perm)
    cv = dict(SQUARE, orthogonal_axis=axis, polygon=poly)
    assert to.crop_v(pts, cv).tolist() == HAND_WANT == to.crop(pts, cv).tolist()


def _adversarial_crop_points(cv, rng, n=4000):
    """Points on the vertices, on the edges (horizontal ones included), on axis_min / axis_max and around them."""
    poly = np.asarray(cv["polygon"])
    nv = len(poly)
    a = rng.randint(0, nv, n)
    b = (a + 1) % nv
    t = rng.choice([0.0, 0.25, 0.5, 1.0, rng.uniform()], n)
    uv = poly[a, :2] + t[:, None] * (poly[b, :2] - poly[a, :2])   # on an edge (t = 0, 1: a vertex)
    uv[n // 2:] += rng.normal(0, 1e-3, (n - n // 2, 2)) * (rng.rand(n - n // 2, 1) < 0.5)
    w = rng.choice([cv["axis_min"], cv["axis_max"], np.nextafter(cv["axis_max"], np.inf), np.nextafter(cv["axis_min"], -np.inf),
                    0.5 * (cv["axis_min"] + cv["axis_max"])], n)
    return np.concatenate([uv, w[:, None]], 1)


@pytest.mark.parametrize("axis,perm", AXIS_PERM, ids=["Z", "Y", "X"])
def test_crop_v_on_vertices_edges_and_axis_bounds(axis, perm):
    rng = np.random.RandomState(11)
    # a concave polygon with two horizontal edges (v constant) and a vertex shared by a horizontal and a slanted edge
    poly_z = np.array([[0.0, 0.0, 0], [4.0, 0.0, 0], [4.0, 3.0, 0], [2.0, 1.0, 0], [1.0, 3.0, 0], [-1.0, 3.0, 0], [0.5, 1.5, 0]])
    cv_z = {"orthogonal_axis": 2, "axis_min": -0.75, "axis_max": 1.25, "polygon": poly_z}
    pts_z = np.concatenate([_adversarial_crop_points(cv_z, rng), HAND_POINTS])
    pts, poly = _moved(pts_z, poly_z, perm)
    cv = dict(cv_z, orthogonal_axis=axis, polygon=poly)
    want = to.crop(pts, cv)
    assert (to.crop_v(pts, cv) == want).all()
    assert 0 < want.sum() < len(pts)


def test_crop_v_on_the_scene_polygon_and_empty_clouds():
    rng = np.random.RandomState(4)
    cv = tnt_cases.crop_volume()
    pts = tnt_cases.OFFSET + rng.uniform(-1.2, 1.2, (50000, 3))
    pts[:1000, :2] = cv["polygon"][rng.randint(0, 6, 1000), :2]
    moved = to.transform(pts, tnt_cases.similarity(1.0003, [1, 1, 0], 1e-4, [1e-3, 0, -2e-3]))
    assert (to.crop_v(moved, cv) == to.crop(moved, cv)).all()
    assert to.crop_v(np.zeros((0, 3)), cv).shape == (0,)
    assert to.crop_v(pts[:10], dict(cv, polygon=np.zeros((0, 3)))).tolist() == [False] * 10  # no polygon: nothing inside


# ---- voxel down-sampling ----------------------------------------------------------------------------------------------------

def _voxel_rows():
    rng = np.random.RandomState(5)
    surf = tnt_cases.surface(rng, 40000)
    dup = np.concatenate([surf[:3000]] * 3)[rng.permutation(9000)]
    far = np.concatenate([rng.uniform(0, 1, (1500, 3)), rng.uniform(0, 1, (1500, 3)) + 4.0e5])
    edges = np.floor(rng.uniform(0, 20, (5000, 3))) * 0.25 + 0.125  # on voxel faces: min 0.125, origin 0, s = 0.25
    one = surf[:1]
    heavy = np.concatenate([surf[:2000], np.repeat(surf[2000:2001], 700, 0) + rng.normal(0, 1e-5, (700, 3))])  # a 700-point voxel
    return {"surface": (surf, 0.01), "duplicates": (dup, 0.02), "split_key": (far, 1e-3), "faces": (edges, 0.25), "one": (one, 0.1),
            "heavy": (heavy, 0.01)}


@pytest.mark.parametrize("row", ["surface", "duplicates", "split_key", "faces", "one", "heavy"])
def test_voxel_downsample_v_is_the_literal_bit_for_bit(row):
    pts, s = _voxel_rows()[row]
    got, want = to.voxel_downsample_v(pts, s), to.voxel_downsample(pts, s)
    assert got.shape == want.shape and got.tobytes() == want.tobytes()
    assert to.voxel_downsample_v(np.zeros((0, 3)), s).shape == (0, 3)


# ---- correspondences --------------------------------------------------------------------------------------------------------

def _lattice_case():
    g = np.arange(-3, 4, dtype=np.float64)
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    tgt = lattice[np.random.RandomState(7).permutation(len(lattice))]
    rng = np.random.RandomState(8)
    src = np.concatenate([np.array([[0.5, 0.0, 0.0], [0.5, 0.5, 0.0], [0.5, 0.5, 0.5], [2.5, -1.5, 0.0], [0.0, 0.0, 0.0], [9.0, 9.0, 9.0]]),
                          rng.randint(-6, 7, (400, 3)) * 0.5])  # half-integer points: up to 8 candidates at one distance
    return src, tgt


@pytest.mark.parametrize("k", [1, 2, 4, 8])
def test_correspondences_v_on_lattice_ties(k):
    src, tgt = _lattice_case()
    for r in (0.5, 0.8660254037844386, 1.0, 3.0):
        want_i, want_d = to.correspondences(src, tgt, r)
        got_i, got_d = to.correspondences_v(src, tgt, r, k=k)
        assert got_i.tolist() == want_i.tolist() and got_d.tobytes() == want_d.tobytes(), r
    assert (want_i >= 0).sum() > 300


def test_correspondences_v_on_duplicates_surfaces_and_empty_clouds():
    rng = np.random.RandomState(6)
    tgt = tnt_cases.surface(rng, 20000)
    tgt = np.concatenate([tgt, tgt[:3000], tgt[:1000]])  # duplicate target points: ties at any distance
    src = np.concatenate([tnt_cases.surface(rng, 15000) + rng.normal(0, 0.01, (15000, 3)), tgt[:500]])  # some exactly on targets
    for r in (0.02, 0.05, 0.4):
        want = to.correspondences(src, tgt, r)
        for k in (2, 8):
            got = to.correspondences_v(src, tgt, r, k=k)
            assert got[0].tolist() == want[0].tolist() and got[1].tobytes() == want[1].tobytes(), (r, k)
    for a, b in ((np.zeros((0, 3)), tgt), (src, np.zeros((0, 3)))):
        i, d = to.correspondences_v(a, b, 0.1)
        assert (i == -1).all() and np.isinf(d).all() and len(i) == len(a)
    i, d = to.correspondences_v(src[:5], tgt[:3], 10.0)  # fewer targets than candidates
    assert i.tolist() == to.correspondences(src[:5], tgt[:3], 10.0)[0].tolist()


# ---- ICP, refinement and scoring --------------------------------------------------------------------------------------------

def _same_icp(got, want):
    assert got["iterations"] == want["iterations"] and got["history"] == want["history"]
    assert got["transformation"].tobytes() == want["transformation"].tobytes()
    assert got["fitness"] == want["fitness"] and got["inlier_rmse"] == want["inlier_rmse"]
    assert got["correspondence_set"].tolist() == want["correspondence_set"].tolist()


def test_icp_v_is_the_literal_loop():
    c = tnt_cases.make_scene(100, n_gt=12000, n_rec=10000)
    s = tnt_cases.apply(c["S"], c["rec"])
    s[:, :2] += 0.01
    s = to.voxel_downsample(s[to.crop(s, c["crop"])], c["tau"])
    g = to.voxel_downsample(c["gt"][to.crop(c["gt"], c["crop"])], c["tau"])
    want = to.icp(s, g, 20 * c["tau"], max_iteration=20)
    got = to.icp_v(s, g, 20 * c["tau"], max_iteration=20)
    _same_icp(got, want)
    assert want["iterations"] > 1 and len(got["deltas"]) == got["iterations"]
    _same_icp(to.icp_v(s + 100.0, g, 0.2, max_iteration=5), to.icp(s + 100.0, g, 0.2, max_iteration=5))  # no correspondence
    _same_icp(to.icp_v(s, np.zeros((0, 3)), 0.2, max_iteration=3), to.icp(s, np.zeros((0, 3)), 0.2, max_iteration=3))


def test_evaluate_scene_v_is_the_literal_chain():
    c = tnt_cases.make_scene(101, n_gt=8000, n_rec=6000)
    init = c["S"].copy()
    init[:3, 3] += [0.01, -0.005, 0.0]
    want = to.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"])
    got = to.evaluate_scene_v(c["rec"], c["gt"], c["crop"], init, c["tau"])
    assert got["transformation"].tobytes() == want["transformation"].tobytes()
    for a, b in zip(got["rounds"], want["rounds"]):
        for k in ("n_source", "n_target", "iterations", "correspondences", "fitness", "history"):
            assert a[k] == b[k], k
        assert a["transformation"].tobytes() == b["transformation"].tobytes()
    for k in ("precision", "recall", "fscore", "n_source_scored", "n_gt_scored", "precision_count", "recall_count"):
        assert got[k] == want[k], k
    assert (got["cum_precision"] == want["cum_precision"]).all() and (got["cum_recall"] == want["cum_recall"]).all()
    assert 0.5 < got["precision"] < 1 and 0.5 < got["recall"] < 1


def test_score_v_on_empty_sides():
    gt = np.array([[1.0, 1.0, 0.0], [1.5, 1.0, 0.0]])
    for rec, g in ((np.zeros((0, 3)), gt), (gt, np.zeros((0, 3))), (np.array([[1.0, 1.9, 0.0]]), gt)):
        got, want = to.score_v(rec, g, SQUARE, np.eye(4), 0.01), to.score(rec, g, SQUARE, np.eye(4), 0.01)
        for k in ("precision", "recall", "fscore", "n_source_scored", "n_gt_scored", "precision_count", "recall_count"):
            assert got[k] == want[k], k
        assert (got["cum_precision"] == want["cum_precision"]).all() and (got["cum_recall"] == want["cum_recall"]).all()
