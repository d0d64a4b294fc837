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
from tests import dtu_cases, dtu_scale_cases


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


def _clouds():
    """The thinning cases of tests/test_gpu_dtu_eval.py."""
    rng = np.random.RandomState(11)
    uniform = rng.uniform(0.0, 10.0, (50000, 3))
    # 220k samples of a 60 x 60 mm surface: ~60 points per mm^2, about 7 neighbours within 0.2 mm
    x, y = rng.uniform(0, 60, 220000), rng.uniform(0, 60, 220000)
    clustered = np.stack([x, y, 3.0 * np.sin(x / 5.0) + 0.01 * x * y], axis=1).astype(np.float32).astype(np.float64)
    base = rng.uniform(0.0, 5.0, (6000, 3)).astype(np.float32).astype(np.float64)
    duplicates = np.concatenate([base, base[:3000], base[:1000]])
    g = np.arange(20) * 0.25  # exact lattice: every neighbour exactly dst = 0.25 apart
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3) + 1000.0
    return [("uniform", uniform, 0.2), ("clustered", clustered, 0.2), ("duplicates", duplicates, 0.2), ("lattice", lattice, 0.25)]


# ---- the checker and the round count of thinning at scan sizes (tests/dtu_scale_cases.py) ------------------------------------

def _thin_rows():
    rows = [(name, {"points": p, "dst": dst, "order": dtu_eval.visiting_order(p.shape[0], 7 + i)})
            for i, (name, p, dst) in enumerate(_clouds())]
    return rows + [("literal", dtu_scale_cases.literal(0))]


def test_thin_violations_accepts_the_sequential_oracle():
    for name, r in _thin_rows():
        keep = do.thin(r["points"], r["order"], r["dst"])
        assert do.thin_violations(r["points"], do.rank_of(r["order"]), keep, r["dst"]).size == 0, name
        assert 0 < keep.sum() < keep.size, name


def test_thin_violations_reports_planted_errors():
    r = dtu_scale_cases.literal(0)
    pts, dst, order = r["points"], r["dst"], r["order"]
    rank = do.rank_of(order)
    keep = do.thin(pts, order, dst)
    removed, kept = np.nonzero(~keep)[0][0], np.nonzero(keep)[0][0]
    flipped = keep.copy()
    flipped[removed] = True
    assert removed in do.thin_violations(pts, rank, flipped, dst)
    flipped = keep.copy()
    flipped[kept] = False
    assert kept in do.thin_violations(pts, rank, flipped, dst)
    # a kept point a and a point b that only a removed trade places in the visiting order: b is kept and a removed in that
    # order's mask, which is wrong for this one
    pairs = do.thin_pairs(pts, dst)
    pairs = np.concatenate([pairs, pairs[:, ::-1]])
    kept_nbrs = np.bincount(pairs[keep[pairs[:, 0]], 1], minlength=keep.size)
    a, b = pairs[keep[pairs[:, 0]] & ~keep[pairs[:, 1]] & (kept_nbrs[pairs[:, 1]] == 1)][0]
    swapped = np.asarray(order).copy()
    swapped[rank[a]], swapped[rank[b]] = b, a
    other = do.thin(pts, swapped, dst)
    assert other[b] and not other[a]
    assert do.thin_violations(pts, rank, other, dst).size > 0
    assert do.thin_violations(pts, do.rank_of(swapped), other, dst).size == 0


def test_thin_sync_rounds_hand_case():
    # 0 accepted; 1 rejected while 2 waits for it; 2 accepted; 3 rejected; 4 accepted
    rounds, keep = do.thin_sync_rounds(_line([0.0, 0.25, 0.5, 0.75, 1.0]), np.arange(5), 0.25)
    assert rounds == 5 and keep.tolist() == [True, False, True, False, True]
    rounds, keep = do.thin_sync_rounds(_line([0.0, 0.25, 0.5, 0.75, 1.0]), do.rank_of([1, 0, 2, 3, 4]), 0.25)
    assert rounds == 4 and keep.tolist() == [False, True, False, True, False]


@pytest.mark.parametrize("row", ["literal", "stack"])
def test_thin_sync_rounds_is_the_oracle_far_below_the_native_round_bound(row):
    """Random visiting orders at DTU densities settle in a few rounds: 12 and 14 here against the bound of 256.  `stack` at
    50k points has the neighbour counts of the 200k row the GPU tests run, at a cost the sequential oracle can pay."""
    r = dtu_scale_cases.literal(0) if row == "literal" else dtu_scale_cases.stack(0, n=50_000)
    rounds, keep = do.thin_sync_rounds(r["points"], do.rank_of(r["order"]), r["dst"])
    assert (keep == do.thin(r["points"], r["order"], r["dst"])).all()
    assert rounds <= 32


@pytest.mark.parametrize("decreasing", [False, True])
def test_chain_needs_more_rounds_than_the_native_bound(decreasing):
    r = dtu_scale_cases.chain(decreasing)
    rounds, keep = do.thin_sync_rounds(r["points"], do.rank_of(r["order"]), r["dst"])
    assert rounds > dtu_scale_cases.THIN_ROUND_BOUND
    assert (keep == do.thin(r["points"], r["order"], r["dst"])).all()
    first = r["order"][0]
    assert keep[first] and (keep[::2] != keep[1::2]).all()  # every other point along the chain, from the first visited


def test_scale_rows_are_pinned():
    sc = dtu_scale_cases
    s = sc.sheets(0)
    assert s["data"].shape[0] > 2 ** 24 and s["stl"].shape[0] == sc.N_STL
    assert (s["data"].astype(np.float32).astype(np.float64) == s["data"]).all()
    rng = np.floor((s["bb"][1] - s["bb"][0]) / 60.0) + 1
    assert rng.tolist() == [6.0, 6.0, 3.0]  # MaxDistCP blocks per axis
    for pts in (s["data"], sc.literal(0)["points"]):  # about 23 neighbours within dst, at most about 50
        counts = sc.neighbour_counts(pts, sc.DST, [-2.5, -2.5, -np.inf], [2.5, 2.5, np.inf])
        assert 18 < counts.mean() < 28 and counts.size > 7000
    st = sc.stack(0)["points"]
    assert st.shape[0] == 200_000 and np.unique(st, axis=0).shape[0] < 0.92 * st.shape[0]
    counts = sc.neighbour_counts(st, sc.DST, [-0.5, -0.5, -np.inf], [0.5, 0.5, np.inf])
    assert 400 < counts.mean() < 1000
    lat = sc.lattice(0)
    inner = sc.neighbour_counts(lat["points"], lat["dst"], [1000.2] * 3, [1024.6] * 3)
    assert lat["points"].shape[0] == 10 ** 6 and (inner == 6).all()  # exactly dst apart along the axes, nothing closer
    ch = sc.chain()
    assert (sc.neighbour_counts(ch["points"], sc.DST, [-np.inf] * 3, [np.inf] * 3) == [1] + [2] * 2998 + [1]).all()


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
