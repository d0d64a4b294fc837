"""The DTU evaluation (csrc/pm_cloud.cu through ops / dtu_eval) at the cloud sizes and densities of real scans, point by point
against the float64 oracle (oracle/dtu_oracle.py).  Rows: tests/dtu_scale_cases.py.

Thinning.  The sequential oracle, dtu_oracle.thin, cannot run at 20M points, so the mask is checked with
dtu_oracle.thin_violations, which holds exactly when the mask is thin's: every point is kept iff no kept point within dst is
visited before it.  `literal` is small enough for thin itself; `chain` needs more rounds than the native bound, so it must
either give thin's mask or raise the round-bound error, never another mask.

Distances.  Both directions of the `sheets` scan over every query against dtu_oracle.max_dist_cp (the literal block loop:
the box is 6 x 6 x 3 blocks of 60 mm), at the default search cell and, on a subsample, at the smallest cell the library
allows (most queries go on to the coarse rings) and at 60/8 (crowded fine cells); queries exactly on the block faces.

evaluate_scan.  Against the oracle chain built from the checked GPU mask: both distances, mask, plane, statistics."""
import numpy as np
import pytest
import torch

from oracle import dtu_oracle as do
from patchmatchnet_b200 import dtu_eval, ops
from tests import dtu_scale_cases as sc
from tests.test_gpu_dtu_eval import _check_distances

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MAX_DIST = 60.0
SUBSAMPLE = 200_000
FACE_QUERIES = 10_000


def _gpu_thin(points, rank, dst):
    keep = ops.thin_points(torch.as_tensor(points, device=DEV), torch.as_tensor(rank.astype(np.int32), device=DEV), dst)
    return keep.cpu().numpy()


def _report(name, points, keep):
    print(f"{name}: {points.shape[0]} points, {int(keep.sum())} kept")


@pytest.fixture(scope="module")
def sheets0():
    """The sheets row of seed 0 with its visiting order and GPU keep mask (checked by test_thinning_sheets_passes_the_checker)."""
    c = sc.sheets(0)
    c["rank"] = do.rank_of(dtu_eval.visiting_order(c["data"].shape[0], 0))
    c["keep"] = _gpu_thin(c["data"], c["rank"], sc.DST)
    return c


# ---- thinning -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [0, 1])
def test_thinning_sheets_passes_the_checker(seed, sheets0):
    if seed == 0:
        pts, rank, keep = sheets0["data"], sheets0["rank"], sheets0["keep"]
    else:
        pts = sc.sheets(seed)["data"]
        rank = do.rank_of(dtu_eval.visiting_order(pts.shape[0], seed))
        keep = _gpu_thin(pts, rank, sc.DST)
    assert pts.shape[0] > 2 ** 24 and keep.dtype == bool
    bad = do.thin_violations(pts, rank, keep, sc.DST)
    assert bad.size == 0, f"{bad.size} of {pts.shape[0]} points decided wrongly, first {bad[:10].tolist()}"
    assert 0 < keep.sum() < pts.shape[0] // 4
    _report(f"sheets seed {seed}", pts, keep)


@pytest.mark.parametrize("row", ["stack", "lattice"])
def test_thinning_dense_rows_pass_the_checker(row):
    r = getattr(sc, row)(3)
    pts, dst = r["points"], r["dst"]
    rank = do.rank_of(r["order"])
    keep = _gpu_thin(pts, rank, dst)
    bad = do.thin_violations(pts, rank, keep, dst)
    assert bad.size == 0, f"{row}: {bad.size} of {pts.shape[0]} points decided wrongly, first {bad[:10].tolist()}"
    assert 0 < keep.sum() < pts.shape[0]
    _report(row, pts, keep)


def test_thinning_literal_matches_the_sequential_oracle_bit_for_bit():
    r = sc.literal(4)
    got = _gpu_thin(r["points"], do.rank_of(r["order"]), r["dst"])
    want = do.thin(r["points"], r["order"], r["dst"])
    assert (got == want).all(), f"{(got != want).sum()} of {got.size} differ"


def test_thinning_sheets_rerun_and_row_permutation(sheets0):
    """The same cloud again gives the same bits; the rows permuted together with their ranks keep the same points, so the
    result does not depend on where a point sits in the input (the key sort and the scatter back)."""
    pts, rank, keep = sheets0["data"], sheets0["rank"], sheets0["keep"]
    assert (_gpu_thin(pts, rank, sc.DST) == keep).all()
    perm = np.random.RandomState(5).permutation(pts.shape[0])
    assert (_gpu_thin(pts[perm], rank[perm], sc.DST) == keep[perm]).all()


@pytest.mark.parametrize("decreasing", [False, True], ids=["along", "against"])
def test_chain_gives_the_oracle_or_the_round_bound_error(decreasing):
    """Each point of the chain waits for the one before it: a synchronous thinning needs about 3000 rounds.  The native one
    may finish sooner (a point reads decisions made earlier in its own round), and must otherwise say so."""
    r = sc.chain(decreasing)
    want = do.thin(r["points"], r["order"], r["dst"])
    try:
        got = _gpu_thin(r["points"], do.rank_of(r["order"]), r["dst"])
    except RuntimeError as e:
        assert "still undecided after the round bound" in str(e)
        return
    assert (got == want).all()


# ---- nearest distances ------------------------------------------------------------------------------------------------------

def _gpu_distances(to, frm, bb, cell=None):
    got = ops.nearest_distance(torch.as_tensor(to, device=DEV), torch.as_tensor(frm, device=DEV), bb, MAX_DIST, cell=cell)
    return got.cpu().numpy()


@pytest.fixture(scope="module")
def oracle_distances(sheets0):
    """dtu_oracle.max_dist_cp on the sheets row, once per direction.  Its value for a query depends on that query alone, so
    a subset of the queries reads a subset of the result.
      data->stl      every data point (20M) to the STL cloud
      stl->thinned   every STL point (3M) to the data the GPU mask keeps (evaluate_scan's completeness side)
      stl->data      the STL points of one column of blocks to all 20M data points (a search grid above 2^24 points)"""
    c = sheets0
    thinned = c["data"][c["keep"]]
    lo = c["bb"][0]
    column = np.nonzero(((c["stl"][:, :2] >= lo[:2] + 2 * MAX_DIST) & (c["stl"][:, :2] < lo[:2] + 3 * MAX_DIST)).all(axis=1))[0]
    cases = {"data->stl": (c["stl"], c["data"]), "stl->thinned": (thinned, c["stl"]), "stl->data": (c["data"], c["stl"][column])}
    return {k: (to, frm, do.max_dist_cp(to, frm, c["bb"], MAX_DIST)) for k, (to, frm) in cases.items()}


@pytest.mark.parametrize("direction", ["data->stl", "stl->thinned", "stl->data"])
def test_distances_on_sheets_match_the_block_oracle(direction, sheets0, oracle_distances):
    """Every query at the default search cell; a subsample at the smallest cell the library allows (60/256: most searches
    go on to the coarse rings) and at 60/8 (hundreds to thousands of points per fine cell)."""
    to, frm, want = oracle_distances[direction]
    bb = sheets0["bb"]
    _check_distances(_gpu_distances(to, frm, bb), want)
    assert (want < 1.0).mean() > 0.9  # most queries have a point nearby: the search's first rings decide
    sub = np.random.RandomState(6).choice(frm.shape[0], min(SUBSAMPLE, frm.shape[0]), replace=False)
    # 60/256 is already the default cell of the 20M-point grid; at 60/8 it would hold about 20 000 points in every fine cell
    cells = [] if direction == "stl->data" else [MAX_DIST / 256, MAX_DIST / 8]
    for cell in cells:
        _check_distances(_gpu_distances(to, frm[sub], bb, cell), want[sub])


def test_distances_of_queries_on_block_faces(sheets0):
    """MaxDistCP's blocks are [bb_lo + k 60, bb_lo + (k + 1) 60) per axis: a query exactly on a lower face belongs to the
    block above it (the oracle and the kernel compute the faces with the same float64 expression), one on the face past the
    last block to no block.  Some queries sit on bb_hi."""
    c = sheets0
    bb, stl = c["bb"], c["stl"]
    rng = np.random.RandomState(7)
    frm = c["data"][rng.randint(0, c["data"].shape[0], FACE_QUERIES)].copy()
    blocks = np.floor((bb[1] - bb[0]) / MAX_DIST)
    axis = rng.randint(0, 3, FACE_QUERIES)
    k = rng.randint(0, blocks[axis] + 2)  # k = blocks + 1 is the face past the last block
    on_hi = rng.rand(FACE_QUERIES) < 0.1
    rows = np.arange(FACE_QUERIES)
    frm[rows, axis] = np.where(on_hi, bb[1][axis], bb[0][axis] + k * MAX_DIST)
    want = do.max_dist_cp(stl, frm, bb, MAX_DIST)
    _check_distances(_gpu_distances(stl, frm, bb), want)
    assert ((k == 0) & ~on_hi & (want < MAX_DIST)).sum() > 100  # on the lower faces of the first blocks, and compared


# ---- evaluate_scan ----------------------------------------------------------------------------------------------------------

def test_evaluate_scan_on_sheets_matches_the_oracle_chain(sheets0, oracle_distances):
    """The oracle chain of dtu_oracle.evaluate_scan from the GPU's (checked) keep mask: MaxDistCP both ways, the mask, the
    plane, the statistics.  Counts exactly, statistics to 1e-9 relative; a rerun gives the same result."""
    c = sheets0
    args = (c["data"], c["stl"], c["obs_mask"], c["bb"], c["res"], c["plane"])
    got = dtu_eval.evaluate_scan(*args, seed=0, device=DEV)
    thinned = c["data"][c["keep"]]
    d_data = oracle_distances["data->stl"][2][c["keep"]]  # the thinned points are a subset of the data->stl queries
    d_stl = oracle_distances["stl->thinned"][2]
    acc = d_data[do.data_in_mask(thinned, c["obs_mask"], c["bb"], c["res"])]
    comp = d_stl[do.stl_above_plane(c["stl"], c["plane"])]
    want = {"n_data": c["data"].shape[0], "n_thinned": int(c["keep"].sum()), "n_stl": c["stl"].shape[0]}
    for name, d in (("acc", acc[acc < 20.0]), ("comp", comp[comp < 20.0])):
        for k, v in do.side_stats(d).items():
            want[f"{name}_{k}"] = v
    assert got.keys() == want.keys()
    for k in want:
        if k.endswith("count") or k.startswith("n_"):
            assert got[k] == want[k], k
        else:
            assert got[k] == pytest.approx(want[k], rel=1e-9), k
    assert want["acc_count"] > 10 ** 6 and want["comp_count"] > 10 ** 6
    assert dtu_eval.evaluate_scan(*args, seed=0, device=DEV) == got
