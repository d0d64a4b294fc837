"""The Tanks and Temples evaluation (csrc/pm_cloud.cu through ops / tnt_eval) at the sizes of real scenes, against the
vectorised float64 oracle (tests/tnt_oracle.py, the *_v forms, shown equal to the literal oracle by
tests/test_tnt_scale_oracle.py).  Rows: tests/tnt_scale_cases.py.

Crop: transformed points and mask bit for bit.  Voxel down-sampling: counts exactly, means within 1e-12 relative (which
also pins the voxel order: neighbouring voxels' means are a voxel apart).  Nearest distances as tnt_eval.score asks for
them (box min / max -+ 5 tau, cap 5 tau, default cell): every query in both directions against cKDTree's uncapped
distance.  ICP: every correspondence index at round-3 size and the 18 moments within the bound of the kernel's summation
order; each refinement round's iteration count and history.  score on rows whose distances are placed exactly, and
evaluate_scene end to end against the oracle chain run from the GPU's estimates, its counts and curves exactly.

Each row is built once per module and each oracle result computed once."""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from patchmatchnet_b200 import _native, ops, tnt_eval
from tests import tnt_cases
from tests import tnt_oracle as to
from tests import tnt_scale_cases as sc
from tests.test_gpu_tnt_eval import _check_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -53  # unit roundoff of float64


def _d(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=DEV)


def _need(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"needs {nbytes} bytes of free device memory, {free} free")


def _ties_at_threshold(deltas, thr=1e-6):
    return [d for d in deltas if abs(d[0] - thr) <= 1e-12 or abs(d[1] - thr) <= 1e-12]


# ---- rows and oracle results, once per module -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def obj():
    _need(12 << 30)
    c = sc.object_row()
    c["init"] = c["S"]
    print(f"object: {len(c['rec'])} reconstruction points, {len(c['gt'])} GT points")
    return c


@pytest.fixture(scope="module")
def obj_oracle(obj):
    """to.evaluate_scene_v on `object`, each round keeping its down-sampled clouds."""
    c = obj
    w = to.evaluate_scene_v(c["rec"], c["gt"], c["crop"], c["init"], c["tau"], keep_inputs=True)
    for k, r in enumerate(w["rounds"]):
        print(f"object round {k + 1}: {r['n_source_cropped']} cropped, {r['n_source']} source, {r['n_target']} target, "
              f"{r['iterations']} iterations")
    return w


@pytest.fixture(scope="module")
def large():
    _need(4 << 30)
    c = sc.large_row()
    print(f"large: {len(c['rec'])} reconstruction points, {len(c['gt'])} GT points")
    return c


@pytest.fixture(scope="module")
def block_gap():
    c = sc.block_gap_row()
    print(f"block_gap: {len(c['rec'])} reconstruction points, {len(c['gt'])} GT points, {len(c['gaps'])} on gaps")
    return c


# ---- crop -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("row", ["object", "large"])
def test_crop_at_scene_size_bit_for_bit(row, obj, large):
    c = obj if row == "object" else large
    t = c["S"] if row == "object" else tnt_cases.similarity(1.0002, [0.3, 1, 0.1], 2e-3, [0.05, -0.02, 0.01])
    out, keep = ops.crop_points(_d(c["rec"]), c["crop"]["orthogonal_axis"], c["crop"]["axis_min"], c["crop"]["axis_max"],
                                c["crop"]["polygon"], t)
    moved = to.transform(c["rec"], t)
    assert out.cpu().numpy().tobytes() == moved.tobytes()
    want = to.crop_v(moved, c["crop"])
    got = keep.cpu().numpy()
    assert (got == want).all(), f"{(got != want).sum()} of {len(want)} differ"
    assert 0 < want.sum() < len(want)
    print(f"{row}: {int(want.sum())} of {len(want)} kept")


@pytest.mark.parametrize("nv", [128, 129])
def test_crop_polygon_limits(nv):
    rng = np.random.RandomState(9)
    poly = sc.star_polygon(nv, (3.0, -2.0))
    pts = np.concatenate([rng.uniform(-1.2, 1.2, (200000, 3)) + [3.0, -2.0, 0.0], poly + [0.0, 0.0, 0.25]])
    cv = {"orthogonal_axis": 2, "axis_min": -0.5, "axis_max": 0.5, "polygon": poly}
    if nv > 128:
        with pytest.raises(RuntimeError, match="128"):
            ops.crop_points(_d(pts), 2, -0.5, 0.5, poly)
        return
    _, keep = ops.crop_points(_d(pts), 2, -0.5, 0.5, poly)
    want = to.crop_v(pts, cv)
    assert (keep.cpu().numpy() == want).all() and 0 < want.sum() < len(pts)


# ---- voxel down-sampling --------------------------------------------------------------------------------------------------

def _check_voxels(pts, s, name):
    want = to.voxel_downsample_v(pts, s)
    got = ops.voxel_downsample(_d(pts), s).cpu().numpy()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0, err_msg=name)
    return got


@pytest.mark.parametrize("row,div", [("object", 1), ("object", 2), ("large", 1), ("large", 2)],
                         ids=["object-tau", "object-tau/2", "large-tau", "large-tau/2"])
def test_voxel_downsample_of_whole_clouds(row, div, obj, large):
    c = obj if row == "object" else large
    got = _check_voxels(c["rec"], c["tau"] / div, row)
    print(f"{row} at tau/{div}: {len(c['rec'])} points -> {len(got)} voxels")


@pytest.mark.parametrize("row", ["64_bits", "65_bits", "x_int32", "x_int32_over"])
def test_voxel_key_widths_and_the_int32_limit(row):
    """22 + 21 + 21 = 64 key bits fit one key; 22 + 21 + 22 is sorted by (y, z), then stably by x.  Open3D's bound check
    refuses an extent beyond voxel_size * (2^31 - 1), so the largest accepted index is 2^31 - 2; one voxel more is refused."""
    pts, s, err = sc.voxel_keys_rows()[row]
    top = np.floor((pts.max(0) - (pts.min(0) - s / 2)) / s).astype(np.int64)
    bits = [int(v).bit_length() for v in top]
    if err:
        with pytest.raises(RuntimeError, match=err):
            ops.voxel_downsample(_d(pts), s)
        return
    assert sum(bits) == {"64_bits": 64, "65_bits": 65, "x_int32": 31 + 14}[row] and (row != "x_int32" or top[0] == 2 ** 31 - 2)
    _check_voxels(pts, s, row)


# ---- nearest distances as score asks for them -----------------------------------------------------------------------------

def _score_distances(to_pts, frm_pts, tau, blocks=False):
    cap = 5 * tau
    allp = np.concatenate([to_pts, frm_pts])
    box = [(allp.min(0) - cap).tolist(), (allp.max(0) + cap).tolist()]
    got = ops.nearest_distance(_d(to_pts), _d(frm_pts), box, cap, blocks=blocks).cpu().numpy()
    return got, box


def _check_capped(got, true, cap, name):
    below = true < cap * (1 - 1e-12)
    above = true > cap * (1 + 1e-12)
    np.testing.assert_allclose(got[below], true[below], rtol=1e-12, atol=0, err_msg=name)
    assert (got[above] == cap).all(), name
    assert (got <= cap).all()


def _in_blocks(q, lo, hi, m):
    """MaxDistCP's block membership per query, Low_k = lo + k m, High_k = Low_k + m, every operation rounded on its own."""
    rng = np.floor((np.asarray(hi) - np.asarray(lo)) / m)
    inside = np.ones(len(q), dtype=bool)
    for a in range(3):
        k0 = np.floor((q[:, a] - lo[a]) / m)
        hit = np.zeros(len(q), dtype=bool)
        for dk in (-1.0, 0.0, 1.0):
            k = k0 + dk
            low = lo[a] + k * m
            hit |= (k >= 0) & (k <= rng[a]) & (q[:, a] >= low) & (q[:, a] < low + m)
        inside &= hit
    return inside


@pytest.mark.parametrize("row", ["object", "large", "block_gap"])
def test_nearest_distance_as_score_calls_it(row, obj, obj_oracle, large, block_gap):
    """Both directions, every query, against the uncapped cKDTree distance: equal to 1e-12 relative below 5 tau, exactly
    5 tau above.  object: the round-2 clouds (voxel tau / 2 of the cropped clouds, the kind score measures)."""
    if row == "object":
        s, g, tau = obj_oracle["rounds"][1]["source"], obj_oracle["rounds"][1]["target"], obj["tau"]
    else:
        c = large if row == "large" else block_gap
        s, g, tau = c["rec"], c["gt"], c["tau"]
    for name, a, b in (("rec->gt", g, s), ("gt->rec", s, g)):
        got, box = _score_distances(a, b, tau)
        true = cKDTree(a).query(b, k=1, workers=-1)[0]
        _check_capped(got, true, 5 * tau, f"{row} {name}")
        print(f"{row} {name}: {len(b)} queries, {(true < 5 * tau).mean():.4f} below 5 tau")
    if row == "block_gap":
        _gap_queries(block_gap)


def _gap_queries(c):
    """The queries on MaxDistCP's gaps get their true distance from the capped search; the blocked search (the DTU
    semantics) gives them 5 tau, as MaxDistCP does."""
    tau, cap = c["tau"], 5 * c["tau"]
    d_rec, box = _score_distances(c["gt"], c["rec"], tau)
    assert box[0] == c["lo"].tolist()  # the anchor holds the minimum: the gaps are the score box's
    true_rec = cKDTree(c["gt"]).query(c["rec"][c["gap_rec"]], k=1)[0]
    assert (true_rec < tau).all()
    np.testing.assert_allclose(d_rec[c["gap_rec"]], true_rec, rtol=1e-12, atol=0)
    blocked, _ = _score_distances(c["gt"], c["rec"], tau, blocks=True)
    member = _in_blocks(c["rec"], box[0], box[1], cap)
    true_all = cKDTree(c["gt"]).query(c["rec"], k=1)[0]
    want_blocked = np.where(member, np.minimum(true_all, cap), cap)
    _check_capped(blocked, want_blocked, cap + 1.0, "blocked rec->gt")  # a cap above every value: compare all to 1e-12
    n_gap = int((~member[c["gap_rec"]]).sum())
    print(f"block_gap: {len(c['gaps'])} queries on gaps; {n_gap} of the {len(c['gap_rec'])} reconstruction ones are in no block "
          f"(the blocked search gives them 5 tau although their true distance is below tau)")
    assert n_gap > 0


def test_cell_faces_of_the_ring_search():
    """Queries whose computed fine cell is off by one, with the true nearest target unvisited after fine ring k yet less
    than k cells away and a visited one just farther (tnt_scale_cases.cell_face_trios), at the default search cell of
    nearest_distance (capped and blocked) and of icp.  The search must end only once the unvisited cells are provably
    farther (the kCellSlack margin); the distance must be the exact nearest one and the index the true nearest target's."""
    tau = 0.003
    cap = 5 * tau
    cell = cap / 8
    q, v, t, k = sc.cell_face_trios(cell)
    corners = np.array([[0.0, -5.0, -5.0], [130.0, 5.0, 5.0]])  # a wide box: the default cell is clamped to max_dist / 8
    targets = np.concatenate([v, t, corners])
    d2 = ((targets[None, :, 0] - q[:, None, 0]) * (targets[None, :, 0] - q[:, None, 0]) +
          (targets[None, :, 1] - q[:, None, 1]) * (targets[None, :, 1] - q[:, None, 1])) + \
         (targets[None, :, 2] - q[:, None, 2]) * (targets[None, :, 2] - q[:, None, 2])
    want_idx = d2.argmin(1)
    want = np.sqrt(d2.min(1))
    assert (want_idx == len(v) + np.arange(len(q))).all() and (want < k * cell).all()
    allp = np.concatenate([targets, q])
    box = [(allp.min(0) - cap).tolist(), (allp.max(0) + cap).tolist()]
    assert ops.default_search_cell(len(targets), box, cap) == cell
    for blocks in (False, True):
        got = ops.nearest_distance(_d(targets), _d(q), box, cap, blocks=blocks).cpu().numpy()
        member = _in_blocks(q, box[0], box[1], cap) if blocks else np.ones(len(q), bool)
        assert (got == np.where(member, want, cap)).all(), (blocks, got - want)
    assert ops.default_search_cell(len(targets), [targets.min(0), targets.max(0)], cap) == cell
    res = ops.icp(_d(q), _d(targets), cap, max_iteration=0, return_correspondences=True)
    assert res["correspondence_set"].cpu().numpy().tolist() == want_idx.tolist()
    print(f"cell faces: {len(q)} queries, rings {k.tolist()}")


# ---- ICP correspondences and moments at round-3 size ----------------------------------------------------------------------

def _icp_query(src, tgt, r):
    """One pmb200_icp_query at the identity, as ops.icp makes it -> (corr int64 [n], moments [18], origin [3])."""
    lib = _native.lib()
    s, t = _d(src), _d(tgt)
    lo, hi = tgt.min(0), tgt.max(0)
    origin = (lo + hi) / 2
    cell = ops.default_search_cell(len(tgt), [lo, hi], r)
    tws = ops._workspace(lib.pmb200_icp_target_workspace_bytes(len(tgt)), "icp_target_workspace_bytes", s.device)
    qws = ops._workspace(lib.pmb200_icp_query_workspace_bytes(len(src)), "icp_query_workspace_bytes", s.device)
    corr = torch.empty(len(src), dtype=torch.int32, device=DEV)
    mom = torch.empty(18, dtype=torch.float64, device=DEV)
    _native.check(lib.pmb200_icp_target(t.data_ptr(), len(tgt), float(cell), tws.data_ptr(), tws.numel(), ops._stream(t)), "icp_target")
    rc = lib.pmb200_icp_query(s.data_ptr(), len(src), ops._host_4x4(None), (ctypes.c_double * 3)(*origin.tolist()), float(r),
                              tws.data_ptr(), len(tgt), float(cell), corr.data_ptr(), mom.data_ptr(), qws.data_ptr(), qws.numel(),
                              ops._stream(s))
    _native.check(rc, "icp_query")
    return corr.cpu().numpy().astype(np.int64), mom.cpu().numpy(), origin


def test_icp_correspondences_and_moments_at_round_3_size(obj, obj_oracle):
    """Round 3 of `object`: the uniform-strided source (over 3M points) against the GT (over 2M), max distance 2 tau, with
    deliberate ties added.

    Every index against to.correspondences_v, ties included.  The moments: the kernel forms each term exactly as numpy does
    here (p = x - o, q = y - o, q_a p_b, ((p0 p0 + p1 p1) + p2 p2), d^2 = ((dx dx + dy dy) + dz dz)), so only the order of
    the additions differs from the exactly rounded sum S* = fsum(t).  That order: each thread adds its L = ceil(n / (G 256))
    terms in a chain from 0.0 (G = min(ceil(n / 256), 65535) blocks), each block sums its 256 threads in a tree of depth 8,
    then thread j of one block adds the partials of blocks j, j + 256, ... (ceil(G / 256) of them) in a chain, and a last
    tree of depth 8 sums those.  A term thus passes through at most D = L + 8 + ceil(G / 256) + 8 rounded additions, and
    the standard bound for any such summation tree gives |S - sum t| <= gamma_D sum |t|, gamma_D = D u / (1 - D u).  With
    |S* - sum t| <= u |S*|:  |S - S*| <= gamma_D sum |t| + u |S*|.  The count moment is an exact integer."""
    rnd = obj_oracle["rounds"][2]
    src, tgt, r = rnd["source"], rnd["target"], 2 * obj["tau"]
    # deliberate ties: 100k target points again under shuffled indices (identical candidates), and an exact 2^-8 lattice
    # beside the cloud with sources on its half-integer positions (distinct candidates at exactly the same distance)
    rng = np.random.RandomState(12)
    lat, lat_src = sc.lattice_ties([33.0, -17.0, 6.0])
    tgt = np.concatenate([tgt, tgt[rng.randint(0, len(tgt), 100_000)], lat])
    tgt = tgt[rng.permutation(len(tgt))]
    src = np.concatenate([src, lat_src])
    corr, mom, o = _icp_query(src, tgt, r)
    want, d2 = to.correspondences_v(src, tgt, r)
    assert (corr == want).all(), f"{(corr != want).sum()} of {len(want)} indices differ"
    dk, ik = cKDTree(tgt).query(src, k=8, distance_upper_bound=r * (1 + 1e-9), workers=-1)
    e = ((tgt[np.minimum(ik, len(tgt) - 1)] - src[:, None, :]) ** 2)
    e = np.where(ik < len(tgt), (e[..., 0] + e[..., 1]) + e[..., 2], np.inf)
    at_best = (e == e.min(1, keepdims=True)) & np.isfinite(e)
    tied = int((at_best.sum(1) >= 2).sum())
    assert tied > 10_000, tied  # rows whose nearest distance is reached by two or more targets
    ok = want >= 0
    n = int(ok.sum())
    assert mom[0] == n and n > 2_000_000
    p, q = src[ok] - o, tgt[want[ok]] - o
    terms = [d2[ok]] + [p[:, a] for a in range(3)] + [q[:, a] for a in range(3)] + \
            [q[:, a] * p[:, b] for a in range(3) for b in range(3)] + [(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) + p[:, 2] * p[:, 2]]
    g = min(-(-len(src) // 256), 65535)
    depth = -(-len(src) // (g * 256)) + 8 + -(-g // 256) + 8
    gamma = depth * U / (1 - depth * U)
    for k, t in enumerate(terms, start=1):
        exact = math.fsum(t.tolist())
        bound = gamma * float(np.abs(t).sum()) + U * abs(exact)
        assert abs(mom[k] - exact) <= bound, (k, mom[k], exact, bound)
    print(f"round 3 correspondences: {len(src)} source, {len(tgt)} target, {n} matched, {tied} tied, summation depth {depth}")


# ---- ICP loop, one round each ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [0, 1, 2], ids=["round1", "round2", "round3"])
def test_icp_rounds_of_object(k, obj, obj_oracle):
    rnd = obj_oracle["rounds"][k]
    dist = (80, 20, 2)[k] * obj["tau"]
    got = ops.icp(_d(rnd["source"]), _d(rnd["target"]), dist, max_iteration=20)
    if got["iterations"] != rnd["iterations"] and _ties_at_threshold(rnd["deltas"]):
        pytest.skip(f"round {k + 1}: a convergence decision within 1e-12 of the 1e-6 threshold: {rnd['deltas']}")
    assert got["iterations"] == rnd["iterations"]
    assert [h[0] for h in got["history"]] == [h[0] for h in rnd["history"]]
    np.testing.assert_allclose([h[1] for h in got["history"]], [h[1] for h in rnd["history"]], rtol=1e-9)
    np.testing.assert_allclose(got["transformation"], rnd["icp"], atol=1e-9, rtol=0)


# ---- score at a fixed transform -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("row", ["block_gap", "hist_edges"])
def test_score_at_the_identity_matches_the_oracle_exactly(row, block_gap):
    c = block_gap if row == "block_gap" else sc.hist_edges_row()
    got = tnt_eval.score(_d(c["rec"]), _d(c["gt"]), c["crop"], np.eye(4), c["tau"])
    want = to.score_v(c["rec"], c["gt"], c["crop"], np.eye(4), c["tau"])
    for k in ("n_source_scored", "n_gt_scored", "precision_count", "recall_count", "precision", "recall", "fscore"):
        assert got[k] == want[k], (k, got[k], want[k])
    assert (np.asarray(got["cum_precision"]) == want["cum_precision"]).all()
    assert (np.asarray(got["cum_recall"]) == want["cum_recall"]).all()
    if row == "hist_edges":
        e = c["distances"]
        assert got["n_source_scored"] == len(e) and got["precision_count"] == int((e < c["tau"]).sum())


# ---- evaluate_scene end to end --------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def stride_half():
    _need(12 << 30)
    c = sc.stride_half_row()
    print(f"stride_half: {len(c['rec'])} reconstruction points, {len(c['gt'])} GT points")
    return c


def _oracle_chain_from(got, c, init, first=None):
    """The oracle's refinement and scoring, each round started from the GPU's estimate before it and the score taken at the
    GPU's final transformation.  The GPU's ICP agrees with the oracle's to about 1e-12 (its moments are summed in another
    order); with millions of points some point lies that close to a voxel face or crop edge, so a chain run on from the
    oracle's own estimates would differ by a voxel for reasons that are not errors.  `first`: the oracle's record of round 1
    (whose start, init, is the same for both)."""
    rec, gt, crop, tau = c["rec"], c["gt"], c["crop"], c["tau"]
    starts = [np.asarray(init, np.float64)] + [np.asarray(r["transformation"]) for r in got["rounds"][:2]]
    rounds = []
    for k, (method, voxel, dist) in enumerate((("voxel", tau, 80 * tau), ("voxel", tau / 2, 20 * tau), ("uniform", None, 2 * tau))):
        if k == 0 and first is not None:
            rounds.append(first)
            continue
        s = to.transform(rec, starts[k])
        s = s[to.crop_v(s, crop)]
        g = gt[to.crop_v(gt, crop)]
        n_cropped = len(s)
        s, g = (to.voxel_downsample_v(s, voxel), to.voxel_downsample_v(g, voxel)) if method == "voxel" else \
               (to.uniform_downsample(s), to.uniform_downsample(g))
        r = to.icp_v(s, g, dist, max_iteration=20)
        if r["iterations"] != got["rounds"][k]["iterations"] and _ties_at_threshold(r["deltas"]):
            pytest.skip(f"round {k + 1}: a convergence decision within 1e-12 of the 1e-6 threshold: {r['deltas']}")
        rounds.append({"n_source": len(s), "n_target": len(g), "iterations": r["iterations"], "correspondences": r["correspondences"],
                       "transformation": r["transformation"] @ starts[k], "n_source_cropped": n_cropped})
    want = {"rounds": rounds, "transformation": rounds[-1]["transformation"]}
    want.update(to.score_v(rec, gt, crop, np.asarray(got["transformation"]), tau))
    return want


@pytest.mark.parametrize("row", ["object", "stride_half"])
def test_evaluate_scene_at_scene_size(row, request):
    """evaluate_scene against the oracle chain of _oracle_chain_from: what test_gpu_tnt_eval's _check_scene asserts (counts,
    precision, recall, F and both curves exactly; each round's sizes, iterations and correspondences exactly, its
    transformation within 1e-9), round 3 strided, and a rerun giving the same result."""
    if row == "object":
        c, oracle = request.getfixturevalue("obj"), request.getfixturevalue("obj_oracle")
        init, first = c["init"], oracle["rounds"][0]
    else:
        c = request.getfixturevalue("stride_half")
        init, first = c["S"], None
    got = tnt_eval.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"], device=DEV)
    want = _oracle_chain_from(got, c, init, first)
    _check_scene(got, want)
    r3 = got["rounds"][2]
    cropped = want["rounds"][2]["n_source_cropped"]
    k = max(int(round(cropped / sc.UNIFORM_MAX_POINTS)), 1)
    assert k >= 2 and r3["n_source"] == -(-cropped // k) < cropped  # round 3 strided
    if row == "stride_half":
        assert cropped == sc.STRIDE_HALF and k == 2
    print(f"{row}: precision {got['precision']:.6f} recall {got['recall']:.6f}; round 3 {cropped} cropped -> {r3['n_source']}")
    again = tnt_eval.evaluate_scene(c["rec"], c["gt"], c["crop"], init, c["tau"], device=DEV)
    assert again == got
