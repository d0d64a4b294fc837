"""The depth-map kernels at the source-view counts and image sizes the evaluation configurations run, element by element
against the oracle evaluated in float64.

View counts.  num_views of the evaluation configurations: DTU 5 sources at 1600x1200, ETH3D high-res 7 at 2688x1792
(image_max_dim 2688), Tanks and Temples 7 at 1920x1080, and reconstruct's default, every source of a pair.txt (10 in the
usual ones), up to PMB200_MAX_VIEWS = 16.  K-A's lane-to-view mapping, its view-weight registers (PMB200_MAX_VIEWS * PIX /
32 per lane in K-A4), the ring slot each item's views start in, the V loops of aggregate_views / aggregate_views_score and
the per-view extents of the ragged pack all depend on V; tests/test_gpu_kernels_at_scale.py runs V = 4 only.

Which K-A kernel runs.  The library's default is generation 3 (kTuneDefaults in pm_kernels.cu: generation 4 measured
slower at every bench shape), so a default call never reaches K-A4; every uniform row is therefore run twice, at the
default and with ka_gen = 4, and the library's record of each call's launch (ops.last_warp_corr_kernel) shows that each
ran as asked.  The ragged rows run warp_corr3_views_kernel: generation 4 takes no per-view extents.

Map sizes.  1920x1080 gives an odd-height stage-3 map (240x135, then 480x270 and 960x540); 2688x1792 gives stage-1
maps of 1344x896.  K-A', K-C and K-B do not depend on V and run at these two sizes only.  Their K-B plans are plans the
at-scale rows already reach (test_new_sizes_select_no_new_kb_branch).

Bounds: the at-scale file's, derived in its docstring, imported unchanged.  The float64 references are evaluated in chunks
of CHUNK_ELEMS elements per intermediate."""
import pytest
import torch
import torch.nn.functional as F

from patchmatchnet_b200 import ops, synthetic
from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet
from tests.test_gpu_kernels_at_scale import (DEV, EPS, F64, KB_ROWS, KC_ROWS, OC_ROWS, SIM_DIMS, SYNTHETIC, STAGE_DOWN,
                                             aggregate_reference, assert_within, check_adaptive_eval, check_init_propagate,
                                             check_ka_ops, check_offset_corr, ka_case, ka_device, ka_references, kb_branch,
                                             kb_plan, random_head, shape_table, smooth)
from tests.test_gpu_kernels_at_scale import row as at_scale_row

# (name, B, image height, image width, source views)
CONFIGS = (("tnt", 1, 1080, 1920, 7), ("eth3d", 1, 1792, 2688, 7), ("dtu", 1, 1200, 1600, 5), ("pair10", 1, 1200, 1600, 10))
FULL = ("tnt", "eth3d")  # every iteration of every stage; the others the first iteration of each stage

# image sizes (H, W) of the sources of the ragged rows: stage s divides each by STAGE_DOWN[s]
ETH3D_MIXED = [(1792, 2688), (2688, 1792), (1792, 2688), (1200, 1600), (2688, 1792), (1792, 2688), (2688, 1792)]
RAGGED16 = [(512, 640), (640, 512), (256, 320), (384, 480)] * 4


def first_iterations(rows):
    return [r for r in rows if r["name"].endswith("/it1")]


def view_count_table():
    rows = []
    for name, B, H, W, V in CONFIGS:
        t = shape_table(((name, B, H, W),), V=V)
        rows += t if name in FULL else first_iterations(t)
    for name, V in (("synthetic/V1", 1), ("synthetic/V9", 9), ("synthetic/V16", 16)):
        rows += first_iterations(shape_table(((name, 1, 512, 640),), V=V))
    for name, sizes, H, W in (("eth3d-mixed", ETH3D_MIXED, 1792, 2688), ("synthetic/V16-ragged", RAGGED16, 512, 640)):
        for r in first_iterations(shape_table(((name, 1, H, W),), V=len(sizes))):
            down = STAGE_DOWN[int(r["name"].split("/s")[-1][0])]
            rows.append(dict(r, sizes=[(h // down, w // down) for h, w in sizes]))
    return rows


def row(name):
    return next(r for r in view_count_table() if r["name"] == name)


KA_ROWS = [r["name"] for r in view_count_table()]
SIZE_ROWS = [r["name"] for r in view_count_table() if r["name"].split("/")[0] in FULL]  # K-A', K-C, K-B


def test_view_count_table():
    t = {r["name"]: r for r in view_count_table()}
    assert len(t) == 5 + 5 + 3 + 3 + 3 * 3 + 3 + 3
    assert (t["tnt/s3/it1"]["H"], t["tnt/s3/it1"]["W"]) == (135, 240) and (t["tnt/s1/it1"]["H"], t["tnt/s1/it1"]["W"]) == (540, 960)
    assert (t["eth3d/s1/it1"]["H"], t["eth3d/s1/it1"]["W"]) == (896, 1344)
    assert {r["V"] for r in t.values()} == {1, 5, 7, 9, 10, 16}
    assert t["eth3d-mixed/s2/it1"]["sizes"][:2] == [(448, 672), (672, 448)] and len(t["synthetic/V16-ragged/s1/it1"]["sizes"]) == 16
    # the at-scale rows are unchanged by the V argument of shape_table
    assert all(r["V"] == 4 for r in shape_table()) and len(shape_table()) == 4 * 5


def test_new_sizes_select_no_new_kb_branch():
    """K-B's planner picks its block shape from the map size.  At the stage maps of 1920x1080 and 2688x1792 it selects
    only plans that the at-scale rows already run (TP=32 with DY = 8 or 4): no new branch."""
    ops.set_tuning("reset")
    plan = lambda r: kb_plan(r["B"], r["D"], r["H"], r["W"], r["K"])
    old = {plan(r) for r in shape_table() + SYNTHETIC}
    new = {name: plan(row(name)) for name in SIZE_ROWS}
    assert set(new.values()) <= old, {n: p for n, p in new.items() if p not in old}
    assert {kb_branch(p, row(n)["D"]) for n, p in new.items()} == {"TP=32 DY=8", "TP=32 DY=4"}
    # the K-A', K-C and K-B rows of the at-scale file exist under the names it uses
    assert all(at_scale_row(n) for n in OC_ROWS + KC_ROWS + KB_ROWS)


def test_last_warp_corr_kernel_is_cleared_by_a_call_that_fails_its_checks():
    from patchmatchnet_b200 import _native

    lib = _native.lib()
    assert lib.pmb200_warp_corr(None, None, None, None, None, None, 1, 1, 8, 8, 4, 4, 4, 4, 1, None) != 0
    assert ops.last_warp_corr_kernel() == -1


def ka_kernels(calls):
    """Run each call -> the K-A kernel each one launched, as the library records it (ops.last_warp_corr_kernel: 4 or 3,
    the generation; 0 the generic kernel)."""
    out = []
    for call in calls:
        call()
        out.append(ops.last_warp_corr_kernel())
    return out


def check_ka_extras(tag, r, case, src, heads):
    """The K-A outputs check_ka_ops does not take: warp_corr_score into the .y lanes of an interleaved xs buffer (the
    score itself is checked there; here it must be the same bits, the .x lanes untouched) and aggregate_views on the
    kernel's own kept similarities and view weights (rounding only: the (2V + 2) eps term of aggregate_reference)."""
    B, D, H, W, G, V = r["B"], r["D"], r["H"], r["W"], r["G"], r["V"]
    ref_n, _, rt, depth, vw = ka_device(case, stack=False)
    sim_head, pw_head = heads
    score = ops.warp_corr_score(ref_n, src, rt, depth, G, vw, sim_head.folded())
    xs = ops.alloc_xs(B, D, H, W, DEV).fill_(-7.0)
    ops.warp_corr_score(ref_n, src, rt, depth, G, vw, sim_head.folded(), xs=xs)
    assert torch.equal(xs[..., 1], score) and bool((xs[..., 0] == -7.0).all()), f"{tag} warp_corr_score into xs"
    del score, xs
    got_vw, kept = ops.warp_corr_view_weights(ref_n, src, rt, depth, G, pw_head.folded(), keep_sims=True)
    kept64 = kept.double()
    agg, agg_b = aggregate_reference(list(kept64), [torch.zeros_like(kept64[0])] * V, got_vw.double())
    del kept64
    assert_within(f"{tag} aggregate_views", ops.aggregate_views(kept, got_vw), agg, agg_b, SIM_DIMS[1:])


@pytest.mark.gpu
@pytest.mark.parametrize("name", KA_ROWS)
def test_warp_corr_ops_at_view_counts(name):
    """Every K-A output (per-view similarities, the weighted average, the score and view-weight epilogues, the kept
    similarities, aggregate_views, aggregate_views_score) at one row, under each K-A kernel that row can run."""
    r = row(name)
    sizes = r.get("sizes")
    case = ka_case(r, seed=r["H"] + r["D"] + r["V"], sizes=sizes)
    sims, bounds = ka_references(case, r["G"])
    heads = (random_head(SimilarityNet, r["G"], 1).to(DEV), random_head(PixelwiseNet, r["G"], 2).to(DEV))
    if sizes is None:
        src = ka_device(case)[1]
        runs = [("default", {}, 3), ("ka_gen=4", {"ka_gen": 4}, 4)]
    else:  # the *_views entry points: generation 3's per-view form
        src = ops.pack_nhwc_views([s.to(DEV) for s in case["src"]])
        runs = [("default", {}, 3)]
    ref_n, _, rt, depth, vw = ka_device(case, stack=False)
    G = r["G"]
    try:
        with torch.no_grad():
            for label, knobs, want_gen in runs:
                ops.set_tuning("reset")
                for k, v in knobs.items():
                    ops.set_tuning(k, v)
                ran = ka_kernels([lambda: ops.warp_corr(ref_n, src, rt, depth, G), lambda: ops.warp_corr(ref_n, src, rt, depth, G, vw),
                                  lambda: ops.warp_corr_score(ref_n, src, rt, depth, G, vw, heads[0].folded()),
                                  lambda: ops.warp_corr_view_weights(ref_n, src, rt, depth, G, heads[1].folded(), keep_sims=True)])
                print(f"[K-A] {name} V={r['V']} {label}: generation {ran} (warp_corr, weighted, score, view weights)")
                assert ran == [want_gen] * 4, (label, ran)
                tag = f"{name} V={r['V']} {label}"
                # check_ka_ops's fp32-oracle check runs on maps up to 200 px, wider ones print the fp32 oracle's distance
                # from float64.  At exactly 200 px its docstring puts the fp32 oracle's own position rounding at about
                # what the check allows, and with 10 views one view exceeds it by itself (3.5e-5 for 3.4e-5 at
                # pair10/s3/it1); there the float64 comparison alone runs.
                fp32_oracle = sizes is None and label == "default" and max(r["H"], r["W"]) != 200
                check_ka_ops(tag, r, case, sims, bounds, heads, fp32_oracle=fp32_oracle, src=None if sizes is None else src)
                check_ka_extras(tag, r, case, src, heads)
    finally:
        ops.set_tuning("reset")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in SIZE_ROWS if n.endswith("/it1")])  # K-A' does not depend on D
def test_offset_corr_at_view_count_sizes(name):
    ops.set_tuning("reset")
    with torch.no_grad():
        check_offset_corr(name, row(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIZE_ROWS)
def test_init_propagate_at_view_count_sizes(name):
    ops.set_tuning("reset")
    check_init_propagate(name, row(name))


@pytest.mark.gpu
@pytest.mark.parametrize("name", SIZE_ROWS)
def test_adaptive_eval_at_view_count_sizes(name):
    ops.set_tuning("reset")
    check_adaptive_eval(name, row(name))


# ------------------------------------------------------------------------------------------------
# helpers of the depth-map forward at these view counts and sizes
# ------------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_relative_projection_up_to_the_view_limit():
    """rt = src @ inv(ref) for V = 1..16 against float64.  The kernel inverts ref in fp64 by Gauss-Jordan with partial
    pivoting and multiplies in fp64, then rounds once to fp32: eps |rt|.  The fp64 inverse X satisfies
    |X - inv| <= c_n u |inv| |A| |X| componentwise (u = 2^-53, c_n <= 4n for n = 4), the 4-term product adds (n + 1) u
    |S| |X|; the float64 reference (torch.linalg.inv) has the same bound, so both terms are counted twice."""
    u, n, B = 2.0 ** -53, 4, 2
    for stage in (3, 1):
        Kc, Ec = synthetic.make_cameras(B, 17, 1792, 2688)
        ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, stage)
        A = ref_proj.double()
        inv = torch.linalg.inv(A)
        dinv = 4 * n * u * (inv.abs() @ A.abs() @ inv.abs())
        for V in range(1, 17):
            got = ops.relative_projection(ref_proj.to(DEV), [m.to(DEV) for m in src_projs[:V]]).cpu()
            assert got.shape == (V, B, 12)
            for v in range(V):
                S = src_projs[v].double()
                want = S @ inv
                bnd = EPS * want.abs() + 2 * (S.abs() @ dinv + (n + 1) * u * (S.abs() @ inv.abs()))
                flat = lambda m: torch.cat([m[:, :3, :3].reshape(B, 9), m[:, :3, 3]], 1)
                assert_within(f"relative_projection s{stage} V={V} view {v}", got[v], flat(want), flat(bnd), ("b", "k"))


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(1080, 1920), (1792, 2688)])
def test_photometric_confidence_at_image_size(H, W):
    """The stage-1 probabilities (D = 8 at half the image size) to a confidence map at the image size.  float64: e =
    sum_d d p_d, k = trunc(e) clamped to [0, D-1], conf = sum of p over k-1..k+2, nearest-upsampled (h / H = 1/2 exactly
    here, so the source pixel is exact).  fp32: e is within (D + 2) eps e of the exact value, so where e lies that close
    to an integer either neighbouring k is right; the 4-term sum adds 3 eps conf (the 0.25 and 4 scalings are exact)."""
    g = torch.Generator().manual_seed(H)
    B, D, h, w = 1, 8, H // 2, W // 2
    prob = torch.softmax(3.0 * smooth(g, B, D, H=h, W=w, cell=2), dim=1).to(DEV)
    got = ops.photometric_confidence(prob, H, W)
    p = prob.double()
    e = (p * torch.arange(D, dtype=F64, device=DEV).view(1, D, 1, 1)).sum(1)
    de = (D + 2) * EPS * e
    padded = F.pad(p, (0, 0, 0, 0, 1, 2))  # p[k + j] for j = -1..2 at padded index k + 1 + j
    mass = lambda k: sum(padded.gather(1, (k + 1 + j).unsqueeze(1)).squeeze(1) for j in range(-1, 3))
    k_lo = torch.trunc(e - de).long().clamp(0, D - 1)
    k_hi = torch.trunc(e + de).long().clamp(0, D - 1)
    c_lo, c_hi = mass(k_lo), mass(k_hi)
    up = lambda t: t.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
    c_lo, c_hi, b_lo, b_hi = up(c_lo), up(c_hi), up(3 * EPS * c_lo), up(3 * EPS * c_hi)
    g64 = got.double()
    use_hi = (g64 - c_hi).abs() * b_lo < (g64 - c_lo).abs() * b_hi
    print(f"[photometric_confidence] {H}x{W}: {int((k_lo != k_hi).sum())} pixels within rounding of an integer index")
    assert_within(f"photometric_confidence {H}x{W}", got, torch.where(use_hi, c_hi, c_lo), torch.where(use_hi, b_hi, b_lo),
                  ("b", "y", "x"))


@pytest.mark.gpu
def test_upsample2x_add_from_an_odd_height_map():
    """FeatureNet's x2 upsample of the stage-3 map of a 1920x1080 view (240x135, 64 channels) plus the lateral map and a
    bias, against float64 F.interpolate(align_corners=False).  The kernel's sample positions and weights (multiples of
    1/4) are exact; the products and sums of the bilinear weights (6 roundings of terms bounded by the bilinear
    sample of |x|) and the two additions (y + bias, then the sum: 3 roundings of |y| + |bias| and the rest)."""
    g = torch.Generator().manual_seed(135)
    N, C, h, w = 1, 64, 135, 240
    x = smooth(g, N, C, H=h, W=w).to(DEV).contiguous(memory_format=torch.channels_last)
    y = smooth(g, N, C, H=2 * h, W=2 * w).to(DEV).contiguous(memory_format=torch.channels_last)
    bias = torch.randn(C, generator=g).to(DEV)
    up = lambda t: F.interpolate(t.double(), size=(2 * h, 2 * w), mode="bilinear", align_corners=False)
    for b in (None, bias):
        bb = torch.zeros(C, dtype=F64, device=DEV) if b is None else b.double()
        want = up(x) + y.double() + bb.view(1, C, 1, 1)
        bnd = 6 * EPS * up(x.abs()) + 3 * EPS * (y.double().abs() + bb.abs().view(1, C, 1, 1))
        assert_within(f"upsample2x_add 240x135 bias={b is not None}", ops.upsample2x_add(x, y, b), want, bnd, ("n", "c", "y", "x"))
