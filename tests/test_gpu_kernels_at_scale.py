"""The PatchMatch hot-path kernels (K-A, K-A', K-C, K-B) at the map sizes reconstruction and training run, and at every
launch shape the library can select, element by element against the oracle evaluated in float64.

Shape table.  Derived from synthetic.DEFAULT_NET_KWARGS and the stage modules: the three stage maps of a 1600x1200 view,
of a 1200x1600 (portrait) view, of the bench's 640x512 with B=1 and of 320x256 with B=2, with 4 source views.  The
launchers choose their block shape from the map size (pmb200_adaptive_eval_plan for K-B, the width rule of
pmb200_init_propagate for K-C), so small maps do not run the code that real images run.  A few synthetic rows reach the
branches the network never selects.

Error bounds.  Every bound is fixed from first principles, per element, before any comparison:
  * eps = 2^-24, the fp32 unit roundoff.  A sum of n products computed in fp32 (any order, fma or not) is within
    (n + 1) eps * sum|terms| of the exact sum; this is evaluated by running the same float64 oracle on the absolute
    values of the inputs (the "abs oracle"), so a bound follows the magnitude of each element rather than a global scale.
  * Coordinates: the kernels round the positions they sample at.  At position p the bilinear sample moves by at most
    dpos * (|df/du| + |df/dv|); the derivative is bounded by the largest neighbour difference of the sampled map around
    the cell (lipschitz_map, sampled at the same position), dpos by the fp32 arithmetic that forms p (project_bound for
    K-A, border_dpos for the border-clamped gathers).
  * The inputs are spatially smooth fields (random values on a 4-pixel lattice, bilinearly interpolated), as feature
    maps, scores and depths are; a coordinate error of a few 1e-4 pixels then moves a sample by ~1e-5 of its scale.
Alongside, the existing tight checks against the fp32 oracle (2e-5 of scale for K-A / K-A', the K-B / K-C bounds of
test_gpu_parity.py) are kept.

All fixtures and helpers live in this file.  The float64 references are evaluated in chunks of hypotheses so that one
chunk allocates well under 4 GB.
"""
import ctypes
import math
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import pm_oracle
from patchmatchnet_b200 import _native, ops, synthetic
from patchmatchnet_b200.net import PatchmatchNet
from patchmatchnet_b200.patchmatch import PixelwiseNet, SimilarityNet

DEV = "cuda:0"
EPS = 2.0 ** -24
F64 = torch.float64
H100_SMS = 132  # the planner's answers on the CPU are for an H100; on the GPU the device's own SM count is used
N_SRC = 4  # source views per reference view
CHUNK_ELEMS = 1 << 25  # float64 elements of one [B,C,d,H,W] intermediate: 256 MB, a chunk holds a handful of them

# ------------------------------------------------------------------------------------------------
# shape table
# ------------------------------------------------------------------------------------------------

VIEWS = (("1600x1200", 1, 1200, 1600), ("1200x1600", 1, 1600, 1200), ("640x512", 1, 512, 640), ("320x256", 2, 256, 320))
STAGE_DOWN = {3: 8, 2: 4, 1: 2}  # FeatureNet's output strides


def stage_config(stage):
    i, kw = stage - 1, synthetic.DEFAULT_NET_KWARGS
    return dict(C=PatchmatchNet.FEATURES[i], G=PatchmatchNet.GROUPS[i], dil=kw["propagation_range"][i],
                K=kw["evaluate_neighbors"][i], iters=kw["patchmatch_iteration"][i], Ns=kw["patchmatch_num_sample"][i],
                Kp=kw["propagate_neighbors"][i], scale=kw["patchmatch_interval_scale"][i])


def stage_iterations(stage):
    """(mode, Ns, Kp, D, inverse) of every iteration, as PatchMatch.forward runs them (patchmatch.py:520-547)."""
    c = stage_config(stage)
    out = []
    for it in range(1, c["iters"] + 1):
        last1 = stage == 1 and it == c["iters"]
        kp = c["Kp"] if c["Kp"] > 0 and not last1 else 0
        if stage == 3 and it == 1:  # the coarsest stage starts without a depth map: 48 random samples
            mode, ns = ops.MODE_RANDOM, 48
        elif c["Ns"] == 1:
            mode, ns = ops.MODE_PASSTHROUGH, 1
        else:
            mode, ns = ops.MODE_PERTURB, c["Ns"]
        out.append(dict(mode=mode, Ns=ns, Kp=kp, D=ns + kp, inverse=last1))
    return out


def shape_table(views=VIEWS, V=N_SRC):
    """Every iteration of every stage of each (name, B, image height, image width) in `views`, with V source views."""
    rows = []
    for view, B, Hi, Wi in views:
        for stage in (3, 2, 1):
            c = stage_config(stage)
            for it, itc in enumerate(stage_iterations(stage), 1):
                rows.append(dict(name=f"{view}/s{stage}/it{it}", B=B, H=Hi // STAGE_DOWN[stage], W=Wi // STAGE_DOWN[stage],
                                 V=V, C=c["C"], G=c["G"], dil=c["dil"], K=c["K"], scale=c["scale"], **itc))
    return rows


# rows for branches the network never selects
SYNTHETIC = [
    # K-B TP=8 (the tile of 32 or 16 pixels exceeds 48 KB: D > 165 with K=9) and K-C's generic kernel (D > 64)
    dict(name="synthetic/D192", B=1, H=150, W=200, V=N_SRC, C=64, G=8, dil=2, K=9, scale=0.025, mode=ops.MODE_PERTURB,
         Ns=176, Kp=16, D=192, inverse=False),
    # K-C init_propagate_kernel<8> (Kp > 0, D <= 8)
    dict(name="synthetic/Ns4Kp4", B=1, H=300, W=400, V=N_SRC, C=32, G=8, dil=4, K=9, scale=0.0125, mode=ops.MODE_PERTURB,
         Ns=4, Kp=4, D=8, inverse=False),
    # K-B TP=32 with DY = D < 4
    dict(name="synthetic/D3", B=1, H=150, W=200, V=N_SRC, C=64, G=8, dil=2, K=9, scale=0.025, mode=ops.MODE_PERTURB,
         Ns=3, Kp=0, D=3, inverse=False),
]


def row(name):
    return next(r for r in shape_table() + SYNTHETIC if r["name"] == name)


def kb_plan(B, D, H, W, K, sms=H100_SMS):
    out = (ctypes.c_int * 3)()
    rc = _native.lib().pmb200_adaptive_eval_plan(B, D, H, W, K, sms, out)
    assert rc == 0, _native.lib().pmb200_last_error().decode()
    return tuple(out)


def kb_branch(plan, D):
    tp, dy, _ = plan
    if tp == 32:
        return "TP=32 DY=D<4" if dy == D and D < 4 else f"TP=32 DY={dy}"
    return f"TP={tp}"


def kc_kernel(Ns, Kp):
    """Which K-C kernel pmb200_init_propagate launches (csrc/pm_kernels.cu, the width rule of the launcher)."""
    D = Ns + Kp
    if Kp == 0 and D <= 64:
        return "init_only"
    for width in (8, 16, 32, 64):
        if D <= width:
            return f"width{width}"
    return "generic"


def test_shape_table_reaches_every_launch_branch():
    ops.set_tuning("reset")
    net = shape_table()
    kb = lambda rows: {kb_branch(kb_plan(r["B"], r["D"], r["H"], r["W"], r["K"]), r["D"]) for r in rows}
    kc = lambda rows: {kc_kernel(r["Ns"], r["Kp"]) for r in rows}
    # the network alone: stage 3 of a 1600x1200 view runs TP=32/DY=8, the bench's stage 3 TP=16
    assert row("1600x1200/s3/it1")["D"] == 64 and row("1600x1200/s3/it2")["D"] == 32
    assert row("1600x1200/s2/it1")["D"] == 16 and row("1600x1200/s1/it1")["D"] == 8
    assert kb_plan(1, 64, 150, 200, 9)[:2] == (32, 8) and kb_plan(1, 32, 150, 200, 9)[:2] == (32, 8)
    assert kb(net) == {"TP=32 DY=4", "TP=32 DY=8", "TP=16"}
    assert kc(net) == {"init_only", "width16", "width32", "width64"}
    # each synthetic row adds a branch the network does not reach, and together they reach all of them
    for r in SYNTHETIC:
        assert not (kb([r]) <= kb(net) and kc([r]) <= kc(net)), r["name"]
    assert kb(net + SYNTHETIC) == {"TP=32 DY=D<4", "TP=32 DY=4", "TP=32 DY=8", "TP=16", "TP=8"}
    assert kc(net + SYNTHETIC) == {"init_only", "width8", "width16", "width32", "width64", "generic"}


KB_KNOB_SHAPES = ((32, 8), (32, 4), (16, 16), (16, 8), (8, 32), (8, 16), (64, 4), (32, 2))  # tools/kbench.py's K-B loop
KA_KNOBS = ([dict(ka_gen=4, ka4_nw=nw, ka4_ctas=c, ka4_stages=st) for nw, c, st in
             ((4, 2, 2), (4, 2, 3), (4, 2, 4), (4, 3, 2), (4, 3, 3), (4, 4, 2), (8, 1, 4), (8, 2, 2), (8, 2, 3))]
            + [dict(ka_gen=3, ka3_dc=d, ka3_dc_vw=d, ka3_pipe=0) for d in (4, 8, 16)]
            + [dict(ka_gen=3, ka3_pipe=1), dict(ka_gen=3, ka3_pipe=1, ka3_minb=5),
               dict(ka_gen=4, ka4_nw=4, ka4_cap=24, ka4_grid=5), dict(ka_gen=4, ka4_nw=8, ka4_cap=40, ka4_grid=3)])


def test_planner_takes_every_kbench_block_shape():
    """The K-B knob test runs at stage 3 of a 1600x1200 view (D=64, K=9): every block shape tools/kbench.py sweeps is
    accepted there (the override is dropped silently when the tile would not fit 48 KB)."""
    try:
        for tp, dy in KB_KNOB_SHAPES:
            ops.set_tuning("reset")
            ops.set_tuning("kb_tp", tp)
            ops.set_tuning("kb_dy", dy)
            assert kb_plan(1, 64, 150, 200, 9)[:2] == (tp, dy)
    finally:
        ops.set_tuning("reset")
    assert kb_plan(1, 64, 150, 200, 9)[:2] == (32, 8)


# ------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------


def smooth(gen, *lead, H, W, cell=4):
    """Spatially smooth fp32 field [*lead, H, W]: N(0,1) values on a `cell`-pixel lattice, bilinearly interpolated."""
    h, w = H // cell + 2, W // cell + 2
    coarse = torch.randn(math.prod(lead), 1, h, w, generator=gen, dtype=F64)
    f = F.interpolate(coarse, size=((h - 1) * cell + 1, (w - 1) * cell + 1), mode="bilinear", align_corners=True)
    return f[..., :H, :W].reshape(*lead, H, W).float()


def lipschitz_map(f, zero_pad):
    """[N,C,H,W] -> [N,C,H,W]: at every texel, an upper bound of |df/du| + |df/dv| of the bilinear interpolant anywhere in
    the cells within two texels of it (zero_pad: the map is continued by zeros, as grid_sample's zeros padding; else by
    its border values).  Sampled bilinearly (border padding) at a position, it bounds the derivative there."""
    p = F.pad(f, (1, 1, 1, 1), mode="constant" if zero_pad else "replicate")
    dx = F.pad((p[..., :, 1:] - p[..., :, :-1]).abs(), (0, 1, 0, 0))
    dy = F.pad((p[..., 1:, :] - p[..., :-1, :]).abs(), (0, 0, 0, 1))
    m = F.max_pool2d(dx, 3, 1) + F.max_pool2d(dy, 3, 1)  # [N,C,H,W]: differences across the cells touching the texel
    return F.max_pool2d(m, 3, 1, padding=1)  # one texel more: the rounded position may sit in the next cell


def sample_pixels(maps, u, v, padding):
    """Bilinear sample of maps [B,C,Hs,Ws] at pixel coordinates u, v [B,d,H,W] (align_corners=True) -> [B,C,d,H,W]."""
    B, C, Hs, Ws = maps.shape
    _, d, H, W = u.shape
    grid = torch.stack((u * (2.0 / (Ws - 1)) - 1.0, v * (2.0 / (Hs - 1)) - 1.0), dim=-1).view(B, d * H, W, 2)
    return F.grid_sample(maps, grid, mode="bilinear", padding_mode=padding, align_corners=True).view(B, C, d, H, W)


def rt_matrix(rt):
    """[B,12] rot (row-major) + trans -> [B,4,4] with that exact relative projection (the oracle then inverts identity)."""
    B = rt.shape[0]
    m = torch.zeros(B, 4, 4, dtype=rt.dtype, device=rt.device)
    m[:, :3, :3] = rt[:, :9].view(B, 3, 3)
    m[:, :3, 3] = rt[:, 9:]
    m[:, 3, 3] = 1.0
    return m


def project_bound(rt, depth, H, W, Hs, Ws):
    """float64 source-pixel positions u, v [B,d,H,W] of project_fast (pm_math.cuh) for rt [B,12] (the fp32 values the
    kernel reads) and depth [B,d,H,W], and a bound on the distance of the kernel's fp32 position from them.

    Kernel arithmetic and its rounding: a = r0 x + r1 y + r2 (2 roundings: |da| <= 2 eps A, A = |r0 x|+|r1 y|+|r2|);
    X = fma(a, d, t) (|dX| <= |d| 2 eps A + eps |X|), same for Y, Z; iz = MUFU.RCP (<= 2 ulp = 4 eps relative);
    u = X * iz * sx (2 roundings; sx = (Ws-1)/(W-1) rounded once).  To first order
        du <= eps [ (2 |d| Ax + |X|) / |Z| * sx + |u| (2 |d| Az / |Z| + 1 + 4 + 3) ]
    and the same for v; the factor 1.01 covers the second-order terms.  Behind the camera (Z <= 1e-3) the kernel uses
    X = W, Y = H, Z = 1 exactly."""
    B, d = depth.shape[:2]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=F64, device=depth.device), torch.arange(W, dtype=F64, device=depth.device),
                            indexing="ij")
    r = rt.view(B, 12, 1, 1, 1)
    a = [r[:, 3 * i] * xs + r[:, 3 * i + 1] * ys + r[:, 3 * i + 2] for i in range(3)]
    A = [(r[:, 3 * i] * xs).abs() + (r[:, 3 * i + 1] * ys).abs() + r[:, 3 * i + 2].abs() for i in range(3)]
    X, Y, Z = [a[i] * depth + r[:, 9 + i] for i in range(3)]
    behind = Z <= 1e-3
    X, Y, Z = torch.where(behind, float(W), X), torch.where(behind, float(H), Y), torch.where(behind, 1.0, Z)
    dd = torch.where(behind, 0.0, depth.abs())
    sx, sy = (Ws - 1) / (W - 1), (Hs - 1) / (H - 1)
    u, v = X / Z * sx, Y / Z * sy
    zt = 2 * dd * A[2] / Z.abs() + 8
    du = EPS * ((2 * dd * A[0] + X.abs()) / Z.abs() * sx + u.abs() * zt)
    dv = EPS * ((2 * dd * A[1] + Y.abs()) / Z.abs() * sy + v.abs() * zt)
    return u, v, 1.01 * torch.maximum(du, dv)


def border_dpos(px, py, H, W):
    """Bound on the fp32 rounding of border_cell's position (pm_math.cuh) for float64 pixel positions px, py.
    p = x + dx + off (1 rounding, eps |p|); g = p / ((size-1)/2) - 1 (2: eps |p| + eps (|p| + size/2));
    i = ((g + 1) size - 1) / 2 (3: eps (|p| + size) each) -> <= eps (6 |p| + 4 size); 10 eps max(|p|, size) covers it."""
    return 10 * EPS * torch.maximum(torch.maximum(px.abs(), py.abs()), torch.tensor(float(max(H, W)), dtype=F64, device=px.device))


def assert_within(what, got, want, bound, dims):
    """got (fp32) vs want (float64) element by element: |got - want| <= bound.  Returns the worst |err| / bound; on failure
    names the worst element's index and both values."""
    got = got.to(want.device, F64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = (got - want).abs()
    ratio = err / bound.expand_as(err).clamp_min(1e-300)
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    worst = float(ratio.max().detach())
    if not worst <= 1.0:
        flat = int(ratio.argmax())
        idx = torch.unravel_index(torch.tensor(flat), err.shape)
        at = ", ".join(f"{n}={int(i)}" for n, i in zip(dims, idx))
        raise AssertionError(f"{what}: worst element ({at}): got {float(got.flatten()[flat]):.9g}, want {float(want.flatten()[flat]):.9g}, "
                             f"|err| {float(err.flatten()[flat]):.3e} > bound {float(bound.expand_as(err).flatten()[flat]):.3e}")
    print(f"[bound] {what}: worst |err|/bound = {worst:.3g}")
    return worst


def assert_tight(what, got, want32, rel=2e-5):
    """The existing check against the fp32 oracle: max-abs <= rel * max(1, scale)."""
    scale = max(1.0, float(want32.abs().max()))
    err = float((got.double() - want32.to(got.device).double()).abs().max())
    assert err <= rel * scale, f"{what}: fp32-oracle max-abs {err:.3e} > {rel} * {scale:.3g}"


# ------------------------------------------------------------------------------------------------
# K-A: warp + group correlation, with its epilogues
# ------------------------------------------------------------------------------------------------


def ka_reference(ref, src, rt, depth, G):
    """float64 oracle of one view's similarities and their bound.  ref [B,C,H,W], src [B,C,Hs,Ws], rt [B,12], depth
    [B,D,H,W] (all float64, on the device).  -> (sim, bound) [B,G,D,H,W].

    Per element: sim = (1/n) sum_c r_c S_c, n = C/G, S_c the zero-padded bilinear sample.  fp32: weights gx*gy (1 - fx and
    the product: 2 roundings, fx = u - floor(u) exact), a 4-term sum (4): |dS_c| <= 7 eps S^abs_c; then n products, n - 1
    sums and the 1/n scale: bound = (n + 9) eps A + dpos (1/n) sum_c |r_c| L_c, A = the abs oracle, L_c = lipschitz_map
    of the source channel sampled at the position."""
    B, C, Hs, Ws = src.shape
    D, H, W = depth.shape[1:]
    n = C // G
    eye = torch.eye(4, dtype=F64, device=ref.device).expand(B, 4, 4)
    M = rt_matrix(rt)
    L = lipschitz_map(src, zero_pad=True)
    sim = torch.empty(B, G, D, H, W, dtype=F64, device=ref.device)
    bound = torch.empty_like(sim)
    step = max(1, CHUNK_ELEMS // (B * C * H * W))
    for d0 in range(0, D, step):
        dch = depth[:, d0:d0 + step]
        sim[:, :, d0:d0 + step] = pm_oracle.groupwise_correlation(pm_oracle.homography_warp(src, M, eye, dch), ref, G)
        A = pm_oracle.groupwise_correlation(pm_oracle.homography_warp(src.abs(), M, eye, dch), ref.abs(), G)
        u, v, dpos = project_bound(rt, dch, H, W, Hs, Ws)
        BL = pm_oracle.groupwise_correlation(sample_pixels(L, u, v, "border"), ref.abs(), G)
        bound[:, :, d0:d0 + step] = (n + 9) * EPS * A + dpos[:, None] * BL
        del A, BL, u, v, dpos
    return sim, bound


def aggregate_reference(sims, bounds, vw):
    """sum_v w_v s_v / (1e-5 + sum_v w_v) in float64 and its bound: the views' bounds carried through the weights, plus
    V products, V - 1 sums, the weight sum (V roundings) and the division: (2V + 2) eps of sum_v (w_v / wsum) |s_v|."""
    V = len(sims)
    wsum = 1e-5 + vw.sum(1)  # [B,H,W]
    agg = sum(sims[v] * (vw[:, v] / wsum)[:, None, None] for v in range(V))
    mag = sum(sims[v].abs() * (vw[:, v] / wsum)[:, None, None] for v in range(V))
    bnd = sum(bounds[v] * (vw[:, v] / wsum)[:, None, None] for v in range(V)) + (2 * V + 2) * EPS * mag
    return agg, bnd


def head_layers(head):
    """BatchNorm folded into the 1x1x1 convs, in float64: [(W0, b0), (W1, b1), (w2, b2)]."""
    def fold(block):
        s = block.bn.weight.detach().double() / torch.sqrt(block.bn.running_var.double() + block.bn.eps)
        return (block.conv.weight.detach().double().flatten(1) * s[:, None],
                block.bn.bias.detach().double() - block.bn.running_mean.double() * s)
    last = getattr(head, head._last)
    return [fold(head.conv0), fold(head.conv1), (last.weight.detach().double().flatten(1), last.bias.detach().double())]


def head_reference(layers, x, dx):
    """MLP G -> 16 -> 8 -> 1 (ReLU between) over dim 1 of x [B,G,...] in float64, and the bound of the fp32 kernel's
    output given |x_kernel - x| <= dx.

    Rounding: a layer with n inputs adds (n + 4) eps (|W| |x_in| + |b|) -- n products and the bias (n + 1 roundings) and
    the fp32 rounding of the folded weights (3 eps relative); these are carried on through |W| (they are ~1e-7).
    The input error dx goes through the layers' linearisation at this voxel, w2 D1 W1 D0 W0, D = diag(relu').  A unit
    is "ambiguous" when its pre-activation is within its own error bound of 0 (the kernel's value may sit on the other
    side of the kink): there relu' is some d in [0, 1] and that unit's paths are bounded by absolute values.  Writing
    D = Ds + E (Ds: relu' of the unambiguous units, 0 at the ambiguous ones; |E| <= A, the ambiguous indicator):
        |w2 D1 W1 D0 W0 dx| <= |w2 Ds1 W1 Ds0 W0| dx + |w2| A1 |W1| (Ds0 + A0) |W0| dx + |w2| Ds1 |W1| A0 |W0| dx."""
    expand = lambda t, h: t.view(1, -1, *([1] * (h.dim() - 2)))
    mm = lambda Wm, h: torch.einsum("oi,bi...->bo...", Wm, h)
    (W0, b0), (W1, b1), (w2, b2) = layers
    # values and the abs-propagated bounds (used for the rounding terms and to find ambiguous units)
    p0 = mm(W0, x) + expand(b0, x)
    e0 = mm(W0.abs(), dx) + (W0.shape[1] + 4) * EPS * (mm(W0.abs(), x.abs()) + expand(b0.abs(), x))
    h0 = p0.clamp_min(0)
    r0 = (W0.shape[1] + 4) * EPS * (mm(W0.abs(), x.abs()) + expand(b0.abs(), x))  # rounding part of e0
    p1 = mm(W1, h0) + expand(b1, h0)
    r1 = mm(W1.abs(), r0) + (W1.shape[1] + 4) * EPS * (mm(W1.abs(), h0) + expand(b1.abs(), h0))
    e1 = mm(W1.abs(), e0) + r1 - mm(W1.abs(), r0)  # r1 already carries |W1| r0, e0 contains r0
    h1 = p1.clamp_min(0)
    o = mm(w2, h1) + expand(b2, h1)
    r2 = mm(w2.abs(), r1) + (w2.shape[1] + 4) * EPS * (mm(w2.abs(), h1) + expand(b2.abs(), h1))
    A0, A1 = (p0.abs() <= e0).to(F64), (p1.abs() <= e1).to(F64)
    S0, S1 = (p0 > e0).to(F64), (p1 > e1).to(F64)
    # signed linearisation row J [B,G,...] of the unambiguous paths, and the absolute rows through ambiguous units
    ones = torch.ones_like(h1[:, :1])
    a = torch.einsum("oi,bo...->bi...", w2, ones) * S1  # [B,8,...]
    J = torch.einsum("oi,bo...->bi...", W0, torch.einsum("oi,bo...->bi...", W1, a) * S0)
    a_amb = torch.einsum("oi,bo...->bi...", w2.abs(), ones) * A1
    g_amb = torch.einsum("oi,bo...->bi...", W1.abs(), a_amb) * (S0 + A0)
    g_amb = g_amb + torch.einsum("oi,bo...->bi...", W1.abs(), torch.einsum("oi,bo...->bi...", w2.abs(), ones) * S1) * A0
    J_amb = torch.einsum("oi,bo...->bi...", W0.abs(), g_amb)
    do = (J.abs() * dx).sum(1) + (J_amb * dx).sum(1) + r2[:, 0]
    return o[:, 0], do


def sigmoid_bound(o, do):
    """sigmoid(o) and its bound: slope <= 1/4; the kernel's exp and division add (4 + 1.5 |o|) eps (the exponent o log2(e)
    is rounded: eps |o| log2(e) relative)."""
    return torch.sigmoid(o), do / 4 + (4 + 1.5 * o.abs()) * EPS


def random_head(cls, G, seed):
    torch.manual_seed(seed)
    head = cls(G)
    for m in head.modules():
        if isinstance(m, torch.nn.BatchNorm3d):  # non-trivial running statistics and affine terms
            m.running_mean.normal_(0, 0.3)
            m.running_var.uniform_(0.5, 1.5)
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.normal_(0, 0.2)
    return head.eval()


def ka_case(r, seed, Hs=None, Ws=None, sizes=None):
    """Inputs of one K-A call at the shape of table row r: smooth features, the synthetic rig's relative projections at
    this stage (computed in float64, rounded once), sorted hypotheses over the depth range, view weights.  sizes: one
    (Hs, Ws) per source view (a list of source maps of different sizes instead of one stacked tensor)."""
    g = torch.Generator().manual_seed(seed)
    B, V, C, H, W, D = r["B"], r["V"], r["C"], r["H"], r["W"], r["D"]
    Hs, Ws = Hs or H, Ws or W
    ref = smooth(g, B, C, H=H, W=W)
    srcs = smooth(g, V, B, C, H=Hs, W=Ws) if sizes is None else [smooth(g, B, C, H=h, W=w) for h, w in sizes]
    down = {64: 8, 32: 4, 16: 2}[C]
    Kc, Ec = synthetic.make_cameras(B, V + 1, H * down, W * down)
    ref_proj, src_projs = synthetic.stage_projections(Kc.double(), Ec.double(), {8: 3, 4: 2, 2: 1}[down])
    rt = torch.stack([torch.cat([(sp @ torch.inverse(ref_proj))[:, :3, :3].reshape(B, 9), (sp @ torch.inverse(ref_proj))[:, :3, 3]], 1)
                      for sp in src_projs]).float()  # [V,B,12]
    lo, hi = synthetic.DEPTH_MIN, synthetic.DEPTH_MAX
    depth = torch.sort(lo + (hi - lo) * torch.rand(B, D, H, W, generator=g), dim=1)[0]
    vw = torch.rand(B, V, H, W, generator=g) + 0.05
    return dict(ref=ref, src=srcs, rt=rt, depth=depth, vw=vw)


def ka_references(case, G):
    dev = DEV
    ref64, depth64 = case["ref"].to(dev, F64), case["depth"].to(dev, F64)
    sims, bounds = [], []
    for v in range(len(case["src"])):
        s, b = ka_reference(ref64, case["src"][v].to(dev, F64), case["rt"][v].to(dev, F64), depth64, G)
        sims.append(s)
        bounds.append(b)
    return sims, bounds


def ka_device(case, stack=True):
    nhwc = lambda x: x.permute(0, 2, 3, 1).contiguous()
    return (nhwc(case["ref"].to(DEV)), torch.stack([nhwc(s.to(DEV)) for s in case["src"]]) if stack else None, case["rt"].to(DEV),
            case["depth"].to(DEV), case["vw"].to(DEV))


SIM_DIMS = ("view", "b", "g", "d", "y", "x")


def check_ka_ops(tag, r, case, sims, bounds, heads, knobs=None, fp32_oracle=True, src=None):
    """Every K-A entry point at one shape against the float64 references.  src: the sources as the kernels take them, in
    place of the stacked case["src"] (an ops.ViewPack for sources of different sizes)."""
    G, V = r["G"], r["V"]
    ref_n, src_n, rt, depth, vw = ka_device(case, stack=src is None)
    if src is not None:
        src_n = src
    sim_head, pw_head = heads
    vw64 = case["vw"].to(DEV, F64)
    want = torch.stack(sims)
    bnd = torch.stack(bounds)
    got = ops.warp_corr(ref_n, src_n, rt, depth, G)
    assert_within(f"{tag} warp_corr", got, want, bnd, SIM_DIMS)
    if fp32_oracle and max(r["W"], r["H"]) <= 200:
        # The fp32 oracle normalises every position (g = u / ((W-1)/2) - 1) and grid_sample un-normalises it
        # ((g + 1) / 2 (Ws-1)): four fp32 roundings at magnitude up to W, ~4 eps W pixels of position error of its own.
        # With these features (slope up to ~1.5 per pixel, |r| ~ 1) that moves a similarity by ~4 * 6e-8 * W * 1.5:
        # 7e-5 at W = 200, about the 2e-5 * scale (scale ~3.5) the check allows; 1.4e-4 and 2.9e-4 at W = 400 and 800.
        # On the wider maps the check is replaced by a printout of the fp32 oracle's own distance from float64.
        eye = torch.eye(4, device=DEV).expand(r["B"], 4, 4)
        for v in range(V):
            w32 = pm_oracle.groupwise_correlation(pm_oracle.homography_warp(case["src"][v].to(DEV), rt_matrix(rt[v]), eye, depth),
                                                  case["ref"].to(DEV), G)
            assert_tight(f"{tag} warp_corr view {v}", got[v], w32)
            del w32
    elif fp32_oracle:
        eye = torch.eye(4, device=DEV).expand(r["B"], 4, 4)
        w32 = pm_oracle.groupwise_correlation(pm_oracle.homography_warp(case["src"][0].to(DEV), rt_matrix(rt[0]), eye, depth),
                                              case["ref"].to(DEV), G)
        print(f"[fp32 oracle] {tag} view 0: fp32 oracle vs float64 max-abs {float((w32.double() - sims[0]).abs().max()):.3e}, "
              f"kernel vs float64 max-abs {float((got[0].double() - sims[0]).abs().max()):.3e}")
        del w32
    del got
    agg, agg_b = aggregate_reference(sims, bounds, vw64)
    assert_within(f"{tag} warp_corr (view-weighted)", ops.warp_corr(ref_n, src_n, rt, depth, G, vw), agg, agg_b, SIM_DIMS[1:])
    # SimilarityNet fused into K-A (every iteration after the first)
    sc, sc_b = head_reference(head_layers(sim_head), agg, agg_b)
    assert_within(f"{tag} warp_corr_score", ops.warp_corr_score(ref_n, src_n, rt, depth, G, vw, sim_head.folded()), sc, sc_b,
                  ("b", "d", "y", "x"))
    del agg, agg_b, sc, sc_b
    # PixelwiseNet fused into K-A (first iteration of the coarsest stage), keeping the similarities
    got_vw, kept = ops.warp_corr_view_weights(ref_n, src_n, rt, depth, G, pw_head.folded(), keep_sims=True)
    assert_within(f"{tag} warp_corr_view_weights (kept sims)", kept, want, bnd, SIM_DIMS)
    layers = head_layers(pw_head)
    vws, vwb = [], []
    for v in range(V):
        o, do = head_reference(layers, sims[v], bounds[v])
        s, ds = sigmoid_bound(o, do)
        vws.append(s.amax(1))
        vwb.append(ds.amax(1))  # the max over hypotheses is 1-Lipschitz
    assert_within(f"{tag} warp_corr_view_weights", got_vw, torch.stack(vws, 1), torch.stack(vwb, 1), ("b", "view", "y", "x"))
    # aggregate_views_score on the kernel's own similarities and view weights: rounding only
    kept64, gvw64 = kept.double(), got_vw.double()
    agg2, agg2_b = aggregate_reference(list(kept64), [torch.zeros_like(kept64[0])] * V, gvw64)
    sc2, sc2_b = head_reference(head_layers(sim_head), agg2, agg2_b)
    assert_within(f"{tag} aggregate_views_score", ops.aggregate_views_score(kept, got_vw, sim_head.folded()), sc2, sc2_b,
                  ("b", "d", "y", "x"))


KA_ROWS = ["1600x1200/s3/it1", "1600x1200/s3/it2", "1200x1600/s2/it1", "1600x1200/s1/it1", "320x256/s3/it1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", KA_ROWS)
def test_warp_corr_ops_at_scale(name):
    r = row(name)
    case = ka_case(r, seed=r["H"] + r["D"])
    sims, bounds = ka_references(case, r["G"])
    heads = (random_head(SimilarityNet, r["G"], 1).to(DEV), random_head(PixelwiseNet, r["G"], 2).to(DEV))
    ops.set_tuning("reset")
    with torch.no_grad():
        check_ka_ops(name, r, case, sims, bounds, heads)


@pytest.mark.gpu
def test_warp_corr_source_maps_of_another_size():
    """Stage 2 of a landscape 1600x1200 reference with portrait 1200x1600 sources (Hs, Ws != H, W)."""
    r = row("1600x1200/s2/it1")
    case = ka_case(r, seed=11, Hs=r["W"], Ws=r["H"])
    sims, bounds = ka_references(case, r["G"])
    heads = (random_head(SimilarityNet, r["G"], 3).to(DEV), random_head(PixelwiseNet, r["G"], 4).to(DEV))
    ops.set_tuning("reset")
    with torch.no_grad():
        check_ka_ops("Hs,Ws != H,W", r, case, sims, bounds, heads, fp32_oracle=False)


def edge_case(seed):
    """Stage 1 of a 1600x1200 view (C=16, G=4, 600x800) with relative projections that are pure x-translations
    rot = I, t = (tx, 0, 0), tx in {+1, -1, +1, 0}.  Then Z = d exactly and u = x + tx / d.

    Hypotheses 0..6 are d = 2^-j, j = -1..5: tx / d = +-2^j, so u = x +- 2^j is exact in fp32 (powers of two: fma, MUFU.RCP
    and the product are exact) and, over the pixel row, lands exactly on u = -1, -0.5, 0, W-1 (the last column the
    interior fast path of zero_pad_cell_fast does not take), W-0.5 and W.  Hypothesis 7 is behind the camera (d = -1).
    Hypotheses 8, 9 sit on both sides of the Z = 1e-3 cut: d = 0.9e-3 and 1.1e-3.  fp32 and float64 disagree on the cut
    only for Z in [1e-3 - 3 eps |Z|, fp32(1e-3) + 3 eps |Z|] = [1e-3 - 2e-10, 1.0000000475e-3 + 2e-10] (fp32(1e-3) is
    1.0000000475e-3, the kernel compares in fp32, the oracle in float64); both hypotheses are 1e-4 away from it.  With
    tx = 0 (view 3) u = x at every hypothesis in front of the camera, so the side of the cut decides zero or the pixel."""
    r = dict(row("1600x1200/s1/it1"))
    B, H, W, C = r["B"], r["H"], r["W"], r["C"]
    r["D"] = 10
    g = torch.Generator().manual_seed(seed)
    rt = torch.zeros(N_SRC, B, 12)
    rt[:, :, [0, 4, 8]] = 1.0
    rt[:, :, 9] = torch.tensor([1.0, -1.0, 1.0, 0.0]).view(N_SRC, 1)
    d = torch.tensor([2.0 ** -j for j in range(-1, 6)] + [-1.0, 0.9e-3, 1.1e-3])
    depth = d.view(1, -1, 1, 1).expand(B, -1, H, W).contiguous()
    case = dict(ref=smooth(g, B, C, H=H, W=W), src=smooth(g, N_SRC, B, C, H=H, W=W), rt=rt, depth=depth,
                vw=torch.rand(B, N_SRC, H, W, generator=g) + 0.05)
    return r, case


def test_edge_case_lands_on_the_borders():
    r, case = edge_case(0)
    W = r["W"]
    u = torch.arange(W, dtype=F64).view(1, -1) + (case["rt"][:, 0, 9].double().view(-1, 1, 1) / case["depth"][0, :7, 0, :1].double().view(1, -1, 1))
    hit = set(float(x) for x in u.flatten().tolist())
    for target in (-1.0, -0.5, 0.0, W - 1.0, W - 0.5, float(W)):
        assert target in hit, target


@pytest.mark.gpu
def test_warp_corr_edges():
    r, case = edge_case(5)
    sims, bounds = ka_references(case, r["G"])
    behind = case["depth"][:, 7:8].expand(-1, 1, -1, -1)
    heads = (random_head(SimilarityNet, r["G"], 5).to(DEV), random_head(PixelwiseNet, r["G"], 6).to(DEV))
    ops.set_tuning("reset")
    with torch.no_grad():
        check_ka_ops("edges", r, case, sims, bounds, heads)
        got = ops.warp_corr(*ka_device(case)[:4], r["G"])
    assert float(behind.max()) < 0 and float(got[:, :, :, 7].abs().max()) == 0.0  # behind the camera: exactly zero
    assert float(got[:, :, :, 8].abs().max()) == 0.0  # Z = 0.9e-3: below the cut
    assert float(got[3, :, :, 9].abs().max()) > 0.1  # Z = 1.1e-3, tx = 0: samples the pixel itself


def ka_kernel_args(fn, sessions=5):
    """Run fn under the CUDA profiler -> [(generation, [template arguments])] of the K-A kernels it launched.

    A profiler session now and then comes back without any device activity at all (its CUPTI records are lost, not the
    launches: fn launches kernels every time and raises when a launch fails).  Such a session says nothing about which
    kernels ran, so fn is profiled again, at most `sessions` times; a session with device activity is taken as it is."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    for _ in range(sessions):
        torch.cuda.synchronize()  # nothing launched before the session runs inside it
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
        if names:
            out = []
            for name in names:
                m = re.search(r"warp_corr([34])_kernel<([^>]*)>", name)
                if m:
                    out.append((int(m.group(1)), [a.strip() for a in m.group(2).split(",")]))
            return out
        print("[profiler] a session recorded no device activity; profiling again")
    raise AssertionError(f"{sessions} profiler sessions recorded no device activity")


def knob_took_effect(knobs, launched):
    """Whether the launches show the variant the knobs ask for: generation 4 with ka4_nw consumer warps
    (warp_corr4_kernel<C, G, EPI, NW, MINB>), or generation 3 with ka3_dc rows per pass, the pipeline, and ka3_minb
    (warp_corr3_kernel<C, G, EPI, DC, PIPE, MINB>).  The ring knobs (ka4_ctas, ka4_stages, ka4_cap, ka4_grid) change no
    template argument; a generation-4 launch that cannot honour them falls back to generation 3, which this catches."""
    if knobs.get("ka_gen") == 4:
        return any(g == 4 and a[3] == str(knobs.get("ka4_nw", 4)) for g, a in launched)
    gen3 = [a for g, a in launched if g == 3]
    if "ka3_dc" in knobs:
        return any(a[3] == str(knobs["ka3_dc"]) for a in gen3)
    if knobs.get("ka3_minb") == 5:
        return any(a[4] == "1" and a[5] == "5" for a in gen3)
    return any(a[4] == "1" for a in gen3)


@pytest.mark.gpu
def test_warp_corr_knobs_match_float64():
    """Every K-A variant tools/kbench.py sweeps, and the other launch knobs the library accepts, within the default's bound,
    at stage 3 of a 1600x1200 view and stage 2 of a 1200x1600 one.  Some knobs do not apply at every shape (ka3_dc = 4 at
    C = 64 and 16 at C = 32 do not fit the lane map or the 40 KB tile, ka3_minb = 5 exists for the stage-2 score kernel
    only): the kernel names show that each variant ran as asked at one of the two shapes at least."""
    took = {i: [] for i in range(len(KA_KNOBS))}
    try:
        for name in ("1600x1200/s3/it1", "1200x1600/s2/it1"):
            r = row(name)
            case = ka_case(r, seed=21)
            sims, bounds = ka_references(case, r["G"])
            heads = (random_head(SimilarityNet, r["G"], 7).to(DEV), random_head(PixelwiseNet, r["G"], 8).to(DEV))
            ref_n, src_n, rt, depth, vw = ka_device(case)
            with torch.no_grad():
                for i, knobs in enumerate(KA_KNOBS):
                    ops.set_tuning("reset")
                    for k, v in knobs.items():
                        ops.set_tuning(k, v)
                    check_ka_ops(f"{name} {knobs}", r, case, sims, bounds, heads, fp32_oracle=False)
                    launched = ka_kernel_args(lambda: (
                        ops.warp_corr_score(ref_n, src_n, rt, depth, r["G"], vw, heads[0].folded()),
                        ops.warp_corr_view_weights(ref_n, src_n, rt, depth, r["G"], heads[1].folded())))
                    print(f"[knobs] {name} {knobs}: {launched}")
                    if knob_took_effect(knobs, launched):
                        took[i].append(name)
            del sims, bounds
    finally:
        ops.set_tuning("reset")
    missing = [KA_KNOBS[i] for i, shapes in took.items() if not shapes]
    assert not missing, f"variants that never ran as asked: {missing}"


# ------------------------------------------------------------------------------------------------
# border-clamped gathers: K-A', K-C, K-B
# ------------------------------------------------------------------------------------------------


def pixel_positions(table, off, H, W):
    """float64 pixel positions (x + dx + off_x, y + dy + off_y) [B,K,H,W] of the neighbour gathers."""
    B = off.shape[0]
    ys, xs = torch.meshgrid(torch.arange(H, dtype=F64, device=off.device), torch.arange(W, dtype=F64, device=off.device),
                            indexing="ij")
    px = torch.stack([xs + dx + off[:, 2 * k] for k, (dy, dx) in enumerate(table)], 1)
    py = torch.stack([ys + dy + off[:, 2 * k + 1] for k, (dy, dx) in enumerate(table)], 1)
    return px, py


def border_sample_bound(f, px, py, H, W):
    """f [B,C,H,W] float64 sampled at the texel position border_cell (pm_math.cuh) computes from the pixel positions px, py
    [B,K,H,W]: the reference's align_corners=False un-normalisation of its align_corners=True grid, i = p size / (size-1)
    - 0.5, clamped to [0, size-1] (both 1-Lipschitz up to the factor size / (size-1), which border_dpos's margin covers).
    -> (value, |f| sampled, bound of the coordinate term dpos * lipschitz) [B,C,K,H,W]."""
    B, C = f.shape[:2]
    K = px.shape[1]
    cx = (px * (W / (W - 1)) - 0.5).clamp(0, W - 1)
    cy = (py * (H / (H - 1)) - 0.5).clamp(0, H - 1)
    grid = torch.stack((cx * (2.0 / (W - 1)) - 1, cy * (2.0 / (H - 1)) - 1), -1).view(B, K * H, W, 2)
    s = lambda m: F.grid_sample(m, grid, mode="bilinear", padding_mode="border", align_corners=True).view(B, C, K, H, W)
    dpos = border_dpos(px, py, H, W)
    return s(f), s(f.abs()), dpos[:, None] * s(lipschitz_map(f, zero_pad=False))


def offsets_reaching_borders(gen, B, K, H, W, reach):
    """Smooth raw offsets [B,2K,H,W] of amplitude `reach` pixels, with exact values placed along the map's edges for the
    first neighbour: x + off_x = 0 on the first row and W - 1 on the last row, y + off_y = -3 on the first column and H + 3
    on the last one.  The table's fixed (dy, dx) of that neighbour (-d, -d, d >= 1) is added on top, and border_cell maps a
    position p to p size / (size-1) - 0.5, so these gathers reach texel 0 through the clamp, sample inside the last
    column, and leave the map beyond both borders in y; together with the smooth part they cover both clamped borders."""
    off = smooth(gen, B, 2 * K, H=H, W=W) * reach
    xs = torch.arange(W, dtype=torch.float32)
    ys = torch.arange(H, dtype=torch.float32)
    off[:, 0, 0, :] = -xs  # x + off = 0 along the first row (first neighbour: dx is added on top, see the tables)
    off[:, 0, -1, :] = (W - 1) - xs  # x + off = W - 1 along the last row
    off[:, 1, :, 0] = -ys - 3.0  # beyond the top border along the first column
    off[:, 1, :, -1] = (H + 3.0) - ys  # beyond the bottom border along the last column
    return off


def oc_reference(ref, off, G, K, dil):
    """K-A' in float64: corr_k = (1/n) sum_c r_c S_c(p_k) with border sampling; bound (n + 9) eps A + coordinate term
    (the same arithmetic as ka_reference, positions from border_dpos)."""
    B, C, H, W = ref.shape
    n = C // G
    table = pm_oracle.neighbour_table("evaluation", K, dil)
    grid = pm_oracle.sampling_grid(table, off.view(B, 2 * K, H * W), H, W)
    want = pm_oracle._FeatureWeightHead(K, G).double().to(ref.device).neighbour_correlation(ref, grid)
    px, py = pixel_positions(table, off, H, W)
    _, sabs, coord = border_sample_bound(ref, px, py, H, W)  # [B,C,K,H,W]
    rabs = ref.abs()[:, :, None]
    A = (sabs * rabs).view(B, G, n, K, H, W).mean(2)
    BL = (coord * rabs).view(B, G, n, K, H, W).mean(2)
    return want, (n + 9) * EPS * A + BL


OC_ROWS = ["1600x1200/s3/it1", "1200x1600/s2/it1", "1600x1200/s1/it1", "320x256/s3/it1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", OC_ROWS)
def test_offset_corr_at_scale(name):
    check_offset_corr(name, row(name))


def check_offset_corr(name, r):
    """K-A' and its fused head at the shape of row r against the float64 references."""
    from patchmatchnet_b200.patchmatch import FeatureWeightNet

    B, C, G, K, dil, H, W = r["B"], r["C"], r["G"], r["K"], r["dil"], r["H"], r["W"]
    g = torch.Generator().manual_seed(H + K)
    ref = smooth(g, B, C, H=H, W=W)
    off = offsets_reaching_borders(g, B, K, H, W, reach=6.0)
    want, bnd = oc_reference(ref.to(DEV, F64), off.to(DEV, F64), G, K, dil)
    ref_n = ref.permute(0, 2, 3, 1).contiguous().to(DEV)
    with torch.no_grad():
        got = ops.offset_corr(ref_n, off.to(DEV), G, K, dil)
        assert_within(f"{name} offset_corr", got, want, bnd, ("b", "g", "k", "y", "x"))
        grid32 = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, dil), off.to(DEV).view(B, 2 * K, H * W), H, W)
        want32 = pm_oracle._FeatureWeightHead(K, G).to(DEV).neighbour_correlation(ref.to(DEV), grid32)
        if max(H, W) <= 800:
            assert_tight(f"{name} offset_corr", got, want32)
        else:
            # the fp32 oracle's own position rounding grows with the map width (its normalised grid, as in
            # check_ka_ops); past the 800 px of the widest rows above it exceeds the 2e-5 check by itself (2.1e-4 at
            # 1344 px, with the kernel within 0.12 of its float64 bound): its distance from float64 is printed instead
            print(f"[fp32 oracle] {name} offset_corr: fp32 oracle vs float64 max-abs {float((want32.double() - want).abs().max()):.3e}, "
                  f"kernel vs float64 max-abs {float((got.double() - want).abs().max()):.3e}")
        del want32
        head = random_head(lambda gg: FeatureWeightNet(K, gg), G, 9).to(DEV)
        o, do = head_reference(head_layers(head), want, bnd)
        s, ds = sigmoid_bound(o, do)
        assert_within(f"{name} offset_corr_weight", ops.offset_corr_weight(ref_n, off.to(DEV), G, K, dil, head.folded()), s, ds,
                      ("b", "k", "y", "x"))


def xnorm_bound(h, dh, dmin, dmax):
    """xn = (1/h - 1/dmax) / (1/dmin - 1/dmax) in float64 and the bound of the fp32 kernel's value for |h_kernel - h| <= dh:
    1/h (2 eps + dh / h^2), the difference (eps |1/h - a|), the range b - a from fp32 1/dmin, 1/dmax (eps (|a| + |b|) each
    and one more for the subtraction), the division (eps |xn|)."""
    B = h.shape[0]
    a, b = (1.0 / dmax).view(B, 1, 1, 1), (1.0 / dmin).view(B, 1, 1, 1)
    xn = (1.0 / h - a) / (b - a)
    dnum = 2 * EPS / h.abs() + dh / h ** 2 + 2 * EPS * (1.0 / h.abs() + a)
    drange = 3 * EPS * (a + b)
    return xn, (dnum + xn.abs() * drange) / (b - a) + EPS * xn.abs()


def kc_reference(seed, off, dmin, dmax, mode, Ns, Kp, dil, scale, H, W):
    """K-C in float64 and its bound.  Initial samples: the fp32 formulas (patchmatch.py:56-94) take <= 8 roundings of the
    inverse depth and one of the division: 16 eps |h| covers them.  Propagated samples gather the centre initial sample
    (border bilinear: 7 eps of |.| sampled, plus its own 16 eps, plus the coordinate term).  Sorting is 1-Lipschitz in the
    max norm, so every sorted output of a pixel is within the largest pre-sort bound of that pixel."""
    B = dmin.shape[0]
    init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, Ns if mode != ops.MODE_RANDOM else 16,
                                     seed if mode != ops.MODE_RANDOM else torch.empty(0, device=seed.device), seed.device,
                                     (lambda size, device: seed) if mode == ops.MODE_RANDOM else None)
    b0 = 16 * EPS * init.abs()
    want, pre = init, b0
    if Kp > 0:
        table = pm_oracle.neighbour_table("propagation", Kp, dil)
        grid = pm_oracle.sampling_grid(table, off.view(B, 2 * Kp, H * W), H, W)
        want = pm_oracle.propagate(init, grid)
        centre = init[:, init.shape[1] // 2:init.shape[1] // 2 + 1]
        px, py = pixel_positions(table, off, H, W)
        _, sabs, coord = border_sample_bound(centre, px, py, H, W)
        pre = torch.cat([b0, (16 + 7) * EPS * sabs[:, 0] + coord[:, 0]], 1)
    bound = pre.amax(1, keepdim=True).expand_as(want)
    xn, xb = xnorm_bound(want, bound, dmin, dmax)
    return want, bound, xn, xb


KC_ROWS = ["1600x1200/s3/it1", "1600x1200/s3/it2", "1200x1600/s2/it1", "1600x1200/s1/it1", "320x256/s2/it2",
           "synthetic/Ns4Kp4", "synthetic/D192"]


def kc_inputs(r, g):
    B, H, W, Kp = r["B"], r["H"], r["W"], r["Kp"]
    dmin = torch.full((B,), synthetic.DEPTH_MIN) + torch.arange(B) * 3.0
    dmax = torch.full((B,), synthetic.DEPTH_MAX) - torch.arange(B) * 4.0
    if r["mode"] == ops.MODE_RANDOM:
        seed = torch.rand(B, 48, H, W, generator=g)
    else:  # a smooth depth map, partly outside [dmin, dmax]: exercises the clamp
        seed = 680.0 + 150.0 * smooth(g, B, 1, H=H, W=W)
    off = offsets_reaching_borders(g, B, Kp, H, W, reach=4.0) if Kp > 0 else None
    return seed, off, dmin, dmax


@pytest.mark.gpu
@pytest.mark.parametrize("name", KC_ROWS)
def test_init_propagate_at_scale(name):
    check_init_propagate(name, row(name))


def check_init_propagate(name, r):
    """K-C (hypotheses, xnorm, the interleaved xs buffer) at the shape of row r against the float64 references."""
    print(f"[plan] {name}: K-C kernel {kc_kernel(r['Ns'], r['Kp'])}")
    B, H, W, Ns, Kp = r["B"], r["H"], r["W"], r["Ns"], r["Kp"]
    g = torch.Generator().manual_seed(H + Ns + Kp)
    seed, off, dmin, dmax = kc_inputs(r, g)
    want, bnd, xn, xb = kc_reference(seed.to(DEV, F64), None if off is None else off.to(DEV, F64), dmin.to(DEV, F64),
                                      dmax.to(DEV, F64), r["mode"], Ns, Kp, r["dil"], r["scale"], H, W)
    dims = ("b", "d", "y", "x")
    args = (seed.to(DEV), None if off is None else off.to(DEV), dmin.to(DEV), dmax.to(DEV), r["mode"], Ns, Kp, r["dil"], r["scale"])
    got, got_x = ops.init_propagate(*args, with_xnorm=True)
    assert_within(f"{name} init_propagate", got, want, bnd, dims)
    assert_within(f"{name} init_propagate xnorm", got_x, xn, xb, dims)
    xs = ops.alloc_xs(B, Ns + Kp, H, W, DEV).fill_(-7.0)
    assert torch.equal(ops.init_propagate(*args, xs=xs), got) and torch.equal(xs[..., 0], got_x) and bool((xs[..., 1] == -7.0).all())


def kb_reference(score0, depth, off, fw, dmin, dmax, dil, scale, inverse, K):
    """K-B in float64 (patchmatch.py:221-237, 509-510, 569-577, 650-669) and bounds of its probabilities and depth.

    S_k, X_k: score and normalised inverse depth gathered at neighbour k (border bilinear): 7 eps of |.| sampled plus the
    coordinate term; X also carries the kernel's own xnorm error (xnorm_bound).  Weight: a = |X_k - x_c| / scale
    (da = (dX_k + dx_c + 2 eps (|X_k| + |x_c|)) / scale + eps a), sigma(4 - 2 clamp(a, 0, 4)) (slope 2 sigma (1 - sigma)
    widened by how far it can change within da, plus the exp / division rounding 6 eps), times the feature weight (eps).  Normalised weights w_k / sum w:
    (dw_k + w^_k sum dw) / sum w + (K + 2) eps w^_k.  s = sum_k w^_k S_k: sum (w^ dS + |S| dw^) + (K + 1) eps sum w^ |S|.
    softmax: log p_d moves by <= ds_d + max_j ds_j (logsumexp is 1-Lipschitz in the max norm), so
    dp_d <= p_d (1.01 (ds_d + max ds) + (D + 4 + 1.5 |s_d - max s|) eps) (exp of a rounded exponent, the sum, the division).
    Depth: sum_d p_d h_d -> sum |h - depth| dp_move + sum |h| dp_round + (D + 1) eps sum p |h| (dp_move, the part from the moved
    scores, sums to zero over d); inverse: idx = sum d p_d, h = 1 / (lo + idx / (D-1) (hi - lo))
    -> h^2 |hi - lo| / (D - 1) didx + 8 eps h (|lo| + |idx (hi - lo) / (D - 1)|) / |q|."""
    B, D, H, W = depth.shape
    table = pm_oracle.neighbour_table("evaluation", K, dil)
    grid = pm_oracle.sampling_grid(table, off.view(B, 2 * K, H * W), H, W)
    xc, dxc = xnorm_bound(depth, torch.zeros_like(depth), dmin, dmax)
    px, py = pixel_positions(table, off, H, W)
    dxc_max = dxc.amax(1, keepdim=True).unsqueeze(2)
    s = torch.empty_like(depth)
    ds = torch.empty_like(depth)
    step = max(1, CHUNK_ELEMS // (B * K * H * W))  # hypotheses per chunk: each [B,d,K,H,W] intermediate stays <= 256 MB
    for d0 in range(0, D, step):
        sl = slice(d0, d0 + step)
        w = pm_oracle.depth_similarity_weight(depth[:, sl], dmin, dmax, grid, scale, K) * fw.unsqueeze(1)
        wsum = w.sum(2, keepdim=True)
        what = w / wsum
        S, Sabs, Scoord = border_sample_bound(score0[:, sl], px, py, H, W)  # [B,d,K,H,W]
        s[:, sl] = (S * what).sum(2)
        dS = 7 * EPS * Sabs + Scoord
        del Sabs, Scoord
        X, Xabs, Xcoord = border_sample_bound(xc[:, sl], px, py, H, W)
        dX = 7 * EPS * Xabs + Xcoord + dxc_max
        del Xabs, Xcoord
        xcc = xc[:, sl].unsqueeze(2)
        a = (X - xcc).abs() / scale
        da = (dX + dxc[:, sl].unsqueeze(2) + 2 * EPS * (X.abs() + xcc.abs())) / scale + EPS * a
        del X, dX
        sig = torch.sigmoid(4.0 - 2.0 * a.clamp(0, 4))
        # slope of sigma(4 - 2 clamp(a)) in a: 2 sigma (1 - sigma) at t = 4 - 2a, which moves by at most 0.1 per unit of t
        # (|d/dt sigma(1 - sigma)| <= 0.1) while t moves by 2 da; the clamp is 1-Lipschitz
        dw = fw.unsqueeze(1) * (2 * (sig * (1 - sig) + 0.2 * da) * da + 6 * EPS * sig) + EPS * w
        del a, da, sig
        dwhat = (dw + what * dw.sum(2, keepdim=True)) / wsum + (K + 2) * EPS * what
        ds[:, sl] = (what * dS + S.abs() * dwhat).sum(2) + (K + 1) * EPS * (what * S.abs()).sum(2)
        del dw, dwhat, dS, S, what, w, wsum
    prob = torch.exp(F.log_softmax(s, dim=1))
    want_depth = pm_oracle._Evaluation.regress(depth, prob, inverse)
    m = s.amax(1, keepdim=True)
    dp_move = prob * 1.01 * (ds + ds.amax(1, keepdim=True))  # the exact softmax of the moved scores: sums to 1 like prob
    dp_round = prob * (D + 4 + 1.5 * (s - m).abs()) * EPS
    dp = dp_move + dp_round
    # sum_d (p'_d - p_d) c_d = sum_d (p'_d - p_d) (c_d - c^) for the moved (exact) softmax: its part of the bound uses |c - c^|
    if not inverse:
        dev_h = (depth - want_depth.unsqueeze(1)).abs()
        dd = (dev_h * dp_move + depth.abs() * dp_round).sum(1) + (D + 1) * EPS * (prob * depth.abs()).sum(1)
    else:
        idxw = torch.arange(D, dtype=F64, device=depth.device).view(1, D, 1, 1)
        idx = (idxw * prob).sum(1)
        didx = ((idxw - idx.unsqueeze(1)).abs() * dp_move + idxw * dp_round).sum(1) + (D + 1) * EPS * idx
        lo, hi = 1.0 / depth[:, 0], 1.0 / depth[:, -1]
        q = lo + idx / (D - 1) * (hi - lo)
        dd = want_depth ** 2 * (hi - lo).abs() / (D - 1) * didx + 8 * EPS * want_depth.abs() * (lo.abs() + (idx * (hi - lo) / (D - 1)).abs()) / q.abs()
    return prob, dp, want_depth, dd


KB_ROWS = ["1600x1200/s3/it1", "1600x1200/s3/it2", "1200x1600/s2/it2", "1600x1200/s1/it1", "640x512/s3/it1", "320x256/s2/it1",
           "synthetic/D192", "synthetic/D3"]


def kb_inputs(r, g):
    B, D, H, W, K = r["B"], r["D"], r["H"], r["W"], r["K"]
    dmin, dmax = torch.full((B,), synthetic.DEPTH_MIN), torch.full((B,), synthetic.DEPTH_MAX)
    # smooth hypotheses (a smooth base map plus sorted smooth offsets, well inside [dmin, dmax]) and scores: the depth
    # weight's slope is 2 / interval_scale per unit of normalised inverse depth, so its coordinate term follows the
    # spatial slope of the hypotheses
    base = 680.0 + 60.0 * smooth(g, B, 1, H=H, W=W, cell=16)
    spread = torch.sort(smooth(g, B, D, H=H, W=W, cell=16), dim=1, descending=bool(r["inverse"]))[0]
    depth = base + 20.0 * spread
    score0 = 2.0 * smooth(g, B, D, H=H, W=W, cell=8)
    off = offsets_reaching_borders(g, B, K, H, W, reach=3.0)
    fw = torch.rand(B, K, H, W, generator=g) + 0.05
    return score0, depth, off, fw, dmin, dmax


def check_kb(tag, r, inputs, refs, sms):
    score0, depth, off, fw, dmin, dmax = [t.to(DEV) for t in inputs]
    prob64, dp, depth64, dd = refs
    B, D, H, W, K = r["B"], r["D"], r["H"], r["W"], r["K"]
    inv_min, inv_max = (1.0 / dmin).view(B, 1, 1, 1), (1.0 / dmax).view(B, 1, 1, 1)
    xnorm = (1.0 / depth - inv_max) / (inv_min - inv_max)
    xs = torch.stack([xnorm, score0], dim=-1).contiguous()
    plan = kb_plan(B, D, H, W, K, sms)
    print(f"[plan] {tag}: K-B TP={plan[0]} DY={plan[1]} smem={plan[2]}")
    for form, (sc, xn, inter, o) in {"score0": (score0, None, None, off), "xnorm": (score0, xnorm, None, off.contiguous(memory_format=torch.channels_last)),
                                     "xs": (None, None, xs, off)}.items():
        got_depth, got_prob = ops.adaptive_eval(sc, depth, o, fw, dmin, dmax, r["dil"], r["scale"], bool(r["inverse"]), xnorm=xn, xs=inter)
        assert_within(f"{tag} adaptive_eval[{form}] prob", got_prob, prob64, dp, ("b", "d", "y", "x"))
        assert_within(f"{tag} adaptive_eval[{form}] depth", got_depth, depth64, dd, ("b", "y", "x"))
    return got_prob, got_depth


@pytest.mark.gpu
@pytest.mark.parametrize("name", KB_ROWS)
def test_adaptive_eval_at_scale(name):
    check_adaptive_eval(name, row(name))


def check_adaptive_eval(name, r):
    """K-B in its three input forms at the shape of row r against the float64 references, and against the fp32 oracle
    on maps up to 200 px."""
    g = torch.Generator().manual_seed(r["H"] + r["D"])
    inputs = kb_inputs(r, g)
    score0, depth, off, fw, dmin, dmax = inputs
    refs = kb_reference(*[t.to(DEV, F64) for t in inputs[:4]], dmin.to(DEV, F64), dmax.to(DEV, F64), r["dil"], r["scale"],
                        bool(r["inverse"]), r["K"])
    ops.set_tuning("reset")
    with torch.no_grad():
        got_prob, got_depth = check_kb(name, r, inputs, refs, torch.cuda.get_device_properties(0).multi_processor_count)
    # the existing fp32-oracle bounds (test_gpu_parity.py), on the maps where the fp32 oracle resolves them.  Its positions
    # are rounded differently from the kernel's (~4 eps W pixels each), and the depth weight amplifies a position
    # difference by its slope 2 / interval_scale times the slope of the normalised inverse depth: at 300x400 and 600x800
    # the fp32 oracle and the kernel differed by 1.0e-5 and 9.8e-5 in probability while the kernel stayed within 0.013 of
    # its float64 bound.
    B, D, H, W, K = r["B"], r["D"], r["H"], r["W"], r["K"]
    if max(H, W) > 200:
        return
    sd, dd_, od, fd, lo, hi = [t.to(DEV) for t in (score0, depth, off, fw, dmin, dmax)]
    grid = pm_oracle.sampling_grid(pm_oracle.neighbour_table("evaluation", K, r["dil"]), od.view(B, 2 * K, H * W), H, W)
    w = pm_oracle.depth_similarity_weight(dd_, lo, hi, grid, r["scale"], K) * fd.unsqueeze(1)
    w = w / torch.sum(w, dim=2).unsqueeze(2)
    s = torch.sum(pm_oracle._border_sample(sd, grid).view(B, D, K, H, W) * w, dim=2)
    p32 = torch.exp(F.log_softmax(s, dim=1))
    assert float((got_prob - p32).abs().max()) <= 5e-6
    d32 = pm_oracle._Evaluation.regress(dd_, p32, bool(r["inverse"]))
    assert float((got_depth - d32).abs().sum() / d32.abs().sum()) <= 1e-6


@pytest.mark.gpu
def test_adaptive_eval_block_shapes_match_float64():
    """tools/kbench.py's eight K-B block shapes (TP=8 and TP=64 included) at stage 3 of a 1600x1200 view, D=64."""
    r = row("1600x1200/s3/it1")
    g = torch.Generator().manual_seed(31)
    inputs = kb_inputs(r, g)
    refs = kb_reference(*[t.to(DEV, F64) for t in inputs[:4]], inputs[4].to(DEV, F64), inputs[5].to(DEV, F64), r["dil"], r["scale"],
                        False, r["K"])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        with torch.no_grad():
            for tp, dy in KB_KNOB_SHAPES:
                ops.set_tuning("reset")
                ops.set_tuning("kb_tp", tp)
                ops.set_tuning("kb_dy", dy)
                assert kb_plan(r["B"], r["D"], r["H"], r["W"], r["K"], sms)[:2] == (tp, dy)
                check_kb(f"TP={tp},DY={dy}", r, inputs, refs, sms)
    finally:
        ops.set_tuning("reset")


# ------------------------------------------------------------------------------------------------
# K-S: FeatureNet's stem at both pixels-per-thread settings
# ------------------------------------------------------------------------------------------------


def stem_case(seed, H, W):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(1, 3, H, W, generator=g)
    w0, b0 = torch.randn(8, 3, 3, 3, generator=g) * 0.3, torch.randn(8, generator=g) * 0.1
    w1, b1 = torch.randn(8, 8, 3, 3, generator=g) * 0.2, torch.randn(8, generator=g) * 0.1
    return x, w0, b0, w1, b1


def stem_reference(x64, W0, B0, W1, B1):
    h0 = F.relu(F.conv2d(x64, W0, B0, padding=1))
    want = F.relu(F.conv2d(h0, W1, B1, padding=1))
    d0 = 30 * EPS * (F.conv2d(x64.abs(), W0.abs(), padding=1) + B0.abs().view(1, -1, 1, 1))
    bnd = F.conv2d(d0, W1.abs(), padding=1) + 75 * EPS * (F.conv2d(h0, W1.abs(), padding=1) + B1.abs().view(1, -1, 1, 1))
    return want, bnd


@pytest.mark.gpu
@pytest.mark.parametrize("ppt", [2, 4])
def test_conv_stem_pixels_per_thread(ppt):
    """relu(conv1(relu(conv0(x)))) on a 1600x1200 image against float64 F.conv2d.  Bound: conv0 has 27 products and the
    bias (28 roundings, + 2 for the order of the fp32 sum): 30 eps (|w0| * |x| + |b0|); conv1 carries that through |w1|
    and adds 75 eps (|w1| * |h0| + |b1|) for its 72 products."""
    x, w0, b0, w1, b1 = stem_case(ppt, 1200, 1600)
    want, bnd = stem_reference(*[t.to(DEV, F64) for t in (x, w0, b0, w1, b1)])
    try:
        ops.set_tuning("reset")
        ops.set_tuning("stem_ppt", ppt)
        got = ops.conv_stem(x.to(DEV), w0, b0, w1, b1)
    finally:
        ops.set_tuning("reset")
    assert_within(f"conv_stem ppt={ppt}", got, want, bnd, ("n", "c", "y", "x"))


# ------------------------------------------------------------------------------------------------
# sensitivity of the comparisons (CPU): one planted error at the last pixel of a partial block is rejected
# ------------------------------------------------------------------------------------------------


def plant_rejected(what, got, want, bound, dims, at):
    """A correct output passes; the same output with one element moved by 10x its bound (at most 1e-3 of scale) fails.
    `at` is the last pixel of the map, with None in place of the slice index (hypothesis or channel group): the last
    slice is used, a choice made without looking at the bound."""
    assert_within(what, got, want, bound, dims)
    if None in at:
        k = at.index(None)
        at = tuple(want.shape[k] - 1 if i == k else a for i, a in enumerate(at))
    scale = float(want.abs().max())
    delta = 10 * float(bound[at])
    assert 0 < delta <= 1e-3 * scale, f"{what}: the bound at the planted element ({float(bound[at]):.3e}) is too loose for scale {scale:.3g}"
    bad = got.clone()
    bad[at] += delta
    with pytest.raises(AssertionError, match="worst element"):
        assert_within(what, bad, want, bound, dims)


def test_sensitivity_warp_corr():
    # 13 x 23 map: 299 pixels, not a multiple of any block; the last pixel (12, 22); one channel group, one hypothesis
    r = dict(B=1, V=2, C=32, G=8, H=13, W=23, D=5)
    case = ka_case(r, seed=3)
    ref64 = case["ref"].double()
    sim, bnd = ka_reference(ref64, case["src"][0].double(), case["rt"][0].double(), case["depth"].double(), r["G"])
    got = sim.float()  # a correct fp32 output: within eps |sim|
    plant_rejected("warp_corr", got, sim, bnd, SIM_DIMS[1:], (0, None, 2, 12, 22))


def test_sensitivity_aggregate_and_heads():
    r = dict(B=1, V=2, C=32, G=8, H=13, W=23, D=5)
    case = ka_case(r, seed=4)
    sims, bounds = zip(*[ka_reference(case["ref"].double(), case["src"][v].double(), case["rt"][v].double(), case["depth"].double(), 8)
                         for v in range(2)])
    agg, agg_b = aggregate_reference(list(sims), list(bounds), case["vw"].double())
    plant_rejected("warp_corr (view-weighted)", agg.float(), agg, agg_b, SIM_DIMS[1:], (0, 5, None, 12, 22))
    sc, sc_b = head_reference(head_layers(random_head(SimilarityNet, 8, 1)), agg, agg_b)
    plant_rejected("warp_corr_score", sc.float(), sc, sc_b, ("b", "d", "y", "x"), (0, None, 12, 22))
    o, do = head_reference(head_layers(random_head(PixelwiseNet, 8, 2)), sims[0], bounds[0])
    s, ds = sigmoid_bound(o, do)
    plant_rejected("warp_corr_view_weights", s.amax(1).float(), s.amax(1), ds.amax(1), ("b", "y", "x"), (0, 12, 22))


def test_sensitivity_offset_corr():
    g = torch.Generator().manual_seed(5)
    B, C, G, K, H, W = 1, 32, 8, 9, 13, 23
    ref = smooth(g, B, C, H=H, W=W).double()
    off = offsets_reaching_borders(g, B, K, H, W, reach=4.0).double()
    want, bnd = oc_reference(ref, off, G, K, 4)
    plant_rejected("offset_corr", want.float(), want, bnd, ("b", "g", "k", "y", "x"), (0, None, 8, 12, 22))
    from patchmatchnet_b200.patchmatch import FeatureWeightNet

    o, do = head_reference(head_layers(random_head(lambda gg: FeatureWeightNet(K, gg), G, 9)), want, bnd)
    s, ds = sigmoid_bound(o, do)
    plant_rejected("offset_corr_weight", s.float(), s, ds, ("b", "k", "y", "x"), (0, None, 12, 22))


def test_sensitivity_init_propagate():
    r = dict(B=1, H=13, W=23, Kp=8, mode=ops.MODE_PERTURB)
    g = torch.Generator().manual_seed(6)
    seed, off, dmin, dmax = kc_inputs(r, g)
    want, bnd, xn, xb = kc_reference(seed.double(), off.double(), dmin.double(), dmax.double(), ops.MODE_PERTURB, 8, 8, 4, 0.0125, 13, 23)
    plant_rejected("init_propagate", want.float(), want, bnd, ("b", "d", "y", "x"), (0, None, 12, 22))
    plant_rejected("init_propagate xnorm", xn.float(), xn, xb, ("b", "d", "y", "x"), (0, None, 12, 22))


@pytest.mark.parametrize("inverse", [False, True])
def test_sensitivity_adaptive_eval(inverse):
    r = dict(B=1, D=8, H=13, W=23, K=9, inverse=inverse)
    g = torch.Generator().manual_seed(7)
    score0, depth, off, fw, dmin, dmax = kb_inputs(r, g)
    prob, dp, dep, dd = kb_reference(score0.double(), depth.double(), off.double(), fw.double(), dmin.double(), dmax.double(), 4,
                                     0.0125, inverse, 9)
    plant_rejected("adaptive_eval prob", prob.float(), prob, dp, ("b", "d", "y", "x"), (0, None, 12, 22))
    plant_rejected("adaptive_eval depth", dep.float(), dep, dd, ("b", "y", "x"), (0, 12, 22))


def test_sensitivity_conv_stem():
    want, bnd = stem_reference(*[t.double() for t in stem_case(2, 13, 23)])
    plant_rejected("conv_stem", want.float(), want, bnd, ("n", "c", "y", "x"), (0, None, 12, 22))
