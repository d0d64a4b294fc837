"""The PatchMatch backward kernels (csrc/pm_backward.cu) at the map sizes training runs, element by element against float64
references, and the argument checks of their launchers.

Shape table.  Derived from train.py's defaults (the per-stage values of synthetic.DEFAULT_NET_KWARGS) and the iteration
logic of PatchMatch.forward: the stage maps of 640x512 (DTU, B=4, V=4, every stage and iteration), of 512x640 (portrait,
one row per stage), train.py's default B=12, V=5 at stage 3 iteration 1, a reference with landscape and portrait sources
of other sizes (the ragged-pack backward), and a uniform pack whose sources are not the reference's size.  Stage 3's first
iteration goes through AggregateViews (K-A without view weights), every later one through K-A with the view weights; stage
1's only iteration is the inverse regression without propagation.  Synthetic rows reach what the defaults never take.

Each backward is called on its own, with fp32 inputs; its float64 reference takes exactly those values, upcast.  The
incoming gradients are smooth fields, so that neighbouring contributions do not cancel into a meaningless scale.

Bounds are fixed per element before any comparison (eps = 2^-24):
  * sums: (m + c) eps * (sum of |terms|), the |terms| from the same reference run on absolute values, m the number of
    contributions an element receives (a count scatter for the atomically accumulated d_src and d_score0: an fp32 sum of m
    terms in any order, or any tree of partial sums, is within (m - 1) eps of the sum of |terms|, with or without fma);
  * sample positions: the bilinear tap weights are 1-Lipschitz tents, continuous across the zero-padded and clamped edges,
    so they move by at most |du| + |dv| (project_bound for K-A, border_dpos for the border-clamped gathers);
  * the position gradients (K-A', K-C, K-B d_offsets) jump where the gather crosses a texel column (row) and at the clamp
    edges, where the multiplier gmx (gmy) drops to 0: within dpos of such a place any value in the hull of the one-sided
    derivatives is accepted, widened by the bound.  Inside a cell the derivative moves with the other coordinate by the
    mixed second difference of the map (curvature_map).
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import pm_oracle
from patchmatchnet_b200 import _native, ops, synthetic
from patchmatchnet_b200.net import PatchmatchNet
from tests.test_emulated_kernels import _aligned
from tests.test_gpu_kernels_at_scale import (CHUNK_ELEMS, EPS, F64, assert_within, border_dpos, border_sample_bound,
                                             ka_case, kb_inputs, kb_reference, lipschitz_map, offsets_reaching_borders,
                                             pixel_positions, plant_rejected, project_bound, smooth,
                                             stage_config, stage_iterations, xnorm_bound)

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE_DOWN = {3: 8, 2: 4, 1: 2}
PASSES = {}  # worst |err| / bound per kernel output over the rows run, printed by each test

# ------------------------------------------------------------------------------------------------
# shape table
# ------------------------------------------------------------------------------------------------

# (tag, B, V, H, W of the images, which iterations)
TRAIN_RUNS = (("dtu", 4, 4, 512, 640, "all"), ("portrait", 4, 4, 640, 512, "it1"), ("default", 12, 5, 512, 640, "s3it1"))
# the ETH3D-style mix of tests/multisize_train_cases.py (multisize_cases.NET_SIZES) scaled to --image-max-dim 640
MIXED_REF = (512, 640)
MIXED_SRC = ((512, 640), (640, 512), (512, 640), (384, 576))


def _row(name, B, V, stage, H, W, it, itc, **kw):
    c = stage_config(stage)
    first = stage == 3 and it == 1  # no view weights yet: K-A without them, then AggregateViews
    r = dict(name=name, B=B, V=V, H=H, W=W, C=c["C"], G=c["G"], dil=c["dil"], K=c["K"], scale=c["scale"], vw=not first,
             agg=first, sizes=None, oc=it == 1, grads="depth", offs="borders", ka="plain", **itc)
    r.update(kw)
    return r


def shape_table():
    rows = []
    for tag, B, V, Hi, Wi, which in TRAIN_RUNS:
        for stage in (3, 2, 1):
            for it, itc in enumerate(stage_iterations(stage), 1):
                if (which == "it1" and it != 1) or (which == "s3it1" and (stage, it) != (3, 1)):
                    continue
                rows.append(_row(f"{tag}/s{stage}/it{it}", B, V, stage, Hi // STAGE_DOWN[stage], Wi // STAGE_DOWN[stage], it, itc))
    for stage, it in ((3, 1), (3, 2), (2, 1), (1, 1)):
        dn = STAGE_DOWN[stage]
        rows.append(_row(f"mixed/s{stage}/it{it}", 2, len(MIXED_SRC), stage, MIXED_REF[0] // dn, MIXED_REF[1] // dn, it,
                         stage_iterations(stage)[it - 1], sizes=[(h // dn, w // dn) for h, w in MIXED_SRC]))
    # one uniform pack whose sources are all of another size than the reference (stage 2 of 640x512, 3/4 x 5/4)
    rows.append(_row("dtu-hs/s2/it1", 2, 4, 2, 128, 160, 1, stage_iterations(2)[0], sizes=[(96, 200)] * 4, uniform=True))
    return rows


def _synthetic(name, stage, H, W, B=2, V=4, it=1, **kw):
    itc = dict(stage_iterations(stage)[it - 1])
    for k in ("mode", "Ns", "Kp", "inverse"):
        if k in kw:
            itc[k] = kw.pop(k)
    itc["D"] = itc["Ns"] + itc["Kp"]
    return _row(name, B, V, stage, H, W, it, itc, **kw)


# rows for branches the defaults never take
SYNTHETIC = [
    _synthetic("synthetic/K17", 2, 128, 160, K=17),
    _synthetic("synthetic/Kp4-perturb", 2, 128, 160, Kp=4),
    _synthetic("synthetic/Kp4-random", 3, 64, 80, Kp=4),
    _synthetic("synthetic/Kp8-random", 3, 64, 80, Kp=8),
    _synthetic("synthetic/Kp4-passthrough", 2, 128, 160, mode=ops.MODE_PASSTHROUGH, Ns=1, Kp=4),
    _synthetic("synthetic/Kp8-passthrough", 2, 128, 160, mode=ops.MODE_PASSTHROUGH, Ns=1, Kp=8),
    _synthetic("synthetic/Kp16-passthrough", 3, 64, 80, mode=ops.MODE_PASSTHROUGH, Ns=1, Kp=16, it=2),
    _synthetic("synthetic/D256", 1, 64, 80, B=1, Ns=240, Kp=16, mode=ops.MODE_PERTURB, inverse=True),
    _synthetic("synthetic/V16", 3, 64, 80, B=2, V=16),
    # K-A without view weights at the stage-2 and stage-1 (C, G), uniform and ragged
    _synthetic("synthetic/s2-no-vw", 2, 128, 160, vw=False),
    _synthetic("synthetic/s1-no-vw", 1, 128, 160, vw=False),
    _synthetic("synthetic/s2-no-vw-views", 2, 128, 160, vw=False, sizes=[(128, 160), (160, 128), (96, 144)]),
    _synthetic("synthetic/s1-no-vw-views", 1, 128, 160, vw=False, sizes=[(128, 160), (160, 128), (96, 144)]),
    _synthetic("synthetic/grad-prob", 3, 64, 80, it=2, grads="prob"),
    _synthetic("synthetic/grad-both", 2, 128, 160, grads="both"),
    _synthetic("synthetic/grad-both-inverse", 1, 128, 160, grads="both"),
]

# edge rows: each reaches its structure by construction (test_edge_rows_reach_their_structure)
EDGES = [
    _synthetic("edge/ka-runs", 3, 64, 80, B=1, it=2, ka="runs"),
    _synthetic("edge/ka-tiny-sources", 3, 64, 80, B=1, it=2, sizes=[(1, 1), (2, 3), (64, 80), (80, 64)]),
    _synthetic("edge/texels", 2, 128, 160, offs="texels"),
    _synthetic("edge/texels-s3", 3, 64, 80, offs="texels", it=2),
    _synthetic("edge/kc-tie", 2, 128, 160, offs="tie"),
]


def all_rows():
    return shape_table() + SYNTHETIC + EDGES


def row(name):
    return next(r for r in all_rows() if r["name"] == name)


def ka_rows():
    return [r["name"] for r in all_rows()]


def agg_rows():
    return [r["name"] for r in all_rows() if r["agg"] or r["name"] == "synthetic/V16"]


def oc_rows():
    return [r["name"] for r in all_rows() if r["oc"]]


def kc_rows():
    return [r["name"] for r in all_rows() if r["Kp"] > 0]


def kb_rows():
    return [r["name"] for r in all_rows()]


def ka_launch(r):
    """(C, G, pack, view weights) of the K-A backward launch of row r."""
    pack = "views" if r["sizes"] and not r.get("uniform") else "uniform"
    return (r["C"], r["G"]), pack, "vw" if r["vw"] else "null"


def test_shape_table_reaches_every_launch_branch():
    rows = all_rows()
    net = shape_table()
    # the training configuration as PatchMatch.forward runs it
    assert row("dtu/s3/it1")["D"] == 64 and row("dtu/s3/it1")["mode"] == ops.MODE_RANDOM and row("dtu/s3/it1")["agg"]
    assert row("dtu/s3/it2")["D"] == 32 and row("dtu/s3/it2")["vw"] and not row("dtu/s3/it2")["agg"]
    assert row("dtu/s2/it2")["D"] == 16 and row("dtu/s1/it1")["Kp"] == 0 and row("dtu/s1/it1")["inverse"]
    assert (row("dtu/s1/it1")["H"], row("dtu/s1/it1")["W"]) == (256, 320) and (row("portrait/s1/it1")["H"], row("portrait/s1/it1")["W"]) == (320, 256)
    assert {(r["B"], r["V"]) for r in net} == {(4, 4), (12, 5), (2, 4)}
    assert {ka_launch(r) for r in rows} == {(cg, p, w) for cg in ((64, 8), (32, 8), (16, 4)) for p in ("uniform", "views")
                                           for w in ("vw", "null")}
    assert any(r.get("uniform") for r in rows)
    assert {r["K"] for r in rows if r["oc"]} == {9, 17}
    assert {(r["Kp"], r["mode"]) for r in rows if r["Kp"] > 0} == {(kp, m) for kp in (4, 8, 16) for m in (0, 1, 2)}
    assert {r["inverse"] for r in rows} == {False, True}
    assert {r["grads"] for r in rows} == {"depth", "prob", "both"}
    assert max(r["D"] for r in rows) == 256 and max(r["V"] for r in rows if r["agg"] or r["name"] == "synthetic/V16") == 16
    assert not any((r["mode"], r["Ns"]) == (ops.MODE_PASSTHROUGH, 1) for r in net)
    # each synthetic row adds something the network rows do not have
    key = lambda r: (ka_launch(r), r["K"], r["Kp"], r["mode"], r["inverse"], r["grads"], r["D"] == 256, r["V"])
    for r in SYNTHETIC:
        assert key(r) not in {key(n) for n in net}, r["name"]


# ------------------------------------------------------------------------------------------------
# where the kernels run: the GPU, or the unmodified kernel bodies under the host emulator
# ------------------------------------------------------------------------------------------------


class Runner:
    """Calls one backward entry point on fp32 inputs (CPU tensors in NCHW) and returns its outputs as float tensors on the
    device the references run on."""

    def __init__(self, emu=None):
        self.emu = emu
        self.dev = "cpu" if emu is not None else "cuda:0"

    def put(self, t):
        if t is None:
            return None
        t = t.detach().float().contiguous()
        return _aligned(t) if self.emu is not None else t.to(self.dev)

    def empty(self, *shape):
        t = torch.full(shape, float("nan"))
        return _aligned(t) if self.emu is not None else t.to(self.dev)

    def call(self, name, *args):
        p = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
        if self.emu is not None:
            rc = getattr(self.emu, "emu_" + name)(*p)
        else:
            rc = getattr(_native.lib(), "pmb200_" + name)(*p, None)
            torch.cuda.synchronize()
        if rc != 0:
            raise RuntimeError(f"{name}: {rc} {_native.lib().pmb200_last_error() if self.emu is None else ''}")

    def ka(self, ref, srcs, rt, depth, vw, gout, G, views):
        B, C, H, W = ref.shape
        V, D = len(srcs), depth.shape[1]
        nhwc = lambda x: x.permute(0, 2, 3, 1)
        ref_n, rt_, dep, vw_, g_ = self.put(nhwc(ref)), self.put(rt), self.put(depth), self.put(vw), self.put(gout)
        d_ref = self.empty(B, H, W, C)
        if not views:
            hs, ws = srcs[0].shape[-2:]
            src = self.put(torch.stack([nhwc(s) for s in srcs]))
            d_src = self.empty(V, B, hs, ws, C)
            self.call("warp_corr_backward", ref_n, src, rt_, dep, vw_, g_, d_ref, d_src, V, B, C, G, H, W, hs, ws, D)
            out = [d_src[v].permute(0, 3, 1, 2) for v in range(V)]
        else:
            shapes = [tuple(s.shape[-2:]) for s in srcs]
            offsets, total = ops.ViewPack.layout(shapes, B, C)
            flat = torch.zeros(total)
            for o, s in zip(offsets, srcs):
                flat[o:o + s.numel()] = nhwc(s).reshape(-1)
            ext = (_native.ViewExtent * V)()
            for v, (o, (h, w)) in enumerate(zip(offsets, shapes)):
                ext[v].offset, ext[v].height, ext[v].width = o, h, w
            data, d_src = self.put(flat), self.empty(total)
            self.call("warp_corr_views_backward", ref_n, data, ext, rt_, dep, vw_, g_, d_ref, d_src, V, B, C, G, H, W, D)
            out = [d_src[o:o + B * h * w * C].view(B, h, w, C).permute(0, 3, 1, 2) for o, (h, w) in zip(offsets, shapes)]
        return d_ref.permute(0, 3, 1, 2), out

    def agg(self, sims, vw, gout):
        V, B, G, D, H, W = sims.shape
        s, w, g = self.put(sims), self.put(vw), self.put(gout)
        d_sims, d_vw = self.empty(V, B, G, D, H, W), self.empty(B, V, H, W)
        self.call("aggregate_views_backward", s, w, g, d_sims, d_vw, V, B, G, D, H, W)
        return d_sims, d_vw

    def oc(self, ref, off, gout, G, K, dil):
        B, C, H, W = ref.shape
        ref_n, o, g = self.put(ref.permute(0, 2, 3, 1)), self.put(off), self.put(gout)
        d_off = self.empty(B, 2 * K, H, W)
        self.call("offset_corr_backward", ref_n, o, g, d_off, B, C, G, H, W, K, dil)
        return d_off

    def kc(self, seed, off, dmin, dmax, gout, mode, Ns, Kp, dil, scale):
        B, _, H, W = seed.shape
        args = [self.put(t) for t in (seed, off, dmin, dmax, gout)]
        d_off = self.empty(B, 2 * Kp, H, W)
        self.call("init_propagate_backward", *args, d_off, mode, B, H, W, Ns, Kp, dil, ctypes.c_float(scale))
        return d_off

    def kb(self, score0, depth, xnorm, off, fw, dmin, dmax, prob, gd, gp, dil, scale, inverse):
        B, D, H, W = score0.shape
        K = fw.shape[1]
        args = [self.put(t) for t in (score0, depth, xnorm, off, fw, dmin, dmax, prob, gd, gp)]
        outs = [self.empty(B, D, H, W), self.empty(B, D, H, W), self.empty(B, 2 * K, H, W), self.empty(B, K, H, W)]
        self.call("adaptive_eval_backward", *args, *outs, B, D, H, W, K, dil, ctypes.c_float(scale), int(inverse))
        return outs


@pytest.fixture(scope="module")
def emu():
    srcs = [os.path.join(REPO, "tests", f) for f in ("emu_backward.cpp", "emu_views_backward.cpp")]
    deps = srcs + [os.path.join(REPO, "tests", "warp_emu.h"), os.path.join(REPO, "include", "patchmatch_b200.h")]
    deps += [os.path.join(REPO, "patchmatchnet_b200", "csrc", f) for f in ("pm_backward.cu", "pm_math.cuh")]
    out = os.path.join(REPO, "tests", "_emu_backward_at_scale.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")  # vector_types.h only
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-I{cuda_inc}", "-o", out] + srcs, check=True,
                       cwd=os.path.join(REPO, "tests"))
    lib = ctypes.CDLL(out)
    P, I, F32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    lib.emu_warp_corr_backward.argtypes = [P] * 8 + [I] * 9
    lib.emu_warp_corr_views_backward.argtypes = [P, P, ctypes.POINTER(_native.ViewExtent)] + [P] * 6 + [I] * 7
    lib.emu_aggregate_views_backward.argtypes = [P] * 5 + [I] * 6
    lib.emu_offset_corr_backward.argtypes = [P] * 4 + [I] * 7
    lib.emu_init_propagate_backward.argtypes = [P] * 6 + [I] * 7 + [F32]
    lib.emu_adaptive_eval_backward.argtypes = [P] * 14 + [I] * 6 + [F32, I]
    for fn in ("emu_warp_corr_backward", "emu_warp_corr_views_backward", "emu_aggregate_views_backward",
               "emu_offset_corr_backward", "emu_init_propagate_backward", "emu_adaptive_eval_backward"):
        getattr(lib, fn).restype = I
    return Runner(lib)


def mini(r):
    """Row r at the emulator's size: 40x56 maps (sources scaled alike), D <= 32, B <= 2, V <= 4 (V = 16 kept for the
    aggregation)."""
    m = dict(r)
    H, W = (40, 56) if r["W"] >= r["H"] else (56, 40)
    m.update(H=H, W=W, B=min(r["B"], 2))
    if r["V"] != 16:
        m["V"] = min(r["V"], 4)
    if r["sizes"]:
        m["sizes"] = [(max(1, h * H // r["H"]) if h > 3 else h, max(1, w * W // r["W"]) if w > 3 else w) for h, w in r["sizes"]][:m["V"]]
    if r["D"] > 32 and r["mode"] == ops.MODE_PERTURB:
        m["Ns"] = 32 - r["Kp"]
        m["D"] = 32
    return m


# ------------------------------------------------------------------------------------------------
# shared pieces of the references
# ------------------------------------------------------------------------------------------------


def _gather(f, idx):
    """f [B,C,H,W], idx [B,*S] flat texel indices -> [B,C,*S]"""
    B, C = f.shape[:2]
    return f.reshape(B, C, -1).gather(2, idx.reshape(B, 1, -1).expand(B, C, -1)).view(B, C, *idx.shape[1:])


def curvature_map(f):
    """[B,C,H,W] -> [B,C,H,W]: at every cell (texel = its top-left corner), an upper bound of the mixed second difference
    |f11 - f10 - f01 + f00| of the cells within one texel of it (border continuation).  Inside a cell d(gix)/d(fy) and
    d(giy)/d(fx) are exactly that difference."""
    p = F.pad(f, (0, 1, 0, 1), mode="replicate")
    m = (p[..., 1:, 1:] - p[..., 1:, :-1] - p[..., :-1, 1:] + p[..., :-1, :-1]).abs()
    return F.max_pool2d(m, 3, 1, padding=1)


def border_grad(f, ix, iy):
    """The backward's view of a border-clamped bilinear gather of f [B,C,H,W] at float64 texel coordinates ix, iy [B,*S]
    (before the clamp): taps and weights, gix, giy (bilinear_grad), the multipliers gmx, gmy (clip_coordinates_set_grad:
    0 at or beyond either border), the absolute terms of gix, giy and the cell's curvature bound.  -> dict of [B,C,*S]
    (gmx, gmy, weights, taps [B,*S])."""
    H, W = f.shape[-2:]
    gmx = torch.where((ix > 0) & (ix < W - 1), W / (W - 1), 0.0)
    gmy = torch.where((iy > 0) & (iy < H - 1), H / (H - 1), 0.0)
    cx, cy = ix.clamp(0, W - 1), iy.clamp(0, H - 1)
    x0, y0 = cx.floor(), cy.floor()
    fx, fy = (cx - x0).unsqueeze(1), (cy - y0).unsqueeze(1)
    dx, dy = (x0 + 1 <= W - 1).long(), (y0 + 1 <= H - 1).long()
    r0 = (y0 * W + x0).long()
    taps = [r0, r0 + dx, r0 + dy * W, r0 + dy * W + dx]
    v00, v01, v10, v11 = [_gather(f, t) for t in taps]
    d1, d0 = v11 - v10, v01 - v00
    e1, e0 = v10 - v00, v11 - v01
    wts = [(1 - fx) * (1 - fy), fx * (1 - fy) * dx.unsqueeze(1), (1 - fx) * fy * dy.unsqueeze(1), fx * fy * (dx * dy).unsqueeze(1)]
    return dict(gix=d0 * (1 - fy) + d1 * fy, giy=e1 * (1 - fx) + e0 * fx, gmx=gmx.unsqueeze(1), gmy=gmy.unsqueeze(1),
                aix=d0.abs() * (1 - fy) + d1.abs() * fy, aiy=e1.abs() * (1 - fx) + e0.abs() * fx,
                mix=_gather(curvature_map(f), r0), taps=taps, wts=wts,
                vabs=[v.abs() for v in (v00, v01, v10, v11)], fx=fx, fy=fy)


def sample_clamped(f, u, v):
    """Bilinear sample of f [B,C,h,w] at pixel coordinates u, v [B,*S], clamped to the map (1-pixel maps included)."""
    h, w = f.shape[-2:]
    cx, cy = u.clamp(0, w - 1), v.clamp(0, h - 1)
    x0, y0 = cx.floor(), cy.floor()
    fx, fy = (cx - x0).unsqueeze(1), (cy - y0).unsqueeze(1)
    x1, y1 = (x0 + 1).clamp(max=w - 1), (y0 + 1).clamp(max=h - 1)
    at = lambda y, x: _gather(f, (y * w + x).long())
    return (at(y0, x0) * (1 - fx) + at(y0, x1) * fx) * (1 - fy) + (at(y1, x0) * (1 - fx) + at(y1, x1) * fx) * fy


def texel_coords(px, py, H, W):
    """border_cell's texel coordinates of pixel positions (align_corners=False un-normalisation of the reference's grid)."""
    return px * (W / (W - 1)) - 0.5, py * (H / (H - 1)) - 0.5


def hull_check(what, got, cands, bound, dims):
    """got within `bound` of the hull [min, max] of the candidate values (one-sided derivatives at a kink; a single
    candidate where there is none)."""
    lo, hi = torch.stack(cands).amin(0), torch.stack(cands).amax(0)
    got64 = got.to(lo.device, F64)
    return assert_within(what, got, torch.minimum(torch.maximum(got64, lo), hi), bound, dims)


def record(op, worst):
    PASSES[op] = max(PASSES.get(op, 0.0), worst)
    print(f"[worst] {op}: {PASSES[op]:.3g}")


def pool_texels(t):
    """[B,C,h,w] -> max over each texel's 3x3 neighbourhood (a rounded position may sit in the next cell)"""
    return F.max_pool2d(t, 3, 1, padding=1)


# ------------------------------------------------------------------------------------------------
# K-A backward
# ------------------------------------------------------------------------------------------------


def ka_bwd_reference(ref, srcs, rt, depth, vw, gout, G):
    """d_ref, d_src of K-A in float64, with their bounds.  ref [B,C,H,W], srcs: V maps [B,C,h_v,w_v], rt [V,B,12], depth
    [B,D,H,W], vw [B,V,H,W] or None, gout [V,B,G,D,H,W] (vw None) or [B,G,D,H,W]; all float64 on one device.

    gamma = gout * s_v / n (s_v = vw_v / (1e-5 + sum vw), 1 without weights; n = C / G); S_c the zero-padded bilinear
    sample of source channel c at the projected position (u, v), taps t with weights w_t.
      d_ref_c  = sum_{v,d} gamma S_c            d_src_c[t] = sum_{pixels, d} gamma r_c w_t
    Rounding.  gamma: s_v (V sums, the division) and two products, (V + 4) eps relative; w_t two roundings (1 - f, the
    product); S_c four products and three sums.  d_ref: V D fused accumulations -> (V D + V + 14) eps sum |gamma| S^abs_c.
    d_src: every term is gamma r w_t rounded (V + 8) eps, then summed in registers while hypotheses stay in one cell and
    by atomics in an arbitrary order, m terms in all -> (m + V + 10) eps sum |gamma r| w_t, m from the count scatter.
    Position.  |dw_t| <= |du| + |dv| <= 2 dpos (project_bound): d_ref moves by dpos sum |gamma| L_c (lipschitz_map of the
    source, sampled there), d_src by 2 dpos sum |gamma r|, scattered to the taps of every position within a texel of the
    map.  A rounded position may use the next cell: the count and the position term are maxed over 3x3 texels."""
    B, C, H, W = ref.shape
    D, V, n = depth.shape[1], len(srcs), C // G
    wsum = 1e-5 + vw.sum(1) if vw is not None else None
    d_ref, a_ref, p_ref = [torch.zeros_like(ref) for _ in range(3)]
    d_srcs, b_srcs = [], []
    step = max(1, CHUNK_ELEMS // (B * C * H * W))
    for v, src in enumerate(srcs):
        hs, ws = src.shape[-2:]
        gv = gout[v] if vw is None else gout * (vw[:, v] / wsum)[:, None, None]
        gam = (gv / n).repeat_interleave(n, 1)  # [B,C,D,H,W]
        L = lipschitz_map(src, zero_pad=True)
        ds, a_s, p_s = [torch.zeros(B, C, hs * ws, dtype=F64, device=ref.device) for _ in range(3)]
        cnt = torch.zeros(B, 1, hs * ws, dtype=F64, device=ref.device)
        for d0 in range(0, D, step):
            u, vv, dpos = project_bound(rt[v], depth[:, d0:d0 + step], H, W, hs, ws)
            g = gam[:, :, d0:d0 + step]
            x0, y0 = u.floor(), vv.floor()
            fx, fy = u - x0, vv - y0
            S = Sa = 0
            gr = g * ref[:, :, None]
            near = (u >= -2) & (u < ws + 1) & (vv >= -2) & (vv < hs + 1)
            for ox, oy in ((0, 0), (1, 0), (0, 1), (1, 1)):
                xi, yi = x0 + ox, y0 + oy
                w = (fx if ox else 1 - fx) * (fy if oy else 1 - fy)
                valid = (xi >= 0) & (xi <= ws - 1) & (yi >= 0) & (yi <= hs - 1)
                w = torch.where(valid, w, 0.0)
                idx = (yi.clamp(0, hs - 1) * ws + xi.clamp(0, ws - 1)).long()
                S = S + w[:, None] * _gather(src, idx)
                Sa = Sa + w[:, None] * _gather(src.abs(), idx)
                ie = idx.reshape(B, 1, -1).expand(B, C, -1)
                ds.scatter_add_(2, ie, (gr * w[:, None]).reshape(B, C, -1))
                a_s.scatter_add_(2, ie, (gr.abs() * w[:, None]).reshape(B, C, -1))
                cnt.scatter_add_(2, idx.reshape(B, 1, -1), valid.to(F64).reshape(B, 1, -1))
                p_s.scatter_add_(2, ie, (gr.abs() * (2 * dpos * near)[:, None]).reshape(B, C, -1))
            d_ref += (g * S).sum(2)
            a_ref += (g.abs() * Sa).sum(2)
            p_ref += (g.abs() * dpos[:, None] * sample_clamped(L, u, vv)).sum(2)
            del S, Sa, gr, g, u, vv, dpos
        m = pool_texels(cnt.view(B, 1, hs, ws))
        d_srcs.append(ds.view(B, C, hs, ws))
        b_srcs.append((m + V + 10) * EPS * a_s.view(B, C, hs, ws) + pool_texels(p_s.view(B, C, hs, ws)))
    return d_ref, (V * D + V + 14) * EPS * a_ref + p_ref, d_srcs, b_srcs


def ka_bwd_inputs(r, seed):
    """Row r's K-A backward inputs (fp32, CPU): ka_case's features, projections, hypotheses and view weights, the sources at
    the row's sizes, a smooth incoming gradient; the "runs" edge row replaces the hypotheses (see ka_runs_depth)."""
    g = torch.Generator().manual_seed(seed)
    case = ka_case(r, seed)
    B, V, C, G, D, H, W = r["B"], r["V"], r["C"], r["G"], r["D"], r["H"], r["W"]
    if r["sizes"]:
        srcs = [smooth(g, B, C, H=h, W=w) for h, w in r["sizes"]]
    else:
        srcs = list(case["src"])
    depth = ka_runs_depth(case["depth"]) if r["ka"] == "runs" else case["depth"]
    vw = case["vw"] if r["vw"] else None
    gout = smooth(g, V, B, G, D, H=H, W=W) if vw is None else smooth(g, B, G, D, H=H, W=W)
    return case["ref"], srcs, case["rt"], depth, vw, gout


def ka_runs_depth(depth):
    """Hypotheses built for the register accumulation of d_src: from each pixel's first hypothesis d, 0-11 within 1e-6 d
    of it (one run in one source cell), 12 behind the camera, 13-19 the run again around 16, which lies beyond the map
    (d = 0.01 puts Z near 0.01 and the projection hundreds of pixels out), 20-27 alternating d and 1.3 d (cells A, B, A,
    ...), the rest close to d again."""
    base = depth[:, :1]
    D = depth.shape[1]
    out = base.repeat(1, D, 1, 1) * (1 + 1e-6 * torch.arange(D, dtype=torch.float32).view(1, D, 1, 1))
    out[:, 12] = -1.0
    out[:, 16] = 0.01
    out[:, 20:28:2] = base * 1.0
    out[:, 21:28:2] = base * 1.3
    return out


def check_ka(tag, rn, r, seed=None, twice=False):
    ref, srcs, rt, depth, vw, gout = ka_bwd_inputs(r, r["H"] + r["D"] if seed is None else seed)
    views = bool(r["sizes"]) and not r.get("uniform")
    got_ref, got_src = rn.ka(ref, srcs, rt, depth, vw, gout, r["G"], views)
    up = lambda t: None if t is None else t.to(rn.dev, F64)
    want_ref, b_ref, want_src, b_src = ka_bwd_reference(up(ref), [up(s) for s in srcs], up(rt), up(depth), up(vw), up(gout), r["G"])
    record("warp_corr_backward d_ref", assert_within(f"{tag} d_ref", got_ref, want_ref, b_ref, ("b", "c", "y", "x")))
    for v in range(len(srcs)):
        record("warp_corr_backward d_src", assert_within(f"{tag} d_src view {v}", got_src[v], want_src[v], b_src[v], ("b", "c", "y", "x")))
    if twice:  # d_ref is written by plain stores: bit-identical; d_src by atomics: within its bound again
        again_ref, again_src = rn.ka(ref, srcs, rt, depth, vw, gout, r["G"], views)
        assert torch.equal(again_ref, got_ref), f"{tag}: d_ref differs between two runs"
        for v in range(len(srcs)):
            assert_within(f"{tag} d_src view {v} (second run)", again_src[v], want_src[v], b_src[v], ("b", "c", "y", "x"))


# ------------------------------------------------------------------------------------------------
# aggregate_views backward
# ------------------------------------------------------------------------------------------------


def agg_bwd_reference(sims, vw, gout):
    """d_sims, d_vw of S = sum_v w_v s_v / wsum (wsum = 1e-5 + sum_v w_v) in float64, sims [V,B,G,D,H,W], vw [B,V,H,W],
    gout [B,G,D,H,W].  d_sims_v = g w_v / wsum: wsum (V roundings), the product and the division: (V + 3) eps.
    d_vw_v = sum_k g_k (s_vk - S_k) / wsum over the G D slices k: S_k is within (V + 2) eps S^abs_k (S^abs = sum_v w_v |s_v|
    / wsum), the difference adds eps |s - S|, each term two more roundings and wsum's V, and the GD fused accumulations one
    each: (GD + 2V + 8) eps sum_k |g_k| (|s_vk - S_k| + S^abs_k) / wsum."""
    V, B, G, D, H, W = sims.shape
    wsum = (1e-5 + vw.sum(1))[:, None, None]  # [B,1,1,H,W]
    w = vw.permute(1, 0, 2, 3)[:, :, None, None]  # [V,B,1,1,H,W]
    S = (sims * w).sum(0) / wsum
    Sa = (sims.abs() * w).sum(0) / wsum
    d_sims = gout * w / wsum
    dev = sims - S
    d_vw = (gout * dev / wsum).sum((2, 3)).permute(1, 0, 2, 3)
    b_vw = (G * D + 2 * V + 8) * EPS * (gout.abs() * (dev.abs() + Sa) / wsum).sum((2, 3)).permute(1, 0, 2, 3)
    return d_sims, (V + 3) * EPS * d_sims.abs(), d_vw, b_vw


def agg_inputs(r, seed):
    g = torch.Generator().manual_seed(seed)
    V, B, G, D, H, W = r["V"], r["B"], r["G"], r["D"], r["H"], r["W"]
    return smooth(g, V, B, G, D, H=H, W=W), torch.rand(B, V, H, W, generator=g) + 0.05, smooth(g, B, G, D, H=H, W=W)


def check_agg(tag, rn, r, twice=False):
    sims, vw, gout = agg_inputs(r, r["V"] + r["H"])
    got_s, got_w = rn.agg(sims, vw, gout)
    ws, bs, wv, bv = agg_bwd_reference(*[t.to(rn.dev, F64) for t in (sims, vw, gout)])
    record("aggregate_views_backward d_sims", assert_within(f"{tag} d_sims", got_s, ws, bs, ("view", "b", "g", "d", "y", "x")))
    record("aggregate_views_backward d_vw", assert_within(f"{tag} d_vw", got_w, wv, bv, ("b", "view", "y", "x")))
    if twice:
        again_s, again_w = rn.agg(sims, vw, gout)
        assert torch.equal(again_s, got_s) and torch.equal(again_w, got_w), f"{tag}: not bit-identical across runs"


# ------------------------------------------------------------------------------------------------
# offsets: smooth with exact values at the borders, on texel boundaries, or the K-C tie
# ------------------------------------------------------------------------------------------------


def offsets_on_texels(gen, B, K, H, W, table, reach):
    """Raw offsets [B,2K,H,W] whose gathers land on integer texel positions (cell boundaries, and 0 / size-1 where they
    reach the clamp edges): the smooth offsets of `reach` pixels moved to the nearest texel, computed in float64 and
    rounded once."""
    off = smooth(gen, B, 2 * K, H=H, W=W).double() * reach
    px, py = pixel_positions(table, off, H, W)
    ix, iy = texel_coords(px, py, H, W)
    tx = (ix.round() + 0.5) * ((W - 1) / W) - (px - off[:, 0::2])
    ty = (iy.round() + 0.5) * ((H - 1) / H) - (py - off[:, 1::2])
    return torch.stack([tx, ty], 2).view(B, 2 * K, H, W).float()


def kc_tie_offsets(gen, B, H, W, dil):
    """Propagation offsets (Kp = 8) with an exact tie between neighbours 0 (dy, dx = -d, -d) and 1 (-d, 0): off_x = +d on
    neighbour 0 and 0 on neighbour 1 give both the x position x + 0, and off_y = -y - 5 pushes both above the map, where
    they clamp to row 0 with fy = 0.  Their propagated values are then bit-equal in the kernel and equal in float64; the
    other six neighbours keep smooth offsets."""
    off = smooth(gen, B, 16, H=H, W=W) * 3.0
    ys = torch.arange(H, dtype=torch.float32).view(1, H, 1)
    off[:, 0], off[:, 2] = float(dil), 0.0
    off[:, 1], off[:, 3] = -ys - 5.0, -ys - 5.0
    return off


def make_offsets(r, g, K, kind_table):
    table = pm_oracle.neighbour_table(kind_table, K, r["dil"])
    B, H, W = r["B"], r["H"], r["W"]
    if r["offs"] == "texels":
        return offsets_on_texels(g, B, K, H, W, table, 3.0)
    if r["offs"] == "tie" and kind_table == "propagation":
        return kc_tie_offsets(g, B, H, W, r["dil"])
    return offsets_reaching_borders(g, B, K, H, W, reach=3.0)


def kink_positions(f, ix, iy, dpos):
    """border_grad at the float64 position and at the position moved by -dpos / +dpos along x and along y."""
    return [border_grad(f, ix + s * dpos, iy) for s in (-1, 0, 1)], [border_grad(f, ix, iy + s * dpos) for s in (-1, 0, 1)]


# ------------------------------------------------------------------------------------------------
# K-A' backward
# ------------------------------------------------------------------------------------------------


def oc_bwd_reference(ref, off, gout, G, K, dil):
    """d_offsets of K-A' (corr_k = (1/n) sum_c r_c B_c(p_k), B the border-clamped sample of the reference itself) in
    float64, as the hull of the one-sided values and its bound.  d_off_x,k = sum_c (gout_{g(c),k} / n) r_c gix_c gmx.
    Rounding: g = gout / n * r (2), gix (the difference, 1 - fy, two products, the sum: 5 relative to its absolute terms
    a_c), gx accumulated over C channels in registers and shuffles (C), times gmx (its own rounding and the product): (C +
    10) eps sum |g| a_c gmx.  Position: inside a cell gix moves with fy only, by the mixed difference (curvature_map): dpos
    sum |g| mix_c gmx.  The bound is the largest over the three candidate positions.  -> ([x, y] candidates lists, bound)
    with d_off laid out [B,2K,H,W]."""
    B, C, H, W = ref.shape
    n = C // G
    table = pm_oracle.neighbour_table("evaluation", K, dil)
    px, py = pixel_positions(table, off, H, W)
    dpos = border_dpos(px, py, H, W)
    ix, iy = texel_coords(px, py, H, W)
    gc = (gout / n).repeat_interleave(n, 1) * ref[:, :, None]  # [B,C,K,H,W]
    xs, ys = kink_positions(ref, ix, iy, dpos)
    cx = [(gc * t["gix"] * t["gmx"]).sum(1) for t in xs]
    cy = [(gc * t["giy"] * t["gmy"]).sum(1) for t in ys]
    bx = torch.stack([(gc.abs() * t["gmx"] * ((C + 10) * EPS * t["aix"] + dpos[:, None] * t["mix"])).sum(1) for t in xs]).amax(0)
    by = torch.stack([(gc.abs() * t["gmy"] * ((C + 10) * EPS * t["aiy"] + dpos[:, None] * t["mix"])).sum(1) for t in ys]).amax(0)
    inter = lambda a, b: torch.stack([a, b], 2).view(B, 2 * K, H, W)
    return [inter(a, b) for a, b in zip(cx, cy)], inter(bx, by)


def check_oc(tag, rn, r, twice=False):
    g = torch.Generator().manual_seed(r["H"] + r["K"])
    B, C, G, K, H, W = r["B"], r["C"], r["G"], r["K"], r["H"], r["W"]
    ref = smooth(g, B, C, H=H, W=W)
    off = make_offsets(r, g, K, "evaluation")
    gout = smooth(g, B, G, K, H=H, W=W)
    got = rn.oc(ref, off, gout, G, K, r["dil"])
    cands, bnd = oc_bwd_reference(*[t.to(rn.dev, F64) for t in (ref, off, gout)], G, K, r["dil"])
    record("offset_corr_backward d_offsets", hull_check(f"{tag} offset_corr d_offsets", got, cands, bnd, ("b", "k2", "y", "x")))
    if twice:
        assert torch.equal(rn.oc(ref, off, gout, G, K, r["dil"]), got), f"{tag}: d_offsets differ between two runs"


# ------------------------------------------------------------------------------------------------
# K-C backward
# ------------------------------------------------------------------------------------------------


def kc_values(seed, off, dmin, dmax, mode, Ns, Kp, dil, scale, H, W):
    """Every hypothesis of K-C in float64 before the sort and its bound (kc_reference's derivation: 16 eps |h| for the
    initial samples, 23 eps of |.| sampled plus the coordinate term for the propagated ones), and the centre map they
    gather.  -> (values [B,Ns+Kp,H,W], bounds, centre [B,1,H,W], px, py, the kernel's fp32 positions [B,Kp,2,H,W])"""
    B = dmin.shape[0]
    init = pm_oracle.init_hypotheses(dmin, dmax, H, W, scale, Ns if mode != ops.MODE_RANDOM else 16,
                                     seed if mode != ops.MODE_RANDOM else torch.empty(0, device=seed.device), seed.device,
                                     (lambda size, device: seed) if mode == ops.MODE_RANDOM else None)
    centre = init[:, init.shape[1] // 2:init.shape[1] // 2 + 1]
    table = pm_oracle.neighbour_table("propagation", Kp, dil)
    px, py = pixel_positions(table, off, H, W)
    S, sabs, coord = border_sample_bound(centre, px, py, H, W)
    # the kernel's fp32 positions: x + ((float)dx + off), two roundings
    off32 = off.float()
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32, device=off.device),
                            torch.arange(W, dtype=torch.float32, device=off.device), indexing="ij")
    pos32 = torch.stack([torch.stack([xs + (float(dx) + off32[:, 2 * k]), ys + (float(dy) + off32[:, 2 * k + 1])], 1)
                         for k, (dy, dx) in enumerate(table)], 1)  # [B,Kp,2,H,W]
    return (torch.cat([init, S[:, 0]], 1), torch.cat([16 * EPS * init.abs(), 23 * EPS * sabs[:, 0] + coord[:, 0]], 1),
            centre, px, py, pos32)


def kc_windows(vals, bnds, Ns, Kp, pos32):
    """Admissible slots [lo, hi] [B,Kp,H,W] of every propagated hypothesis.  Slot = number of hypotheses sorted before it;
    one whose value interval lies strictly below counts, one whose interval overlaps widens the window.  Two neighbours
    whose fp32 positions are identical gather bit-equal values in the kernel: when they are also equal in float64 the
    stable order decides (the lower neighbour index first), with no ambiguity."""
    D = Ns + Kp
    los, his = [], []
    for kk in range(Kp):
        j = Ns + kk
        v, b = vals[:, j], bnds[:, j]
        lo = torch.zeros_like(v, dtype=torch.long)
        amb = torch.zeros_like(lo)
        for i in range(D):
            if i == j:
                continue
            vi, bi = vals[:, i], bnds[:, i]
            eq = (vi == v) & (pos32[:, i - Ns] == pos32[:, kk]).all(1) if i >= Ns else torch.zeros_like(v, dtype=torch.bool)
            before = (vi + bi < v - b) | (eq & (i < j))
            overlap = ~eq & (vi + bi >= v - b) & (vi - bi <= v + b)
            lo += before.long()
            amb += (overlap & ~before).long()
        los.append(lo)
        his.append(lo + amb)
    return torch.stack(los, 1), torch.stack(his, 1)


def kc_bwd_reference(seed, off, dmin, dmax, gout, mode, Ns, Kp, dil, scale):
    """d_offsets of K-C in float64: for propagated hypothesis kk, gout[slot] gix gmx (gix of the centre map at its gather),
    the slot where the stable sort puts it.  Accepted: the hull of gout[r] * (gix gmx at the one-sided positions) over the
    admissible slots r (kc_windows).  Bound: max |gout| over the window times the error of gix gmx: the centre values carry
    16 eps |v| each, so gix is within 16 eps (|v00| + |v01|) (1 - fy) + 16 eps (|v10| + |v11|) fy + 5 eps a + dpos mix
    (a: its absolute terms, mix: curvature_map), and the two products and gmx add 3 eps |gix gmx|.
    -> (candidates, bound, windows (lo, hi), dict of the float64 gix gmx, giy gmy and their bounds)"""
    B, _, H, W = gout.shape
    vals, bnds, centre, px, py, pos32 = kc_values(seed, off, dmin, dmax, mode, Ns, Kp, dil, scale, H, W)
    lo, hi = kc_windows(vals, bnds, Ns, Kp, pos32)
    dpos = border_dpos(px, py, H, W)
    ix, iy = texel_coords(px, py, H, W)
    gmin = torch.full_like(vals[:, Ns:], float("inf"))
    gmax = torch.full_like(gmin, -float("inf"))
    for r in range(Ns + Kp):
        inwin = (lo <= r) & (r <= hi)
        gr = gout[:, r:r + 1].expand_as(gmin)
        gmin = torch.where(inwin, torch.minimum(gmin, gr), gmin)
        gmax = torch.where(inwin, torch.maximum(gmax, gr), gmax)
    gabs = torch.maximum(gmin.abs(), gmax.abs())
    xs, ys = kink_positions(centre, ix, iy, dpos)

    def err(t, axis):
        va = t["vabs"]
        if axis == "x":  # the centre values' own rounding, through the differences gix takes
            dv = 16 * EPS * ((va[0] + va[1]) * (1 - t["fy"]) + (va[2] + va[3]) * t["fy"])
            gi, gm, a = t["gix"], t["gmx"], t["aix"]
        else:
            dv = 16 * EPS * ((va[0] + va[2]) * (1 - t["fx"]) + (va[1] + va[3]) * t["fx"])
            gi, gm, a = t["giy"], t["gmy"], t["aiy"]
        return (gm * (dv + 5 * EPS * a + dpos[:, None] * t["mix"]) + 3 * EPS * (gi * gm).abs())[:, 0]

    Gx = [(t["gix"] * t["gmx"])[:, 0] for t in xs]
    Gy = [(t["giy"] * t["gmy"])[:, 0] for t in ys]
    ex = torch.stack([err(t, "x") for t in xs]).amax(0)
    ey = torch.stack([err(t, "y") for t in ys]).amax(0)
    cx = [gg * G for gg in (gmin, gmax) for G in Gx]
    cy = [gg * G for gg in (gmin, gmax) for G in Gy]
    inter = lambda a, b: torch.stack([a, b], 2).view(B, 2 * Kp, H, W)
    cands = [inter(a, b) for a, b in zip(cx, cy)]
    return cands, inter(gabs * ex, gabs * ey), (lo, hi), dict(Gx=Gx, Gy=Gy, ex=ex, ey=ey)


def kc_inputs(r, g):
    B, H, W, Kp = r["B"], r["H"], r["W"], r["Kp"]
    dmin = torch.full((B,), synthetic.DEPTH_MIN) + torch.arange(B) * 3.0
    dmax = torch.full((B,), synthetic.DEPTH_MAX) - torch.arange(B) * 4.0
    if r["mode"] == ops.MODE_RANDOM:
        seed = torch.rand(B, 48, H, W, generator=g)
    else:  # a smooth depth map, partly outside [dmin, dmax]: the perturbed samples are clamped there
        seed = 680.0 + 150.0 * smooth(g, B, 1, H=H, W=W)
    return seed, make_offsets(r, g, Kp, "propagation"), dmin, dmax


def check_kc(tag, rn, r, twice=False):
    g = torch.Generator().manual_seed(r["H"] + r["Ns"] + r["Kp"])
    B, H, W, Ns, Kp, D = r["B"], r["H"], r["W"], r["Ns"], r["Kp"], r["D"]
    seed, off, dmin, dmax = kc_inputs(r, g)
    gout = smooth(g, B, D, H=H, W=W)
    args = (r["mode"], Ns, Kp, r["dil"], r["scale"])
    got = rn.kc(seed, off, dmin, dmax, gout, *args)
    up = [t.to(rn.dev, F64) for t in (seed, off, dmin, dmax)]
    cands, bnd, (lo, hi), G = kc_bwd_reference(*up, gout.to(rn.dev, F64), *args)
    record("init_propagate_backward d_offsets", hull_check(f"{tag} init_propagate d_offsets", got, cands, bnd, ("b", "k2", "y", "x")))
    if twice:
        assert torch.equal(rn.kc(seed, off, dmin, dmax, gout, *args), got), f"{tag}: d_offsets differ between two runs"
    # rank probe: gout[b, r] = r + 1, so each propagated hypothesis's d_offset is (slot + 1) gix gmx
    probe = (torch.arange(D, dtype=torch.float32) + 1).view(1, D, 1, 1).expand(B, D, H, W)
    d = rn.kc(seed, off, dmin, dmax, probe, *args).to(rn.dev, F64).view(B, Kp, 2, H, W)
    ok_x = (G["Gx"][0] == G["Gx"][2]) & (G["Gx"][1].abs() > 1e3 * G["ex"])
    ok_y = (G["Gy"][0] == G["Gy"][2]) & (G["Gy"][1].abs() > 1e3 * G["ey"])
    slot_x = (d[:, :, 0] / G["Gx"][1]).round() - 1
    slot_y = (d[:, :, 1] / G["Gy"][1]).round() - 1
    ok = ok_x | ok_y  # [B,Kp,H,W]: hypotheses whose slot can be read
    slot = torch.where(ok_x, slot_x, slot_y)
    assert int(ok.sum()) > 0.2 * ok.numel(), f"{tag}: only {int(ok.sum())} of {ok.numel()} hypotheses probed"
    assert bool(((slot >= lo) & (slot <= hi))[ok].all()), f"{tag}: a slot outside its admissible window"
    # within a pixel the slots read are distinct (the unread ones get distinct negative stand-ins)
    stand_in = -1.0 - torch.arange(Kp, dtype=F64, device=slot.device).view(1, Kp, 1, 1)
    srt = torch.where(ok, slot, stand_in).sort(1)[0]
    assert bool((srt[:, 1:] > srt[:, :-1]).all()), f"{tag}: two propagated hypotheses routed to one slot"
    pixels = int(ok.any(1).sum())
    print(f"[rank probe] {tag}: {pixels} pixels probed ({int(ok.sum())} hypotheses), {int((hi > lo)[ok].sum())} ambiguous windows met")
    return lo, hi


# ------------------------------------------------------------------------------------------------
# K-B backward
# ------------------------------------------------------------------------------------------------


def kb_bwd_reference(score0, depth, xnorm, off, fw, prob, gd, gp_in, dil, scale, inverse, K):
    """K-B backward in float64, all inputs the kernel's fp32 values upcast (prob: fp32 of the float64 forward; xnorm: the
    normalised inverse depth map the forward gathers).  gd [B,H,W] or None, gp_in [B,D,H,W] or None.

    Regression: gp_d = gp_in + gd h_d (inverse: gp_in + gd didx d, didx = -h^2 (1/h_last - 1/h_0) / (D - 1) with h the
    regressed depth); d_hyp = gd p_d (inverse: only the two end hypotheses).  Softmax: ds_d = p_d (gp_d - <gp, p>).
    Aggregation per hypothesis d: w_k = sigma(4 - 2 clamp(|X_k - x_c| / scale, 0, 4)) fw_k, S_k the gathered score,
    s = sum w S / sum w; dsn_k = ds w_k / sum w goes to the score taps (d_score0, atomics), dsn_k gix gmx to d_offsets,
    ds sigma (S_k - s) / sum w to d_fw.
    Bounds.  gp: 2 eps (|gp_in| + |gd h|) (inverse: the relative error of didx -- q = 1/h_0 + idx (1/h_last - 1/h_0)/(D-1)
    within eps (2 |1/h_0| + 4 idx/(D-1) (|1/h_0| + |1/h_last|) + D idx/(D-1) |1/h_last - 1/h_0|), h = 1/q two eps more,
    didx twice that, plus the cancellation 3 eps (|1/h_0| + |1/h_last|) / |1/h_last - 1/h_0|).  <gp, p>: sum of the
    errors plus (D + 1) eps sum |gp| p.  ds: p (dgp + ddot + 2 eps (|gp| + |dot|)) -- the cancellation in gp - <gp, p>
    is bounded through the absolute terms, not the result.  The weights, s and the gathered scores repeat the forward's
    arithmetic (kb_reference's derivation, with the x map read rather than computed).  dsn: |ds| (dw + w (dden / den +
    3 eps)) / den + dds w / den.  d_score0 at a texel: sum of dsn errors times the tap weight and of |dsn| 2 dpos (the tap
    weight's move, dpos per coordinate that is not clamped), maxed over 3x3 texels, plus (m + 4) eps sum |dsn| w_t with m from the count scatter.  d_offsets: per
    hypothesis the dsn error times |gix| gmx, |dsn| gmx (5 eps a + dpos mix), then (D + 4) eps of the absolute sum; the
    hull over the one-sided positions as for K-A'.  d_fw: each term's error from dds, dsigma, dS, ds, dden, then
    (D + 1) eps of the absolute sum.  -> dict of (want or candidates, bound) per output."""
    B, D, H, W = depth.shape
    dev = depth.device
    table = pm_oracle.neighbour_table("evaluation", K, dil)
    px, py = pixel_positions(table, off, H, W)
    dpos = border_dpos(px, py, H, W)  # [B,K,H,W]
    ix, iy = texel_coords(px, py, H, W)
    zero = torch.zeros_like(depth)
    gdv = torch.zeros(B, H, W, dtype=F64, device=dev) if gd is None else gd
    gpi = zero if gp_in is None else gp_in
    p, h = prob, depth
    gdx = gdv.unsqueeze(1)
    if not inverse:
        gp = gpi + gdx * h
        dgp = 2 * EPS * (gpi.abs() + (gdx * h).abs())
        dhyp = gdx * p
        bhyp = EPS * dhyp.abs()
    else:
        dw_ = torch.arange(D, dtype=F64, device=dev).view(1, D, 1, 1)
        idx = (dw_ * p).sum(1)
        lo_, hi_ = 1.0 / h[:, 0], 1.0 / h[:, -1]
        t = idx / (D - 1)
        q = lo_ + t * (hi_ - lo_)
        do = 1.0 / q
        rq = EPS * (2 * lo_.abs() + 4 * t * (lo_.abs() + hi_.abs()) + D * t * (hi_ - lo_).abs()) / q.abs()
        rdo = rq + 2 * EPS
        didx = -do ** 2 * (hi_ - lo_) / (D - 1)
        rdidx = 2 * rdo + 3 * EPS * (lo_.abs() + hi_.abs()) / (hi_ - lo_).abs() + 4 * EPS
        gterm = gdx * didx.unsqueeze(1) * dw_
        gp = gpi + gterm
        dgp = gterm.abs() * (rdidx.unsqueeze(1) + 3 * EPS) + EPS * (gpi.abs() + gp.abs())
        dhyp = zero.clone()
        bhyp = zero.clone()
        for dd, frac in ((0, 1 - t), (D - 1, t)):
            c = gdv * do ** 2 / h[:, dd] ** 2
            dhyp[:, dd] += c * frac
            bhyp[:, dd] += c.abs() * ((2 * rdo + 8 * EPS) * frac.abs() + (D + 2) * EPS * t)
    dot = (gp * p).sum(1, keepdim=True)
    ddot = (dgp * p).sum(1, keepdim=True) + (D + 1) * EPS * (gp.abs() * p).sum(1, keepdim=True)
    ds = p * (gp - dot)
    dds = p * (dgp + ddot + 2 * EPS * (gp.abs() + dot.abs()))

    dsc, asc, esc = [torch.zeros(B, D, H * W, dtype=F64, device=dev) for _ in range(3)]
    cnt = torch.zeros(B, 1, H * W, dtype=F64, device=dev)
    cx, cy = [torch.zeros(B, K, H, W, dtype=F64, device=dev) for _ in range(3)], [torch.zeros(B, K, H, W, dtype=F64, device=dev) for _ in range(3)]
    ex, ey, ax, ay = [torch.zeros(3, B, K, H, W, dtype=F64, device=dev) for _ in range(4)]
    dfw, efw, afw = [torch.zeros(B, K, H, W, dtype=F64, device=dev) for _ in range(3)]
    step = max(1, CHUNK_ELEMS // (4 * B * K * H * W))
    for d0 in range(0, D, step):
        sl = slice(d0, d0 + step)
        S, Sabs, Scoord = border_sample_bound(score0[:, sl], px, py, H, W)  # [B,d,K,H,W]
        eS = 7 * EPS * Sabs + Scoord
        X, Xabs, Xcoord = border_sample_bound(xnorm[:, sl], px, py, H, W)
        eX = 7 * EPS * Xabs + Xcoord
        xc = xnorm[:, sl].unsqueeze(2)
        a = (X - xc).abs() / scale
        da = (eX + 2 * EPS * (X.abs() + xc.abs())) / scale + EPS * a
        sig = torch.sigmoid(4.0 - 2.0 * a.clamp(0, 4))
        dsig = 2 * (sig * (1 - sig) + 0.2 * da) * da + 6 * EPS * sig
        f = fw.unsqueeze(1)
        w = sig * f
        dw = f * dsig + EPS * w
        den = w.sum(2, keepdim=True)
        dden = dw.sum(2, keepdim=True) + K * EPS * den
        s = (S * w).sum(2, keepdim=True) / den
        dnum = (S.abs() * dw + w * eS).sum(2, keepdim=True) + (K + 1) * EPS * (w * S.abs()).sum(2, keepdim=True)
        es = (dnum + s.abs() * dden) / den + EPS * s.abs()
        dsd, ddsd = ds[:, sl].unsqueeze(2), dds[:, sl].unsqueeze(2)
        dsn = dsd * w / den
        edsn = dsd.abs() * (dw + w * (dden / den + 3 * EPS)) / den + ddsd * w / den
        # d_fw
        tf = dsd * sig * (S - s) / den
        dfw += tf.sum(1)
        afw += tf.abs().sum(1)
        efw += (ddsd * sig * (S - s).abs() / den + dsd.abs() * (dsig * (S - s).abs() / den + sig * (eS + es + EPS * (S.abs() + s.abs())) / den
                                                                 + sig * (S - s).abs() * dden / den ** 2) + 3 * EPS * tf.abs()).sum(1)
        del X, Xabs, Xcoord, eX, a, da, Sabs, Scoord
        # d_score0: the scatter of dsn through the tap weights of the float64 position
        f_s = score0[:, sl]
        xs, ys = kink_positions(f_s, ix, iy, dpos)
        t0 = xs[1]
        dn = f_s.shape[1]
        # the tap weights move with the position only where it is not clamped: by dpos per coordinate
        move = (dpos * (((ix > -dpos) & (ix < W - 1 + dpos)).to(F64) + ((iy > -dpos) & (iy < H - 1 + dpos)).to(F64))).unsqueeze(1)
        for tap, wt in zip(t0["taps"], t0["wts"]):
            ie = tap.reshape(B, 1, -1).expand(B, dn, -1)
            dsc[:, sl].scatter_add_(2, ie, (dsn * wt).reshape(B, dn, -1))
            asc[:, sl].scatter_add_(2, ie, (dsn.abs() * wt).reshape(B, dn, -1))
            esc[:, sl].scatter_add_(2, ie, (edsn * wt + dsn.abs() * move).reshape(B, dn, -1))
            if d0 == 0:
                cnt.scatter_add_(2, tap.reshape(B, 1, -1), torch.ones_like(tap, dtype=F64).reshape(B, 1, -1))
        # d_offsets
        for i, (tx, ty) in enumerate(zip(xs, ys)):
            cx[i] += (dsn * tx["gix"] * tx["gmx"]).sum(1)
            cy[i] += (dsn * ty["giy"] * ty["gmy"]).sum(1)
            ex[i] += (tx["gmx"] * (edsn * tx["gix"].abs() + dsn.abs() * (5 * EPS * tx["aix"] + dpos.unsqueeze(1) * tx["mix"]))).sum(1)
            ey[i] += (ty["gmy"] * (edsn * ty["giy"].abs() + dsn.abs() * (5 * EPS * ty["aiy"] + dpos.unsqueeze(1) * ty["mix"]))).sum(1)
            ax[i] += (dsn * tx["gix"] * tx["gmx"]).abs().sum(1)
            ay[i] += (dsn * ty["giy"] * ty["gmy"]).abs().sum(1)
        del xs, ys, t0, S, w, dw, sig, dsig, dsn, edsn, tf
    m = pool_texels(cnt.view(B, 1, H, W))  # every hypothesis plane receives the same count
    b_sc = pool_texels(esc.view(B, D, H, W)) + (m + 4) * EPS * asc.view(B, D, H, W)
    bx = (ex + (D + 4) * EPS * ax).amax(0)
    by = (ey + (D + 4) * EPS * ay).amax(0)
    inter = lambda a, b: torch.stack([a, b], 2).view(B, 2 * K, H, W)
    return dict(d_score0=(dsc.view(B, D, H, W), b_sc), d_hyp=(dhyp, bhyp),
                d_offsets=([inter(a, b) for a, b in zip(cx, cy)], inter(bx, by)),
                d_fw=(dfw, efw + (D + 1) * EPS * afw))


def kb_bwd_inputs(r, g):
    """kb_inputs' smooth scores, hypotheses (descending for the inverse regression), offsets and feature weights; the fp32
    x map of the hypotheses; prob = fp32 of the float64 forward (kb_reference); smooth incoming gradients."""
    B, D, H, W, K = r["B"], r["D"], r["H"], r["W"], r["K"]
    score0, depth, off, fw, dmin, dmax = kb_inputs(r, g)
    if r["offs"] != "borders":
        off = make_offsets(r, g, K, "evaluation")
    xn, _ = xnorm_bound(depth.double(), torch.zeros_like(depth.double()), dmin.double(), dmax.double())
    prob64 = kb_reference(score0.double(), depth.double(), off.double(), fw.double(), dmin.double(), dmax.double(), r["dil"],
                          r["scale"], bool(r["inverse"]), K)[0]
    gd = smooth(g, B, H=H, W=W) if r["grads"] in ("depth", "both") else None
    gp = smooth(g, B, D, H=H, W=W) if r["grads"] in ("prob", "both") else None
    return score0, depth, xn.float(), off, fw, dmin, dmax, prob64.float(), gd, gp


def check_kb(tag, rn, r, twice=False):
    g = torch.Generator().manual_seed(r["H"] + r["D"] + r["K"])
    score0, depth, xn, off, fw, dmin, dmax, prob, gd, gp = kb_bwd_inputs(r, g)
    got = rn.kb(score0, depth, xn, off, fw, dmin, dmax, prob, gd, gp, r["dil"], r["scale"], r["inverse"])
    up = lambda t: None if t is None else t.to(rn.dev, F64)
    ref = kb_bwd_reference(up(score0), up(depth), up(xn), up(off), up(fw), up(prob), up(gd), up(gp), r["dil"], r["scale"],
                           bool(r["inverse"]), r["K"])
    dims4 = ("b", "d", "y", "x")
    for name, out, dims in (("d_score0", got[0], dims4), ("d_hyp", got[1], dims4), ("d_fw", got[3], ("b", "k", "y", "x"))):
        want, bnd = ref[name]
        record(f"adaptive_eval_backward {name}", assert_within(f"{tag} adaptive_eval {name}", out, want, bnd, dims))
    cands, bnd = ref["d_offsets"]
    record("adaptive_eval_backward d_offsets", hull_check(f"{tag} adaptive_eval d_offsets", got[2], cands, bnd, ("b", "k2", "y", "x")))
    if twice:
        again = rn.kb(score0, depth, xn, off, fw, dmin, dmax, prob, gd, gp, r["dil"], r["scale"], r["inverse"])
        for i in (1, 2, 3):
            assert torch.equal(again[i], got[i]), f"{tag}: output {i} differs between two runs"
        assert_within(f"{tag} adaptive_eval d_score0 (second run)", again[0], *ref["d_score0"], dims4)


# ------------------------------------------------------------------------------------------------
# edge rows reach their structure
# ------------------------------------------------------------------------------------------------


def test_edge_rows_reach_their_structure():
    # K-A runs: float64 cells of every hypothesis at the GPU row's size
    r = row("edge/ka-runs")
    ref, srcs, rt, depth, vw, gout = ka_bwd_inputs(r, 1)
    u, v, _ = project_bound(rt[0].double(), depth.double(), r["H"], r["W"], r["H"], r["W"])
    inside = (u >= -1) & (u < r["W"]) & (v >= -1) & (v < r["H"])
    key = torch.where(inside, u.floor() * 100000 + v.floor(), -1.0)
    n_in = float(inside[:, 0].sum())
    assert n_in > 0.5 * inside[:, 0].numel()
    run = (key[:, 1:12] == key[:, :1]).all(1) & inside[:, 0]
    assert float(run.sum()) > 0.9 * n_in  # 12 consecutive hypotheses in one cell
    assert not bool(inside[:, 12].any()) and not bool(inside[:, 16].any())  # behind the camera, beyond the map
    assert float(((key[:, 13] == key[:, 11]) & run).sum()) > 0.9 * n_in  # the run goes on across the break
    aba = (key[:, 20] == key[:, 22]) & (key[:, 21] != key[:, 20]) & inside[:, 21]
    assert float(aba.sum()) > 0.5 * n_in
    # tiny sources
    assert {(1, 1), (2, 3)} <= set(row("edge/ka-tiny-sources")["sizes"])
    # texel-aligned gathers: on integer texel positions within dpos, and on both clamp edges
    r = row("edge/texels")
    g = torch.Generator().manual_seed(0)
    table = pm_oracle.neighbour_table("evaluation", r["K"], r["dil"])
    off = offsets_on_texels(g, r["B"], r["K"], r["H"], r["W"], table, 3.0).double()
    px, py = pixel_positions(table, off, r["H"], r["W"])
    ix, _ = texel_coords(px, py, r["H"], r["W"])
    dpos = border_dpos(px, py, r["H"], r["W"])
    assert float(((ix - ix.round()).abs() <= dpos).double().mean()) > 0.99
    assert bool((ix.round() == 0).any()) and bool((ix.round() == r["W"] - 1).any())
    # K-C exact tie: neighbours 0 and 1 compute the same position, above the map
    r = row("edge/kc-tie")
    seed, off, dmin, dmax = kc_inputs(r, torch.Generator().manual_seed(2))
    table = pm_oracle.neighbour_table("propagation", r["Kp"], r["dil"])
    assert table[0] == (-r["dil"], -r["dil"]) and table[1] == (-r["dil"], 0)
    px, py = pixel_positions(table, off.double(), r["H"], r["W"])
    assert torch.equal(px[:, 0], px[:, 1]) and bool((py[:, :2] < 0).all())
    vals, _, centre, _, _, _ = kc_values(*[t.double() for t in (seed, off, dmin, dmax)], r["mode"], r["Ns"], r["Kp"], r["dil"], r["scale"],
                                      r["H"], r["W"])
    assert torch.equal(vals[:, r["Ns"]], vals[:, r["Ns"] + 1])
    # the seed leaves [dmin, dmax]: some centre samples are clamped
    inv = 1.0 / centre
    assert bool(((inv - 1.0 / dmax.double().view(-1, 1, 1, 1)).abs() < 1e-12).any() | ((inv - 1.0 / dmin.double().view(-1, 1, 1, 1)).abs() < 1e-12).any())


# ------------------------------------------------------------------------------------------------
# the emulator: every reference, bound, edge row and the rank probe at reduced sizes (CPU)
# ------------------------------------------------------------------------------------------------

EMU_KA = sorted({r["name"] for r in all_rows() if r["name"].startswith(("dtu/", "mixed/", "dtu-hs/", "synthetic/s", "edge/ka"))})


@pytest.mark.parametrize("name", EMU_KA)
def test_emulated_warp_corr_backward(emu, name):
    check_ka(f"emu {name}", emu, mini(row(name)))


@pytest.mark.parametrize("name", agg_rows())
def test_emulated_aggregate_views_backward(emu, name):
    check_agg(f"emu {name}", emu, mini(row(name)))


@pytest.mark.parametrize("name", sorted(set(oc_rows()) & {"dtu/s3/it1", "dtu/s2/it1", "dtu/s1/it1", "synthetic/K17", "edge/texels"}))
def test_emulated_offset_corr_backward(emu, name):
    check_oc(f"emu {name}", emu, mini(row(name)))


@pytest.mark.parametrize("name", kc_rows())
def test_emulated_init_propagate_backward(emu, name):
    check_kc(f"emu {name}", emu, mini(row(name)))


@pytest.mark.parametrize("name", ["dtu/s3/it1", "dtu/s3/it2", "dtu/s2/it1", "dtu/s1/it1", "synthetic/K17", "synthetic/grad-prob",
                                  "synthetic/grad-both", "synthetic/grad-both-inverse", "edge/texels-s3"])
def test_emulated_adaptive_eval_backward(emu, name):
    check_kb(f"emu {name}", emu, mini(row(name)))


# ------------------------------------------------------------------------------------------------
# the GPU at training sizes
# ------------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", ka_rows())
def test_warp_corr_backward_at_scale(name):
    check_ka(name, Runner(), row(name), twice=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", agg_rows())
def test_aggregate_views_backward_at_scale(name):
    check_agg(name, Runner(), row(name), twice=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", oc_rows())
def test_offset_corr_backward_at_scale(name):
    check_oc(name, Runner(), row(name), twice=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", kc_rows())
def test_init_propagate_backward_at_scale(name):
    check_kc(name, Runner(), row(name), twice=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", kb_rows())
def test_adaptive_eval_backward_at_scale(name):
    check_kb(name, Runner(), row(name), twice=True)


# ------------------------------------------------------------------------------------------------
# sensitivity (CPU): a 13 x 23 map, not a multiple of any block
# ------------------------------------------------------------------------------------------------

SMALL = dict(B=1, H=13, W=23)


def test_sensitivity_warp_corr_backward():
    r = dict(SMALL, V=2, C=32, G=8, D=5, vw=True, sizes=None, ka="plain")
    ref, srcs, rt, depth, vw, gout = [None if t is None else (t.double() if isinstance(t, torch.Tensor) else [s.double() for s in t])
                                      for t in ka_bwd_inputs(r, 3)]
    d_ref, b_ref, d_src, b_src = ka_bwd_reference(ref, srcs, rt, depth, vw, gout, 8)
    plant_rejected("d_ref", d_ref.float(), d_ref, b_ref, ("b", "c", "y", "x"), (0, None, 12, 22))
    # the source texel the last pixel's hypotheses reach most
    c = b_src[1][0, -1]
    at = divmod(int((d_src[1][0, -1].abs() / c.clamp_min(1e-300) * (c > 0)).argmax()), 23)
    plant_rejected("d_src", d_src[1].float(), d_src[1], b_src[1], ("b", "c", "y", "x"), (0, None) + at)


def test_sensitivity_aggregate_views_backward():
    r = dict(SMALL, V=3, G=8, D=5)
    sims, vw, gout = [t.double() for t in agg_inputs(r, 4)]
    ws, bs, wv, bv = agg_bwd_reference(sims, vw, gout)
    plant_rejected("d_sims", ws.float(), ws, bs, ("view", "b", "g", "d", "y", "x"), (2, 0, 7, None, 12, 22))
    plant_rejected("d_vw", wv.float(), wv, bv, ("b", "view", "y", "x"), (0, None, 12, 22))


def test_sensitivity_offset_corr_backward():
    g = torch.Generator().manual_seed(5)
    B, C, G, K, H, W = 1, 32, 8, 9, 13, 23
    ref, gout = smooth(g, B, C, H=H, W=W).double(), smooth(g, B, G, K, H=H, W=W).double()
    off = offsets_reaching_borders(g, B, K, H, W, reach=3.0).double()
    cands, bnd = oc_bwd_reference(ref, off, gout, G, K, 4)
    plant_rejected("offset_corr d_offsets", cands[1].float(), cands[1], bnd, ("b", "k2", "y", "x"), (0, 0, 12, 22))
    # a clamped gather (neighbour 0 leaves the map upwards on the first column: gmy = 0) given the interior value
    t = border_grad(ref, *texel_coords(*pixel_positions(pm_oracle.neighbour_table("evaluation", K, 4), off, H, W), H, W))
    assert float(t["gmy"][0, 0, 0, 5, 0]) == 0.0
    interior = ((gout / 4).repeat_interleave(4, 1) * ref[:, :, None] * t["giy"] * (H / (H - 1))).sum(1)
    bad = cands[1].clone()
    bad[0, 1, 5, 0] = interior[0, 0, 5, 0]
    assert float(interior[0, 0, 5, 0].abs()) > 10 * float(bnd[0, 1, 5, 0])
    with pytest.raises(AssertionError, match="worst element"):
        hull_check("offset_corr d_offsets (clamped)", bad.float(), cands, bnd, ("b", "k2", "y", "x"))


def kc_small(mode=ops.MODE_PERTURB, offs="tie"):
    r = dict(SMALL, Kp=8, Ns=8, D=16, mode=mode, dil=4, scale=0.0125, offs=offs)
    g = torch.Generator().manual_seed(6)
    seed, off, dmin, dmax = kc_inputs(r, g)
    gout = smooth(g, 1, 16, H=13, W=23)
    return r, [t.double() for t in (seed, off, dmin, dmax, gout)]


def test_sensitivity_init_propagate_backward():
    r, (seed, off, dmin, dmax, gout) = kc_small()
    cands, bnd, (lo, hi), G = kc_bwd_reference(seed, off, dmin, dmax, gout, r["mode"], 8, 8, 4, 0.0125)
    want = cands[1]  # no slot ambiguity and no kink at the planted element
    assert float(lo[0, 3, 12, 22]) == float(hi[0, 3, 12, 22])
    plant_rejected("init_propagate d_offsets", want.float(), want, bnd, ("b", "k2", "y", "x"), (0, 6, 12, 22))
    # the tied pair (neighbours 0 and 1): the stable order gives neighbour 0 the earlier slot; swapping their gradients fails
    assert bool((lo[:, 1] == lo[:, 0] + 1).all() and (hi[:, 1] == hi[:, 0] + 1).all())
    swapped = want.clone()
    swapped[:, 0] = gout.gather(1, lo[:, 1:2])[:, 0] * G["Gx"][1][:, 0]
    swapped[:, 2] = gout.gather(1, lo[:, 0:1])[:, 0] * G["Gx"][1][:, 1]
    with pytest.raises(AssertionError, match="worst element"):
        hull_check("init_propagate d_offsets (tied slots swapped)", swapped.float(), cands, bnd, ("b", "k2", "y", "x"))
    # the tied pair is clamped in y: d_off_y is 0 there, the interior value is rejected
    clamped = want.clone()
    centre = kc_values(seed, off, dmin, dmax, r["mode"], 8, 8, 4, 0.0125, 13, 23)[2]
    t = border_grad(centre, *texel_coords(*pixel_positions(pm_oracle.neighbour_table("propagation", 8, 4), off, 13, 23), 13, 23))
    interior = gout.gather(1, lo[:, 0:1])[:, 0] * t["giy"][:, 0, 0] * (13 / 12)
    clamped[:, 1] = interior
    assert float(interior.abs().max()) > 10 * float(bnd[:, 1].max())
    with pytest.raises(AssertionError, match="worst element"):
        hull_check("init_propagate d_offsets (clamped)", clamped.float(), cands, bnd, ("b", "k2", "y", "x"))


@pytest.mark.parametrize("grads,inverse", [("depth", False), ("prob", False), ("both", True)])
def test_sensitivity_adaptive_eval_backward(grads, inverse):
    r = dict(SMALL, D=8, K=9, dil=4, scale=0.0125, inverse=inverse, grads=grads, offs="borders")
    g = torch.Generator().manual_seed(7)
    ins = [None if t is None else t.double() for t in kb_bwd_inputs(r, g)]
    score0, depth, xn, off, fw, dmin, dmax, prob, gd, gp = ins
    ref = kb_bwd_reference(score0, depth, xn, off, fw, prob, gd, gp, 4, 0.0125, inverse, 9)
    want, bnd = ref["d_score0"]
    plant_rejected("d_score0", want.float(), want, bnd, ("b", "d", "y", "x"), (0, None, 12, 22))
    want, bnd = ref["d_fw"]
    plant_rejected("d_fw", want.float(), want, bnd, ("b", "k", "y", "x"), (0, None, 12, 22))
    cands, bnd = ref["d_offsets"]
    plant_rejected("d_offsets", cands[1].float(), cands[1], bnd, ("b", "k2", "y", "x"), (0, 0, 12, 22))
    want, bnd = ref["d_hyp"]
    at = (0, 0 if inverse else 7, 12, 22)
    if grads != "prob":
        plant_rejected("d_hyp", want.float(), want, bnd, ("b", "d", "y", "x"), at)
    else:
        assert float(want.abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------
# launcher checks (CPU): every rejection happens before anything is written or launched
# ------------------------------------------------------------------------------------------------

_FAKE = 1 << 20  # pointers that are never dereferenced: the checks run first
_BIG = (1 << 15, 1 << 14)  # H * W = 2^29: one past the 29-bit texel index of the tap keys
# entry point, arguments after the pointers, number of pointers, expected message
LAUNCHER_CHECKS = {
    "warp_corr_backward source too large": ("pmb200_warp_corr_backward", 8, [1, 1, 32, 8, 8, 8, *_BIG, 1],
                                            "warp_corr_backward: source map too large"),
    "init_propagate_backward random Ns": ("pmb200_init_propagate_backward", 6, [0, 1, 8, 8, 8, 8, 4, 0.0125],
                                          "init_propagate_backward: random init has 48 samples"),
    "init_propagate_backward passthrough Ns": ("pmb200_init_propagate_backward", 6, [2, 1, 8, 8, 4, 8, 4, 0.0125],
                                               "init_propagate_backward: passthrough needs Ns == 1"),
    "init_propagate_backward too many hypotheses": ("pmb200_init_propagate_backward", 6, [1, 1, 8, 8, 250, 8, 4, 0.0125],
                                                    "init_propagate_backward: too many hypotheses"),
    "init_propagate_backward map too large": ("pmb200_init_propagate_backward", 6, [1, 1, *_BIG, 8, 8, 4, 0.0125],
                                              "init_propagate_backward: map too large"),
    "adaptive_eval_backward inverse D=1": ("pmb200_adaptive_eval_backward", 14, [1, 1, 8, 8, 9, 2, 0.025, 1],
                                           "adaptive_eval_backward: inverse regression needs D >= 2"),
    "adaptive_eval_backward map too large": ("pmb200_adaptive_eval_backward", 14, [1, 1, *_BIG, 9, 2, 0.025, 0],
                                             "adaptive_eval_backward: map too large"),
    "init_propagate map too large": ("pmb200_init_propagate", None, [1, 1, *_BIG, 8, 8, 4, 0.0125],
                                     "init_propagate: map too large"),
    "adaptive_eval map too large": ("pmb200_adaptive_eval", None, [1, 1, *_BIG, 9, 2, 0.025, 0], "adaptive_eval: map too large"),
}
# the forward launchers' pointer arguments, with their flags (offsets_channels_last) in place
_FORWARD_HEAD = {"pmb200_init_propagate": [_FAKE, _FAKE, 0, _FAKE, _FAKE, _FAKE, _FAKE, 1],
                 "pmb200_adaptive_eval": [_FAKE] * 5 + [0] + [_FAKE] * 5}


def _have_library():
    try:
        _native.lib()
        return True
    except _native.NativeLibraryMissing:
        return False


@pytest.mark.skipif(not _have_library(), reason="libpmb200.so is not built")
@pytest.mark.parametrize("case", list(LAUNCHER_CHECKS))
def test_launcher_rejects_before_anything_runs(case):
    """Run in a process that sees no GPU, so that a launcher that does not check would fail on its zero fill or its launch
    with another message instead of reaching a device."""
    fn, nptr, tail, msg = LAUNCHER_CHECKS[case]
    head = [_FAKE] * nptr if nptr is not None else _FORWARD_HEAD[fn]
    script = ("import ctypes, sys\n"
              f"sys.path.insert(0, {REPO!r})\n"
              "from patchmatchnet_b200 import _native\n"
              "lib = _native.lib()\n"
              f"args = {head!r} + {tail!r}\n"
              f"fn = getattr(lib, {fn!r})\n"
              "args = [ctypes.c_float(a) if t is ctypes.c_float else a for a, t in zip(args, fn.argtypes)]\n"
              "rc = fn(*args, None)\n"
              "print(rc, lib.pmb200_last_error().decode())\n")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, env=env, timeout=120)
    assert res.returncode == 0, res.stderr
    rc, text = res.stdout.strip().split(" ", 1)
    assert int(rc) == -1 and msg in text, res.stdout
