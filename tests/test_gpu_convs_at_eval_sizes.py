"""The convolution kernels (K-S, the mma.sync kernel conv2d_nhwc, the wgmma forms K-D5 / K-D5h, K-R) at the view counts and
image sizes the evaluation configurations run, element by element against float64 F.conv2d.

Rows.  FeatureNet runs the views of one request stacked (PatchmatchNet.stack_views): N = V + 1 images of Tanks and Temples
(8 x 1080x1920), ETH3D (8 x 1792x2688), DTU (6 x 1200x1600) and a 10-source pair.txt (11 x 1200x1600), plus one ETH3D
portrait view alone (1 x 2688x1792, the per-view path of views of different sizes).  Every FeatureNet layer runs at the map
size and N it sees there, in the form ops.conv_form picks (asserted per row), in the fp32-accurate mode and, for the layers
ops.conv_prefers_native keeps native there, in the TF32 mode (conv2d_nhwc at precision 1).  The offset convs of each stage
run at the stage maps of 1920x1080 and 2688x1792 with their dilations, Refinement at the image sizes and at one size the
sizing rule of reconstruct makes (an image scaled to image_max_dim, then each side rounded to a multiple of 8) whose width is
not a multiple of 16.  One row runs the whole FeatureNet fast path against the module in float64, link by link (see
feature_net_links: a bound carried through all eleven layers is vacuous).

Bounds, per element.  eps = 2^-24.  S = |W| * |x| + |b| (the conv of the absolute values), K = Cin KS^2 products.
  * 3xTF32 (conv2d_nhwc precision 3, K-D5, K-D5h): a x w is computed as a_hi w_hi + a_hi w_lo + a_lo' w_hi, a_hi = a with
    its 13 low mantissa bits cleared (|a_lo| < 2^-10 |a|), a_lo' = a_lo as the tensor core reads it (truncated to TF32:
    |a_lo - a_lo'| < 2^-10 |a_lo| <= 2^-20 |a|), w_hi = rna(w), w_lo = rna(w - w_hi) (|w - w_hi - w_lo| <= 2^-22 |w|).  The
    terms left out are a_hi (w - w_hi - w_lo) (4 eps |a w|), a_lo w_lo (8 eps) and (a_lo - a_lo') w_hi (16 eps): 28 eps, and
    one more for the products of the error terms.  The TF32 x TF32 products are exact in fp32; the accumulator takes 3K + 1
    additions (the bias included), each, if the tensor core truncates, within 2 eps of the partial sum, which is at most S.
        |got - want| <= c3(K) eps S,   c3(K) = 2 (3K + 1) + 29.
  * TF32 (precision 1): a truncated (2^-10 = 16384 eps), w rounded (2^-11 = 8192 eps), their product (8 eps), K + 1
    additions: c1(K) = 16384 + 8192 + 8 + 2 (K + 1).
  * Exact fp32 FFMA (K-S, K-R): K products and the bias, K + 3 (the stem's own 30 and 75 of the at-scale file).
  * Chained rows (the top-down path, Refinement) carry the bound through each layer: |W| * bound_in, plus the layer's own term taken over |x| + bound_in.
    ReLU and the nearest / bilinear x2 upsampling are 1-Lipschitz; the bilinear epilogue of add_up2x adds 8 eps of the
    upsampled |u| (the 6 roundings of the at-scale upsample2x_add bound and the final addition), BatchNorm folded into fp32
    weights one more eps of S per layer.
The element bound grows like K eps.  A result computed with a dropped split term (plain TF32 operands, or a_lo w_hi left
out) is off by about 2^-11 |a w| per product with a random sign: its error grows like sqrt(K) and stays under the element
bound.  Hence the second check.

Precision statistic, 3xTF32 single-layer rows.  r = RMS over the tensor of (got - want) / S.  Treating the 3K + 1
accumulator roundings and the K split residuals as uncorrelated, each rounding of second moment at most (2 eps S)^2 and the
residuals of second moment at most (28 eps |a_k w_k|)^2 with sqrt(sum_k (a_k w_k)^2) <= S:
        r <= tau(K) = (2 sqrt(3K + 1) + 28) eps.
It is shown to bite below: a float64 emulation with a_lo w_hi dropped fails it at K = 72, 576 and 1600, and on the GPU the
precision-1 output of conv2d_nhwc on the same inputs fails the fp32-accurate checks.

The float64 references run on the device, per image and per band of output rows with its input halo, so that no
intermediate exceeds CHUNK_ELEMS elements."""
import contextlib
import ctypes
import math
import time

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from patchmatchnet_b200 import _native, data_io, ops
from patchmatchnet_b200 import net as pm_net
from patchmatchnet_b200.net import FeatureNet, PackedConv
from tests.test_conv import LAYERS as CONV_TEST_LAYERS
from tests.test_emulated_conv import _random_refinement
from tests.test_gpu_conv5h_schedule import plan_of as tc5h_plan
from tests.test_gpu_conv5h_schedule import units_of
from tests.test_gpu_kernels_at_scale import CHUNK_ELEMS, DEV, EPS, F64, assert_within, plant_rejected, stem_reference

H100_SMS = 132

# (name, N = views per launch, image height, image width)
CONFIGS = (("tnt", 8, 1080, 1920), ("eth3d", 8, 1792, 2688), ("dtu", 6, 1200, 1600), ("pair10", 11, 1200, 1600),
           ("eth3d-portrait", 1, 2688, 1792))

# (name, Cin, Cout, KS, stride, pad, halvings of the image size at its input, ReLU, bias).  conv3 / conv4, conv6 / conv7 and
# conv9 / conv10 are one shape at one size each.
FEATURE_LAYERS = (("conv0", 3, 8, 3, 1, 1, 0, True, True), ("conv1", 8, 8, 3, 1, 1, 0, True, True),
                  ("conv2", 8, 16, 5, 2, 2, 0, True, True), ("conv3/4", 16, 16, 3, 1, 1, 1, True, True),
                  ("conv5", 16, 32, 5, 2, 2, 1, True, True), ("conv6/7", 32, 32, 3, 1, 1, 2, True, True),
                  ("conv8", 32, 64, 5, 2, 2, 2, True, True), ("conv9/10", 64, 64, 3, 1, 1, 3, True, True),
                  ("output1", 64, 64, 1, 1, 0, 3, False, False))
# the form each layer runs in the fp32-accurate mode (conv0 / conv1 run fused in K-S there)
FP32_FORMS = {"conv2": 0, "conv3/4": 2, "conv5": 1, "conv6/7": 2, "conv8": 1, "conv9/10": 2, "output1": 0}
# the layers conv2d_nhwc serves at precision 1 in the TF32 mode (the others go to cuDNN: out of scope)
TF32_NATIVE = {"conv0", "conv1", "conv2", "conv3/4", "output1"}

# offset convs: (stage, Cin, Cout, dilation) -- propa_conv (2 x propagate_neighbors outputs) and eval_conv (18) of stages 3 / 2,
# eval_conv of stage 1 (stage 1 propagates nothing); stage s runs at the image size halved s times
OFFSET_LAYERS = (("s3.propa", 3, 64, 32, 2), ("s3.eval", 3, 64, 18, 2), ("s2.propa", 2, 32, 16, 4), ("s2.eval", 2, 32, 18, 4),
                 ("s1.eval", 1, 16, 18, 6))
OFFSET_IMAGES = (("tnt", 1080, 1920), ("eth3d", 1792, 2688))


def halve(n, times):
    for _ in range(times):
        n = (n - 1) // 2 + 1  # a 5x5 stride-2 conv with pad 2
    return n


def c3(K):
    return 2 * (3 * K + 1) + 29


def c1(K):
    return 16384 + 8192 + 8 + 2 * (K + 1)


def tau(K):
    return (2 * math.sqrt(3 * K + 1) + 28) * EPS


def odd_refinement_size():
    """The image size reconstruct runs for an ETH3D 6048x4032 view at image_max_dim 1000: data_io.scale_to_max_dim, then
    PatchmatchNet's rounding of each side to a multiple of 8 (net._round_dims_to_8)."""
    import numpy as np

    img, _, _ = data_io.scale_to_max_dim(np.zeros((4032, 6048, 3), np.float32), 1000)
    images, _, _, _ = pm_net._round_dims_to_8([torch.zeros(1, 3, img.shape[0], img.shape[1])], torch.ones(1, 1, 3, 3))
    return tuple(images[0].shape[-2:])


REFINE_SIZES = ((1080, 1920), (1792, 2688), (1200, 1600))


@contextlib.contextmanager
def precision(p):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = p == 1
    try:
        assert ops.conv_precision() == p
        yield
    finally:
        torch.backends.cudnn.allow_tf32 = old


def layer_rows():
    rows = []
    for cfg, N, H, W in CONFIGS:
        for name, cin, cout, ks, s, pad, down, relu, bias in FEATURE_LAYERS:
            r = dict(cfg=cfg, layer=name, N=N, H=halve(H, down), W=halve(W, down), cin=cin, cout=cout, ks=ks, stride=s, pad=pad, dil=1,
                     relu=relu, bias=bias, signed=False)
            if name in FP32_FORMS:
                rows.append(dict(r, name=f"{cfg}/{name}/fp32", prec=3, form=FP32_FORMS[name]))
            if name in TF32_NATIVE:
                rows.append(dict(r, name=f"{cfg}/{name}/tf32", prec=1, form=0))
    for cfg, H, W in OFFSET_IMAGES:
        for name, stage, cin, cout, dil in OFFSET_LAYERS:
            r = dict(cfg=cfg, layer=name, N=1, H=halve(H, stage), W=halve(W, stage), cin=cin, cout=cout, ks=3, stride=1, pad=dil,
                     dil=dil, relu=False, bias=True, signed=True)
            rows.append(dict(r, name=f"{cfg}/{name}/fp32", prec=3, form=2))
            if name == "s1.eval":
                rows.append(dict(r, name=f"{cfg}/{name}/tf32", prec=1, form=0))
    return rows


ROWS = {r["name"]: r for r in layer_rows()}


def out_size(r):
    Ho = (r["H"] + 2 * r["pad"] - r["dil"] * (r["ks"] - 1) - 1) // r["stride"] + 1
    Wo = (r["W"] + 2 * r["pad"] - r["dil"] * (r["ks"] - 1) - 1) // r["stride"] + 1
    return Ho, Wo


# ------------------------------------------------------------------------------------------------
# CPU: the row table, the forms and the launch plans
# ------------------------------------------------------------------------------------------------


def test_rows_run_the_forms_the_library_picks():
    """A change to ops.TC5_LAYERS / TC5H_LAYERS or conv_prefers_native that moves a layer out of its form fails here, not
    silently in a row that would then test another kernel."""
    for r in ROWS.values():
        with precision(r["prec"]):
            native = ops.conv_prefers_native(r["cin"], r["cout"], r["ks"])
            assert native and ops.conv_form(r["cin"], r["cout"], r["ks"], r["stride"]) == r["form"], r["name"]
    with precision(1):
        for name, cin, cout, ks, *_ in FEATURE_LAYERS:
            assert ops.conv_prefers_native(cin, cout, ks) == (name in TF32_NATIVE), name
        for name, _, cin, cout, _ in OFFSET_LAYERS:
            assert ops.conv_prefers_native(cin, cout, 3) == (name == "s1.eval"), name
    assert (ROWS["tnt/conv9/10/fp32"]["H"], ROWS["tnt/conv9/10/fp32"]["W"]) == (135, 240)
    assert (ROWS["dtu/output1/fp32"]["H"], ROWS["dtu/output1/fp32"]["W"]) == (150, 200)
    assert (ROWS["eth3d/s1.eval/fp32"]["H"], ROWS["eth3d/s1.eval/fp32"]["W"]) == (896, 1344)


def test_refinement_size_from_the_sizing_rule():
    H, W = odd_refinement_size()
    assert (H, W) == (664, 1000)
    assert W % 8 == 0 and W % 16 != 0 and H % 8 == 0 and H % 16 != 0
    assert all(w % 32 == 0 and h % 8 == 0 for h, w in REFINE_SIZES)


def nhwc_plan(N, H, W, cin, cout, ks, stride, pad, dil, rows_per_warp=0, sms=H100_SMS):
    out = (ctypes.c_int * 5)()
    rc = _native.lib().pmb200_conv2d_nhwc_plan(N, H, W, cin, cout, ks, stride, pad, dil, rows_per_warp, sms, out)
    assert rc == 0, _native.lib().pmb200_last_error().decode()
    return tuple(out)


def form0_launches():
    """(name, N, H, W, Cin, Cout, KS, stride, pad, dil) of every conv2d_nhwc launch of the new rows (transposed form: the
    zero-stuffed input size)."""
    out = [(n, r["N"], r["H"], r["W"], r["cin"], r["cout"], r["ks"], r["stride"], r["pad"], r["dil"]) for n, r in ROWS.items() if r["form"] == 0]
    for cfg, N, H, W in CONFIGS[:5]:
        e, q, h = halve(H, 3), halve(H, 2), halve(H, 1)
        ew, qw, hw = halve(W, 3), halve(W, 2), halve(W, 1)
        out += [(f"{cfg}/u_o", N, e, ew, 64, 32, 1, 1, 0, 1), (f"{cfg}/u_t", N, e, ew, 64, 16, 1, 1, 0, 1),
                (f"{cfg}/l2", N, q, qw, 32, 32, 1, 1, 0, 1), (f"{cfg}/l2_t", N, q, qw, 32, 16, 1, 1, 0, 1), (f"{cfg}/l1", N, h, hw, 16, 16, 1, 1, 0, 1)]
    for H, W in REFINE_SIZES + (odd_refinement_size(),):
        h, w = H // 2, W // 2
        out += [(f"refine{H}x{W}/conv1", 1, h, w, 1, 8, 3, 1, 1, 1), (f"refine{H}x{W}/conv2", 1, h, w, 8, 8, 3, 1, 1, 1),
                (f"refine{H}x{W}/deconv", 1, H, W, 8, 8, 3, 1, 1, 1), (f"refine{H}x{W}/conv0", 1, H, W, 3, 8, 3, 1, 1, 1),
                (f"refine{H}x{W}/conv3", 1, H, W, 16, 8, 3, 1, 1, 1), (f"refine{H}x{W}/res", 1, H, W, 8, 1, 3, 1, 1, 1)]
    return out


def test_conv2d_nhwc_plans_of_the_eval_rows():
    """The plan conv2d_nhwc launches with (warp groups, rows per warp, halo buffers, CTAs, shared memory) for test_conv.py's
    rows (2 x 37x53) and for every conv2d_nhwc launch of this file's rows.  The small maps never prefetch a second halo
    tile; the evaluation maps do, with the most rows per warp the accumulators allow, and with one warp group even for
    Cout = 32."""
    old = {}
    for name, (cin, cout, ks, s, pad, dil, _) in CONV_TEST_LAYERS.items():
        for mt in (0, 1, 2, 4):
            old[(name, mt)] = nhwc_plan(2, 37, 53, cin, cout, ks, s, pad, dil, mt)
    new = {n: nhwc_plan(*a) for n, *a in form0_launches()}
    for k, p in sorted(new.items()):
        print(f"[plan] {k}: nsplit {p[0]} mt {p[1]} nbuf {p[2]} ctas {p[3]} smem {p[4]}")
    old_default = {k[0]: p for k, p in old.items() if k[1] == 0}
    assert {p[2] for p in old_default.values()} == {1}
    assert {p[2] for p in new.values()} == {1, 2}
    assert {(p[0], p[1], p[2]) for p in new.values()} - {(p[0], p[1], p[2]) for p in old_default.values()} >= {(1, 4, 2), (1, 2, 2)}
    assert new["eth3d/conv1/tf32"][:3] == (1, 4, 2) and new["eth3d/conv2/fp32"][:3] == (1, 2, 2)
    assert new["tnt/l2"][0] == 1  # Cout 32 (nt 4): one warp group on a large map
    assert old_default["feature.output2"][0] == 2  # and two on test_conv.py's small one
    # the planner's answer is the one the launcher uses: the same plan for the transposed form's zero-stuffed size
    assert nhwc_plan(1, 1080, 1920, 8, 8, 3, 1, 1, 1) == new["refine1080x1920/deconv"]
    for p in new.values():
        assert p[4] <= 200 * 1024 * p[2] and 1 <= p[3]


def test_conv2d_nhwc_plan_rejects_bad_sizes():
    out = (ctypes.c_int * 5)()
    assert _native.lib().pmb200_conv2d_nhwc_plan(1, 8, 8, 65, 8, 3, 1, 1, 1, 0, 132, out) != 0
    assert _native.lib().pmb200_conv2d_nhwc_plan(1, 8, 8, 8, 8, 3, 1, 1, 1, 0, 0, out) != 0
    assert _native.lib().pmb200_conv2d_nhwc_plan(1, 2, 2, 8, 8, 5, 1, 0, 1, 0, 132, out) != 0  # empty output


def test_tc5h_plans_of_the_eval_rows():
    """K-D5h at the evaluation sizes: units per CTA reach the hundreds (the at-scale tests reach about 6,400 units per
    launch, a few dozen per CTA), so each CTA's persistent loop, mbarrier phases and filter ring turn hundreds of times."""
    most = 0
    for n, r in ROWS.items():
        if r["form"] != 2:
            continue
        units = units_of(r["N"], *out_size(r))
        p = tc5h_plan(r["cin"], r["cout"], r["ks"], r["dil"], units)
        per_cta = units / min(units, H100_SMS * p["ctas"])
        most = max(most, per_cta)
        print(f"[tc5h plan] {n}: {units} units, {p}, {per_cta:.0f} units per CTA")
    assert most >= 200
    assert units_of(8, 896, 1344) == 150528  # ETH3D's half-resolution map: 8 x 112 x 168 units
    assert units_of(8, 896, 1344) // (H100_SMS * 4) >= 200


# ------------------------------------------------------------------------------------------------
# checks: the float64 reference in bands of output rows
# ------------------------------------------------------------------------------------------------


def smooth_dev(g, N, C, H, W, signed):
    """Smooth field on the device: N(0,1) on a 4-pixel lattice, bilinearly interpolated; |.| unless signed."""
    coarse = torch.randn(N, C, H // 4 + 2, W // 4 + 2, generator=g).to(DEV)
    f = F.interpolate(coarse, size=(H // 4 * 4 + 8, W // 4 * 4 + 8), mode="bilinear", align_corners=False)[..., :H, :W]
    f = f if signed else f.abs()
    return f.contiguous(memory_format=torch.channels_last)


def random_layer(g, cin, cout, ks, bias):
    w = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    b = torch.randn(cout, generator=g) * 0.5 if bias else None
    return w, b


def bands(x, w, b, stride, pad, dil):
    """Yields (n, r0, r1, want, S) for output rows r0:r1 of image n: float64 F.conv2d of the input band with its halo (zero
    rows only outside the image) and of the absolute values, S = |W| * |x| + |b|."""
    N, C, H, W = x.shape
    cout, _, ks, _ = w.shape
    Ho = (H + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    rows = max(1, CHUNK_ELEMS // (max(cout, C * stride) * max(W, Wo)))
    w64 = w.to(DEV, F64)
    b64 = torch.zeros(cout, dtype=F64, device=DEV) if b is None else b.to(DEV, F64)
    for n in range(N):
        for r0 in range(0, Ho, rows):
            r1 = min(Ho, r0 + rows)
            lo, hi = r0 * stride - pad, (r1 - 1) * stride - pad + dil * (ks - 1) + 1
            xb = F.pad(x[n:n + 1, :, max(lo, 0):min(hi, H)].to(F64), (pad, pad, max(0, -lo), max(0, hi - H)))
            want = F.conv2d(xb, w64, b64, stride, 0, dil)
            S = F.conv2d(xb.abs(), w64.abs(), None, stride, 0, dil) + b64.abs().view(1, -1, 1, 1)
            yield n, r0, r1, want, S


class Tally:
    """The worst |err| / bound and the RMS of (got - want) / S of one output, over its bands."""

    def __init__(self, tag, K=None):
        self.tag, self.K, self.worst, self.sq, self.n = tag, K, 0.0, 0.0, 0

    def add(self, got, want, bound, S):
        self.worst = max(self.worst, assert_within(self.tag, got, want, bound, ("n", "c", "y", "x")))
        if self.K is not None:
            e = (got.to(DEV, F64) - want) / S.clamp_min(1e-300)
            self.sq += float(e.square().sum())
            self.n += e.numel()

    def finish(self, form=None):
        msg = f"[row] {self.tag}: form {form}, worst |err|/bound {self.worst:.3g}"
        if self.K is None:
            print(msg)
            return self.worst, None
        r = math.sqrt(self.sq / max(self.n, 1))
        print(f"{msg}, precision statistic {r / EPS:.3g} eps <= tau {tau(self.K) / EPS:.3g} eps")
        assert r <= tau(self.K), f"{self.tag}: precision statistic {r / EPS:.3g} eps > tau(K={self.K}) = {tau(self.K) / EPS:.3g} eps"
        return self.worst, r


def check_conv(tag, got, x, w, b, stride, pad, dil, relu, c, K_stat=None, form=None):
    t = Tally(tag, K_stat)
    for n, r0, r1, want, S in bands(x, w, b, stride, pad, dil):
        t.add(got[n:n + 1, :, r0:r1], want.relu() if relu else want, c * EPS * S, S)
    return t.finish(form)


def run_conv(x, w, b, r):
    conv = nn.Conv2d(r["cin"], r["cout"], r["ks"], r["stride"], r["pad"], r["dil"], bias=b is not None).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(w)
        if b is not None:
            conv.bias.copy_(b)
    packed = PackedConv()
    form = packed.packed(conv)[0]
    with torch.no_grad():
        return packed(conv, x, relu=r["relu"]), form


# ------------------------------------------------------------------------------------------------
# GPU rows
# ------------------------------------------------------------------------------------------------


@pytest.fixture()
def timed():
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"[cost] {time.perf_counter() - t0:.2f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GB")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(ROWS))
def test_layer_at_eval_size(name, timed):
    r = ROWS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = smooth_dev(g, r["N"], r["cin"], r["H"], r["W"], r["signed"])
    w, b = random_layer(g, r["cin"], r["cout"], r["ks"], r["bias"])
    K = r["cin"] * r["ks"] ** 2
    with precision(r["prec"]):
        got, form = run_conv(x, w.to(DEV), None if b is None else b.to(DEV), r)
    assert form == r["form"], (name, form)
    assert got.shape == (r["N"], r["cout"], *out_size(r))
    c = c3(K) if r["prec"] == 3 else c1(K)
    check_conv(name, got, x, w, b, r["stride"], r["pad"], r["dil"], r["relu"], c, K if r["prec"] == 3 else None, form)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [c[0] for c in CONFIGS])
def test_stem_at_eval_size(cfg, timed):
    """K-S (conv0 -> conv1 in one launch, exact fp32) on the stacked views, against stem_reference per image."""
    _, N, H, W = next(c for c in CONFIGS if c[0] == cfg)
    g = torch.Generator().manual_seed(N * H + W)
    x = torch.rand(N, 3, H, W, generator=g).to(DEV)
    w0, b0 = torch.randn(8, 3, 3, 3, generator=g) * 0.3, torch.randn(8, generator=g) * 0.1
    w1, b1 = torch.randn(8, 8, 3, 3, generator=g) * 0.2, torch.randn(8, generator=g) * 0.1
    got = ops.conv_stem(x, w0, b0, w1, b1)
    t = Tally(f"{cfg}/K-S")
    for n in range(N):
        want, bnd = stem_reference(x[n:n + 1].double(), *[v.to(DEV, F64) for v in (w0, b0, w1, b1)])
        t.add(got[n:n + 1], want, bnd, None)
        del want, bnd
    t.finish("K-S")


def top_down_case(seed, N, H, W):
    g = torch.Generator().manual_seed(seed)
    fn = FeatureNet().eval()
    with torch.no_grad():
        for name in ("output1", "inner1", "inner2", "output2", "output3"):
            m = getattr(fn, name)
            m.weight.copy_(torch.randn(m.weight.shape, generator=g) / m.in_channels ** 0.5)
            if m.bias is not None:
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.5)
    maps = [smooth_dev(g, N, C, halve(H, k), halve(W, k), False) for C, k in ((64, 3), (32, 2), (16, 1))]
    return fn.to(DEV), maps


def up2(t):
    return F.interpolate(t, scale_factor=2.0, mode="bilinear", align_corners=False)


def top_down_reference(h, e, q, hf):
    """The composed top-down path of FeatureNet._fused_top_down in float64 on one image (e, q, hf: the trunk maps), with the
    chained bounds: (out2, bound2, out1, bound1, S of u_o, u_t)."""
    w = {k: v.to(DEV, F64) for k, v in h.items()}
    e, q, hf = e.double(), q.double(), hf.double()
    out = {}
    for name, W_, x in (("u_o", w["u_o"], e), ("u_t", w["u_t"], e)):
        out[name] = (F.conv2d(x, W_), F.conv2d(x, W_.abs()))
        out[name] = out[name] + (c3(64) * EPS * out[name][1],)

    def lateral(W_, c, x, u):
        uw, us, ub = u
        conv = F.conv2d(x, W_, c)
        S = F.conv2d(x, W_.abs()) + c.abs().view(1, -1, 1, 1)
        want = conv + up2(uw)
        bound = up2(ub) + 8 * EPS * up2(us + ub) + (c3(W_.shape[1]) + 1) * EPS * S
        return want, S + up2(us), bound

    o2 = lateral(w["l2_o"], w["c2_o"], q, out["u_o"])
    t = lateral(w["l2_t"], w["c2_t"], q, out["u_t"])
    o1 = lateral(w["l1"], w["c1"], hf, t)
    return out, o2, o1


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", [c[0] for c in CONFIGS])
def test_top_down_path_at_eval_size(cfg, timed):
    """fp32-accurate mode: FeatureNet._fused_top_down itself (u_o / u_t, then the three lateral 1x1 convs with the add_up2x
    epilogue, each on the kernel's own previous output), against float64 per image.  The TF32 mode: the same launches at
    precision 1 (plus 1 eps of the composed weights' rounding, carried in c1)."""
    _, N, H, W = next(c for c in CONFIGS if c[0] == cfg)
    fn, (e, q, hf) = top_down_case(N + H, N, H, W)
    h = fn.composed_heads()
    for prec in (3, 1):
        with precision(prec), torch.no_grad():
            got = fn._fused_top_down(e, q, hf)
            u_o = ops.conv2d_nhwc(e, ops.pack_conv_filter(h["u_o"].to(DEV), prec), None, 32, 1)
            u_t = ops.conv2d_nhwc(e, ops.pack_conv_filter(h["u_t"].to(DEV), prec), None, 16, 1)
        scale = (lambda K: c1(K) / c3(K)) if prec == 1 else (lambda K: 1.0)
        tag = f"{cfg}/top-down/{'fp32' if prec == 3 else 'tf32'}"
        tallies = {k: Tally(f"{tag}/{k}", 64 if prec == 3 and k.startswith("u_") else None) for k in ("u_o", "u_t", "out2", "out1")}
        for n in range(N):
            u, o2, o1 = top_down_reference(h, e[n:n + 1], q[n:n + 1], hf[n:n + 1])
            s = scale(64)
            tallies["u_o"].add(u_o[n:n + 1], u["u_o"][0], s * u["u_o"][2], u["u_o"][1])
            tallies["u_t"].add(u_t[n:n + 1], u["u_t"][0], s * u["u_t"][2], u["u_t"][1])
            tallies["out2"].add(got[2][n:n + 1], o2[0], scale(32) * o2[2], o2[1])
            tallies["out1"].add(got[1][n:n + 1], o1[0], scale(32) * o1[2], o1[1])
            del u, o2, o1
        for t in tallies.values():
            t.finish("0 (add_up2x)" if "out" in t.tag else 0)


def refine_case(seed, N, H, W):
    m = _random_refinement(seed).to(DEV)
    g = torch.Generator().manual_seed(seed)
    h, w = H // 2, W // 2
    img = torch.rand(N, 3, H, W, generator=g).to(DEV)
    dmin = torch.full((N,), 400.0, device=DEV)
    dmax = torch.full((N,), 900.0, device=DEV)
    depth = dmin.view(N, 1, 1, 1) + smooth_dev(g, N, 1, h, w, True).sigmoid().contiguous() * (dmax - dmin).view(N, 1, 1, 1)
    return m, img, depth, dmin, dmax


def refine_reference(hw, img, depth, lo, hi, cK):
    """Refinement in float64 from its folded weights hw (Refinement.host_weights order) on one image band, with the chained
    bound; cK(K) is the per-layer constant of the arithmetic that runs it."""
    w1, b1, w2, b2, wd, bd, w0, b0, w3, b3, wr = [t.to(DEV, F64) for t in hw]
    span = hi - lo
    d = (depth - lo) / span
    dd = 4 * EPS * (depth.abs() + abs(lo)) / span

    def layer(x, bx, W_, B, K, relu=True, transposed=False):
        if transposed:
            f = lambda t, ww, bb: F.conv_transpose2d(t, ww, bb, stride=2, padding=1, output_padding=1)  # noqa: E731
        else:
            f = lambda t, ww, bb: F.conv2d(t, ww, bb, padding=1)  # noqa: E731
        y = f(x, W_, B)
        S = f(x.abs() + bx, W_.abs(), None if B is None else B.abs())
        return (y.relu() if relu else y), f(bx, W_.abs(), None) + (cK(K) + 1) * EPS * S

    h1, bh1 = layer(d, dd, w1, b1, 9)
    h2, bh2 = layer(h1, bh1, w2, b2, 72)
    up, bup = layer(h2, bh2, wd, bd, 72, transposed=True)
    i0, bi0 = layer(img, torch.zeros_like(img), w0, b0, 27)
    h3, bh3 = layer(torch.cat((up, i0), 1), torch.cat((bup, bi0), 1), w3, b3, 144)
    res, bres = layer(h3, bh3, wr, None, 72, relu=False)
    nd = F.interpolate(d, scale_factor=2.0, mode="nearest")
    ndd = F.interpolate(dd, scale_factor=2.0, mode="nearest")
    want = (nd + res) * span + lo
    bound = span * (ndd + bres) + 4 * EPS * (span * (nd.abs() + res.abs()) + abs(lo))
    return want, bound


def check_refinement(tag, got, hw, img, depth, dmin, dmax, cK):
    """Against refine_reference in bands of full-resolution rows: each band is computed with 8 half-resolution rows of
    margin (more than the chain's reach) and the margin is dropped, except at the image's own borders."""
    N, _, H, W = got.shape
    h = H // 2
    band = max(8, CHUNK_ELEMS // (64 * W) // 2 * 2)
    t = Tally(tag)
    for n in range(N):
        for R0 in range(0, H, band):
            R1 = min(H, R0 + band)
            a, b = max(0, R0 // 2 - 8), min(h, R1 // 2 + 8)
            want, bound = refine_reference(hw, img[n:n + 1, :, 2 * a:2 * b].double(), depth[n:n + 1, :, a:b].double(), float(dmin[n]),
                                           float(dmax[n]), cK)
            k0 = R0 - 2 * a
            t.add(got[n:n + 1, :, R0:R1], want[:, :, k0:k0 + R1 - R0], bound[:, :, k0:k0 + R1 - R0], None)
    return t.finish()


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", REFINE_SIZES + (odd_refinement_size(),))
def test_refinement_at_image_size(H, W, timed):
    """K-R (refine_low + refine_full, exact fp32) and, in the TF32 mode, Refinement._native_tail (six conv2d_nhwc launches at
    precision 1, the transposed form writing channels 0..7 of the 16-channel buffer) with the module's own tail."""
    m, img, depth, dmin, dmax = refine_case(H + W, 1, H, W)
    hw = m.host_weights()
    with precision(3), torch.no_grad():
        got = m(img, depth, dmin, dmax)
    check_refinement(f"refine {H}x{W} K-R", got, hw, img, depth, dmin, dmax, lambda K: K + 3)
    with precision(1), torch.no_grad():
        got = m(img, depth, dmin, dmax)
    check_refinement(f"refine {H}x{W} tf32 native tail", got, hw, img, depth, dmin, dmax, c1)


def random_feature_net(seed):
    g = torch.Generator().manual_seed(seed)
    fn = FeatureNet().eval()
    with torch.no_grad():
        for mod in fn.modules():
            if isinstance(mod, nn.Conv2d):
                fan = mod.in_channels * mod.kernel_size[0] ** 2
                mod.weight.copy_(torch.randn(mod.weight.shape, generator=g) / fan ** 0.5)
                if mod.bias is not None:
                    mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.5)
            elif isinstance(mod, nn.BatchNorm2d):
                mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.3)
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.3)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
    return fn


def feature_net_links(fn64, x, got):
    """Each link of the fast path against the module's own float64 layers applied to the fast path's own input of that
    link (LIBRARY_FAST_PATH = False: conv, BatchNorm, ReLU as the reference runs them), one image: K-S on the image, conv2..10
    on the previous layer's fp32 output, output1 and the top-down path (output2 / output3 of the upsampled sums of inner1 /
    inner2) on the fp32 trunk maps.  A bound carried through all eleven layers grows by about sqrt(K) per layer (|W| * bound):
    some 10^10 at the outputs, no check at all; per link it stays c3(K) + 1 (the folded weights' rounding).  -> {tag: (got,
    want, bound)}."""
    old = pm_net.LIBRARY_FAST_PATH
    pm_net.LIBRARY_FAST_PATH = False
    out = {}
    try:
        with torch.no_grad():
            def folded(i):
                m = getattr(fn64, f"conv{i}")
                sc = m.bn.weight / torch.sqrt(m.bn.running_var + m.bn.eps)
                return m.conv.weight * sc.view(-1, 1, 1, 1), m.bn.bias - m.bn.running_mean * sc, m.conv.stride[0], m.conv.padding[0]

            w0, b0, _, _ = folded(0)
            w1, b1, _, _ = folded(1)
            want, bnd = stem_reference(x, w0, b0, w1, b1)
            s0 = EPS * F.conv2d(x.abs(), w0.abs(), b0.abs(), padding=1)
            bnd = bnd + F.conv2d(s0, w1.abs(), padding=1) + 2 * EPS * F.conv2d(want + s0, w1.abs(), b1.abs(), padding=1)
            assert torch.allclose(want, fn64.conv1(fn64.conv0(x)), rtol=1e-12, atol=1e-12)
            out["K-S"] = (got["stem"], want, bnd)
            for i in range(2, 11):
                xin = got[i - 1].double()
                W_, B, st, pd = folded(i)
                K = W_.shape[1] * W_.shape[2] ** 2
                out[f"conv{i}"] = (got[i], getattr(fn64, f"conv{i}")(xin), (c3(K) + 1) * EPS * F.conv2d(xin.abs(), W_.abs(), B.abs(), st, pd))
            e, q, hf = got[10].double(), got[7].double(), got[4].double()
            lin = lambda t, m_: F.conv2d(t, m_.abs())  # noqa: E731
            out["out3"] = (got["out3"], fn64.output1(e), (c3(64) + 1) * EPS * lin(e.abs(), fn64.output1.weight))
            top2 = up2(e) + fn64.inner1(q)
            out2, out1 = fn64.output2(top2), fn64.output3(up2(top2) + fn64.inner2(hf))
            Wf = lambda conv: conv.weight.flatten(1)  # noqa: E731
            W2, W3, Wi1, Wi2 = Wf(fn64.output2), Wf(fn64.output3), Wf(fn64.inner1), Wf(fn64.inner2)
            as4 = lambda m_: m_.reshape(m_.shape[0], m_.shape[1], 1, 1)  # noqa: E731
            h = {"u_o": as4(W2), "u_t": as4(W3), "l2_o": as4(W2 @ Wi1), "l2_t": as4(W3 @ Wi1), "l1": as4(W3 @ Wi2),
                 "c2_o": W2 @ fn64.inner1.bias, "c2_t": W3 @ fn64.inner1.bias, "c1": W3 @ fn64.inner2.bias}
            _, o2, o1 = top_down_reference(h, e, q, hf)
            # the composed weights are rounded once to fp32: one more eps of each S
            out["out2"] = (got["out2"], out2, o2[2] + EPS * o2[1])
            out["out1"] = (got["out1"], out1, o1[2] + 2 * EPS * o1[1])
    finally:
        pm_net.LIBRARY_FAST_PATH = old
    return out


@pytest.mark.gpu
def test_whole_feature_net_at_tnt(timed):
    """The fast path (K-S, then every trunk layer in its form, output1, the composed top-down path) on 8 x 1080x1920 against
    the module in float64 with the reference's op sequence, link by link: BatchNorm folding, composed heads, chained
    epilogues."""
    _, N, H, W = CONFIGS[0]
    fn = random_feature_net(7).to(DEV)
    fn64 = random_feature_net(7).double().to(DEV)
    g = torch.Generator().manual_seed(8)
    x = torch.rand(N, 3, H, W, generator=g).to(DEV)
    got = {}
    hooks = [getattr(fn, f"conv{i}").register_forward_hook(lambda m, i_, o, k=i: got.__setitem__(k, o)) for i in range(2, 11)]
    hooks.append(fn.conv2.register_forward_pre_hook(lambda m, i_: got.__setitem__("stem", i_[0])))
    try:
        with precision(3), torch.no_grad():
            outs = fn(x)
    finally:
        for hk in hooks:
            hk.remove()
    got[1] = got["stem"]
    got.update({"out3": outs[3], "out2": outs[2], "out1": outs[1]})
    tallies = {}
    for n in range(N):
        links = feature_net_links(fn64, x[n:n + 1].double(), {k: v[n:n + 1] for k, v in got.items()})
        for k, (gg, want, bound) in links.items():
            tallies.setdefault(k, Tally(f"tnt/FeatureNet/{k}")).add(gg, want, bound, None)
        del links
    for t in tallies.values():
        t.finish("fast path")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tnt/conv2/fp32", "eth3d/conv8/fp32", "dtu/conv9/10/fp32", "tnt/conv3/4/fp32"])
def test_tf32_output_fails_the_fp32_checks(name):
    """The same layer and inputs through conv2d_nhwc at precision 1 (plain TF32 operands) must be rejected by the
    fp32-accurate checks; on a quarter of the views, enough for the statistic."""
    r = ROWS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = smooth_dev(g, r["N"], r["cin"], r["H"], r["W"], r["signed"])[:2]
    w, b = random_layer(g, r["cin"], r["cout"], r["ks"], r["bias"])
    K = r["cin"] * r["ks"] ** 2
    got = ops.conv2d_nhwc(x, ops.pack_conv_filter(w.to(DEV), 1), b.to(DEV), r["cout"], r["ks"], r["stride"], r["pad"], r["dil"],
                          relu=r["relu"], precision=1)
    with pytest.raises(AssertionError) as err:
        check_conv(f"{name} at precision 1", got, x, w, b, r["stride"], r["pad"], r["dil"], r["relu"], c3(K), K)
    print(f"[sensitivity] {name}: rejected: {str(err.value).splitlines()[0]}")


# ------------------------------------------------------------------------------------------------
# CPU: the checks bite
# ------------------------------------------------------------------------------------------------


def test_sensitivity_conv():
    g = torch.Generator().manual_seed(1)
    x = torch.rand(1, 8, 13, 23, generator=g, dtype=F64)
    w, b = random_layer(g, 8, 16, 3, True)
    want = F.conv2d(x, w.double(), b.double(), padding=1)
    S = F.conv2d(x, w.double().abs(), b.double().abs(), padding=1)
    plant_rejected("conv 8->16", want.float(), want, c3(72) * EPS * S, ("n", "c", "y", "x"), (0, None, 12, 22))


def test_sensitivity_add_up2x_epilogue():
    g = torch.Generator().manual_seed(2)
    fn, _ = _cpu(top_down_case, 2, 1, 8, 8)
    h = fn.composed_heads()
    maps = [torch.rand(1, C, 13 * 2 ** (2 - k), 23 * 2 ** (2 - k), generator=g, dtype=F64) for C, k in ((64, 2), (32, 1), (16, 0))]
    u, o2, o1 = _cpu(top_down_reference, h, *maps)
    plant_rejected("add_up2x out2", o2[0].float(), o2[0], o2[2], ("n", "c", "y", "x"), (0, None, 25, 45))
    plant_rejected("add_up2x out1", o1[0].float(), o1[0], o1[2], ("n", "c", "y", "x"), (0, None, 51, 91))


def test_sensitivity_refinement_chain():
    m = _random_refinement(4)
    g = torch.Generator().manual_seed(4)
    img = torch.rand(1, 3, 26, 46, generator=g, dtype=F64)
    depth = 400 + 500 * torch.rand(1, 1, 13, 23, generator=g, dtype=F64)
    want, bound = _cpu(refine_reference, m.host_weights(), img, depth, 400.0, 900.0, lambda K: K + 3)
    plant_rejected("refinement chain", want.float(), want, bound, ("n", "c", "y", "x"), (0, 0, 25, 45))


def _cpu(fn, *args):
    """Run a float64 reference on the CPU (its tensors follow DEV)."""
    global DEV
    saved, DEV = DEV, "cpu"
    try:
        return fn(*args)
    finally:
        DEV = saved


def trunc_tf32(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


@pytest.mark.parametrize("cin,ks", [(8, 3), (64, 3), (64, 5)])
def test_precision_statistic_rejects_a_dropped_split_term(cin, ks):
    """float64 emulation of the 3xTF32 conv (ops._tf32_round for the filter split, the activations split by truncation as
    the kernels do), K = 72, 576, 1600: complete, it passes tau(K); with a_lo w_hi dropped it fails."""
    K = cin * ks * ks
    g = torch.Generator().manual_seed(K)
    x = torch.rand(1, cin, 40, 40, generator=g)
    w, b = random_layer(g, cin, 16, ks, True)
    hi, whi = trunc_tf32(x), ops._tf32_round(w)
    wlo = ops._tf32_round(w - whi)
    lo = trunc_tf32(x - hi)
    d = lambda t: t.double()  # noqa: E731
    want = F.conv2d(d(x), d(w), d(b))
    S = F.conv2d(d(x), d(w).abs(), d(b).abs())
    kept = F.conv2d(d(hi), d(whi) + d(wlo), d(b))
    rms = lambda got: float((((got - want) / S) ** 2).mean().sqrt())  # noqa: E731
    complete, dropped = rms(kept + F.conv2d(d(lo), d(whi))), rms(kept)
    print(f"[emulated] K={K}: complete {complete / EPS:.3g} eps, a_lo w_hi dropped {dropped / EPS:.3g} eps, tau {tau(K) / EPS:.3g} eps")
    assert complete <= tau(K) < dropped
