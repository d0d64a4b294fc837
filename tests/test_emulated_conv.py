"""The channels-last tensor-core conv family (csrc/pm_conv.cu) -- kernel AND launch planning of pmb200_conv2d_nhwc -- executed
on the CPU by the warp emulator (tests/warp_emu.h, tests/emu_conv.cpp): mma.sync.m16n8k8 TF32 is a warp collective with the
hardware's fragment layout and TF32 operand truncation, cp.async an immediate copy / zero fill.  The CPU twin of the GPU
cases in tests/test_conv.py, at the same tolerances: 3xTF32 (precision 3) <= 2e-5 of the output scale, TF32 (precision 1)
<= 3e-3, against torch's fp32 conv2d.  tests/conv_emulator.py (Python) checks the fragment ALGEBRA; this runs the source."""
import ctypes
import os
import subprocess

import pytest
import torch
import torch.nn.functional as F

from patchmatchnet_b200 import ops
from tests.test_conv import LAYERS, _ref_conv

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="session")
def emu_conv():
    src = os.path.join(REPO, "tests", "emu_conv.cpp")
    deps = [src, os.path.join(REPO, "tests", "warp_emu.h"), os.path.join(REPO, "include", "patchmatch_b200.h"),
            os.path.join(REPO, "patchmatchnet_b200", "csrc", "pm_conv.cu"), os.path.join(REPO, "patchmatchnet_b200", "csrc", "pm_stem.cu"),
            os.path.join(REPO, "patchmatchnet_b200", "csrc", "pm_refine.cu")]
    out = os.path.join(REPO, "tests", "_emu_conv.so")
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", f"-I{cuda_inc}", "-o", out, src], check=True, cwd=os.path.join(REPO, "tests"))
    lib = ctypes.CDLL(out)
    P, I = ctypes.c_void_p, ctypes.c_int
    lib.emu_conv2d_nhwc.argtypes = [P] * 5 + [I] * 15 + [P]
    lib.emu_conv2d_nhwc.restype = I
    lib.emu_conv2d_filter_floats.argtypes = [I] * 4
    lib.emu_conv2d_filter_floats.restype = I
    lib.emu_conv_last_error.restype = ctypes.c_char_p
    lib.emu_conv_stem.argtypes = [P] * 6 + [I] * 3 + [P]
    lib.emu_conv_stem.restype = I
    lib.emu_refine_low.argtypes = [P] * 8 + [I] * 3 + [P]
    lib.emu_refine_low.restype = I
    lib.emu_refine_full.argtypes = [P] * 13 + [I] * 3 + [P]
    lib.emu_refine_full.restype = I
    lib.emu_conv_set_stem_ppt.argtypes = [I]
    lib.emu_conv_set_stem_ppt.restype = None
    return lib


def _cl(x):
    return x.contiguous(memory_format=torch.channels_last)


def _run(lib, x, frag, bias, cout, ks, S=1, pad=0, dil=1, relu=False, prec=3, transposed2x=False, out=None, yco=0, mt=0, add_up2x=None):
    x = _cl(x)
    N, cin, H, W = x.shape
    assert frag.numel() == lib.emu_conv2d_filter_floats(cin, cout, ks, prec)
    Hv, Wv = (2 * H, 2 * W) if transposed2x else (H, W)
    Ho = (Hv + 2 * pad - dil * (ks - 1) - 1) // S + 1
    Wo = (Wv + 2 * pad - dil * (ks - 1) - 1) // S + 1
    if out is None:
        out = _cl(torch.full((N, cout, Ho, Wo), float("nan")))
    ycs = out.shape[1]
    frag = frag.contiguous()
    rc = lib.emu_conv2d_nhwc(x.data_ptr(), frag.data_ptr(), None if bias is None else bias.data_ptr(),
                             None if add_up2x is None else add_up2x.data_ptr(), out.data_ptr(), N, H, W, cin, cout, ks, S, pad, dil,
                             1 if relu else 0, prec, 1 if transposed2x else 0, ycs, yco, mt, None)
    assert rc == 0, lib.emu_conv_last_error()
    return out


def _scaled_err(got, want):
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-6))


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_emulated_source_matches_conv2d(emu_conv, name):
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    # ragged: neither dimension a multiple of the 16 x (4*MT) tile; two images for the light layers (the MMA emulation
    # costs ~1 us per fiber switch, so the 64-channel layers get one image)
    N, H, W = (2 if cin * cout * ks * ks <= 8 * 16 * 25 else 1), 13, 21
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    b = torch.randn(cout, generator=g)
    want = _ref_conv(x, w, b, S, pad, dil, relu)
    for prec, tol in ((3, 2e-5), (1, 3e-3)):
        frag = ops.pack_conv_filter(w, prec)
        for mt in ((0, 1, 2, 4) if (prec == 3 and cin * cout * ks * ks <= 32 * 32 * 9) else (0,)):
            got = _run(emu_conv, x, frag, b, cout, ks, S, pad, dil, relu=relu, prec=prec, mt=mt)
            assert got.shape == want.shape
            err = _scaled_err(got, want)
            assert err <= tol, f"{name} precision {prec} rows_per_warp {mt}: scaled max err {err:.3e}"


@pytest.mark.parametrize("name", ["feature.conv0", "feature.conv1", "feature.conv2", "feature.conv3", "feature.conv9", "stage1.eval_conv"])
def test_emulated_persistent_double_buffered_path(emu_conv, name, monkeypatch):
    """On a pretend 1-SM device the planner gives the same small map several tiles per CTA and two halo buffers: the
    persistent loop with the next tile's prefetch in flight (what every full-size layer runs on the GPU)."""
    monkeypatch.setenv("PM_EMU_SMS", "1")
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 1)
    N, H, W = 2, 29, 37
    x = torch.randn(N, cin, H, W, generator=g)
    w = torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5
    b = torch.randn(cout, generator=g)
    want = _ref_conv(x, w, b, S, pad, dil, relu)
    got = _run(emu_conv, x, ops.pack_conv_filter(w, 3), b, cout, ks, S, pad, dil, relu=relu, prec=3, mt=0)
    assert _scaled_err(got, want) <= 2e-5


def test_emulated_transposed_conv_and_channel_slices(emu_conv):
    g = torch.Generator().manual_seed(5)
    low = torch.randn(2, 8, 11, 19, generator=g)
    img = torch.randn(2, 3, 22, 38, generator=g)
    wt = torch.randn(8, 8, 3, 3, generator=g) / 8
    bt = torch.randn(8, generator=g)
    w0 = torch.randn(8, 3, 3, 3, generator=g) / 5
    b0 = torch.randn(8, generator=g)
    want = torch.cat((F.conv_transpose2d(low, wt, bt, stride=2, padding=1, output_padding=1).relu(), F.conv2d(img, w0, b0, padding=1).relu()), dim=1)
    both = _cl(torch.full((2, 16, 22, 38), float("nan")))
    _run(emu_conv, low, ops.pack_conv_filter(wt, 3, transposed=True), bt, 8, 3, 1, 1, 1, relu=True, transposed2x=True, out=both, yco=0)
    assert torch.isnan(both[:, 8:]).all(), "the other half of the buffer must be untouched"
    _run(emu_conv, img, ops.pack_conv_filter(w0, 3), b0, 8, 3, 1, 1, 1, relu=True, out=both, yco=8)
    assert _scaled_err(both, want) <= 2e-5


def test_emulated_conv_with_fused_upsample_add(emu_conv):
    g = torch.Generator().manual_seed(9)
    for cin, cout, (h, w) in ((32, 32, (9, 13)), (16, 16, (16, 20)), (32, 16, (8, 8))):
        fine = torch.randn(2, cin, 2 * h, 2 * w, generator=g)
        coarse = _cl(torch.randn(2, cout, h, w, generator=g))
        wt = torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5
        b = torch.randn(cout, generator=g)
        want = F.interpolate(coarse, scale_factor=2.0, mode="bilinear", align_corners=False) + F.conv2d(fine, wt, b)
        got = _run(emu_conv, fine, ops.pack_conv_filter(wt, 3), b, cout, 1, prec=3, add_up2x=coarse)
        assert _scaled_err(got, want) <= 2e-5


def test_emulated_planner_rejects_bad_arguments(emu_conv):
    x = _cl(torch.zeros(1, 8, 8, 8))
    y = _cl(torch.zeros(1, 8, 8, 8))
    f = torch.zeros(emu_conv.emu_conv2d_filter_floats(8, 8, 3, 1))
    args = lambda **kw: [x.data_ptr(), f.data_ptr(), None, None, y.data_ptr(), 1, 8, 8, 8, 8, kw.get("ks", 3), kw.get("S", 1), 1, 1, 0,
                         kw.get("prec", 1), 0, 8, kw.get("yco", 0), 0, None]
    assert emu_conv.emu_conv2d_nhwc(*args(S=3)) == -1
    assert emu_conv.emu_conv2d_nhwc(*args(prec=2)) == -1
    assert emu_conv.emu_conv2d_nhwc(*args(yco=4)) == -1 and b"channel slice" in emu_conv.emu_conv_last_error()


@pytest.mark.parametrize("ppt", [2, 4])
@pytest.mark.parametrize("shape", [(2, 21, 45), (1, 16, 32), (1, 37, 70), (3, 5, 9)])
def test_emulated_stem_matches_two_convs(emu_conv, shape, ppt):
    """K-S (csrc/pm_stem.cu, the kernel's own source under the warp emulator): relu(conv1(relu(conv0(x)))) with folded biases
    against the two F.conv2d calls, ragged sizes (partial 32 x 16 tiles, image borders inside the conv0 halo), exact fp32
    arithmetic -> agreement to rounding-order noise."""
    N, H, W = shape
    g = torch.Generator().manual_seed(N * 1000 + H * 10 + W)
    x = torch.randn(N, 3, H, W, generator=g)
    w0, b0 = torch.randn(8, 3, 3, 3, generator=g) / 27 ** 0.5, torch.randn(8, generator=g) * 0.5
    w1, b1 = torch.randn(8, 8, 3, 3, generator=g) / 72 ** 0.5, torch.randn(8, generator=g) * 0.5
    y = torch.full((N, H, W, 8), float("nan"))
    emu_conv.emu_conv_set_stem_ppt(ppt)  # output pixels per thread: 256- or 128-thread CTAs
    rc = emu_conv.emu_conv_stem(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr(), N, H, W, None)
    assert rc == 0, emu_conv.emu_conv_last_error()
    want = F.relu(F.conv2d(F.relu(F.conv2d(x.double(), w0.double(), b0.double(), padding=1)), w1.double(), b1.double(), padding=1)).float()
    emu_conv.emu_conv_set_stem_ppt(2)
    got = y.permute(0, 3, 1, 2)
    assert torch.isfinite(got).all()
    assert _scaled_err(got, want) <= 2e-6


def test_emulated_stem_argument_errors(emu_conv):
    x, y = torch.zeros(1, 3, 4, 4), torch.zeros(1, 4, 4, 8)
    w0, b0, w1, b1 = torch.zeros(8, 3, 3, 3), torch.zeros(8), torch.zeros(8, 8, 3, 3), torch.zeros(8)
    assert emu_conv.emu_conv_stem(None, w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr(), 1, 4, 4, None) == -1
    assert emu_conv.emu_conv_stem(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr(), 1, 0, 4, None) == -1
    assert emu_conv.emu_conv_stem(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr() + 4, 1, 4, 4, None) == -1


def _random_refinement(seed):
    from patchmatchnet_b200.net import Refinement

    torch.manual_seed(seed)
    m = Refinement().eval()
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.weight.uniform_(0.5, 1.5)
                mod.bias.normal_(0, 0.3)
                mod.running_mean.normal_(0, 0.3)
                mod.running_var.uniform_(0.5, 1.5)
    return m


@pytest.mark.parametrize("shape", [(2, 10, 22), (1, 8, 16), (1, 13, 35), (2, 3, 5)])
def test_emulated_refinement_matches_the_module(emu_conv, shape):
    """K-R (pm_stem.cu one-plane form + pm_refine.cu, the kernels' own source under the warp emulator) against the Refinement
    module's reference op sequence in float64 (reference models/net.py:73-122): transposed conv by output parity, halo
    recompute across tile borders, image borders inside every halo, the residual tail; ragged sizes, two images."""
    N, h, w = shape
    m = _random_refinement(N * 100 + h)
    g = torch.Generator().manual_seed(h * 7 + w)
    img = torch.rand(N, 3, 2 * h, 2 * w, generator=g)
    dmin = torch.tensor([400.0, 425.0][:N])
    dmax = torch.tensor([900.0, 935.0][:N])
    depth = dmin.view(N, 1, 1, 1) + torch.rand(N, 1, h, w, generator=g) * (dmax - dmin).view(N, 1, 1, 1)
    with torch.no_grad():
        want = m.double()(img.double(), depth.double(), dmin.double(), dmax.double()).float()
        m.float()
        hw = m.host_weights()
    low = torch.full((N, h, w, 8), float("nan"))
    rc = emu_conv.emu_refine_low(depth.data_ptr(), dmin.data_ptr(), dmax.data_ptr(), *(t.data_ptr() for t in hw[:4]), low.data_ptr(), N, h, w, None)
    assert rc == 0, emu_conv.emu_conv_last_error()
    assert torch.isfinite(low).all()
    out = torch.full((N, 1, 2 * h, 2 * w), float("nan"))
    rc = emu_conv.emu_refine_full(low.data_ptr(), img.data_ptr(), depth.data_ptr(), dmin.data_ptr(), dmax.data_ptr(), *(t.data_ptr() for t in hw[4:]),
                                  out.data_ptr(), N, 2 * h, 2 * w, None)
    assert rc == 0, emu_conv.emu_conv_last_error()
    assert torch.isfinite(out).all()
    # depths are ~400..935 and the residual is O(span): compare on the normalised scale
    span = (dmax - dmin).view(N, 1, 1, 1)
    assert float(((out - want).abs() / span).max()) <= 2e-6


def test_emulated_refinement_argument_errors(emu_conv):
    z = torch.zeros(1, 4, 4, 8)
    hw = _random_refinement(0).host_weights()
    img, depth, lo, hi, out = torch.zeros(1, 3, 8, 8), torch.zeros(1, 1, 4, 4), torch.zeros(1), torch.ones(1), torch.zeros(1, 1, 8, 8)
    args = [z.data_ptr(), img.data_ptr(), depth.data_ptr(), lo.data_ptr(), hi.data_ptr(), *(t.data_ptr() for t in hw[4:]), out.data_ptr()]
    assert emu_conv.emu_refine_full(*args, 1, 7, 8, None) == -1 and b"even" in emu_conv.emu_conv_last_error()
    assert emu_conv.emu_refine_full(None, *args[1:], 1, 8, 8, None) == -1
    assert emu_conv.emu_refine_low(depth.data_ptr(), None, hi.data_ptr(), *(t.data_ptr() for t in hw[:4]), z.data_ptr(), 1, 4, 4, None) == -1
