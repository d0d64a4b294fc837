"""Native channels-last tensor-core conv (csrc/pm_conv.cu, ops.conv2d_nhwc): the offset convs of the hot path
(reference models/patchmatch.py:288-311) and the FeatureNet / Refinement convs either side of it (models/net.py:9-122).

CPU part: the host-side filter packing and the kernel's index math (staging, fragment addresses, lane <-> element
mapping, epilogue ownership, zero-stuffed transposed form) through the lane-level emulator in tests/conv_emulator.py,
against torch's conv2d / conv_transpose2d.  GPU part (-m gpu): the kernel itself against cuDNN in full fp32 for
every layer shape of the network plus ragged sizes, channel slices and forced tile heights.
Tolerances: precision 3 (3xTF32) is fp32-accurate -> 2e-5 of the output scale; precision 1 (TF32 operands, the
library's default behaviour) -> 3e-3 of the output scale (10-bit mantissas, K <= 1600 products)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from patchmatchnet_b200 import _native, ops
from tests.conv_emulator import emulate_conv, pixel_stride

# (cin, cout, ks, stride, pad, dil, relu): every conv shape of the model
LAYERS = {
    "feature.conv0": (3, 8, 3, 1, 1, 1, True),
    "feature.conv1": (8, 8, 3, 1, 1, 1, True),
    "feature.conv2": (8, 16, 5, 2, 2, 1, True),
    "feature.conv3": (16, 16, 3, 1, 1, 1, True),
    "feature.conv5": (16, 32, 5, 2, 2, 1, True),
    "feature.conv6": (32, 32, 3, 1, 1, 1, True),
    "feature.conv8": (32, 64, 5, 2, 2, 1, True),
    "feature.conv9": (64, 64, 3, 1, 1, 1, True),
    "feature.output1": (64, 64, 1, 1, 0, 1, False),
    "feature.inner1": (32, 64, 1, 1, 0, 1, False),
    "feature.inner2": (16, 64, 1, 1, 0, 1, False),
    "feature.output2": (64, 32, 1, 1, 0, 1, False),
    "feature.output3": (64, 16, 1, 1, 0, 1, False),
    "refine.conv1": (1, 8, 3, 1, 1, 1, True),
    "refine.conv3": (16, 8, 3, 1, 1, 1, True),
    "refine.res": (8, 1, 3, 1, 1, 1, False),
    "stage3.propa_conv": (64, 32, 3, 1, 2, 2, False),
    "stage3.eval_conv": (64, 18, 3, 1, 2, 2, False),
    "stage2.propa_conv": (32, 16, 3, 1, 4, 4, False),
    "stage2.eval_conv": (32, 18, 3, 1, 4, 4, False),
    "stage1.eval_conv": (16, 18, 3, 1, 6, 6, False),
    "stage1.propa_conv": (16, 1, 3, 1, 6, 6, False),
}


def _ref_conv(x, w, b, S, pad, dil, relu):
    y = F.conv2d(x, w, b, stride=S, padding=pad, dilation=dil)
    return y.relu() if relu else y


# ------------------------------------------------------------------------------------------------
# CPU: packing + index math
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", ["feature.conv0", "feature.conv2", "feature.conv9", "refine.res", "stage2.eval_conv", "stage1.eval_conv",
                                  "feature.inner2", "refine.conv1"])
def test_emulated_kernel_matches_conv2d(name):
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    H, W = (7, 19) if cin >= 32 else (11, 21)
    x = torch.randn(1, cin, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(cout, cin, ks, ks, generator=g).double()
    b = torch.randn(cout, generator=g).double()
    want = _ref_conv(x, w.float().double(), b, S, pad, dil, relu).permute(0, 2, 3, 1).numpy()
    scale = np.abs(want).max()
    for prec, tol in ((3, 2e-6), (1, 2e-3)):  # hi+lo restores the fp32 weight to 2^-22; TF32 weights carry 2^-11
        frag = ops.pack_conv_filter(w.float(), prec)
        assert frag.numel() == _native.lib().pmb200_conv2d_filter_floats(cin, cout, ks, prec)
        for mt in (1, 4):
            got = emulate_conv(x.permute(0, 2, 3, 1).numpy(), frag.numpy(), b.numpy(), cout, ks, S, pad, dil, relu, False, mt)
            assert got.shape == want.shape
            assert not np.isnan(got).any(), "an output element was never written"
            assert np.abs(got - want).max() <= tol * scale
            assert emulate_conv.last_banks_ok, "the 64-bit A-fragment loads of each half-warp must hit 32 distinct banks"


def test_emulated_transposed_form_matches_conv_transpose2d():
    """ConvTranspose2d(8, 8, 3, stride=2, padding=1, output_padding=1) (reference net.py:89) == stride-1 conv with the
    flipped filter and pad 1 over the zero-stuffed input; written into channels 0..7 of a 16-channel buffer."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 6, 9, generator=g, dtype=torch.float64)
    wt = torch.randn(8, 8, 3, 3, generator=g).double()
    b = torch.randn(8, generator=g).double()
    want = F.conv_transpose2d(x, wt, b, stride=2, padding=1, output_padding=1).relu().permute(0, 2, 3, 1).numpy()
    want = F.conv_transpose2d(x, wt.float().double(), b, stride=2, padding=1, output_padding=1).relu().permute(0, 2, 3, 1).numpy()
    frag = ops.pack_conv_filter(wt.float(), 3, transposed=True)
    y = np.full((2, 12, 18, 16), np.nan)
    got = emulate_conv(x.permute(0, 2, 3, 1).numpy(), frag.numpy(), b.numpy(), 8, 3, 1, 1, 1, True, True, 4, ycs=16, yco=0, y=y)
    assert np.abs(got[..., :8] - want).max() <= 2e-6 * np.abs(want).max()
    assert np.isnan(got[..., 8:]).all(), "channels outside the slice must not be touched"


def test_pixel_stride_rule():
    for kc in (8, 16, 32, 64):
        for S in (1, 2):
            ps = pixel_stride(kc, S)
            assert ps >= kc and ps % 4 == 0 and (S * ps) % 32 in (8, 24)


def test_tf32_rounding_matches_cvt_rna():
    """The host-side TF32 rounding of the filter: nearest 10-bit mantissa, ties away from zero."""
    x = torch.tensor([1.0, 1.0 + 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, 1.0 + 2.0 ** -12, -(1.0 + 2.0 ** -11), 3.0e-5, -7.25, 0.0])
    r = ops._tf32_round(x)
    want = torch.tensor([1.0, 1.0 + 2.0 ** -10, 1.0 + 2.0 ** -10, 1.0, -(1.0 + 2.0 ** -10), 0.0, -7.25, 0.0])
    want[5] = r[5]
    assert torch.equal(r, want)
    assert (r.view(torch.int32) & 0x1FFF).eq(0).all()
    assert ((r - x).abs() <= x.abs() * 2.0 ** -11).all()
    g = torch.Generator().manual_seed(0)
    w = torch.randn(1000, generator=g)
    hi = ops._tf32_round(w)
    lo = ops._tf32_round(w - hi)
    assert ((hi + lo - w).abs() <= w.abs() * 2.0 ** -21).all()


def test_conv_entry_rejects_bad_arguments_without_gpu():
    lib = _native.lib()
    one = ctypes.c_void_p(64)
    ok_tail = (1, 8, 8, 8, 8, 3, 1, 1, 1, 0, 1, 0, 0, 0, 0, None)
    assert lib.pmb200_conv2d_nhwc(None, one, None, None, one, *ok_tail) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_conv2d_nhwc(one, one, None, None, one, 1, 8, 8, 65, 8, 3, 1, 1, 1, 0, 1, 0, 0, 0, 0, None) == -1  # Cin > 64
    assert lib.pmb200_conv2d_nhwc(one, one, None, None, one, 1, 8, 8, 8, 8, 3, 3, 1, 1, 0, 1, 0, 0, 0, 0, None) == -1   # stride 3
    assert lib.pmb200_conv2d_nhwc(one, one, None, None, one, 1, 8, 8, 8, 8, 3, 1, 1, 1, 0, 2, 0, 0, 0, 0, None) == -1   # precision 2
    assert lib.pmb200_conv2d_nhwc(one, one, None, None, one, 1, 8, 8, 8, 8, 3, 1, 1, 1, 0, 1, 0, 12, 8, 0, None) == -1  # slice outside
    assert lib.pmb200_conv2d_nhwc(one, one, None, one, one, 1, 7, 8, 8, 8, 1, 1, 0, 1, 0, 1, 0, 0, 0, 0, None) == -1  # add_up2x: odd Ho
    assert lib.pmb200_conv2d_filter_floats(64, 64, 3, 1) == 9 * 8 * 8 * 64
    assert lib.pmb200_conv2d_filter_floats(3, 18, 3, 3) == 9 * 1 * 3 * 128
    assert lib.pmb200_conv2d_filter_floats(0, 8, 3, 1) == -1
    assert lib.pmb200_conv2d_filter_floats(8, 8, 3, 2) == -1


def test_conv_wrapper_has_no_cpu_fallback():
    x = torch.zeros(1, 8, 4, 4)
    frag = ops.pack_conv_filter(torch.zeros(8, 8, 3, 3), 1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.conv2d_nhwc(x, frag, None, 8, 3, 1, 1, precision=1)


# ------------------------------------------------------------------------------------------------
# GPU: the kernel against cuDNN in full fp32
# ------------------------------------------------------------------------------------------------


@pytest.fixture()
def fp32_library():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _scaled_err(got, want):
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-6))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LAYERS))
def test_gpu_conv_matches_cudnn_fp32(name, fp32_library):
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    dev = "cuda:0"
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    # ragged map: neither dimension a multiple of the 16 x (4*MT) tile; two images
    N, H, W = 2, 37, 53
    x = torch.randn(N, cin, H, W, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    want = _ref_conv(x, w, b, S, pad, dil, relu)
    for prec, tol in ((3, 2e-5), (1, 3e-3)):
        frag = ops.pack_conv_filter(w, prec)
        for mt in (0, 1, 2, 4):
            got = ops.conv2d_nhwc(x, frag, b, cout, ks, S, pad, dil, relu=relu, precision=prec, rows_per_warp=mt)
            assert got.shape == want.shape
            err = _scaled_err(got, want)
            assert err <= tol, f"{name} precision {prec} rows_per_warp {mt}: scaled max err {err:.3e}"
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_gpu_conv_full_size_layers(fp32_library):
    """The three heaviest shapes at their BASELINE config-2 sizes (5 stacked views of 640x512)."""
    dev = "cuda:0"
    g = torch.Generator().manual_seed(11)
    for name, (H, W) in (("feature.conv1", (512, 640)), ("feature.conv5", (256, 320)), ("feature.conv9", (64, 80))):
        cin, cout, ks, S, pad, dil, relu = LAYERS[name]
        x = torch.randn(5, cin, H, W, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        want = _ref_conv(x, w, b, S, pad, dil, relu)
        got = ops.conv2d_nhwc(x, ops.pack_conv_filter(w, 3), b, cout, ks, S, pad, dil, relu=relu, precision=3)
        assert _scaled_err(got, want) <= 2e-5, name


TC5_LAYERS = sorted(n for n, (cin, cout, ks, S, pad, dil, relu) in LAYERS.items() if cin in (8, 16, 32, 64))


def test_tc5_filter_image_matches_the_address_swizzle():
    """ops.pack_conv_filter_tc5 against the element-by-element definition in include/patchmatch_b200.h: byte offset `off` of
    the dense [Npad][row bytes] tile moves to off ^ ((off >> 3) & mask), mask 0x70 / 0x30 / 0x10 for 128 / 64 / 32-byte rows
    (what TMA writes and wgmma reads for a K-major operand); hi + lo restores the weight to 2^-22."""
    torch.manual_seed(0)
    for (cout, cin, ks) in [(16, 8, 5), (18, 32, 3), (64, 64, 3), (8, 16, 3), (32, 16, 5), (64, 64, 1)]:
        w = torch.randn(cout, cin, ks, ks)
        got = ops.pack_conv_filter_tc5(w)
        npad, cblk = (cout + 15) // 16 * 16, min(cin, 32)
        kb, RB = cin // cblk, cblk * 4
        assert got.numel() == ks * ks * 2 * npad * cin
        hi = ops._tf32_round(w)
        lo = ops._tf32_round(w - hi)
        assert float((hi + lo - w).abs().max()) <= 2.0 ** -21 * float(w.abs().max())
        ref = torch.zeros(ks * ks, kb, 2, npad * RB // 4)
        mask = {128: 0x70, 64: 0x30, 32: 0x10}[RB]
        for t in range(ks * ks):
            ky, kx = divmod(t, ks)
            for si, ww in enumerate((hi, lo)):
                for k in range(kb):
                    blk = ww[:, k * cblk:(k + 1) * cblk, ky, kx]
                    for n in range(cout):
                        for c in range(cblk):
                            off = n * RB + c * 4
                            ref[t, k, si, (off ^ ((off >> 3) & mask)) // 4] = blk[n, c]
        assert torch.equal(got, ref.view(-1)), (cout, cin, ks)
    with pytest.raises(RuntimeError):
        ops.pack_conv_filter_tc5(torch.zeros(8, 3, 3, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("name", TC5_LAYERS)
def test_gpu_tc5_conv_matches_cudnn_fp32(name, fp32_library):
    """K-D5 (wgmma / TMA implicit GEMM, 3xTF32) against cuDNN in full fp32: every layer shape it can take, ragged
    map sizes (partial tiles on both axes, zero padding from the TMA's out-of-bounds fill), two images, strides 1 and 2,
    dilation up to 6, output channels that are not a multiple of 16."""
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    dev = "cuda:0"
    assert _native.lib().pmb200_conv2d_tc5_supported(cin, cout, ks, S) == 1
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 1)
    for (N, H, W) in ((2, 37, 53), (1, 16, 32), (3, 9, 70)):
        x = torch.randn(N, cin, H, W, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        want = _ref_conv(x, w, b, S, pad, dil, relu)
        got = ops.conv2d_tc5(x, ops.pack_conv_filter_tc5(w), b, cout, ks, S, pad, dil, relu=relu)
        torch.cuda.synchronize()
        assert got.shape == want.shape
        err = _scaled_err(got, want)
        assert err <= 2e-5, f"{name} {N}x{H}x{W}: scaled max err {err:.3e}"
        got_nb = ops.conv2d_tc5(x, ops.pack_conv_filter_tc5(w), None, cout, ks, S, pad, dil, relu=False)
        assert _scaled_err(got_nb, F.conv2d(x, w, None, S, pad, dil)) <= 2e-5


TC5H_LAYERS = sorted(n for n in TC5_LAYERS if LAYERS[n][3] == 1)


def test_tc5h_filter_image_layout():
    torch.manual_seed(1)
    w = torch.randn(18, 32, 3, 3)
    got = ops.pack_conv_filter_tc5h(w).view(9, 8, 2, 32, 4)
    hi = ops._tf32_round(w)
    lo = ops._tf32_round(w - hi)
    for (t, s_, c, n, e) in ((0, 0, 0, 0, 0), (4, 1, 7, 17, 3), (8, 0, 3, 5, 2)):
        ky, kx = divmod(t, 3)
        assert float(got[t, c, s_, n, e]) == float((hi, lo)[s_][n, 4 * c + e, ky, kx])
    assert float(got[:, :, :, 18:].abs().max()) == 0.0
    assert ops.pack_conv_filter_tc5h(w).numel() == ops.pack_conv_filter_tc5(w).numel()


@pytest.mark.gpu
@pytest.mark.parametrize("name", TC5H_LAYERS)
def test_gpu_tc5h_conv_matches_cudnn_fp32(name, fp32_library):
    """K-D5h (stride-1 halo-tile form: one 5-D TMA box per tile, filter taps as shifted no-swizzle descriptors) against cuDNN
    fp32 on every stride-1 layer shape, ragged sizes (partial 8 x 16 tiles, zero padding from the TMA fill), dilation up to 6."""
    cin, cout, ks, S, pad, dil, relu = LAYERS[name]
    dev = "cuda:0"
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 2)
    for (N, H, W) in ((2, 37, 53), (1, 16, 8), (3, 9, 70)):
        x = torch.randn(N, cin, H, W, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        want = _ref_conv(x, w, b, S, pad, dil, relu)
        got = ops.conv2d_tc5(x, ops.pack_conv_filter_tc5h(w), b, cout, ks, 1, pad, dil, relu=relu, halo=True)
        torch.cuda.synchronize()
        assert got.shape == want.shape
        err = _scaled_err(got, want)
        assert err <= 2e-5, f"{name} {N}x{H}x{W}: scaled max err {err:.3e}"


@pytest.mark.gpu
def test_gpu_tc5_conv_full_size_layers_and_channel_slice(fp32_library):
    dev = "cuda:0"
    g = torch.Generator().manual_seed(12)
    for name, (H, W) in (("feature.conv2", (512, 640)), ("feature.conv5", (256, 320)), ("feature.conv9", (64, 80)), ("stage3.eval_conv", (64, 80))):
        cin, cout, ks, S, pad, dil, relu = LAYERS[name]
        x = torch.randn(5, cin, H, W, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        w = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        want = _ref_conv(x, w, b, S, pad, dil, relu)
        got = ops.conv2d_tc5(x, ops.pack_conv_filter_tc5(w), b, cout, ks, S, pad, dil, relu=relu)
        assert _scaled_err(got, want) <= 2e-5, name
    # written into channels 8..15 of a wider channels-last tensor; the rest untouched
    cin, cout = 16, 8
    x = torch.randn(2, cin, 38, 54, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    w = (torch.randn(cout, cin, 3, 3, generator=g) / 12).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    both = torch.full((2, 16, 38, 54), float("nan"), device=dev).contiguous(memory_format=torch.channels_last)
    ops.conv2d_tc5(x, ops.pack_conv_filter_tc5(w), b, cout, 3, 1, 1, 1, relu=True, out=both, out_channel_offset=8)
    torch.cuda.synchronize()
    assert torch.isnan(both[:, :8]).all()
    assert _scaled_err(both[:, 8:], F.conv2d(x, w, b, padding=1).relu()) <= 2e-5


@pytest.mark.gpu
def test_gpu_transposed_conv_and_channel_slices(fp32_library):
    dev = "cuda:0"
    g = torch.Generator().manual_seed(5)
    low = torch.randn(2, 8, 19, 27, generator=g).to(dev)
    img = torch.randn(2, 3, 38, 54, generator=g).to(dev)
    wt = (torch.randn(8, 8, 3, 3, generator=g) / 8).to(dev)
    bt = torch.randn(8, generator=g).to(dev)
    w0 = (torch.randn(8, 3, 3, 3, generator=g) / 5).to(dev)
    b0 = torch.randn(8, generator=g).to(dev)
    want = torch.cat((F.conv_transpose2d(low, wt, bt, stride=2, padding=1, output_padding=1).relu(),
                      F.conv2d(img, w0, b0, padding=1).relu()), dim=1)
    both = torch.full((2, 16, 38, 54), float("nan"), device=dev).contiguous(memory_format=torch.channels_last)
    ops.conv2d_nhwc(low, ops.pack_conv_filter(wt, 3, transposed=True), bt, 8, 3, 1, 1, 1, relu=True, transposed2x=True,
                    out=both, out_channel_offset=0, precision=3)
    assert torch.isnan(both[:, 8:]).all(), "the other half of the buffer must be untouched"
    ops.conv2d_nhwc(img, ops.pack_conv_filter(w0, 3), b0, 8, 3, 1, 1, 1, relu=True, out=both, out_channel_offset=8, precision=3)
    assert _scaled_err(both, want) <= 2e-5


@pytest.mark.gpu
def test_gpu_net_native_convs_match_library_convs(fp32_library, golden_weights):
    """Whole network, eval mode: native convs (3xTF32) vs the folded cuDNN convs in fp32 -- same depth map."""
    from patchmatchnet_b200 import synthetic
    from patchmatchnet_b200.net import PatchmatchNet, load_reference_state

    dev = "cuda:0"
    net = PatchmatchNet(**synthetic.DEFAULT_NET_KWARGS)
    load_reference_state(net, golden_weights)
    net = net.eval().to(dev)
    inp = synthetic.make_inputs(1, 3, 128, 160, seed=3)
    args = lambda: ([i.to(dev) for i in inp["images"]], inp["intrinsics"].to(dev), inp["extrinsics"].to(dev),
                    inp["depth_min"].to(dev), inp["depth_max"].to(dev))
    outs = {}
    old = ops.NATIVE_CONVS
    try:
        for flag in (True, False):
            ops.NATIVE_CONVS = flag
            torch.manual_seed(0)
            with torch.no_grad():
                depth, conf, _ = net(*args())
            outs[flag] = (depth, conf)
    finally:
        ops.NATIVE_CONVS = old
    rel = float((outs[True][0] - outs[False][0]).abs().sum() / outs[False][0].abs().sum())
    assert rel <= 1e-4, rel


@pytest.mark.gpu
def test_gpu_conv_with_fused_upsample_add(fp32_library):
    """Lateral 1x1 conv + bias + bilinear x2 upsample of the coarser map in one launch (reference net.py:60-66)."""
    dev = "cuda:0"
    g = torch.Generator().manual_seed(9)
    for cin, cout, (h, w) in ((32, 32, (19, 27)), (16, 16, (32, 40)), (32, 16, (8, 8))):
        fine = torch.randn(2, cin, 2 * h, 2 * w, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        coarse = torch.randn(2, cout, h, w, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
        wt = (torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5).to(dev)
        b = torch.randn(cout, generator=g).to(dev)
        want = F.interpolate(coarse, scale_factor=2.0, mode="bilinear", align_corners=False) + F.conv2d(fine, wt, b)
        got = ops.conv2d_nhwc(fine, ops.pack_conv_filter(wt, 3), b, cout, 1, precision=3, add_up2x=coarse)
        assert _scaled_err(got, want) <= 2e-5
    with pytest.raises(RuntimeError, match="add_up2x"):
        ops.conv2d_nhwc(fine, ops.pack_conv_filter(wt, 3), b, cout, 1, precision=3, add_up2x=coarse[:, :, :-1])


def test_conv_stem_rejects_what_it_cannot_serve():
    w0, b0, w1, b1 = torch.zeros(8, 3, 3, 3), torch.zeros(8), torch.zeros(8, 8, 3, 3), torch.zeros(8)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.conv_stem(torch.zeros(1, 3, 8, 8), w0, b0, w1, b1)


def test_fused_refinement_wrappers_reject_cpu_tensors_and_device_weights():
    """ops.refine_low / ops.refine_full: no CPU fallback for the maps, and the weights must be HOST tensors (they travel in the
    kernel parameter block)."""
    from patchmatchnet_b200.net import Refinement

    hw = Refinement().eval().host_weights()
    assert [tuple(t.shape) for t in hw] == [(8, 1, 3, 3), (8,), (8, 8, 3, 3), (8,), (8, 8, 3, 3), (8,), (8, 3, 3, 3), (8,), (8, 16, 3, 3), (8,), (1, 8, 3, 3)]
    assert all(t.device.type == "cpu" and t.dtype == torch.float32 and t.is_contiguous() for t in hw)
    depth, lo, hi = torch.zeros(1, 1, 4, 4), torch.zeros(1), torch.ones(1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.refine_low(depth, lo, hi, *hw[:4])
    low = torch.zeros(1, 8, 4, 4).contiguous(memory_format=torch.channels_last)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        ops.refine_full(low, torch.zeros(1, 3, 8, 8), depth, lo, hi, *hw[4:])


def test_refinement_host_weights_fold_batchnorm_like_the_module():
    """Refinement.host_weights(): conv + eval-mode BatchNorm folded (transposed conv over its OUTPUT channel) reproduce the
    module's own layers on random inputs."""
    from tests.test_emulated_conv import _random_refinement

    m = _random_refinement(11)
    w1, b1, w2, b2, wd, bd, w0, b0, w3, b3, wr = m.host_weights()
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        x1 = torch.randn(1, 1, 6, 7, generator=g)
        assert torch.allclose(F.relu(F.conv2d(x1, w1, b1, padding=1)), m.conv1(x1), atol=1e-5)
        x8 = torch.randn(1, 8, 6, 7, generator=g)
        assert torch.allclose(F.relu(F.conv2d(x8, w2, b2, padding=1)), m.conv2(x8), atol=1e-5)
        up = F.relu(F.conv_transpose2d(x8, wd, bd, stride=2, padding=1, output_padding=1))
        assert torch.allclose(up, F.relu(m.bn(m.deconv(x8))), atol=1e-5)
        x3 = torch.randn(1, 3, 6, 7, generator=g)
        assert torch.allclose(F.relu(F.conv2d(x3, w0, b0, padding=1)), m.conv0(x3), atol=1e-5)
        x16 = torch.randn(1, 16, 6, 7, generator=g)
        assert torch.allclose(F.relu(F.conv2d(x16, w3, b3, padding=1)), m.conv3(x16), atol=1e-5)
        assert torch.equal(wr, m.res.weight)


@pytest.mark.gpu
def test_gpu_conv_stem_matches_cudnn_fp32(fp32_library):
    """K-S (fused conv0 -> conv1 of FeatureNet, exact fp32 FFMA with the weights in the constant bank) against the two cuDNN
    fp32 convolutions: ragged sizes and the bench's 5 x 640 x 512; strided-batch input (views of one buffer)."""
    dev = "cuda:0"
    g = torch.Generator().manual_seed(77)
    w0, b0 = torch.randn(8, 3, 3, 3, generator=g) / 27 ** 0.5, torch.randn(8, generator=g) * 0.5
    w1, b1 = torch.randn(8, 8, 3, 3, generator=g) / 72 ** 0.5, torch.randn(8, generator=g) * 0.5
    for (N, H, W) in ((2, 37, 53), (1, 16, 32), (3, 9, 70), (5, 512, 640)):
        x = torch.randn(N, 3, H, W, generator=g).to(dev)
        want = F.relu(F.conv2d(F.relu(F.conv2d(x, w0.to(dev), b0.to(dev), padding=1)), w1.to(dev), b1.to(dev), padding=1))
        got = ops.conv_stem(x, w0, b0, w1, b1)
        torch.cuda.synchronize()
        assert got.shape == want.shape and got.is_contiguous(memory_format=torch.channels_last)
        assert _scaled_err(got, want) <= 2e-6, (N, H, W)
    with pytest.raises(RuntimeError, match="HOST"):
        ops.conv_stem(x, w0.to(dev), b0, w1, b1)


@pytest.mark.gpu
def test_gpu_fused_refinement_matches_the_layerwise_path(fp32_library, monkeypatch):
    """K-R (two exact-fp32 launches) against the same module run layer by layer on cuDNN fp32 kernels, and against the
    conv-family path it replaces; bench size and a ragged one."""
    from patchmatchnet_b200 import net as pm_net
    from tests.test_emulated_conv import _random_refinement

    dev = "cuda:0"
    m = _random_refinement(3).to(dev)
    g = torch.Generator().manual_seed(5)
    for (N, h, w) in ((1, 256, 320), (2, 21, 37)):
        img = torch.rand(N, 3, 2 * h, 2 * w, generator=g).to(dev)
        dmin = torch.tensor([400.0, 425.0][:N], device=dev)
        dmax = torch.tensor([900.0, 935.0][:N], device=dev)
        depth = dmin.view(N, 1, 1, 1) + torch.rand(N, 1, h, w, generator=g).to(dev) * (dmax - dmin).view(N, 1, 1, 1)
        span = (dmax - dmin).view(N, 1, 1, 1)
        with torch.no_grad():
            got = m(img, depth, dmin, dmax)
            monkeypatch.setattr(ops, "REFINE_FUSED", False)
            family = m(img, depth, dmin, dmax)                 # conv-family launches + ATen tail
            monkeypatch.setattr(pm_net, "LIBRARY_FAST_PATH", False)
            want = m(img, depth, dmin, dmax)                   # the reference's own op sequence on cuDNN fp32
            monkeypatch.setattr(pm_net, "LIBRARY_FAST_PATH", True)
            monkeypatch.setattr(ops, "REFINE_FUSED", True)
        torch.cuda.synchronize()
        assert got.shape == want.shape == (N, 1, 2 * h, 2 * w)
        assert float(((got - want).abs() / span).max()) <= 5e-6, (N, h, w)
        assert float(((family - want).abs() / span).max()) <= 5e-5
