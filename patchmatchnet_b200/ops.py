"""Tensor-level wrappers over the C ABI (``include/patchmatch_b200.h``).

PyTorch is plumbing here: it owns the device buffers and the CUDA stream.  Each
wrapper checks dtype / device / layout, allocates the output with the caching
allocator, and enqueues ONE native kernel on the tensor's current stream via
ctypes -- capturable in a CUDA graph, no host synchronisation.  A CPU tensor is
an error (there is no fallback path).
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple, Union

import torch

from . import _native

Tensor = torch.Tensor


def _on_device(t: Tensor) -> bool:
    """The one place that decides whether a tensor may be handed to the native library.  (tests/emu_backend.py replaces
    this, `_device_guard` and `_stream` to run the wrappers against the CPU-emulated kernels; the product has no such path.)"""
    return t.is_cuda


def _device_guard(t: Tensor):
    """Context that makes `t`'s GPU current for the duration of a native call."""
    return torch.cuda.device(t.device)


def _require(t: Tensor, name: str, ndim: Optional[int] = None) -> Tensor:
    if not _on_device(t):
        raise RuntimeError(f"{name}: the H100 path needs a CUDA tensor (got {t.device}); there is no CPU fallback")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name}: expected float32, got {t.dtype}")
    if ndim is not None and t.dim() != ndim:
        raise RuntimeError(f"{name}: expected {ndim} dims, got shape {tuple(t.shape)}")
    return t if t.is_contiguous() else t.contiguous()


def _offsets_arg(off: Tensor, shape, name: str):
    """(tensor, channels_last flag) for a raw offset-conv output: planar NCHW memory or channels-last memory are both
    consumed in place; anything else is made NCHW-contiguous."""
    if not _on_device(off) or off.dtype != torch.float32:
        raise RuntimeError(f"{name}: offsets must be a CUDA float32 tensor (got {off.dtype} on {off.device}); there is no CPU fallback")
    if tuple(off.shape) != tuple(shape):
        raise RuntimeError(f"{name}: offsets must be {tuple(shape)}, got {tuple(off.shape)}")
    if off.is_contiguous():
        return off, 0
    if off.is_contiguous(memory_format=torch.channels_last):
        return off, 1
    return off.contiguous(), 0


def _stream(t: Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _rowmajor_4x4(m: Tensor, name: str) -> Tensor:
    """[B,4,4] with contiguous 4x4 blocks; the batch stride may be anything (torch.unbind views)."""
    if not _on_device(m) or m.dtype != torch.float32 or m.dim() != 3 or m.shape[1:] != (4, 4):
        raise RuntimeError(f"{name}: expected a CUDA float32 [B,4,4] tensor, got {m.dtype} {tuple(m.shape)} on {m.device}")
    if m.stride(1) != 4 or m.stride(2) != 1:
        m = m.contiguous()
    return m


def set_tuning(key: str, value: int = 0) -> None:
    """Measurement aid (tools/kbench.py, A/B tests): override a launch-configuration knob of the library for this process;
    `set_tuning("reset")` restores every default.  Keys: include/patchmatch_b200.h, pmb200_set_tuning.  Results never depend
    on these knobs, only launch shapes do."""
    _native.check(_native.lib().pmb200_set_tuning(key.encode(), int(value)), "set_tuning")


def relative_projection(ref_proj: Tensor, src_projs: Sequence[Tensor]) -> Tensor:
    """[V,B,12] rotation/translation of src_proj @ inv(ref_proj); reference module.py:148-150."""
    B = ref_proj.shape[0]
    V = len(src_projs)
    ref = _rowmajor_4x4(ref_proj, "ref_proj")
    mats = [_rowmajor_4x4(m, "src_proj") for m in src_projs]
    if any(m.shape[0] != B for m in mats):
        raise RuntimeError("relative_projection: batch size mismatch")
    if B > 1 and len({m.stride(0) for m in mats}) != 1:
        mats = [m.contiguous() for m in mats]
    out = torch.empty((V, B, 12), dtype=torch.float32, device=ref.device)
    arr, keep = _native.pointer_array([m.data_ptr() for m in mats])
    with _device_guard(ref):
        rc = _native.lib().pmb200_relative_projection(
            ref.data_ptr(), ref.stride(0), arr, mats[0].stride(0), V, B, out.data_ptr(), _stream(ref)
        )
    _native.check(rc, "relative_projection")
    return out


def _is_packed_nhwc(maps: Sequence[Tensor]) -> bool:
    """True when the maps are channels-last views laid out back to back in ONE storage (e.g. slices of one
    stacked channels-last FeatureNet output), so that packing would be a no-op."""
    first = maps[0]
    B, C, H, W = first.shape
    want = (H * W * C, 1, W * C, C)
    store = first.untyped_storage().data_ptr()
    if first.dtype != torch.float32 or first.data_ptr() % 32 != 0:  # the kernels read a lane's 8 channels with one 256-bit load
        return False
    for i, m in enumerate(maps):
        if (m.shape != first.shape or m.stride() != want or m.untyped_storage().data_ptr() != store
                or m.storage_offset() != first.storage_offset() + i * first.numel()):
            return False
    return True


def pack_nhwc(maps: Sequence[Tensor]) -> Tensor:
    """[n,B,H,W,C] channels-last copy of n NCHW maps of equal shape (one launch)."""
    first = maps[0]
    B, C, H, W = first.shape
    if _is_packed_nhwc(maps):
        return torch.as_strided(first, (len(maps), B, H, W, C), (B * H * W * C, H * W * C, W * C, C, 1))
    srcs = [_require(m, "feature map", 4) for m in maps]
    for m in srcs:
        if m.shape != first.shape:
            raise RuntimeError("pack_nhwc: maps must share one shape")
    out = torch.empty((len(srcs), B, H, W, C), dtype=torch.float32, device=first.device)
    arr, keep = _native.pointer_array([m.data_ptr() for m in srcs])
    with _device_guard(first):
        rc = _native.lib().pmb200_pack_nhwc(arr, len(srcs), B, C, H, W, out.data_ptr(), _stream(first))
    _native.check(rc, "pack_nhwc")
    return out


class ViewPack:
    """A ragged channels-last source pack: source view v, batch item b, is [heights[v], widths[v], C] starting at float
    offsets[v] + b * heights[v] * widths[v] * C of `data` (flat float32).  What the *_views entry points take
    (pmb200_view_extent)."""

    # every view starts on a 256-byte boundary: the gathers need 16 bytes, whole 128-byte lines keep a texel in one line
    ALIGN_FLOATS = 64

    def __init__(self, data: Tensor, offsets: Sequence[int], heights: Sequence[int], widths: Sequence[int], B: int, C: int) -> None:
        self.data, self.B, self.C = data, int(B), int(C)
        self.offsets, self.heights, self.widths = [int(o) for o in offsets], [int(h) for h in heights], [int(w) for w in widths]
        ext = (_native.ViewExtent * len(self.offsets))()
        for v, (o, h, w) in enumerate(zip(self.offsets, self.heights, self.widths)):
            ext[v].offset, ext[v].height, ext[v].width = o, h, w
        self.extents = ext  # host array, read by the entry points at call time

    def __len__(self) -> int:
        return len(self.offsets)

    @property
    def device(self):
        return self.data.device

    @staticmethod
    def layout(shapes: Sequence[Tuple[int, int]], B: int, C: int) -> Tuple[List[int], int]:
        """(float offset of every view, total floats) of a pack of views of the given (H, W)."""
        offsets, n = [], 0
        for h, w in shapes:
            offsets.append(n)
            n += -(-(B * h * w * C) // ViewPack.ALIGN_FLOATS) * ViewPack.ALIGN_FLOATS
        return offsets, n

    @classmethod
    def from_shapes(cls, data: Tensor, shapes: Sequence[Tuple[int, int]], B: int, C: int) -> "ViewPack":
        """The pack of views of the given (H, W) over `data`, laid out by `layout` (what pack_nhwc_views builds)."""
        offsets, _ = cls.layout(shapes, B, C)
        return cls(data, offsets, [h for h, _ in shapes], [w for _, w in shapes], B, C)

    def view(self, v: int) -> Tensor:
        """[B,H_v,W_v,C] view of source v (no copy)."""
        h, w = self.heights[v], self.widths[v]
        n = self.B * h * w * self.C
        return self.data[self.offsets[v]:self.offsets[v] + n].view(self.B, h, w, self.C)


def pack_nhwc_views(maps: Sequence[Tensor]) -> ViewPack:
    """Ragged channels-last pack of n NCHW maps [B,C,H_v,W_v] that share B and C but not their size: one pmb200_pack_nhwc
    launch per map into its slice of one buffer.  Views start on ViewPack.ALIGN_FLOATS-float boundaries."""
    srcs = [_require(m, "feature map", 4) for m in maps]
    B, C = srcs[0].shape[:2]
    if any(m.shape[:2] != (B, C) for m in srcs):
        raise RuntimeError("pack_nhwc_views: maps must share batch size and channels")
    shapes = [tuple(m.shape[2:]) for m in srcs]
    offsets, total = ViewPack.layout(shapes, B, C)
    data = torch.empty(total, dtype=torch.float32, device=srcs[0].device)
    pack = ViewPack.from_shapes(data, shapes, B, C)
    with _device_guard(srcs[0]):
        for v, m in enumerate(srcs):
            arr, keep = _native.pointer_array([m.data_ptr()])
            rc = _native.lib().pmb200_pack_nhwc(arr, 1, B, C, shapes[v][0], shapes[v][1], data.data_ptr() + 4 * offsets[v], _stream(m))
            _native.check(rc, "pack_nhwc_views")
    return pack


def photometric_confidence(prob: Tensor, out_h: int, out_w: int) -> Tensor:
    """[B,D,h,w] probabilities -> [B,out_h,out_w] confidence (reference net.py:289-299)."""
    pr = _require(prob, "prob", 4)
    B, D, h, w = pr.shape
    out = torch.empty((B, out_h, out_w), dtype=torch.float32, device=pr.device)
    with _device_guard(pr):
        rc = _native.lib().pmb200_photometric_confidence(pr.data_ptr(), out.data_ptr(), B, D, h, w, out_h, out_w, _stream(pr))
    _native.check(rc, "photometric_confidence")
    return out


def upsample2x_add(x: Tensor, y: Tensor, bias: Optional[Tensor] = None) -> Tensor:
    """bilinear x2 upsample of `x` plus `y` (plus a per-channel `bias`), channels-last 4-D CUDA tensors (logical NCHW)."""
    N, C, h, w = x.shape
    if y.shape != (N, C, 2 * h, 2 * w):
        raise RuntimeError("upsample2x_add: y must be [N,C,2h,2w]")
    for t, nm in ((x, "x"), (y, "y")):
        if not _on_device(t) or t.dtype != torch.float32:
            raise RuntimeError(f"upsample2x_add: {nm} must be a CUDA float32 tensor (no CPU fallback)")
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    if not y.is_contiguous(memory_format=torch.channels_last):
        y = y.contiguous(memory_format=torch.channels_last)
    b_ptr = None
    if bias is not None:
        bias = _require(bias, "bias", 1)
        if bias.numel() != C:
            raise RuntimeError("upsample2x_add: bias must have C elements")
        b_ptr = bias.data_ptr()
    out = torch.empty_like(y, memory_format=torch.channels_last)
    with _device_guard(x):
        rc = _native.lib().pmb200_upsample2x_add_nhwc(x.data_ptr(), y.data_ptr(), b_ptr, out.data_ptr(), N, h, w, C, _stream(x))
    _native.check(rc, "upsample2x_add_nhwc")
    return out


# The small learned convs (offset convs of the hot path, FeatureNet, Refinement) run through csrc/pm_conv.cu in eval
# mode.  False (or PMB200_NATIVE_CONVS=0) hands them back to cuDNN -- kept only for A/B measurements.
NATIVE_CONVS = os.environ.get("PMB200_NATIVE_CONVS", "1") != "0"
NATIVE_CONVS_ALL = os.environ.get("PMB200_NATIVE_CONVS", "1") == "all"  # A/B aid: native even where the library is faster


def conv_prefers_native(cin: int, cout: int, ks: int) -> bool:
    """Which implementation runs a small conv in eval mode (per-layer timings: tools/convbench.py).  The native
    channels-last kernel takes the memory-bound layers -- every 1x1 conv and every layer with at most 3200 multiply-adds
    per output pixel (full-resolution 3->8 / 8->8 / 8->16 convs, the refinement head, the stage-1 offset conv) -- while in
    the TF32 mode the FLOP-heavy 16..64-channel 3x3 / 5x5 layers stay with cuDNN's implicit-GEMM kernels."""
    if not NATIVE_CONVS:
        return False
    # fp32-accurate mode (cudnn.allow_tf32 off): the library's fp32 kernels for the FLOP-bound layers do not use the tensor
    # cores at all, the native 3xTF32 kernels do -> every conv native.  The parity configuration and the bench default are
    # this mode (the depth maps of the TF32 mode are outside north_star's 1e-3: tests/test_gpu_bench_mode.py).
    return NATIVE_CONVS_ALL or conv_precision() == 3 or ks == 1 or cin * cout * ks * ks <= 3200


def _round_kcin(cin: int) -> int:
    return 8 if cin <= 8 else (16 if cin <= 16 else (32 if cin <= 32 else 64))


def _round_nt(cout: int) -> int:
    nt = (cout + 7) // 8
    return nt if nt <= 4 else 8


def _tf32_round(x: Tensor) -> Tensor:
    """fp32 -> nearest TF32 value (10-bit mantissa), ties away from zero -- the arithmetic of PTX cvt.rna.tf32.f32 for
    finite inputs: add half an ulp to the magnitude bits, clear the 13 low bits."""
    bits = x.contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def pack_conv_filter(weight: Tensor, precision: int, transposed: bool = False) -> Tensor:
    """Conv filter [Cout,Cin,KS,KS] -> the tensor-core fragment order `pmb200_conv2d_nhwc` reads for `precision`
    (include/patchmatch_b200.h): [tap][k-slice][n-tile][lane][2 or 4] with lane = 4*g + t holding the weights of
    output channel nt*8+g for the adjacent input channels ks*8+2t, ks*8+2t+1 of that tap (the MMA's k slots t, t+4),
    zero padded.  precision 1: values rounded to TF32; precision 3: (b0_hi, b1_hi, b0_lo, b1_lo) with
    hi = tf32(w), lo = tf32(w - hi).  `transposed`: `weight` is a ConvTranspose2d filter [Cin,Cout,KS,KS]; the
    equivalent direct filter is its spatial flip with the channel axes swapped.  Pure layout/rounding work on the
    weight's own device (host logic, CPU-testable)."""
    if weight.dim() != 4 or weight.shape[2] != weight.shape[3]:
        raise RuntimeError(f"pack_conv_filter: expected [Cout,Cin,KS,KS], got {tuple(weight.shape)}")
    if precision not in (1, 3):
        raise RuntimeError("pack_conv_filter: precision must be 1 (TF32) or 3 (3xTF32)")
    w = weight.detach().float()
    if transposed:
        w = w.flip(2, 3).permute(1, 0, 2, 3)
    cout, cin, ks, _ = w.shape
    if not (1 <= cin <= 64 and 1 <= cout <= 64):
        raise RuntimeError("pack_conv_filter: 1 <= Cin, Cout <= 64")
    kc, nt = _round_kcin(cin), _round_nt(cout)
    wp = torch.zeros((ks * ks, kc, nt * 8), dtype=torch.float32, device=w.device)
    wp[:, :cin, :cout] = w.permute(2, 3, 1, 0).reshape(ks * ks, cin, cout)
    # channel = ks8*8 + 2*t + half ; n = j*8 + g  ->  [tap][ks8][j][g][t][half]
    frag = wp.view(ks * ks, kc // 8, 4, 2, nt, 8).permute(0, 1, 4, 5, 2, 3).contiguous()
    hi = _tf32_round(frag)
    if precision == 1:
        return hi.view(-1)
    lo = _tf32_round(frag - hi)
    return torch.cat((hi, lo), dim=-1).contiguous().view(-1)


# K-D5 (csrc/pm_conv5.cu): wgmma / TMA implicit-GEMM convolution, fp32-accurate (3xTF32).  Used in the
# fp32-accurate mode for the layers it serves when TC5_CONVS is on (PMB200_TC5=0 hands them back to the mma.sync kernel).
TC5_CONVS = os.environ.get("PMB200_TC5", "1") != "0"


# (Cin, Cout, KS, stride) of the layers a wgmma form serves instead of the mma.sync kernel's 3xTF32 mode (cold time per launch
# at the 640x512 sizes: tools/convbench.py).  Per-tap form K-D5 (the only one for stride 2): the 16->32 and 32->64 5x5 stride-2
# layers; not conv2 (Cin = 8: one K slice per tap, the instruction count is the cost).  PMB200_TC5=all takes every supported
# layer (A/B measurements), PMB200_TC5=0 none.
TC5_LAYERS = {(16, 32, 5, 2), (32, 64, 5, 2)}
TC5_ALL = os.environ.get("PMB200_TC5", "1") == "all"
# Stride-1 layers served by the halo-tile form K-D5h (one TMA box + one split per output tile, taps as shifted descriptors,
# [w_hi | w_lo] as one operand): FeatureNet conv3/4, conv6/7, conv9/10, output2/3 and the offset convs of every stage.  Not
# where Cin = 8 (conv1: one K slice per tap, the instruction count is the cost) nor Refinement.
# PMB200_TC5H=all: every stride-1 layer the kernel takes (A/B measurements); =0: none.
TC5H_LAYERS = {(16, 16, 3, 1), (32, 32, 3, 1), (64, 64, 3, 1), (64, 32, 1, 1), (64, 16, 1, 1),
               (64, 32, 3, 1), (64, 18, 3, 1), (32, 16, 3, 1), (32, 18, 3, 1), (16, 18, 3, 1)}
TC5H_ALL = os.environ.get("PMB200_TC5H", "1") == "all"
TC5H_OFF = os.environ.get("PMB200_TC5H", "1") == "0"


def conv_tc5_mode(cin: int, cout: int, ks: int, stride: int = 1, transposed: bool = False, fused_add: bool = False) -> str:
    """"" (mma.sync kernel), "halo" (K-D5h) or "tap" (K-D5): which wgmma form, if any, runs this conv.  Only in the
    fp32-accurate mode (the arithmetic of both IS the 3xTF32 split), never with a fused transposed / upsample-add epilogue, and
    only for layers on the measured lists above."""
    if not (NATIVE_CONVS and TC5_CONVS) or transposed or fused_add or conv_precision() != 3:
        return ""
    if not _native.lib().pmb200_conv2d_tc5_supported(cin, cout, ks, stride):
        return ""
    key = (cin, cout, ks, stride)
    if stride == 1 and not TC5H_OFF and (TC5H_ALL or key in TC5H_LAYERS):
        return "halo"
    if TC5_ALL or key in TC5_LAYERS:
        return "tap"
    return ""


def conv_uses_tc5(cin: int, cout: int, ks: int, stride: int = 1, transposed: bool = False, fused_add: bool = False) -> bool:
    return conv_tc5_mode(cin, cout, ks, stride, transposed, fused_add) != ""


def pack_conv_filter_tc5_for(weight: Tensor, mode: str) -> Tensor:
    return pack_conv_filter_tc5h(weight) if mode == "halo" else pack_conv_filter_tc5(weight)


def pack_conv_filter_tc5(weight: Tensor) -> Tensor:
    """Conv filter [Cout,Cin,KS,KS] -> the shared-memory image `pmb200_conv2d_tc5` copies per tap (include/patchmatch_b200.h):
    [tap][Cin/32 blocks][2 Npad rows][min(Cin,32) channels], rows 0..Npad-1 = w_hi (TF32-rounded weight), Npad..2Npad-1 = w_lo
    (TF32-rounded remainder) -- ONE K-major wgmma operand of N = 2 Npad whose first Npad rows double as the N = Npad operand --
    in the swizzle of the tensor core for its row size.  Pure layout / rounding work on the weight's device (CPU-testable)."""
    if weight.dim() != 4 or weight.shape[2] != weight.shape[3]:
        raise RuntimeError(f"pack_conv_filter_tc5: expected [Cout,Cin,KS,KS], got {tuple(weight.shape)}")
    w = weight.detach().float()
    cout, cin, ks, _ = w.shape
    if cin not in (8, 16, 32, 64) or not (1 <= cout <= 64):
        raise RuntimeError("pack_conv_filter_tc5: Cin in {8,16,32,64}, 1 <= Cout <= 64")
    npad = (cout + 15) // 16 * 16
    cblk = min(cin, 32)
    kb = cin // cblk
    hi = _tf32_round(w)
    lo = _tf32_round(w - hi)
    both = torch.stack((hi, lo))  # [2, Cout, Cin, KS, KS]
    t = torch.zeros((ks * ks, kb, 2, npad, cblk), dtype=torch.float32, device=w.device)
    t[:, :, :, :cout] = both.permute(3, 4, 0, 1, 2).reshape(ks * ks, 2, cout, kb, cblk).permute(0, 3, 1, 2, 4)
    # swizzle: 16-byte chunk j of row r moves to chunk j ^ f(r); Npad is a multiple of 8, so f(Npad + r) = f(r)
    chunks = cblk // 4
    rows = torch.arange(npad, device=w.device)
    f = {8: rows % 8, 4: (rows // 2) % 4, 2: (rows // 4) % 2}[chunks]
    j = torch.arange(chunks, device=w.device)
    src = (j.view(1, chunks) ^ f.view(npad, 1))  # physical chunk p of row r holds logical chunk p ^ f(r)
    t = t.view(ks * ks, kb, 2, npad, chunks, 4)
    idx = src.view(1, 1, 1, npad, chunks, 1).expand(ks * ks, kb, 2, npad, chunks, 4)
    return torch.gather(t, 4, idx).contiguous().view(-1)


def pack_conv_filter_tc5h(weight: Tensor) -> Tensor:
    """Conv filter [Cout,Cin,KS,KS] -> the image `pmb200_conv2d_tc5h` streams per tap: [tap][Cin/4 chunks][2 Npad rows][4 floats],
    rows 0..Npad-1 = w_hi, Npad..2Npad-1 = w_lo: ONE wgmma operand of N = 2 Npad (a_hi x [w_hi | w_lo] is a single MMA), whose
    first Npad rows double as the N = Npad operand of a_lo x w_hi.  No swizzle: 8 rows of one chunk are one core matrix."""
    if weight.dim() != 4 or weight.shape[2] != weight.shape[3]:
        raise RuntimeError(f"pack_conv_filter_tc5h: expected [Cout,Cin,KS,KS], got {tuple(weight.shape)}")
    w = weight.detach().float()
    cout, cin, ks, _ = w.shape
    if cin not in (8, 16, 32, 64) or not (1 <= cout <= 64):
        raise RuntimeError("pack_conv_filter_tc5h: Cin in {8,16,32,64}, 1 <= Cout <= 64")
    npad = (cout + 15) // 16 * 16
    hi = _tf32_round(w)
    lo = _tf32_round(w - hi)
    both = torch.stack((hi, lo))  # [2, Cout, Cin, KS, KS]
    t = torch.zeros((ks * ks, cin // 4, 2, npad, 4), dtype=torch.float32, device=w.device)
    t[:, :, :, :cout] = both.permute(3, 4, 0, 1, 2).reshape(ks * ks, 2, cout, cin // 4, 4).permute(0, 3, 1, 2, 4)
    return t.contiguous().view(-1)


# K-S (csrc/pm_stem.cu): FeatureNet's conv0 -> conv1 as one exact-fp32 launch; PMB200_STEM=0 keeps the two K-D launches.
STEM_FUSED = os.environ.get("PMB200_STEM", "1") != "0"


def conv_stem(x: Tensor, w0: Tensor, b0: Tensor, w1: Tensor, b1: Tensor) -> Tensor:
    """relu(conv1(relu(conv0(x)))) of FeatureNet (3 -> 8 -> 8, 3x3, pad 1; reference models/net.py:18-19, :44) in one launch.
    `x` [N,3,H,W] contiguous NCHW on the device; the BatchNorm-folded weights `w0` [8,3,3,3], `b0` [8], `w1` [8,8,3,3], `b1` [8]
    are HOST float32 tensors (they travel in the kernel's parameter block).  Returns [N,8,H,W] in channels-last memory."""
    if not _on_device(x) or x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
        raise RuntimeError(f"conv_stem: x must be a CUDA float32 [N,3,H,W] tensor (got {x.dtype} {tuple(x.shape)} on {x.device}); no CPU fallback")
    if not x.is_contiguous():
        x = x.contiguous()
    for name, t, shape in (("w0", w0, (8, 3, 3, 3)), ("b0", b0, (8,)), ("w1", w1, (8, 8, 3, 3)), ("b1", b1, (8,))):
        if t.device.type != "cpu" or t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous():
            raise RuntimeError(f"conv_stem: {name} must be a contiguous float32 HOST tensor of shape {shape}")
    N, _, H, W = x.shape
    y = torch.empty((N, 8, H, W), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
    with _device_guard(x):
        rc = _native.lib().pmb200_conv_stem(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), y.data_ptr(), N, H, W,
                                            _stream(x))
    _native.check(rc, "conv_stem")
    return y


# K-R (csrc/pm_refine.cu + the one-plane form of csrc/pm_stem.cu): Refinement as two exact-fp32 launches; PMB200_REFINE=0 keeps
# the six conv-family launches and the ATen tail.
REFINE_FUSED = os.environ.get("PMB200_REFINE", "1") != "0"


def _host_weights(name: str, pairs) -> None:
    for nm, t, shape in pairs:
        if t.device.type != "cpu" or t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous():
            raise RuntimeError(f"{name}: {nm} must be a contiguous float32 HOST tensor of shape {shape}")


def refine_low(depth_half: Tensor, depth_min: Tensor, depth_max: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor) -> Tensor:
    """relu(conv2(relu(conv1((depth - lo) / span)))) of Refinement at half resolution (reference models/net.py:104-110), one launch.
    depth_half [N,1,h,w], depth_min / depth_max [N] on the device; BatchNorm-folded HOST weights.  -> [N,8,h,w], channels-last."""
    if not _on_device(depth_half) or depth_half.dtype != torch.float32 or depth_half.dim() != 4 or depth_half.shape[1] != 1:
        raise RuntimeError(f"refine_low: depth_half must be a CUDA float32 [N,1,h,w] tensor (got {depth_half.dtype} {tuple(depth_half.shape)} on {depth_half.device}); no CPU fallback")
    _host_weights("refine_low", (("w1", w1, (8, 1, 3, 3)), ("b1", b1, (8,)), ("w2", w2, (8, 8, 3, 3)), ("b2", b2, (8,))))
    N, _, h, w = depth_half.shape
    dh = depth_half if depth_half.is_contiguous() else depth_half.contiguous()
    lo, hi = _require(depth_min.reshape(-1), "depth_min", 1), _require(depth_max.reshape(-1), "depth_max", 1)
    if lo.numel() != N or hi.numel() != N:
        raise RuntimeError("refine_low: depth_min / depth_max must have one value per image")
    y = torch.empty((N, 8, h, w), dtype=torch.float32, device=dh.device, memory_format=torch.channels_last)
    with _device_guard(dh):
        rc = _native.lib().pmb200_refine_low(dh.data_ptr(), lo.data_ptr(), hi.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr(),
                                             y.data_ptr(), N, h, w, _stream(dh))
    _native.check(rc, "refine_low")
    return y


def refine_full(low: Tensor, img: Tensor, depth_half: Tensor, depth_min: Tensor, depth_max: Tensor, wd: Tensor, bd: Tensor, w0: Tensor, b0: Tensor,
                w3: Tensor, b3: Tensor, wr: Tensor) -> Tensor:
    """The full-resolution half of Refinement (reference models/net.py:103, :112-120) in one launch: transposed conv of `low`,
    conv0 of the image, conv3 over their concatenation, the residual conv, `(nearest_up2x(d) + res) * span + lo`.
    low [N,8,h,w] channels-last (refine_low), img [N,3,2h,2w] NCHW, depth_half [N,1,h,w]; HOST weights.  -> depth [N,1,2h,2w]."""
    if not _on_device(low) or low.dtype != torch.float32 or low.dim() != 4 or low.shape[1] != 8 or not low.is_contiguous(memory_format=torch.channels_last):
        raise RuntimeError("refine_full: low must be a channels-last CUDA float32 [N,8,h,w] tensor; no CPU fallback")
    N, _, h, w = low.shape
    if not _on_device(img) or img.dtype != torch.float32 or tuple(img.shape) != (N, 3, 2 * h, 2 * w):
        raise RuntimeError(f"refine_full: img must be a CUDA float32 [{N},3,{2 * h},{2 * w}] tensor, got {tuple(img.shape)}")
    if tuple(depth_half.shape) != (N, 1, h, w) or depth_half.dtype != torch.float32 or not _on_device(depth_half):
        raise RuntimeError(f"refine_full: depth_half must be a CUDA float32 [{N},1,{h},{w}] tensor")
    _host_weights("refine_full", (("wd", wd, (8, 8, 3, 3)), ("bd", bd, (8,)), ("w0", w0, (8, 3, 3, 3)), ("b0", b0, (8,)),
                                  ("w3", w3, (8, 16, 3, 3)), ("b3", b3, (8,)), ("wr", wr, (1, 8, 3, 3))))
    img = img if img.is_contiguous() else img.contiguous()
    dh = depth_half if depth_half.is_contiguous() else depth_half.contiguous()
    lo, hi = _require(depth_min.reshape(-1), "depth_min", 1), _require(depth_max.reshape(-1), "depth_max", 1)
    out = torch.empty((N, 1, 2 * h, 2 * w), dtype=torch.float32, device=low.device)
    with _device_guard(low):
        rc = _native.lib().pmb200_refine_full(low.data_ptr(), img.data_ptr(), dh.data_ptr(), lo.data_ptr(), hi.data_ptr(), wd.data_ptr(), bd.data_ptr(),
                                              w0.data_ptr(), b0.data_ptr(), w3.data_ptr(), b3.data_ptr(), wr.data_ptr(), out.data_ptr(), N, 2 * h, 2 * w,
                                              _stream(low))
    _native.check(rc, "refine_full")
    return out


def conv2d_tc5(x: Tensor, filter_tc5: Tensor, bias: Optional[Tensor], cout: int, ks: int, stride: int = 1, pad: int = 0, dil: int = 1,
               relu: bool = False, out: Optional[Tensor] = None, out_channel_offset: int = 0, halo: bool = False) -> Tensor:
    """Channels-last convolution on the 5th-generation tensor cores (csrc/pm_conv5.cu), fp32-accurate.  Same calling
    convention as conv2d_nhwc; `filter_tc5` comes from pack_conv_filter_tc5, or from pack_conv_filter_tc5h with `halo=True`
    (stride 1 only: the halo-tile form K-D5h)."""
    if halo and stride != 1:
        raise RuntimeError("conv2d_tc5: the halo-tile form serves stride 1")
    if not _on_device(x) or x.dtype != torch.float32 or x.dim() != 4:
        raise RuntimeError(f"conv2d_tc5: x must be a 4-D CUDA float32 tensor (got {x.dtype} {tuple(x.shape)} on {x.device}); no CPU fallback")
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    N, cin, H, W = x.shape
    want = _native.lib().pmb200_conv2d_tc5_filter_floats(cin, cout, ks)
    if want <= 0 or filter_tc5.numel() != want or filter_tc5.dtype != torch.float32 or filter_tc5.device != x.device:
        raise RuntimeError(f"conv2d_tc5: filter must be {want} float32 values on {x.device} (pack_conv_filter_tc5)")
    Ho = (H + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    Wo = (W + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    if out is None:
        out = torch.empty((N, cout, Ho, Wo), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
        ycs, yco = cout, 0
    else:
        if (out.dim() != 4 or out.shape[0] != N or out.shape[2:] != (Ho, Wo) or out.dtype != torch.float32 or out.device != x.device
                or not out.is_contiguous(memory_format=torch.channels_last)):
            raise RuntimeError("conv2d_tc5: `out` must be a channels-last CUDA float32 [N,C,Ho,Wo] tensor")
        ycs, yco = out.shape[1], out_channel_offset
    b_ptr = None
    if bias is not None:
        bias = _require(bias, "bias", 1)
        if bias.numel() != cout:
            raise RuntimeError("conv2d_tc5: bias must have Cout elements")
        b_ptr = bias.data_ptr()
    with _device_guard(x):
        if halo:
            rc = _native.lib().pmb200_conv2d_tc5h(x.data_ptr(), filter_tc5.data_ptr(), b_ptr, out.data_ptr(), N, H, W, cin, cout, ks, pad,
                                                  dil, 1 if relu else 0, ycs, yco, _stream(x))
        else:
            rc = _native.lib().pmb200_conv2d_tc5(x.data_ptr(), filter_tc5.data_ptr(), b_ptr, out.data_ptr(), N, H, W, cin, cout, ks, stride,
                                                 pad, dil, 1 if relu else 0, ycs, yco, _stream(x))
    _native.check(rc, "conv2d_tc5h" if halo else "conv2d_tc5")
    return out


def conv_precision() -> int:
    """1 (TF32 operands) when the library would use TF32 for convolutions (torch.backends.cudnn.allow_tf32, torch's
    default), else 3 (3xTF32, fp32-accurate): the native convs honour the same switch as the cuDNN ones they replace."""
    return 1 if torch.backends.cudnn.allow_tf32 else 3


def conv2d_nhwc(x: Tensor, filter_frag: Tensor, bias: Optional[Tensor], cout: int, ks: int, stride: int = 1, pad: int = 0,
                dil: int = 1, relu: bool = False, transposed2x: bool = False, out: Optional[Tensor] = None,
                out_channel_offset: int = 0, precision: Optional[int] = None, rows_per_warp: int = 0,
                add_up2x: Optional[Tensor] = None) -> Tensor:
    """Channels-last convolution on the tensor cores (csrc/pm_conv.cu).  `x` is a logical-NCHW CUDA tensor in
    channels-last memory (made so if not); returns a logical-NCHW channels-last tensor [N,cout,Ho,Wo], or writes the
    channels out_channel_offset..+cout of `out` (a wider channels-last tensor: concat fusion) and returns `out`.
    `add_up2x`: a coarser channels-last map [N,cout,Ho/2,Wo/2] whose bilinear x2 upsample is added in the epilogue."""
    if not _on_device(x) or x.dtype != torch.float32 or x.dim() != 4:
        raise RuntimeError(f"conv2d_nhwc: x must be a 4-D CUDA float32 tensor (got {x.dtype} {tuple(x.shape)} on {x.device}); no CPU fallback")
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    N, cin, H, W = x.shape
    prec = conv_precision() if precision is None else precision
    up_ptr = None
    if add_up2x is not None:
        if (not _on_device(add_up2x) or add_up2x.dtype != torch.float32 or add_up2x.dim() != 4
                or not add_up2x.is_contiguous(memory_format=torch.channels_last)):
            raise RuntimeError("conv2d_nhwc: add_up2x must be a channels-last CUDA float32 tensor")
        up_ptr = add_up2x.data_ptr()
    want = _native.lib().pmb200_conv2d_filter_floats(cin, cout, ks, prec)
    if want <= 0 or filter_frag.numel() != want or filter_frag.dtype != torch.float32 or filter_frag.device != x.device:
        raise RuntimeError(f"conv2d_nhwc: filter must be {want} float32 values on {x.device} in fragment order for precision {prec} "
                           "(pack_conv_filter)")
    Hv, Wv = (2 * H, 2 * W) if transposed2x else (H, W)
    Ho = (Hv + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    Wo = (Wv + 2 * pad - dil * (ks - 1) - 1) // stride + 1
    if add_up2x is not None and tuple(add_up2x.shape) != (N, cout, Ho // 2, Wo // 2):
        raise RuntimeError(f"conv2d_nhwc: add_up2x must be [N,cout,Ho/2,Wo/2] = {(N, cout, Ho // 2, Wo // 2)}, got {tuple(add_up2x.shape)}")
    if out is None:
        out = torch.empty((N, cout, Ho, Wo), dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
        ycs, yco = cout, 0
    else:
        if (out.dim() != 4 or out.shape[0] != N or out.shape[2:] != (Ho, Wo) or out.dtype != torch.float32 or out.device != x.device
                or not out.is_contiguous(memory_format=torch.channels_last)):
            raise RuntimeError("conv2d_nhwc: `out` must be a channels-last CUDA float32 [N,C,Ho,Wo] tensor")
        ycs, yco = out.shape[1], out_channel_offset
    b_ptr = None
    if bias is not None:
        bias = _require(bias, "bias", 1)
        if bias.numel() != cout:
            raise RuntimeError("conv2d_nhwc: bias must have Cout elements")
        b_ptr = bias.data_ptr()
    with _device_guard(x):
        rc = _native.lib().pmb200_conv2d_nhwc(
            x.data_ptr(), filter_frag.data_ptr(), b_ptr, up_ptr, out.data_ptr(), N, H, W, cin, cout, ks, stride, pad, dil,
            1 if relu else 0, prec, 1 if transposed2x else 0, ycs, yco, rows_per_warp, _stream(x),
        )
    _native.check(rc, "conv2d_nhwc")
    return out


def warp_corr(
    ref_nhwc: Tensor, src_nhwc: Union[Tensor, ViewPack], rt: Tensor, depth: Tensor, G: int, view_weights: Optional[Tensor] = None
) -> Tensor:
    """K-A.  ref [B,H,W,C], src [V,B,Hs,Ws,C] or a ViewPack (sources of different sizes, pack_nhwc_views), rt [V,B,12],
    depth [B,D,H,W].

    Without view weights: per-view similarities [V,B,G,D,H,W].  With view_weights [B,V,H,W]:
    the weighted average over views [B,G,D,H,W] (reference patchmatch.py:192-217)."""
    if isinstance(src_nhwc, ViewPack):
        return _warp_corr_views(ref_nhwc, src_nhwc, rt, depth, G, view_weights)
    ref = _require(ref_nhwc, "ref_nhwc", 4)
    src = _require(src_nhwc, "src_nhwc", 5)
    rt = _require(rt, "rt", 3)
    depth = _require(depth, "depth", 4)
    B, H, W, C = ref.shape
    V, Bs, Hs, Ws, Cs = src.shape
    D = depth.shape[1]
    if Bs != B or Cs != C or rt.shape != (V, B, 12) or depth.shape != (B, D, H, W):
        raise RuntimeError("warp_corr: inconsistent shapes")
    if view_weights is not None:
        vw = _require(view_weights, "view_weights", 4)
        if vw.shape != (B, V, H, W):
            raise RuntimeError("warp_corr: view_weights must be [B,V,H,W]")
        out = torch.empty((B, G, D, H, W), dtype=torch.float32, device=ref.device)
        vw_ptr = vw.data_ptr()
    else:
        out = torch.empty((V, B, G, D, H, W), dtype=torch.float32, device=ref.device)
        vw_ptr = None
    with _device_guard(ref):
        rc = _native.lib().pmb200_warp_corr(
            ref.data_ptr(), src.data_ptr(), rt.data_ptr(), depth.data_ptr(), vw_ptr, out.data_ptr(),
            V, B, C, G, H, W, Hs, Ws, D, _stream(ref),
        )
    _native.check(rc, "warp_corr")
    return out


def _views_args(ref_nhwc, pack: ViewPack, rt, depth):
    ref = _require(ref_nhwc, "ref_nhwc", 4)
    if not _on_device(pack.data) or pack.data.dtype != torch.float32:
        raise RuntimeError("warp_corr: the view pack must hold CUDA float32 data")
    rt = _require(rt, "rt", 3)
    depth = _require(depth, "depth", 4)
    B, H, W, C = ref.shape
    V, D = len(pack), depth.shape[1]
    if pack.B != B or pack.C != C or rt.shape != (V, B, 12) or depth.shape != (B, D, H, W):
        raise RuntimeError("warp_corr: inconsistent shapes")
    return ref, rt, depth, (V, B, C, H, W, D)


def _warp_corr_views(ref_nhwc, pack: ViewPack, rt, depth, G: int, view_weights: Optional[Tensor]) -> Tensor:
    ref, rt, depth, (V, B, C, H, W, D) = _views_args(ref_nhwc, pack, rt, depth)
    vw_ptr = None
    if view_weights is not None:
        vw = _require(view_weights, "view_weights", 4)
        if vw.shape != (B, V, H, W):
            raise RuntimeError("warp_corr: view_weights must be [B,V,H,W]")
        out = torch.empty((B, G, D, H, W), dtype=torch.float32, device=ref.device)
        vw_ptr = vw.data_ptr()
    else:
        out = torch.empty((V, B, G, D, H, W), dtype=torch.float32, device=ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_warp_corr_views(
            ref.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth.data_ptr(), vw_ptr, out.data_ptr(),
            V, B, C, G, H, W, D, _stream(ref),
        )
    _native.check(rc, "warp_corr_views")
    return out


def _warp_args(ref_nhwc, src_nhwc, rt, depth):
    ref = _require(ref_nhwc, "ref_nhwc", 4)
    src = _require(src_nhwc, "src_nhwc", 5)
    rt = _require(rt, "rt", 3)
    depth = _require(depth, "depth", 4)
    B, H, W, C = ref.shape
    V, Bs, Hs, Ws, Cs = src.shape
    D = depth.shape[1]
    if Bs != B or Cs != C or rt.shape != (V, B, 12) or depth.shape != (B, D, H, W):
        raise RuntimeError("warp_corr: inconsistent shapes")
    return ref, src, rt, depth, (V, B, C, H, W, Hs, Ws, D)


def _score_target(xs: Optional[Tensor], B: int, D: int, H: int, W: int, device):
    if xs is None:
        out = torch.empty((B, D, H, W), dtype=torch.float32, device=device)
        return out, out.data_ptr(), 1
    if xs.shape != (B, D, H, W, 2) or not xs.is_contiguous() or xs.dtype != torch.float32 or xs.device != device:
        raise RuntimeError("xs must be a contiguous float32 [B,D,H,W,2] buffer on the same device")
    return xs, xs.data_ptr() + 4, 2  # the .y lanes


def warp_corr_score(ref_nhwc: Tensor, src_nhwc: Tensor, rt: Tensor, depth: Tensor, G: int, view_weights: Tensor,
                    head: "_native.MlpStruct", xs: Optional[Tensor] = None) -> Tensor:
    """K-A with the SimilarityNet head fused (eval mode): -> raw score [B,D,H,W]; the similarity
    tensor is never written.  `head` holds the BN-folded weights (host struct, see PointwiseHead.folded).  src_nhwc may be a
    ViewPack (sources of different sizes)."""
    if isinstance(src_nhwc, ViewPack):
        ref, rt, depth, (V, B, C, H, W, D) = _views_args(ref_nhwc, src_nhwc, rt, depth)
        vw = _require(view_weights, "view_weights", 4)
        if vw.shape != (B, V, H, W):
            raise RuntimeError("warp_corr_score: view_weights must be [B,V,H,W]")
        out, out_ptr, stride = _score_target(xs, B, D, H, W, ref.device)
        with _device_guard(ref):
            rc = _native.lib().pmb200_warp_corr_score_views(
                ref.data_ptr(), src_nhwc.data.data_ptr(), src_nhwc.extents, rt.data_ptr(), depth.data_ptr(), vw.data_ptr(), head,
                out_ptr, stride, V, B, C, G, H, W, D, _stream(ref),
            )
        _native.check(rc, "warp_corr_score_views")
        return out
    ref, src, rt, depth, (V, B, C, H, W, Hs, Ws, D) = _warp_args(ref_nhwc, src_nhwc, rt, depth)
    vw = _require(view_weights, "view_weights", 4)
    if vw.shape != (B, V, H, W):
        raise RuntimeError("warp_corr_score: view_weights must be [B,V,H,W]")
    out, out_ptr, stride = _score_target(xs, B, D, H, W, ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_warp_corr_score(
            ref.data_ptr(), src.data_ptr(), rt.data_ptr(), depth.data_ptr(), vw.data_ptr(), head, out_ptr, stride,
            V, B, C, G, H, W, Hs, Ws, D, _stream(ref),
        )
    _native.check(rc, "warp_corr_score")
    return out


def warp_corr_view_weights(ref_nhwc: Tensor, src_nhwc: Tensor, rt: Tensor, depth: Tensor, G: int,
                           head: "_native.MlpStruct", keep_sims: bool = False):
    """K-A with PixelwiseNet fused (eval mode): -> pixel-wise view weights [B,V,H,W]
    (and, keep_sims, the per-view similarities [V,B,G,D,H,W] for aggregate_views_score).  src_nhwc may be a ViewPack."""
    if isinstance(src_nhwc, ViewPack):
        ref, rt, depth, (V, B, C, H, W, D) = _views_args(ref_nhwc, src_nhwc, rt, depth)
        out = torch.empty((B, V, H, W), dtype=torch.float32, device=ref.device)
        sims = torch.empty((V, B, G, D, H, W), dtype=torch.float32, device=ref.device) if keep_sims else None
        with _device_guard(ref):
            rc = _native.lib().pmb200_warp_corr_view_weights_views(
                ref.data_ptr(), src_nhwc.data.data_ptr(), src_nhwc.extents, rt.data_ptr(), depth.data_ptr(), head, out.data_ptr(),
                None if sims is None else sims.data_ptr(), V, B, C, G, H, W, D, _stream(ref),
            )
        _native.check(rc, "warp_corr_view_weights_views")
        return (out, sims) if keep_sims else out
    ref, src, rt, depth, (V, B, C, H, W, Hs, Ws, D) = _warp_args(ref_nhwc, src_nhwc, rt, depth)
    out = torch.empty((B, V, H, W), dtype=torch.float32, device=ref.device)
    sims = torch.empty((V, B, G, D, H, W), dtype=torch.float32, device=ref.device) if keep_sims else None
    with _device_guard(ref):
        rc = _native.lib().pmb200_warp_corr_view_weights(
            ref.data_ptr(), src.data_ptr(), rt.data_ptr(), depth.data_ptr(), head, out.data_ptr(),
            None if sims is None else sims.data_ptr(), V, B, C, G, H, W, Hs, Ws, D, _stream(ref),
        )
    _native.check(rc, "warp_corr_view_weights")
    return (out, sims) if keep_sims else out


def aggregate_views_score(sims: Tensor, view_weights: Tensor, head: "_native.MlpStruct", xs: Optional[Tensor] = None) -> Tensor:
    """MLP(sum_v sims[v]*w[:,v] / (1e-5 + sum_v w[:,v])) -> raw score [B,D,H,W]."""
    sims = _require(sims, "sims", 6)
    vw = _require(view_weights, "view_weights", 4)
    V, B, G, D, H, W = sims.shape
    if vw.shape != (B, V, H, W):
        raise RuntimeError("aggregate_views_score: view_weights must be [B,V,H,W]")
    out, out_ptr, stride = _score_target(xs, B, D, H, W, sims.device)
    with _device_guard(sims):
        rc = _native.lib().pmb200_aggregate_views_score(
            sims.data_ptr(), vw.data_ptr(), head, out_ptr, stride, V, B, G, D, H, W, _stream(sims)
        )
    _native.check(rc, "aggregate_views_score")
    return out


def offset_corr_weight(ref_nhwc: Tensor, offsets: Tensor, G: int, K: int, dilation: int, head: "_native.MlpStruct") -> Tensor:
    """K-A' with the FeatureWeightNet head fused (eval mode): -> feature weight [B,K,H,W]."""
    ref = _require(ref_nhwc, "ref_nhwc", 4)
    B, H, W, C = ref.shape
    off, off_cl = _offsets_arg(offsets, (B, 2 * K, H, W), "offset_corr_weight")
    out = torch.empty((B, K, H, W), dtype=torch.float32, device=ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_offset_corr_weight(
            ref.data_ptr(), off.data_ptr(), off_cl, head, out.data_ptr(), B, C, G, H, W, K, dilation, _stream(ref)
        )
    _native.check(rc, "offset_corr_weight")
    return out


FUSED_HEAD_SHAPES = ((64, 8), (32, 8), (16, 4))


def aggregate_views(sims: Tensor, view_weights: Tensor) -> Tensor:
    """sum_v sims[v]*w[:,v] / (1e-5 + sum_v w[:,v]) -> [B,G,D,H,W]."""
    sims = _require(sims, "sims", 6)
    vw = _require(view_weights, "view_weights", 4)
    V, B, G, D, H, W = sims.shape
    if vw.shape != (B, V, H, W):
        raise RuntimeError("aggregate_views: view_weights must be [B,V,H,W]")
    out = torch.empty((B, G, D, H, W), dtype=torch.float32, device=sims.device)
    with _device_guard(sims):
        rc = _native.lib().pmb200_aggregate_views(
            sims.data_ptr(), vw.data_ptr(), out.data_ptr(), V, B, G, D, H, W, _stream(sims)
        )
    _native.check(rc, "aggregate_views")
    return out


def offset_corr(ref_nhwc: Tensor, offsets: Tensor, G: int, K: int, dilation: int) -> Tensor:
    """K-A'.  ref [B,H,W,C], offsets [B,2K,H,W] -> [B,G,K,H,W]."""
    ref = _require(ref_nhwc, "ref_nhwc", 4)
    B, H, W, C = ref.shape
    off, off_cl = _offsets_arg(offsets, (B, 2 * K, H, W), "offset_corr")
    out = torch.empty((B, G, K, H, W), dtype=torch.float32, device=ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_offset_corr(
            ref.data_ptr(), off.data_ptr(), off_cl, out.data_ptr(), B, C, G, H, W, K, dilation, _stream(ref)
        )
    _native.check(rc, "offset_corr")
    return out


MODE_RANDOM, MODE_PERTURB, MODE_PASSTHROUGH = 0, 1, 2


def alloc_xs(B: int, D: int, H: int, W: int, device) -> Tensor:
    """Interleaved (normalised inverse depth, raw score) buffer [B,D,H,W,2]: K-C fills the .x lanes, the K-A score
    epilogue the .y lanes, K-B then gathers both with one 8-byte load per tap."""
    return torch.empty((B, D, H, W, 2), dtype=torch.float32, device=device)


def init_propagate(
    seed_map: Tensor,
    offsets: Optional[Tensor],
    depth_min: Tensor,
    depth_max: Tensor,
    mode: int,
    Ns: int,
    Kp: int,
    dilation: int,
    interval_scale: float,
    with_xnorm: bool = False,
    xs: Optional[Tensor] = None,
):
    """K-C.  seed_map: U[0,1) noise [B,48,H,W] (mode 0) or current depth [B,1,H,W]; -> [B,Ns+Kp,H,W]
    (and, with_xnorm, the normalised inverse depth of every hypothesis, same shape).  With `xs` (an interleaved
    (xnorm, score) buffer [B,Ns+Kp,H,W,2] from alloc_xs) the normalised inverse depth goes into its .x lanes."""
    seed = _require(seed_map, "seed_map", 4)
    B, S, H, W = seed.shape
    if S != (48 if mode == MODE_RANDOM else 1):
        raise RuntimeError("init_propagate: seed_map has the wrong number of channels")
    dmin = _require(depth_min.reshape(-1), "depth_min", 1)
    dmax = _require(depth_max.reshape(-1), "depth_max", 1)
    if dmin.numel() != B or dmax.numel() != B:
        raise RuntimeError("init_propagate: depth_min/max must have B elements")
    off_ptr, off_cl = None, 0
    if Kp > 0:
        off, off_cl = _offsets_arg(offsets, (B, 2 * Kp, H, W), "init_propagate")
        off_ptr = off.data_ptr()
    out = torch.empty((B, Ns + Kp, H, W), dtype=torch.float32, device=seed.device)
    if xs is not None:
        if xs.shape != (B, Ns + Kp, H, W, 2) or not xs.is_contiguous() or xs.dtype != torch.float32 or not _on_device(xs):
            raise RuntimeError("init_propagate: xs must be a contiguous CUDA float32 [B,Ns+Kp,H,W,2] buffer")
        xn, xn_ptr, xstride = None, xs.data_ptr(), 2
    else:
        xn = torch.empty_like(out) if with_xnorm else None
        xn_ptr, xstride = (None if xn is None else xn.data_ptr()), 1
    with _device_guard(seed):
        rc = _native.lib().pmb200_init_propagate(
            seed.data_ptr(), off_ptr, off_cl, dmin.data_ptr(), dmax.data_ptr(), out.data_ptr(), xn_ptr, xstride,
            mode, B, H, W, Ns, Kp, dilation, float(interval_scale), _stream(seed),
        )
    _native.check(rc, "init_propagate")
    if xs is not None:
        return out
    return (out, xn) if with_xnorm else out


def adaptive_eval(
    score0: Tensor,
    depth_sample: Tensor,
    offsets: Tensor,
    feature_weight: Tensor,
    depth_min: Tensor,
    depth_max: Tensor,
    dilation: int,
    interval_scale: float,
    is_inverse: bool,
    xnorm: Optional[Tensor] = None,
    xs: Optional[Tensor] = None,
):
    """K-B.  -> (depth [B,H,W], prob [B,D,H,W]).  xnorm: normalised inverse depth from init_propagate.
    With `xs` (interleaved (xnorm, score) buffer) `score0` is ignored and may be None."""
    if xs is not None:
        if xs.dim() != 5 or xs.shape[-1] != 2 or not xs.is_contiguous() or not _on_device(xs) or xs.dtype != torch.float32:
            raise RuntimeError("adaptive_eval: xs must be a contiguous CUDA float32 [B,D,H,W,2] buffer")
        score0 = xs[..., 1]  # shape carrier only; never made contiguous below
        sc = score0
    else:
        sc = _require(score0, "score0", 4)
    ds = _require(depth_sample, "depth_sample", 4)
    fw = _require(feature_weight, "feature_weight", 4)
    B, D, H, W = sc.shape
    K = fw.shape[1]
    off, off_cl = _offsets_arg(offsets, (B, 2 * K, H, W), "adaptive_eval")
    if ds.shape != sc.shape or fw.shape != (B, K, H, W):
        raise RuntimeError("adaptive_eval: inconsistent shapes")
    dmin = _require(depth_min.reshape(-1), "depth_min", 1)
    dmax = _require(depth_max.reshape(-1), "depth_max", 1)
    xn_ptr = None
    if xnorm is not None:
        xn = _require(xnorm, "xnorm", 4)
        if xn.shape != sc.shape:
            raise RuntimeError("adaptive_eval: xnorm must match depth_sample")
        xn_ptr = xn.data_ptr()
    prob = torch.empty((B, D, H, W), dtype=torch.float32, device=sc.device)
    depth = torch.empty((B, H, W), dtype=torch.float32, device=sc.device)
    with _device_guard(sc):
        rc = _native.lib().pmb200_adaptive_eval(
            None if xs is not None else sc.data_ptr(), ds.data_ptr(), xn_ptr, None if xs is None else xs.data_ptr(), off.data_ptr(), off_cl, fw.data_ptr(), dmin.data_ptr(), dmax.data_ptr(),
            prob.data_ptr(), depth.data_ptr(), B, D, H, W, K, dilation, float(interval_scale),
            1 if is_inverse else 0, _stream(sc),
        )
    _native.check(rc, "adaptive_eval")
    return depth, prob


def compose_filter_cameras(ref_K, ref_E, src_Ks, src_Es) -> Tensor:
    """[V,60] float64 (CPU): the camera matrices `pmb200_geometric_filter` takes, composed the way the reference composes
    them -- numpy float32 inverses and products (eval.py:116-139) -- and then widened to float64 without rounding."""
    import numpy as np

    f32 = lambda m: np.asarray(m.detach().cpu().numpy() if isinstance(m, torch.Tensor) else m, dtype=np.float32)
    Kr, Er = f32(ref_K), f32(ref_E)
    rows = []
    for K, E in zip(src_Ks, src_Es):
        Ks, Es = f32(K), f32(E)
        t1 = np.matmul(Es, np.linalg.inv(Er))
        t2 = np.matmul(Er, np.linalg.inv(Es))
        rows.append(np.concatenate([np.linalg.inv(Kr).ravel(), t1[:3, :4].ravel(), Ks.ravel(), np.linalg.inv(Ks).ravel(),
                                    t2[:3, :4].ravel(), Kr.ravel()]).astype(np.float64))
    return torch.from_numpy(np.stack(rows))


def geometric_filter(ref_depth: Tensor, confidence: Tensor, src_depths: Union[Tensor, Sequence[Tensor]], cams: Tensor,
                     geo_pixel_thres: float = 1.0, geo_depth_thres: float = 0.01, photo_thres: float = 0.8, geo_mask_thres: int = 3):
    """Geometric-consistency filtering of one reference view against V source views in one launch (reference
    eval.py:86-190, :220-256).  ref_depth / confidence [H,W], src_depths [V,Hs,Ws] CUDA float32, or a list of V source maps
    [Hs_v,Ws_v] of different sizes (pmb200_geometric_filter_views); cams [V,60] float64 from
    compose_filter_cameras (moved to the device here).  -> (photo_mask bool [H,W], geo_mask_sum int32 [H,W],
    final_mask bool [H,W], depth_averaged float64 [H,W])."""
    if not isinstance(src_depths, torch.Tensor):
        return _geometric_filter_views(ref_depth, confidence, list(src_depths), cams, geo_pixel_thres, geo_depth_thres,
                                       photo_thres, geo_mask_thres)
    ref = _require(ref_depth, "ref_depth", 2)
    conf = _require(confidence, "confidence", 2)
    src = _require(src_depths, "src_depths", 3)
    H, W = ref.shape
    V, Hs, Ws = src.shape
    if conf.shape != (H, W):
        raise RuntimeError("geometric_filter: confidence must match ref_depth")
    if cams.shape != (V, 60) or cams.dtype != torch.float64:
        raise RuntimeError("geometric_filter: cams must be a [V,60] float64 tensor (compose_filter_cameras)")
    cams = cams.to(ref.device).contiguous()
    mask_sum = torch.empty((H, W), dtype=torch.int32, device=ref.device)
    photo = torch.empty((H, W), dtype=torch.uint8, device=ref.device)
    final = torch.empty((H, W), dtype=torch.uint8, device=ref.device)
    avg = torch.empty((H, W), dtype=torch.float64, device=ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_geometric_filter(
            ref.data_ptr(), conf.data_ptr(), src.data_ptr(), cams.data_ptr(), V, H, W, Hs, Ws, float(geo_pixel_thres),
            float(geo_depth_thres), float(photo_thres), int(geo_mask_thres), mask_sum.data_ptr(), photo.data_ptr(),
            final.data_ptr(), avg.data_ptr(), _stream(ref),
        )
    _native.check(rc, "geometric_filter")
    return photo.bool(), mask_sum, final.bool(), avg


def _geometric_filter_views(ref_depth: Tensor, confidence: Tensor, src_depths: List[Tensor], cams: Tensor, geo_pixel_thres: float,
                            geo_depth_thres: float, photo_thres: float, geo_mask_thres: int):
    ref = _require(ref_depth, "ref_depth", 2)
    conf = _require(confidence, "confidence", 2)
    srcs = [_require(s, "src_depths", 2) for s in src_depths]
    H, W = ref.shape
    V = len(srcs)
    if conf.shape != (H, W):
        raise RuntimeError("geometric_filter: confidence must match ref_depth")
    if V < 1 or cams.shape != (V, 60) or cams.dtype != torch.float64:
        raise RuntimeError("geometric_filter: cams must be a [V,60] float64 tensor (compose_filter_cameras)")
    flat = torch.cat([s.reshape(-1) for s in srcs])
    ext = (_native.ViewExtent * V)()
    off = 0
    for v, s in enumerate(srcs):
        ext[v].offset, ext[v].height, ext[v].width = off, s.shape[0], s.shape[1]
        off += s.numel()
    cams = cams.to(ref.device).contiguous()
    mask_sum = torch.empty((H, W), dtype=torch.int32, device=ref.device)
    photo = torch.empty((H, W), dtype=torch.uint8, device=ref.device)
    final = torch.empty((H, W), dtype=torch.uint8, device=ref.device)
    avg = torch.empty((H, W), dtype=torch.float64, device=ref.device)
    with _device_guard(ref):
        rc = _native.lib().pmb200_geometric_filter_views(
            ref.data_ptr(), conf.data_ptr(), flat.data_ptr(), ext, cams.data_ptr(), V, H, W, float(geo_pixel_thres),
            float(geo_depth_thres), float(photo_thres), int(geo_mask_thres), mask_sum.data_ptr(), photo.data_ptr(),
            final.data_ptr(), avg.data_ptr(), _stream(ref),
        )
    _native.check(rc, "geometric_filter_views")
    return photo.bool(), mask_sum, final.bool(), avg


def compose_fusion_camera(ref_K, ref_E) -> Tensor:
    """[25] float64 (CPU): inverse(ref_intrinsics) (9) then inverse(ref_extrinsics) (16), inverted in float32 as numpy does
    on the reference's float32 camera files (eval.py:278-279) and then widened without rounding."""
    import numpy as np

    f32 = lambda m: np.asarray(m.detach().cpu().numpy() if isinstance(m, torch.Tensor) else m, dtype=np.float32)
    return torch.from_numpy(np.concatenate([np.linalg.inv(f32(ref_K)).ravel(), np.linalg.inv(f32(ref_E)).ravel()]).astype(np.float64))


def fuse_points(final_mask: Tensor, depth_averaged: Tensor, ref_img: Tensor, cam25: Tensor, normals: Optional[Tensor] = None) -> Tensor:
    """Point-cloud half of the fusion for one reference view (reference eval.py:273-296): -> uint8 [n,15] CUDA tensor, the
    binary little-endian PLY vertex records (float32 x, y, z, uint8 r, g, b) of the surviving pixels in row-major order.
    final_mask bool / uint8 [H,W], depth_averaged float64 [H,W] (as geometric_filter returns them), ref_img float32
    [H,W,3] in [0,1].  One host synchronisation at the end (the vertex count sizes the result).

    With `normals`, the reference view's camera-frame normal map (float32 [H,W,3], estimate_normals), the records are the
    27-byte oriented ones, uint8 [n,27] (pmb200_fuse_points_oriented): float32 x, y, z, nx, ny, nz, uint8 r, g, b, the
    normal rotated into the world frame; the same pixels in the same order."""
    if not _on_device(final_mask) or not _on_device(depth_averaged) or not _on_device(ref_img):
        raise RuntimeError("fuse_points: the H100 path needs CUDA tensors; there is no CPU fallback")
    H, W = depth_averaged.shape
    if depth_averaged.dtype != torch.float64 or tuple(final_mask.shape) != (H, W) or tuple(ref_img.shape) != (H, W, 3) or ref_img.dtype != torch.float32:
        raise RuntimeError("fuse_points: final_mask [H,W], depth_averaged float64 [H,W], ref_img float32 [H,W,3]")
    if cam25.shape != (25,) or cam25.dtype != torch.float64:
        raise RuntimeError("fuse_points: cam25 must be a [25] float64 tensor (compose_fusion_camera)")
    if normals is not None:
        normals = _require(normals, "fuse_points: normals", 3)
        if tuple(normals.shape) != (H, W, 3):
            raise RuntimeError(f"fuse_points: normals must be [H,W,3] = [{H},{W},3], got {tuple(normals.shape)}")
    mask = final_mask.to(torch.uint8).contiguous()
    depth = depth_averaged.contiguous()
    img = ref_img.contiguous()
    cam = cam25.to(depth.device).contiguous()
    body = torch.empty((H * W, 15 if normals is None else 27), dtype=torch.uint8, device=depth.device)
    count = torch.zeros(1, dtype=torch.int32, device=depth.device)
    scratch = torch.empty(((H * W + 255) // 256,), dtype=torch.int32, device=depth.device)
    with _device_guard(depth):
        if normals is None:
            rc = _native.lib().pmb200_fuse_points(mask.data_ptr(), depth.data_ptr(), img.data_ptr(), cam.data_ptr(), H, W, body.data_ptr(),
                                                  count.data_ptr(), scratch.data_ptr(), _stream(depth))
        else:
            rc = _native.lib().pmb200_fuse_points_oriented(mask.data_ptr(), depth.data_ptr(), img.data_ptr(), normals.data_ptr(),
                                                           cam.data_ptr(), H, W, body.data_ptr(), count.data_ptr(), scratch.data_ptr(),
                                                           _stream(depth))
    _native.check(rc, "fuse_points" if normals is None else "fuse_points_oriented")
    return body[: int(count.item())]


def _kinv_host(K):
    """K^-1 as pmb200_depth_normals takes it: the float32 inverse numpy computes (as compose_fusion_camera inverts), widened
    to 9 float64 values in a host array."""
    import ctypes

    import numpy as np

    k = np.asarray(K.detach().cpu().numpy() if isinstance(K, torch.Tensor) else K, dtype=np.float32)
    if k.shape != (3, 3):
        raise RuntimeError(f"estimate_normals: K must be [3,3], got {k.shape}")
    return (ctypes.c_double * 9)(*np.linalg.inv(k).astype(np.float64).ravel().tolist())


def estimate_normals(depth: Tensor, K, radius: int = 3, depth_thres: float = 0.01, min_inliers: int = 6) -> Tensor:
    """Per-pixel unit normals of a depth map in the camera frame (pmb200_depth_normals; this project's own definition, see
    include/patchmatch_b200.h): the least-spread direction of the back-projected points of the pixels within `radius` whose
    depth is within depth_thres * D(p) of the pixel's, facing the camera; (0, 0, 0) where there is no estimate.
    depth CUDA float32 [H,W]; K float32 [3,3] (array or tensor) at the map's size.  -> CUDA float32 [H,W,3], the layout of
    COLMAP's normal maps.  radius 1..7 (PMB200_EINVAL otherwise, before any launch)."""
    d = _require(depth, "estimate_normals: depth", 2)
    H, W = d.shape
    kinv = _kinv_host(K)
    out = torch.empty((H, W, 3), dtype=torch.float32, device=d.device)
    with _device_guard(d):
        rc = _native.lib().pmb200_depth_normals(d.data_ptr(), kinv, H, W, int(radius), float(depth_thres), int(min_inliers),
                                                out.data_ptr(), _stream(d))
    _native.check(rc, "depth_normals")
    return out


MESH_VOXEL_BYTES = 12  # tsdf float32, weight float32, colour uchar4 per voxel (pmb200_tsdf_integrate)


def _mesh_grid_args(voxel_size, trunc, what: str) -> Tuple[float, int]:
    import math

    if isinstance(voxel_size, bool) or not isinstance(voxel_size, (int, float)) or not math.isfinite(voxel_size) or voxel_size <= 0:
        raise ValueError(f"{what}: voxel_size must be a positive finite number, got {voxel_size!r}")
    if isinstance(trunc, bool) or not isinstance(trunc, int) or not 1 <= trunc <= 4:
        raise ValueError(f"{what}: trunc must be an int in 1..4 (voxels), got {trunc!r}")
    return float(voxel_size), int(trunc)


def tsdf_allocate(points: Tensor, voxel_size: float, trunc: int = 3) -> Tensor:
    """The sorted unique keys (int64 [n_blocks], the uint64 keys' bits) of every 8^3-voxel block that the cube
    [p - trunc * voxel_size, p + trunc * voxel_size] of some seed point p meets (pmb200_tsdf_alloc).  points CUDA float32
    [n,3].  One host synchronisation (the block count).  ValueError for bad arguments and for a point whose voxel index does
    not fit in [-2^23, 2^23)."""
    import ctypes

    s, trunc = _mesh_grid_args(voxel_size, trunc, "tsdf_allocate")
    if not isinstance(points, Tensor) or not _on_device(points) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] != 3:
        raise ValueError("tsdf_allocate: points must be a CUDA float32 [n,3] tensor")
    pts = points.contiguous()
    n = pts.shape[0]
    lib = _native.lib()
    ws_bytes = lib.pmb200_tsdf_alloc_workspace_bytes(n)
    if ws_bytes < 0:
        raise ValueError("tsdf_allocate: " + lib.pmb200_last_error().decode("utf-8", "replace"))
    ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=pts.device)
    nb = ctypes.c_int64(0)
    with _device_guard(pts):
        rc = lib.pmb200_tsdf_alloc(pts.data_ptr(), n, s, trunc, ctypes.byref(nb), ws.data_ptr(), int(ws_bytes), _stream(pts))
    if rc == -1:
        raise ValueError(lib.pmb200_last_error().decode("utf-8", "replace"))
    _native.check(rc, "tsdf_alloc")
    return ws[: 8 * nb.value].view(torch.int64).clone()


def tsdf_view_table(depths: Sequence[Tensor], images: Sequence[Tensor], Ks, Es):
    """(ctypes array of pmb200_tsdf_view, depth base pointer, image base pointer, tensors to keep alive) for the integration.
    The maps are read in place: each view's offsets are counted in float32 elements from the lowest-addressed map, so
    views in separate allocations (an image bank) need no copy.  depths CUDA float32 [H_v,W_v] (0 where a pixel is not an
    observation), images CUDA float32 [3,H_v,W_v] in [0,1], Ks [3,3] and Es [4,4] (world -> camera) float32 arrays or
    tensors."""
    import numpy as np

    V = len(depths)
    if V == 0 or len(images) != V or len(Ks) != V or len(Es) != V:
        raise ValueError(f"tsdf_mesh: need one depth, image, K and E per view and at least one view (got {len(depths)}, "
                         f"{len(images)}, {len(Ks)}, {len(Es)})")
    f32 = lambda m: np.asarray(m.detach().cpu().numpy() if isinstance(m, Tensor) else m, dtype=np.float32)
    keep, dev = [], None
    table = (_native.TsdfView * V)()
    for v in range(V):
        d, img = depths[v], images[v]
        for t, what in ((d, "depth"), (img, "image")):
            if not isinstance(t, Tensor) or not _on_device(t) or t.dtype != torch.float32:
                raise ValueError(f"tsdf_mesh: view {v}: the {what} must be a CUDA float32 tensor")
        if d.dim() != 2 or tuple(img.shape) != (3,) + tuple(d.shape) or d.shape[0] < 1 or d.shape[1] < 1:
            raise ValueError(f"tsdf_mesh: view {v}: depth [H,W] and image [3,H,W], got {tuple(d.shape)} and {tuple(img.shape)}")
        if dev is None:
            dev = d.device
        if d.device != dev or img.device != dev:
            raise ValueError("tsdf_mesh: every map must be on one device")
        k, e = f32(Ks[v]), f32(Es[v])
        if k.shape != (3, 3) or e.shape != (4, 4):
            raise ValueError(f"tsdf_mesh: view {v}: K must be [3,3] and E [4,4], got {k.shape} and {e.shape}")
        table[v].K[:] = k.astype(np.float64).ravel().tolist()
        table[v].Rt[:] = e[:3, :4].astype(np.float64).ravel().tolist()
        table[v].height, table[v].width = int(d.shape[0]), int(d.shape[1])
        keep += [d.contiguous(), img.contiguous()]
    dbase = min(t.data_ptr() for t in keep[0::2])
    ibase = min(t.data_ptr() for t in keep[1::2])
    for v in range(V):
        table[v].depth_offset = (keep[2 * v].data_ptr() - dbase) // 4
        table[v].image_offset = (keep[2 * v + 1].data_ptr() - ibase) // 4
    return table, dbase, ibase, keep


def tsdf_integrate(keys: Tensor, depths: Sequence[Tensor], images: Sequence[Tensor], Ks, Es, voxel_size: float,
                   trunc: int = 3) -> Tuple[Tensor, Tensor, Tensor]:
    """TSDF integration of every view into the blocks `keys` (tsdf_allocate), one launch (pmb200_tsdf_integrate; definition
    in include/patchmatch_b200.h).  -> (tsdf float32, weight float32, colour uint8 [.,4]) per voxel, [n_blocks * 512],
    voxel index block * 512 + x + 8 y + 64 z."""
    import ctypes

    s, trunc = _mesh_grid_args(voxel_size, trunc, "tsdf_integrate")
    if not isinstance(keys, Tensor) or not _on_device(keys) or keys.dtype != torch.int64 or keys.dim() != 1 or keys.shape[0] < 1:
        raise ValueError("tsdf_integrate: keys must be a non-empty CUDA int64 [n_blocks] tensor (tsdf_allocate)")
    table, dbase, ibase, keep = tsdf_view_table(depths, images, Ks, Es)
    if keep[0].device != keys.device:
        raise ValueError("tsdf_integrate: the maps must be on the keys' device")
    nb, V = keys.shape[0], len(depths)
    lib = _native.lib()
    ws = _workspace(lib.pmb200_tsdf_integrate_workspace_bytes(V), "tsdf_integrate_workspace_bytes", keys.device)
    tsdf = torch.empty(nb * 512, dtype=torch.float32, device=keys.device)
    weight = torch.empty_like(tsdf)
    colour = torch.empty((nb * 512, 4), dtype=torch.uint8, device=keys.device)
    with _device_guard(keys):
        rc = lib.pmb200_tsdf_integrate(keys.data_ptr(), nb, s, trunc, ctypes.addressof(table), V, dbase, ibase, tsdf.data_ptr(),
                                       weight.data_ptr(), colour.data_ptr(), ws.data_ptr(), ws.numel(), _stream(keys))
    _native.check(rc, "tsdf_integrate")
    return tsdf, weight, colour


def tsdf_extract(keys: Tensor, tsdf: Tensor, weight: Tensor, colour: Tensor, voxel_size: float, min_weight: int = 1
                 ) -> Tuple[Tensor, Tensor]:
    """Marching cubes over the integrated blocks (pmb200_tsdf_mesh_count / _write): -> (vertex records uint8 [nv,15], the
    layout of the plain fused.ply, faces int32 [nf,3]) on the device, in the documented order.  One host synchronisation
    (the counts size the outputs)."""
    s, _ = _mesh_grid_args(voxel_size, 1, "tsdf_extract")
    if isinstance(min_weight, bool) or not isinstance(min_weight, int) or min_weight < 1:
        raise ValueError(f"tsdf_extract: min_weight must be an int >= 1, got {min_weight!r}")
    nb = keys.shape[0]
    if tsdf.shape != (nb * 512,) or weight.shape != (nb * 512,) or colour.shape != (nb * 512, 4):
        raise ValueError("tsdf_extract: tsdf, weight [n_blocks*512] and colour [n_blocks*512,4] as tsdf_integrate returns them")
    lib = _native.lib()
    ws_bytes = lib.pmb200_tsdf_mesh_workspace_bytes(nb)
    ws = _workspace(ws_bytes, "tsdf_mesh_workspace_bytes", keys.device)
    totals = torch.zeros(2, dtype=torch.int64, device=keys.device)
    with _device_guard(keys):
        rc = lib.pmb200_tsdf_mesh_count(keys.data_ptr(), nb, tsdf.data_ptr(), weight.data_ptr(), min_weight, totals.data_ptr(),
                                        ws.data_ptr(), int(ws_bytes), _stream(keys))
    _native.check(rc, "tsdf_mesh_count")
    nv, nf = (int(v) for v in totals.tolist())
    if nv >= 2 ** 31:
        raise ValueError(f"tsdf_extract: {nv} vertices do not fit int32 face indices; use a larger voxel size")
    verts = torch.empty((nv, 15), dtype=torch.uint8, device=keys.device)
    faces = torch.empty((nf, 3), dtype=torch.int32, device=keys.device)
    if nv == 0 and nf == 0:
        return verts, faces
    with _device_guard(keys):
        rc = lib.pmb200_tsdf_mesh_write(keys.data_ptr(), nb, s, tsdf.data_ptr(), weight.data_ptr(), colour.data_ptr(), min_weight,
                                        verts.data_ptr(), faces.data_ptr(), ws.data_ptr(), int(ws_bytes), _stream(keys))
    _native.check(rc, "tsdf_mesh_write")
    return verts, faces


def tsdf_mesh_bytes(n_blocks: int) -> int:
    """Device memory the volume and the extraction need for n_blocks allocated blocks (the views' maps not included):
    n_blocks * 512 * 12 bytes of volume, plus 3 bytes per voxel and a few per block of extraction workspace."""
    return n_blocks * 512 * (MESH_VOXEL_BYTES + 3) + n_blocks * 40


def tsdf_mesh(points: Tensor, depths: Sequence[Tensor], images: Sequence[Tensor], Ks, Es, voxel_size: float, trunc: int = 3,
              min_weight: int = 1) -> Tuple[Tensor, Tensor]:
    """A coloured triangle mesh of the views' depth maps: TSDF integration over the blocks the seed points allocate, then
    marching cubes (this project's own definition, include/patchmatch_b200.h).  points CUDA float32 [n,3] (e.g. the xyz of
    the fused points); per view the depth float32 [H,W] (0 where there is no observation), the image float32 [3,H,W] in
    [0,1], K [3,3] and E [4,4] (world -> camera); voxel_size in world units, trunc in voxels (1..4), min_weight the views a
    voxel needs.  -> (vertex records uint8 [nv,15], faces int32 [nf,3]) on the device.

    ValueError before any launch on bad arguments, and before the volume is allocated when its memory would exceed the
    device's free memory (the message gives the block count: use a larger voxel size)."""
    _mesh_grid_args(voxel_size, trunc, "tsdf_mesh")
    if isinstance(min_weight, bool) or not isinstance(min_weight, int) or min_weight < 1:
        raise ValueError(f"tsdf_mesh: min_weight must be an int >= 1, got {min_weight!r}")
    tsdf_view_table(depths, images, Ks, Es)  # the views' checks, before any launch
    keys = tsdf_allocate(points, voxel_size, trunc)
    nb = keys.shape[0]
    if nb == 0:
        return torch.empty((0, 15), dtype=torch.uint8, device=points.device), torch.empty((0, 3), dtype=torch.int32, device=points.device)
    need = tsdf_mesh_bytes(nb)
    with _device_guard(keys):
        free = torch.cuda.mem_get_info(keys.device)[0] + torch.cuda.memory_reserved(keys.device) - torch.cuda.memory_allocated(keys.device)
    if nb >= 2 ** 22 or need > free:
        raise ValueError(f"tsdf_mesh: the volume has {nb} blocks of 8^3 voxels and needs {need / 2 ** 30:.2f} GiB "
                         f"({free / 2 ** 30:.2f} GiB free, at most 4194303 blocks); use a larger voxel size")
    tsdf, weight, colour = tsdf_integrate(keys, depths, images, Ks, Es, voxel_size, trunc)
    return tsdf_extract(keys, tsdf, weight, colour, voxel_size, min_weight)


def render_camera_arrays(P):
    """A 3 x 4 float64 camera K [R | t] -> (P rounded to float32, row-major [12]; camera centre -M^-1 p4 computed in float64
    and rounded to float32 [3]), the HOST values pmb200_render_points / _mesh take.  ValueError for a camera that is not
    finite or whose left 3 x 3 is singular."""
    import numpy as np

    P64 = np.asarray(P.detach().cpu().numpy() if isinstance(P, Tensor) else P, dtype=np.float64)
    if P64.shape != (3, 4) or not np.isfinite(P64).all():
        raise ValueError(f"render: the camera must be a finite 3 x 4 matrix K [R | t], got shape {P64.shape}")
    try:
        centre = -np.linalg.solve(P64[:, :3], P64[:, 3])
    except np.linalg.LinAlgError:
        raise ValueError("render: the camera's left 3 x 3 is singular") from None
    return P64.astype(np.float32).ravel(), centre.astype(np.float32)


def _render_args(P, width: int, height: int, near: float, background, what: str):
    import ctypes
    import math

    for name, v in (("width", width), ("height", height)):
        if isinstance(v, bool) or not isinstance(v, int) or not 1 <= v <= 16384:
            raise ValueError(f"{what}: {name} must be an int in 1..16384, got {v!r}")
    if not (isinstance(near, (int, float)) and math.isfinite(near) and near > 0):
        raise ValueError(f"{what}: near must be a positive finite number, got {near!r}")
    bg = [int(c) for c in background]
    if len(bg) != 3 or any(not 0 <= c <= 255 for c in bg):
        raise ValueError(f"{what}: background must be three values in 0..255, got {background!r}")
    p, c = render_camera_arrays(P)
    return (ctypes.c_float * 12)(*p.tolist()), (ctypes.c_float * 3)(*c.tolist()), (ctypes.c_ubyte * 3)(*bg)


def _render_attr(t: Optional[Tensor], n: int, dtype, device, name: str, what: str) -> Optional[Tensor]:
    if t is None:
        return None
    if not isinstance(t, Tensor) or not _on_device(t) or t.dtype != dtype or tuple(t.shape) != (n, 3) or t.device != device:
        raise ValueError(f"{what}: {name} must be a CUDA {dtype} [{n},3] tensor on the vertices' device")
    return t.contiguous()


def _render_xyz(xyz: Tensor, what: str) -> Tensor:
    if not isinstance(xyz, Tensor) or not _on_device(xyz) or xyz.dtype != torch.float32 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise ValueError(f"{what}: xyz must be a CUDA float32 [n,3] tensor (there is no CPU fallback)")
    return xyz.contiguous()


def render_points(xyz: Tensor, rgb: Optional[Tensor], normals: Optional[Tensor], P, width: int, height: int, near: float,
                  point_size: int = 1, shade: bool = False, background=(255, 255, 255)) -> Tuple[Tensor, Tensor]:
    """Z-buffered square splats of a point cloud (pmb200_render_points; definition in include/patchmatch_b200.h).  xyz CUDA
    float32 [n,3]; rgb uint8 [n,3] or None (grey); normals float32 [n,3] or None (used by shade=True); P the 3 x 4 float64
    camera K [R | t] (pixel (x, y) sampled at (x, y)); near > 0 the depth at or below which points are skipped; point_size
    odd 1..15.  -> (rgb uint8 [H,W,3], depth float32 [H,W], 0 where nothing was drawn) on the device.  Bit-identical to
    tests/render_oracle.py and from run to run.  ValueError before any launch on bad arguments."""
    what = "render_points"
    pts = _render_xyz(xyz, what)
    n = pts.shape[0]
    if n >= 2 ** 32:
        raise ValueError(f"{what}: at most 2^32 - 1 points, got {n}")
    if isinstance(point_size, bool) or not isinstance(point_size, int) or not (1 <= point_size <= 15 and point_size % 2 == 1):
        raise ValueError(f"{what}: point_size must be an odd int in 1..15, got {point_size!r}")
    col = _render_attr(rgb, n, torch.uint8, pts.device, "rgb", what)
    nrm = _render_attr(normals, n, torch.float32, pts.device, "normals", what)
    p_host, c_host, bg = _render_args(P, width, height, near, background, what)
    lib = _native.lib()
    ws = _workspace(lib.pmb200_render_points_workspace_bytes(width, height), "render_points_workspace_bytes", pts.device)
    out_rgb = torch.empty((height, width, 3), dtype=torch.uint8, device=pts.device)
    out_depth = torch.empty((height, width), dtype=torch.float32, device=pts.device)
    with _device_guard(pts):
        rc = lib.pmb200_render_points(pts.data_ptr(), None if col is None else col.data_ptr(), None if nrm is None else nrm.data_ptr(),
                                      n, p_host, c_host, width, height, point_size, float(near), 1 if shade else 0, bg,
                                      out_rgb.data_ptr(), out_depth.data_ptr(), ws.data_ptr(), ws.numel(), _stream(pts))
    _native.check(rc, what)
    return out_rgb, out_depth


def render_mesh(xyz: Tensor, rgb: Optional[Tensor], faces: Tensor, P, width: int, height: int, near: float, shade: bool = False,
                background=(255, 255, 255), check_faces: bool = True) -> Tuple[Tensor, Tensor]:
    """Z-buffered rasterisation of a triangle mesh with perspective-correct colours and flat headlight shading
    (pmb200_render_mesh; definition in include/patchmatch_b200.h).  xyz CUDA float32 [nv,3]; rgb uint8 [nv,3] or None (grey);
    faces int32 [nf,3]; P, near, shade and background as for render_points.  -> (rgb uint8 [H,W,3], depth float32 [H,W]) on
    the device.  A face with a vertex at or behind `near` is dropped, not clipped.  With check_faces (the default) a face
    index outside 0..nv-1 raises ValueError (one host read); without it such faces are skipped by the kernel."""
    what = "render_mesh"
    pts = _render_xyz(xyz, what)
    nv = pts.shape[0]
    if not isinstance(faces, Tensor) or not _on_device(faces) or faces.dtype != torch.int32 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"{what}: faces must be a CUDA int32 [nf,3] tensor")
    if faces.device != pts.device:
        raise ValueError(f"{what}: faces must be on the vertices' device")
    fc = faces.contiguous()
    nf = fc.shape[0]
    if nv >= 2 ** 31 or nf >= 2 ** 31:
        raise ValueError(f"{what}: at most 2^31 - 1 vertices and faces, got {nv} and {nf}")
    if check_faces and nf:
        lo, hi = (int(v) for v in torch.aminmax(fc))
        if lo < 0 or hi >= nv:
            raise ValueError(f"{what}: a face refers to a vertex outside 0..{nv - 1}")
    col = _render_attr(rgb, nv, torch.uint8, pts.device, "rgb", what)
    p_host, c_host, bg = _render_args(P, width, height, near, background, what)
    lib = _native.lib()
    ws = _workspace(lib.pmb200_render_mesh_workspace_bytes(width, height, nv, nf), "render_mesh_workspace_bytes", pts.device)
    out_rgb = torch.empty((height, width, 3), dtype=torch.uint8, device=pts.device)
    out_depth = torch.empty((height, width), dtype=torch.float32, device=pts.device)
    with _device_guard(pts):
        rc = lib.pmb200_render_mesh(pts.data_ptr(), None if col is None else col.data_ptr(), nv, fc.data_ptr(), nf, p_host, c_host,
                                    width, height, float(near), 1 if shade else 0, bg, out_rgb.data_ptr(), out_depth.data_ptr(),
                                    ws.data_ptr(), ws.numel(), _stream(pts))
    _native.check(rc, what)
    return out_rgb, out_depth


def split_ply_body(body: Tensor):
    """uint8 [n,15] vertex records -> (vertices float32 [n,3], colours uint8 [n,3]) on the CPU."""
    b = body.detach().cpu().contiguous()
    return b[:, :12].contiguous().view(torch.float32).view(-1, 3), b[:, 12:].contiguous()


def _points_arg(p: Tensor, name: str) -> Tensor:
    if not _on_device(p):
        raise RuntimeError(f"{name}: the H100 path needs a CUDA tensor (got {p.device}); there is no CPU fallback")
    if p.dtype != torch.float64 or p.dim() != 2 or p.shape[1] != 3:
        raise RuntimeError(f"{name}: expected a float64 [n,3] tensor, got {p.dtype} {tuple(p.shape)}")
    return p.contiguous()


def thin_points(points: Tensor, rank: Tensor, dst: float) -> Tensor:
    """Thinning of a point cloud to a minimum distance (reference evaluations/dtu/reducePts_haa.m): the points visited in the
    order of `rank` (int32 [n], a permutation of 0..n-1) that survive, i.e. that no surviving earlier point lies within
    distance <= dst of.  points float64 [n,3] CUDA -> keep bool [n].  One host synchronisation at the end (the round-bound
    check)."""
    pts = _points_arg(points, "thin_points")
    n = pts.shape[0]
    if rank.shape != (n,) or rank.dtype != torch.int32 or rank.device != pts.device:
        raise RuntimeError("thin_points: rank must be an int32 [n] tensor on the points' device")
    rk = rank.contiguous()
    keep = torch.empty(n, dtype=torch.uint8, device=pts.device)
    undecided = torch.empty(1, dtype=torch.int32, device=pts.device)
    lib = _native.lib()
    ws_bytes = lib.pmb200_thin_points_workspace_bytes(n)
    if ws_bytes < 0:
        _native.check(int(ws_bytes), "thin_points_workspace_bytes")
    ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=pts.device)
    with _device_guard(pts):
        rc = lib.pmb200_thin_points(pts.data_ptr(), rk.data_ptr(), n, float(dst), keep.data_ptr(), undecided.data_ptr(),
                                    ws.data_ptr(), int(ws_bytes), _stream(pts))
    _native.check(rc, "thin_points")
    left = int(undecided.item())
    if left:
        raise RuntimeError(f"thin_points: {left} points still undecided after the round bound of the native thinning")
    return keep.bool()


def default_search_cell(n_to: int, bb, max_dist: float) -> float:
    """Fine cell edge for nearest_distance: about twice the spacing of n_to points spread over a surface the size of the box.
    It only sets the speed of the search, never its result."""
    import math

    ext = [max(float(bb[1][a]) - float(bb[0][a]), 1e-9) for a in range(3)]
    side = (ext[0] * ext[1] * ext[2]) ** (1.0 / 3.0)
    cell = 2.0 * side / math.sqrt(max(n_to, 1))
    return min(max(cell, max_dist / 256.0), max_dist / 8.0)  # the library requires cell >= max_dist / 256


def nearest_distance(to_points: Tensor, from_points: Tensor, bb, max_dist: float = 60.0, cell: Optional[float] = None) -> Tensor:
    """Distance from every `from` point to the nearest `to` point, capped at max_dist, with the block membership of the
    reference's evaluations/dtu/MaxDistCP.m: a point outside its max_dist blocks over the box `bb` ([[x,y,z] lo, [x,y,z] hi])
    gets max_dist.  Exact float64 distances.  to_points [m,3], from_points [n,3] float64 CUDA -> float64 [n]."""
    import ctypes

    to = _points_arg(to_points, "nearest_distance (to)")
    frm = _points_arg(from_points, "nearest_distance (from)")
    if to.device != frm.device:
        raise RuntimeError("nearest_distance: both clouds must be on the same device")
    box = [float(v) for row in bb for v in row]
    if len(box) != 6:
        raise RuntimeError("nearest_distance: bb must be 2 x 3 (lo, hi)")
    if cell is None:
        cell = default_search_cell(to.shape[0], [box[:3], box[3:]], max_dist)
    out = torch.empty(frm.shape[0], dtype=torch.float64, device=frm.device)
    lib = _native.lib()
    ws_bytes = lib.pmb200_nearest_distance_workspace_bytes(to.shape[0])
    if ws_bytes < 0:
        _native.check(int(ws_bytes), "nearest_distance_workspace_bytes")
    ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=frm.device)
    bb_host = (ctypes.c_double * 6)(*box)
    with _device_guard(frm):
        rc = lib.pmb200_nearest_distance(to.data_ptr(), to.shape[0], frm.data_ptr(), frm.shape[0], bb_host, float(max_dist), float(cell),
                                         out.data_ptr(), ws.data_ptr(), int(ws_bytes), _stream(frm))
    _native.check(rc, "nearest_distance")
    return out


def _host_4x4(transform):
    """A 4 x 4 (array-like, or None for the identity) -> HOST ctypes array of 16 doubles, row-major."""
    import ctypes

    import numpy as np

    m = np.eye(4) if transform is None else np.asarray(transform, dtype=np.float64).reshape(4, 4)
    return (ctypes.c_double * 16)(*m.reshape(16).tolist())


def crop_points(points: Tensor, orthogonal_axis: int, axis_min: float, axis_max: float, polygon, transform=None):
    """Open3D's SelectionPolygonVolume crop (include/patchmatch_b200.h, pmb200_crop_polygon) after the 4 x 4 `transform`
    (last row 0 0 0 1; None = identity).  points float64 [n,3] CUDA; polygon [k,3] vertices (k <= 128); orthogonal_axis
    0 / 1 / 2 for "X" / "Y" / "Z".  -> (transformed points float64 [n,3], keep bool [n]); kept points keep their order."""
    import ctypes

    import numpy as np

    pts = _points_arg(points, "crop_points")
    n = pts.shape[0]
    poly = np.ascontiguousarray(np.asarray(polygon, dtype=np.float64).reshape(-1, 3))
    out = torch.empty_like(pts)
    keep = torch.empty(n, dtype=torch.uint8, device=pts.device)
    with _device_guard(pts):
        rc = _native.lib().pmb200_crop_polygon(pts.data_ptr(), n, _host_4x4(transform), int(orthogonal_axis), float(axis_min),
                                               float(axis_max), (ctypes.c_double * max(poly.size, 1))(*poly.reshape(-1).tolist()),
                                               poly.shape[0], out.data_ptr(), keep.data_ptr(), _stream(pts))
    _native.check(rc, "crop_points")
    return out, keep.bool()


def voxel_downsample(points: Tensor, voxel_size: float) -> Tensor:
    """Open3D's VoxelDownSample (include/patchmatch_b200.h, pmb200_voxel_downsample): one point per occupied voxel of edge
    voxel_size anchored at the cloud's min bound - voxel_size / 2, the mean of its points, voxels in ascending (x, y, z)
    index order.  points float64 [n,3] CUDA -> float64 [m,3].  Two host reads: the cloud's bounds and the voxel count."""
    import ctypes

    pts = _points_arg(points, "voxel_downsample")
    n = pts.shape[0]
    if n == 0:
        return pts.new_empty((0, 3))
    lo, hi = torch.aminmax(pts, dim=0)
    bounds = (ctypes.c_double * 6)(*torch.cat([lo, hi]).cpu().tolist())
    out = torch.empty_like(pts)
    count = torch.empty(1, dtype=torch.int64, device=pts.device)
    lib = _native.lib()
    ws = _workspace(lib.pmb200_voxel_downsample_workspace_bytes(n), "voxel_downsample_workspace_bytes", pts.device)
    with _device_guard(pts):
        rc = lib.pmb200_voxel_downsample(pts.data_ptr(), n, bounds, float(voxel_size), out.data_ptr(), count.data_ptr(),
                                         ws.data_ptr(), ws.numel(), _stream(pts))
    _native.check(rc, "voxel_downsample")
    return out[: int(count.item())]


def beam_observed(queries: Tensor, scan_points: Tensor, origin, beam_start_radius: float, tan_half_angle: float,
                  observed: Optional[Tensor] = None, mask: Optional[Tensor] = None) -> Tensor:
    """Which queries lie in the free beam of some point of one laser scan (include/patchmatch_b200.h, pmb200_beam_observed):
    the scan's angular index around `origin` (3 numbers) is built, then every query under `mask` (bool or uint8 [n], None =
    all) that `observed` does not already mark is tested.  queries [n,3] and scan_points [m,3] float64 CUDA, scan points in
    the scene frame; beam_start_radius r0 and tan_half_angle T >= 0.  -> observed uint8 [n], updated in place when given (so
    one call per scan ORs the scans).  Exact: the result equals a brute-force evaluation of the predicate, bit for bit."""
    import ctypes

    q = _points_arg(queries, "beam_observed (queries)")
    s = _points_arg(scan_points, "beam_observed (scan points)")
    if s.device != q.device:
        raise RuntimeError("beam_observed: queries and scan points must be on the same device")
    o = [float(v) for v in origin]
    if len(o) != 3:
        raise RuntimeError("beam_observed: origin must have 3 coordinates")
    n = q.shape[0]
    if observed is None:
        observed = torch.zeros(n, dtype=torch.uint8, device=q.device)
    elif observed.dtype != torch.uint8 or observed.shape != (n,) or observed.device != q.device or not observed.is_contiguous():
        raise RuntimeError("beam_observed: observed must be a contiguous uint8 [n] tensor on the queries' device")
    m = None
    if mask is not None:
        if mask.shape != (n,) or mask.device != q.device or mask.dtype not in (torch.bool, torch.uint8):
            raise RuntimeError("beam_observed: mask must be a bool or uint8 [n] tensor on the queries' device")
        m = mask.to(torch.uint8).contiguous()
    lib = _native.lib()
    ws = _workspace(lib.pmb200_beam_index_workspace_bytes(s.shape[0]), "beam_index_workspace_bytes", q.device)
    o_host = (ctypes.c_double * 3)(*o)
    with _device_guard(q):
        rc = lib.pmb200_beam_index(s.data_ptr(), s.shape[0], o_host, ws.data_ptr(), ws.numel(), _stream(q))
        _native.check(rc, "beam_index")
        rc = lib.pmb200_beam_observed(q.data_ptr(), n, m.data_ptr() if m is not None else None, ws.data_ptr(), s.shape[0], o_host,
                                      float(beam_start_radius), float(tan_half_angle), observed.data_ptr(), _stream(q))
    _native.check(rc, "beam_observed")
    return observed


def voxel_score(points: Tensor, dist: Tensor, tau: float, observed: Optional[Tensor] = None) -> dict:
    """Density-normalised score of a cloud at tolerance tau (include/patchmatch_b200.h, pmb200_voxel_score): a point is good
    when dist <= tau, bad when dist > tau and `observed` marks it (every such point when observed is None), else excluded;
    voxels of edge tau anchored at the world origin.  points float64 [n,3], dist float64 [n], observed uint8/bool [n] or None,
    all CUDA.  -> {"good", "bad", "excluded", "voxels", "fraction_sum"}: the counts and the sum over voxels holding a good or
    bad point of good / (good + bad).  Two host reads: the counted points' bounds and the result."""
    import ctypes

    pts = _points_arg(points, "voxel_score")
    n = pts.shape[0]
    if dist.dtype != torch.float64 or dist.shape != (n,) or dist.device != pts.device:
        raise RuntimeError("voxel_score: dist must be a float64 [n] tensor on the points' device")
    d = dist.contiguous()
    obs = None
    if observed is not None:
        if observed.shape != (n,) or observed.device != pts.device or observed.dtype not in (torch.bool, torch.uint8):
            raise RuntimeError("voxel_score: observed must be a bool or uint8 [n] tensor on the points' device")
        obs = observed.to(torch.uint8).contiguous()
    counted = (d <= tau) | (obs.bool() if obs is not None else True)
    inf = torch.tensor(float("inf"), dtype=torch.float64, device=pts.device)
    lo = torch.where(counted[:, None], pts, inf).amin(0) if n else inf.expand(3)
    hi = torch.where(counted[:, None], pts, -inf).amax(0) if n else -inf.expand(3)
    b = torch.cat([lo, hi]).cpu().tolist()
    if not b[0] <= b[3]:  # nothing counts: any valid box
        b = [0.0] * 6
    counts = torch.empty(4, dtype=torch.int64, device=pts.device)
    fsum = torch.empty(1, dtype=torch.float64, device=pts.device)
    lib = _native.lib()
    ws = _workspace(lib.pmb200_voxel_score_workspace_bytes(n), "voxel_score_workspace_bytes", pts.device)
    with _device_guard(pts):
        rc = lib.pmb200_voxel_score(pts.data_ptr(), d.data_ptr(), n, float(tau), obs.data_ptr() if obs is not None else None,
                                    (ctypes.c_double * 6)(*b), counts.data_ptr(), fsum.data_ptr(), ws.data_ptr(), ws.numel(),
                                    _stream(pts))
    _native.check(rc, "voxel_score")
    c = counts.cpu().tolist()
    return {"good": c[0], "bad": c[1], "excluded": c[2], "voxels": c[3], "fraction_sum": float(fsum.cpu())}


def umeyama_from_moments(m) -> "np.ndarray":
    """The similarity (with scaling) that best maps the correspondences' source points onto their targets (Umeyama 1991, the
    estimate of Eigen::umeyama with scaling), from the 18 sums of pmb200_icp_query taken relative to an origin o:
        mu_p = S_p / n, mu_q = S_q / n, Sigma = S_qp / n - mu_q mu_p^T, var_p = S_pp / n - |mu_p|^2,
        Sigma = U D V^T (numpy's SVD), S = diag(1, 1, -1 if det(U) det(V) < 0 else 1),
        R = U S V^T, c = trace(D S) / var_p, t = mu_q - c R mu_p.
    -> float64 [4,4] acting on coordinates relative to o.  The identity when there is no correspondence."""
    import numpy as np

    m = np.asarray(m, dtype=np.float64)
    n = m[0]
    if n == 0:
        return np.eye(4)
    mu_p, mu_q = m[2:5] / n, m[5:8] / n
    sigma = m[8:17].reshape(3, 3) / n - np.outer(mu_q, mu_p)
    var_p = m[17] / n - mu_p @ mu_p
    u, d, vt = np.linalg.svd(sigma)
    s = np.ones(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        s[2] = -1.0
    r = (u * s) @ vt
    c = (d @ s) / var_p
    out = np.eye(4)
    out[:3, :3] = c * r
    out[:3, 3] = mu_q - c * (r @ mu_p)
    return out


def icp(source: Tensor, target: Tensor, max_dist: float, max_iteration: int = 30, init=None, relative_fitness: float = 1e-6,
        relative_rmse: float = 1e-6, cell: Optional[float] = None, return_correspondences: bool = False) -> dict:
    """Point-to-point ICP with scaling, Open3D's registration_icp loop (INTEGRATION.md "Tanks and Temples evaluation"):
    correspondences of T = init (nearest target point within distance <= max_dist, ties to the smallest target index),
    fitness = |C| / |source| and inlier RMSE = sqrt(sum d^2 / |C|) (0 without correspondences); then per iteration the
    Umeyama similarity of the correspondences is composed onto T and the correspondences are recomputed, stopping once
    |delta fitness| < relative_fitness and |delta RMSE| < relative_rmse, or after max_iteration updates.  The target is
    sorted into its cell hash once; each evaluation is one query launch (the source transformed in the kernel) and one
    device-to-host copy of 18 sums.  source [n,3], target [m,3] float64 CUDA ->
    {"transformation" float64 [4,4], "fitness", "inlier_rmse", "iterations", "correspondences" (final |C|),
     "history" [(|C|, sum d^2)] of every evaluation, and "correspondence_set" int32 [n] (-1 = none) when asked}."""
    import ctypes
    import math

    import numpy as np

    src = _points_arg(source, "icp (source)")
    tgt = _points_arg(target, "icp (target)")
    if src.device != tgt.device:
        raise RuntimeError("icp: both clouds must be on the same device")
    if not (max_dist > 0 and math.isfinite(max_dist)):
        raise ValueError("icp: max_dist must be positive and finite")
    n_src, n_tgt = src.shape[0], tgt.shape[0]
    lib = _native.lib()
    if n_tgt > 0:
        lo, hi = torch.aminmax(tgt, dim=0)
        lo, hi = lo.cpu().numpy(), hi.cpu().numpy()
    else:
        lo = hi = np.zeros(3)
    origin = (ctypes.c_double * 3)(*((lo + hi) / 2).tolist())
    if cell is None:
        cell = default_search_cell(n_tgt, [lo, hi], max_dist)
    tws = _workspace(lib.pmb200_icp_target_workspace_bytes(n_tgt), "icp_target_workspace_bytes", src.device)
    qws = _workspace(lib.pmb200_icp_query_workspace_bytes(n_src), "icp_query_workspace_bytes", src.device)
    moments = torch.empty(18, dtype=torch.float64, device=src.device)
    corr = torch.empty(n_src, dtype=torch.int32, device=src.device) if return_correspondences else None
    with _device_guard(src):
        _native.check(lib.pmb200_icp_target(tgt.data_ptr(), n_tgt, float(cell), tws.data_ptr(), tws.numel(), _stream(tgt)), "icp_target")

    def evaluate(t):
        with _device_guard(src):
            rc = lib.pmb200_icp_query(src.data_ptr(), n_src, _host_4x4(t), origin, float(max_dist), tws.data_ptr(), n_tgt, float(cell),
                                      corr.data_ptr() if corr is not None else None, moments.data_ptr(), qws.data_ptr(), qws.numel(),
                                      _stream(src))
        _native.check(rc, "icp_query")
        m = moments.cpu().numpy()
        fit = m[0] / n_src if n_src else 0.0
        return m, fit, (math.sqrt(m[1] / m[0]) if m[0] > 0 else 0.0)

    t = np.eye(4) if init is None else np.asarray(init, dtype=np.float64).reshape(4, 4).copy()
    m, fitness, rmse = evaluate(t)
    history = [(int(m[0]), float(m[1]))]
    o = np.asarray(origin[:])
    iterations = 0
    for _ in range(max_iteration):
        rel = umeyama_from_moments(m)  # acts on coordinates relative to the origin
        upd = np.eye(4)
        upd[:3, :3] = rel[:3, :3]
        upd[:3, 3] = rel[:3, 3] + o - rel[:3, :3] @ o
        t = upd @ t
        m, f2, r2 = evaluate(t)
        history.append((int(m[0]), float(m[1])))
        iterations += 1
        done = abs(fitness - f2) < relative_fitness and abs(rmse - r2) < relative_rmse
        fitness, rmse = f2, r2
        if done:
            break
    out = {"transformation": t, "fitness": fitness, "inlier_rmse": rmse, "iterations": iterations,
           "correspondences": int(m[0]), "history": history}
    if corr is not None:
        out["correspondence_set"] = corr
    return out


def _model_args(xyz: Tensor, obs_offsets: Tensor, obs_points: Tensor, per_image: Tensor, per_image_shape, name: str):
    """Checks of a sparse model held on the device (ops.view_scores / ops.depth_ranges) -> contiguous tensors and N, M."""
    for t, what in ((xyz, "xyz"), (obs_offsets, "obs_offsets"), (obs_points, "obs_points"), (per_image, "per-image cameras")):
        if not _on_device(t):
            raise RuntimeError(f"{name}: {what} must be a CUDA tensor (got {t.device}); there is no CPU fallback")
        if t.device != xyz.device:
            raise RuntimeError(f"{name}: every tensor must be on xyz's device")
    if xyz.dtype != torch.float64 or xyz.dim() != 2 or xyz.shape[1] != 3:
        raise RuntimeError(f"{name}: xyz must be float64 [P,3], got {xyz.dtype} {tuple(xyz.shape)}")
    if obs_offsets.dtype != torch.int32 or obs_offsets.dim() != 1 or obs_offsets.shape[0] < 2:
        raise RuntimeError(f"{name}: obs_offsets must be int32 [N+1] with N >= 1")
    if obs_points.dtype != torch.int32 or obs_points.dim() != 1:
        raise RuntimeError(f"{name}: obs_points must be int32 [M]")
    n = obs_offsets.shape[0] - 1
    if per_image.dtype != torch.float64 or tuple(per_image.shape) != (n,) + tuple(per_image_shape):
        raise RuntimeError(f"{name}: expected float64 {(n,) + tuple(per_image_shape)} per-image cameras, got {per_image.dtype} "
                           f"{tuple(per_image.shape)}")
    return xyz.contiguous(), obs_offsets.contiguous(), obs_points.contiguous(), per_image.contiguous(), n, obs_points.shape[0]


def _workspace(nbytes: int, what: str, device) -> Tensor:
    if nbytes < 0:
        _native.check(int(nbytes), what)
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=device)


def view_scores(xyz: Tensor, obs_offsets: Tensor, obs_points: Tensor, centers: Tensor, theta0: float = 5.0, sigma1: float = 1.0,
                sigma2: float = 10.0) -> Tensor:
    """View selection scores of a sparse model (reference colmap_input.py:336-373): float64 [N,N], symmetric, zero diagonal.
    xyz float64 [P,3], obs_offsets int32 [N+1], obs_points int32 [M] (dense point indices, -1 entries removed), centers
    float64 [N,3]; all CUDA.  One host read: the number of contributions, which sizes the second phase."""
    xyz, offs, pts, ctr, n, m = _model_args(xyz, obs_offsets, obs_points, centers, (3,), "view_scores")
    lib = _native.lib()
    total = torch.empty(1, dtype=torch.int64, device=xyz.device)
    with _device_guard(xyz):
        ws_bytes = int(lib.pmb200_view_scores_workspace_bytes(n, m, 0))
        ws = _workspace(ws_bytes, "view_scores_workspace_bytes", xyz.device)
        rc = lib.pmb200_view_scores_count(offs.data_ptr(), pts.data_ptr(), n, m, total.data_ptr(), ws.data_ptr(), ws_bytes, _stream(xyz))
        _native.check(rc, "view_scores_count")
        t = int(total.item())
        need = int(lib.pmb200_view_scores_workspace_bytes(n, m, t))
        if need < 0:
            _native.check(need, "view_scores_workspace_bytes")
        if need > ws_bytes:  # grow, keeping the first part the count call filled
            grown = torch.empty(need, dtype=torch.uint8, device=xyz.device)
            grown[:ws_bytes].copy_(ws[:ws_bytes])
            ws, ws_bytes = grown, need
        score = torch.empty((n, n), dtype=torch.float64, device=xyz.device)
        rc = lib.pmb200_view_scores(xyz.data_ptr(), xyz.shape[0], offs.data_ptr(), pts.data_ptr(), ctr.data_ptr(), n, m, t, float(theta0),
                                    float(sigma1), float(sigma2), score.data_ptr(), ws.data_ptr(), ws_bytes, _stream(xyz))
    _native.check(rc, "view_scores")
    return score


def depth_ranges(xyz: Tensor, obs_offsets: Tensor, obs_points: Tensor, extrinsics: Tensor) -> Tensor:
    """Relaxed depth range per image (reference colmap_input.py:318-333): float64 [N,2] = the 1 % and 99 % order statistics of
    the z of the image's observations (duplicates included), NaN for an image without observations.  Arguments as
    view_scores, with extrinsics float64 [N,4,4] (world -> camera) instead of the centres."""
    xyz, offs, pts, ext, n, m = _model_args(xyz, obs_offsets, obs_points, extrinsics, (4, 4), "depth_ranges")
    lib = _native.lib()
    out = torch.empty((n, 2), dtype=torch.float64, device=xyz.device)
    with _device_guard(xyz):
        ws_bytes = int(lib.pmb200_depth_ranges_workspace_bytes(n, m))
        ws = _workspace(ws_bytes, "depth_ranges_workspace_bytes", xyz.device)
        rc = lib.pmb200_depth_ranges(xyz.data_ptr(), xyz.shape[0], offs.data_ptr(), pts.data_ptr(), ext.data_ptr(), n, m, out.data_ptr(),
                                     ws.data_ptr(), ws_bytes, _stream(xyz))
    _native.check(rc, "depth_ranges")
    return out


def _camera_struct(camera) -> "_native.CameraStruct":
    """A colmap_input.Camera (model name, width, height, params in COLMAP's order) -> pmb200_camera."""
    from .colmap_input import CAMERA_MODELS

    ids = {name: (k, n) for k, (name, n) in CAMERA_MODELS.items()}
    if camera.model not in ids:
        raise ValueError(f"camera {camera.id}: unknown model {camera.model}")
    model_id, n = ids[camera.model]
    if len(camera.params) != n:
        raise ValueError(f"camera {camera.id}: {camera.model} has {n} parameters, got {len(camera.params)}")
    s = _native.CameraStruct()
    s.model, s.width, s.height = model_id, int(camera.width), int(camera.height)
    for i, v in enumerate(camera.params):
        s.params[i] = float(v)
    return s


def undistort_extents(cameras: Sequence, device="cuda:0") -> Tensor:
    """Border extents of COLMAP's UndistortCamera for each camera (include/patchmatch_b200.h, pmb200_undistort_extents):
    float64 [n,8] on `device` = (left min, left max, right min, right max) of the mapped x, then (top min, top max, bottom
    min, bottom max) of the mapped y.  cameras: colmap_input.Camera tuples.  One upload and one launch."""
    import ctypes

    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"undistort_extents: the H100 path needs a CUDA device (got {dev}); there is no CPU fallback")
    n = len(cameras)
    host = (_native.CameraStruct * max(n, 1))(*[_camera_struct(c) for c in cameras])
    staging = torch.empty(max(n, 1) * ctypes.sizeof(_native.CameraStruct), dtype=torch.uint8, device=dev)
    out = torch.empty((n, 8), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        rc = _native.lib().pmb200_undistort_extents(host, n, staging.data_ptr(), out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        _native.check(rc, "undistort_extents")
        torch.cuda.current_stream(dev).synchronize()  # `host` is pageable and goes out of scope
    return out


UNDISTORT_MIN_SCALE = 0.2
UNDISTORT_MAX_SCALE = 2.0


def undistorted_camera(camera, extents, blank_pixels: float = 0.0):
    """COLMAP's UndistortCamera with its defaults (min_scale 0.2, max_scale 2.0, no ROI, no max_image_size): the PINHOLE
    colmap_input.Camera (same id) with fx, fy kept, size sx W x sy H and the principal point scaled with it, from the
    camera's 8 extents (undistort_extents).  blank_pixels in [0, 1]: 0 keeps only valid pixels, 1 keeps the whole view.
    ValueError naming the camera when a scale is not finite."""
    import math

    import numpy as np

    from .colmap_input import Camera, intrinsic_matrix

    if not 0.0 <= blank_pixels <= 1.0:
        raise ValueError(f"blank_pixels must be in [0, 1], got {blank_pixels}")
    k = intrinsic_matrix(camera)
    fx, fy, cx, cy = float(k[0, 0]), float(k[1, 1]), float(k[0, 2]), float(k[1, 2])
    e = np.asarray(extents.tolist() if hasattr(extents, "tolist") else extents, dtype=np.float64).reshape(8)
    b = np.float64(blank_pixels)
    size = []
    # numpy scalars divide as IEEE doubles (inf / nan, no ZeroDivisionError); Python's min / max pick like std::min / std::max
    for c, n, (lo_min, lo_max, hi_min, hi_max) in ((np.float64(cx), camera.width, e[0:4]), (np.float64(cy), camera.height, e[4:8])):
        with np.errstate(all="ignore"):
            min_s = min(c / (c - lo_min), (n - 0.5 - c) / (hi_max - c))
            max_s = max(c / (c - lo_max), (n - 0.5 - c) / (hi_min - c))
            s = float(1.0 / (min_s * b + max_s * (1.0 - b)))
        if not math.isfinite(s):
            raise ValueError(f"camera {camera.id} ({camera.model}): the undistorted scale is not finite ({s}); check its "
                             "distortion parameters")
        s = max(UNDISTORT_MIN_SCALE, min(s, UNDISTORT_MAX_SCALE))
        size.append(int(max(1.0, s * n)))
    w, h = size
    return Camera(camera.id, "PINHOLE", w, h, [fx, fy, cx * w / camera.width, cy * h / camera.height])


def undistort_image(image: Tensor, camera, pinhole) -> Tensor:
    """Resample an image of the distorted `camera` into the PINHOLE camera `pinhole` (include/patchmatch_b200.h,
    pmb200_undistort_image).  image uint8 [H,W,3] RGB CUDA with H, W the camera's size; camera, pinhole: colmap_input.Camera
    (pinhole: the result of undistorted_camera).  -> uint8 [pinhole.height, pinhole.width, 3] on image's device.  One launch."""
    import ctypes

    if not _on_device(image):
        raise RuntimeError(f"undistort_image: the H100 path needs a CUDA tensor (got {image.device}); there is no CPU fallback")
    if image.dtype != torch.uint8 or tuple(image.shape) != (camera.height, camera.width, 3):
        raise RuntimeError(f"undistort_image: expected uint8 [{camera.height},{camera.width},3] for camera {camera.id}, got "
                           f"{image.dtype} {tuple(image.shape)}")
    if pinhole.model != "PINHOLE":
        raise ValueError(f"undistort_image: the target camera must be PINHOLE, got {pinhole.model}")
    src = image.contiguous()
    out = torch.empty((pinhole.height, pinhole.width, 3), dtype=torch.uint8, device=src.device)
    cam = _camera_struct(camera)
    kp = (ctypes.c_double * 4)(*[float(v) for v in pinhole.params])
    with _device_guard(src):
        rc = _native.lib().pmb200_undistort_image(src.data_ptr(), ctypes.byref(cam), kp, int(pinhole.width), int(pinhole.height),
                                                  out.data_ptr(), _stream(src))
    _native.check(rc, "undistort_image")
    return out


DEPTH_LOSS_MAX_MAPS = 16
DEPTH_METRICS_MAX_THRESHOLDS = 8


def _ground_truth_args(depth_gt: Tensor, mask: Tensor, name: str):
    """float32 [B,H,W] ground truth and uint8 / bool [B,H,W] mask on one device -> contiguous (gt, uint8 mask)."""
    gt = _require(depth_gt, f"{name} (depth_gt)", 3)
    if not _on_device(mask) or mask.device != gt.device or tuple(mask.shape) != tuple(gt.shape):
        raise RuntimeError(f"{name}: mask must be a CUDA tensor of depth_gt's shape {tuple(gt.shape)} on its device, got "
                           f"{tuple(mask.shape)} on {mask.device}")
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    if mask.dtype != torch.uint8:
        raise RuntimeError(f"{name}: mask must be uint8 or bool, got {mask.dtype}")
    return gt, mask.contiguous()


def _level_maps(maps: Sequence[Tensor], levels: Sequence[int], shape, device, name: str):
    """Maps at pyramid levels: each float32 [B, H >> l, W >> l] (a [B,1,h,w] map is taken as [B,h,w]) -> contiguous [B,h,w]."""
    B, H, W = shape
    out = []
    for m, l in zip(maps, levels):
        if not 0 <= int(l) <= 3:
            raise RuntimeError(f"{name}: level {l} outside 0..3")
        want = (B, H >> int(l), W >> int(l))
        t = _require(m, name)
        if t.device != device or t.numel() != want[0] * want[1] * want[2] or tuple(t.shape[-2:]) != want[1:] or t.shape[0] != B:
            raise RuntimeError(f"{name}: a level-{l} map must be {want} (or [B,1,h,w]) on {device}, got {tuple(m.shape)} on {m.device}")
        out.append(t)
    return out


def depth_loss_terms(maps: Sequence[Tensor], levels: Sequence[int], depth_gt: Tensor, mask: Tensor) -> Tensor:
    """The sums behind patchmatchnet_loss (reference models/net.py:321-342) without a host synchronisation: float64
    [n_maps + 4] = for each map, the sum of smooth-L1(d - gt) (beta 1) over the masked pixels of its level, then the mask
    counts of levels 0..3.  Map m is at pyramid level levels[m]; depth_gt float32 [B,H,W] and mask (uint8 or bool) [B,H,W] are
    full resolution, and level l reads them at (y << l, x << l) as F.interpolate(scale_factor=0.5**l, mode="nearest") does.
    Deterministic: reruns are bit-identical."""
    import ctypes

    gt, mk = _ground_truth_args(depth_gt, mask, "depth_loss_terms")
    n = len(maps)
    if len(levels) != n or not 1 <= n <= DEPTH_LOSS_MAX_MAPS:
        raise RuntimeError(f"depth_loss_terms: 1..{DEPTH_LOSS_MAX_MAPS} maps, one level each (got {n} maps, {len(levels)} levels)")
    ms = _level_maps(maps, levels, tuple(gt.shape), gt.device, "depth_loss_terms")
    B, H, W = gt.shape
    lv = (ctypes.c_int * n)(*[int(l) for l in levels])
    lib = _native.lib()
    terms = torch.empty(n + 4, dtype=torch.float64, device=gt.device)
    with _device_guard(gt):
        ws_bytes = int(lib.pmb200_depth_loss_workspace_bytes(lv, n, B, H, W))
        ws = _workspace(ws_bytes, "depth_loss_workspace_bytes", gt.device)
        ptrs, keep = _native.pointer_array([m.data_ptr() for m in ms])
        rc = lib.pmb200_depth_loss(ptrs, lv, n, gt.data_ptr(), mk.data_ptr(), B, H, W, terms.data_ptr(), ws.data_ptr(), ws_bytes,
                                   _stream(gt))
    _native.check(rc, "depth_loss")
    return terms


def depth_loss_backward(maps: Sequence[Tensor], levels: Sequence[int], depth_gt: Tensor, mask: Tensor, terms: Tensor,
                        grad_loss: Tensor, scale: float = 1.0) -> list:
    """Gradient of  loss = sum_m terms[m] / terms[n_maps + levels[m]]  with respect to every map, in one launch:
    mask ? clamp(d - gt, -1, 1) * grad_loss * scale / count_level : 0, each of its map's shape.  grad_loss is a device scalar."""
    gt, mk = _ground_truth_args(depth_gt, mask, "depth_loss_backward")
    n = len(maps)
    if len(levels) != n or not 1 <= n <= DEPTH_LOSS_MAX_MAPS:
        raise RuntimeError(f"depth_loss_backward: 1..{DEPTH_LOSS_MAX_MAPS} maps, one level each")
    ms = _level_maps(maps, levels, tuple(gt.shape), gt.device, "depth_loss_backward")
    if terms.dtype != torch.float64 or tuple(terms.shape) != (n + 4,) or terms.device != gt.device:
        raise RuntimeError(f"depth_loss_backward: terms must be float64 [{n + 4}] on {gt.device}")
    g = _require(grad_loss.reshape(()), "depth_loss_backward (grad_loss)")
    import ctypes

    B, H, W = gt.shape
    grads = [torch.empty_like(m) for m in ms]
    lv = (ctypes.c_int * n)(*[int(l) for l in levels])
    with _device_guard(gt):
        ptrs, keep_m = _native.pointer_array([m.data_ptr() for m in ms])
        gptrs, keep_g = _native.pointer_array([t.data_ptr() for t in grads])
        rc = _native.lib().pmb200_depth_loss_backward(ptrs, lv, n, gt.data_ptr(), mk.data_ptr(), B, H, W, terms.contiguous().data_ptr(),
                                                      g.data_ptr(), float(scale), gptrs, _stream(gt))
    _native.check(rc, "depth_loss_backward")
    return [t.view_as(m) for t, m in zip(grads, maps)]


def depth_metrics(maps: Sequence[Tensor], depth_gt: Tensor, mask: Tensor, thresholds: Sequence[float] = (1.0, 2.0, 4.0, 8.0)) -> Tensor:
    """Per-image sums behind the reference's absolute_depth_error_metrics and threshold_metrics (utils.py:187-221), without a
    host synchronisation.  maps: the four maps of levels 0..3 (float32 [B, H >> l, W >> l]); -> float64 [B, 8 + n_thr]:
    the sum of |d - gt| over the masked pixels of levels 0..3, the mask counts of levels 0..3, and per threshold the number
    of masked level-0 pixels with float32 |d - gt| > t.  Exact counts: rates formed from them match the reference bit for bit."""
    import ctypes

    gt, mk = _ground_truth_args(depth_gt, mask, "depth_metrics")
    if len(maps) != 4:
        raise RuntimeError("depth_metrics: one map for each of the levels 0..3")
    if len(thresholds) > DEPTH_METRICS_MAX_THRESHOLDS:
        raise RuntimeError(f"depth_metrics: at most {DEPTH_METRICS_MAX_THRESHOLDS} thresholds")
    ms = _level_maps(maps, range(4), tuple(gt.shape), gt.device, "depth_metrics")
    B, H, W = gt.shape
    thr = (ctypes.c_float * max(len(thresholds), 1))(*[float(t) for t in thresholds])
    out = torch.empty((B, 8 + len(thresholds)), dtype=torch.float64, device=gt.device)
    with _device_guard(gt):
        ptrs, keep = _native.pointer_array([m.data_ptr() for m in ms])
        rc = _native.lib().pmb200_depth_metrics(ptrs, gt.data_ptr(), mk.data_ptr(), B, H, W, thr, len(thresholds), out.data_ptr(),
                                                _stream(gt))
    _native.check(rc, "depth_metrics")
    return out
