"""Caller-side shell: ``PatchmatchNet`` with the reference constructor / forward
signatures and parameter names (reference ``models/net.py:125-301``).

Only ``PatchMatch`` (the hot path) is native H100 code.  The dense 2-D convs of
the feature pyramid and the refinement head stay library ops (cuDNN), as the
scope table (SURVEY.md 8a/8f) says; they are here because the reference's
``models/net.py`` does not exist on the GPU box and the end-to-end metric
(depth-maps/s) is quoted on the full cascade.  When the reference *is*
importable, ``patchmatchnet_b200.PatchMatch`` drops into its unmodified
``models/net.py`` instead (see INTEGRATION.md, tests/test_dropin_reference.py).

The stage module class is a constructor argument so that the oracle
(``oracle.pm_oracle.PatchMatchOracle``) can be timed/checked behind the very
same shell by tests and by bench.py's CPU-baseline leg.
"""
from __future__ import annotations

from typing import Dict, List, Tuple, Type

import torch
import torch.nn as nn
import torch.nn.functional as F

Tensor = torch.Tensor


def _fold_bn(weight: Tensor, bn: nn.BatchNorm2d, out_dim: int = 0):
    """Eval-mode BatchNorm folded into the preceding (bias-free) convolution: returns (weight', bias')."""
    scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    shape = [1] * weight.dim()
    shape[out_dim] = -1
    w = (weight.double() * scale.view(shape)).float()
    b = (bn.bias.double() - bn.running_mean.double() * scale).float()
    return w, b


# The caller-side shell (FeatureNet, Refinement, stage glue) has CUDA eval fast paths: BatchNorm folded into cuDNN
# conv+bias+ReLU calls on channels-last data, views stacked into one batch, batched projection matrices, native
# upsample+add and confidence tail.  Setting this False makes the shell issue the reference's own op sequence
# (bench.py uses that, with the oracle stage module, to time "the reference in eager PyTorch on this GPU").
LIBRARY_FAST_PATH = True


def _fast(x: Tensor) -> bool:
    """Inference fast paths (BatchNorm folded into constant weights, cuDNN fused conv+ReLU, native convs) have no
    derivative: they are taken only when autograd is off.  In eval() with grad enabled -- frozen-BN fine-tuning,
    gradient analysis -- the shell issues the reference's own differentiable op sequence, as the reference does."""
    return LIBRARY_FAST_PATH and x.is_cuda and not torch.is_grad_enabled()


class _FoldCache:
    """Caches derived (folded / packed) weights until any source tensor is modified or moved.  The (stamp, value)
    pair is one attribute, read and written whole: module replicas (nn.DataParallel threads) may share a cache object,
    and then at worst recompute -- a caller never gets another device's value."""

    def __init__(self) -> None:
        self._entry = (None, None)

    def get(self, tensors, make, key=None):
        stamp = (key,) + tuple((t.data_ptr(), t._version, t.device) for t in tensors)
        have, value = self._entry
        if stamp != have:
            with torch.no_grad():
                value = make()
            self._entry = (stamp, value)
        return value


_FUSED_CONV_RELU = hasattr(torch, "cudnn_convolution_relu")

def _native_convs(x: Tensor) -> bool:
    """Eval mode on CUDA: every conv of the shell (FeatureNet, Refinement) runs through the native channels-last
    tensor-core conv (csrc/pm_conv.cu, ops.conv2d_nhwc) instead of cuDNN, unless ops.NATIVE_CONVS is False
    (PMB200_NATIVE_CONVS=0), which keeps the folded cuDNN calls -- bench.py uses that for an A/B line."""
    from . import ops

    return ops.NATIVE_CONVS and _fast(x) and not torch.is_grad_enabled()


def ops_prefers(conv: nn.Conv2d) -> bool:
    from . import ops

    return ops.conv_prefers_native(conv.in_channels, conv.out_channels, conv.kernel_size[0])


class _PackedConv:
    """Fragment-ordered filter (+ bias) of a plain nn.Conv2d, cached until the weights change or move."""

    def __init__(self) -> None:
        self._cache = _FoldCache()

    def __call__(self, conv: nn.Conv2d, x: Tensor, relu: bool = False, with_bias: bool = True) -> Tensor:
        from . import ops

        srcs = [conv.weight] + ([conv.bias] if conv.bias is not None else [])
        mode = ops.conv_tc5_mode(conv.in_channels, conv.out_channels, conv.kernel_size[0], conv.stride[0])
        if mode:
            frag, bias = self._cache.get(
                srcs, lambda: (ops.pack_conv_filter_tc5_for(conv.weight, mode), None if conv.bias is None else conv.bias.detach().clone()),
                key="tc5" + mode)
            return ops.conv2d_tc5(x, frag, bias if with_bias else None, conv.out_channels, conv.kernel_size[0], conv.stride[0],
                                  conv.padding[0], conv.dilation[0], relu=relu, halo=mode == "halo")
        prec = ops.conv_precision()
        frag, bias = self._cache.get(
            srcs, lambda: (ops.pack_conv_filter(conv.weight, prec), None if conv.bias is None else conv.bias.detach().clone()), key=prec)
        return ops.conv2d_nhwc(x, frag, bias if with_bias else None, conv.out_channels, conv.kernel_size[0], conv.stride[0],
                               conv.padding[0], conv.dilation[0], relu=relu)


class _ConvBnReLU2d(nn.Module):
    """conv2d (no bias) + BatchNorm2d + ReLU; children named ``conv`` / ``bn`` as in the reference
    checkpoints (reference models/module.py:11-40).

    Training, or CPU: the three ops as written in the reference.  Eval on CUDA: BatchNorm is folded into
    the conv weights (cached) and conv + bias + ReLU run as ONE cuDNN call on channels-last data -- the
    separate cudnn bn_fw_inf kernel would otherwise be a launch (and a full activation pass) per layer."""

    def __init__(self, cin: int, cout: int, k: int = 3, stride: int = 1, pad: int = 1) -> None:
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=pad, bias=False)
        self.bn = nn.BatchNorm2d(cout)
        self._cache = _FoldCache()
        self._frag_cache = _FoldCache()
        self._tc5_cache = _FoldCache()

    def folded_frag(self):
        """(fragment-ordered folded filter, folded bias) for the native conv."""
        from . import ops

        bn = self.bn
        srcs = [self.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        prec = ops.conv_precision()

        def make():
            w, b = _fold_bn(self.conv.weight, bn)
            return ops.pack_conv_filter(w, prec), b.contiguous()

        return self._frag_cache.get(srcs, make, key=prec)

    def folded_tc5(self, mode: str):
        """(filter image for the wgmma conv in the given form, folded bias)."""
        from . import ops

        bn = self.bn
        srcs = [self.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        def make():
            w, b = _fold_bn(self.conv.weight, bn)
            return ops.pack_conv_filter_tc5_for(w, mode), b.contiguous()

        return self._tc5_cache.get(srcs, make, key=mode)

    def native(self, x: Tensor, out: Tensor = None, out_channel_offset: int = 0) -> Tensor:
        from . import ops

        c = self.conv
        mode = ops.conv_tc5_mode(c.in_channels, c.out_channels, c.kernel_size[0], c.stride[0])
        if mode:
            frag, b = self.folded_tc5(mode)
            return ops.conv2d_tc5(x, frag, b, c.out_channels, c.kernel_size[0], c.stride[0], c.padding[0], c.dilation[0],
                                  relu=True, out=out, out_channel_offset=out_channel_offset, halo=mode == "halo")
        frag, b = self.folded_frag()
        return ops.conv2d_nhwc(x, frag, b, c.out_channels, c.kernel_size[0], c.stride[0], c.padding[0], c.dilation[0],
                               relu=True, out=out, out_channel_offset=out_channel_offset)

    def folded(self):
        bn = self.bn
        srcs = [self.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        def make():
            w, b = _fold_bn(self.conv.weight, bn)
            return w.contiguous(memory_format=torch.channels_last), b

        return self._cache.get(srcs, make)

    def forward(self, x: Tensor) -> Tensor:
        if self.training or not _fast(x):
            return F.relu(self.bn(self.conv(x)), inplace=True)
        c = self.conv
        if _native_convs(x) and ops_prefers(c):
            return self.native(x)
        w, b = self.folded()
        c = self.conv
        if _FUSED_CONV_RELU:
            return torch.cudnn_convolution_relu(x, w, b, c.stride, c.padding, c.dilation, 1)
        return F.relu_(F.conv2d(x, w, b, c.stride, c.padding, c.dilation))


class FeatureNet(nn.Module):
    """Three-level feature pyramid (reference models/net.py:9-70): 1/8 x 64ch,
    1/4 x 32ch, 1/2 x 16ch, keyed 3 / 2 / 1."""

    def __init__(self) -> None:
        super().__init__()
        spec = [  # (cin, cout, k, stride, pad)
            (3, 8, 3, 1, 1), (8, 8, 3, 1, 1),
            (8, 16, 5, 2, 2), (16, 16, 3, 1, 1), (16, 16, 3, 1, 1),
            (16, 32, 5, 2, 2), (32, 32, 3, 1, 1), (32, 32, 3, 1, 1),
            (32, 64, 5, 2, 2), (64, 64, 3, 1, 1), (64, 64, 3, 1, 1),
        ]
        for i, s in enumerate(spec):
            setattr(self, f"conv{i}", _ConvBnReLU2d(*s))
        self.output1 = nn.Conv2d(64, 64, 1, bias=False)
        self.inner1 = nn.Conv2d(32, 64, 1, bias=True)
        self.inner2 = nn.Conv2d(16, 64, 1, bias=True)
        self.output2 = nn.Conv2d(64, 32, 1, bias=False)
        self.output3 = nn.Conv2d(64, 16, 1, bias=False)
        self._packed = {n: _PackedConv() for n in ("output1", "inner1", "inner2", "output2", "output3")}
        self._composed_cache = _FoldCache()
        self._stem_cache = _FoldCache()
        self.fuse_top_down = True  # eval mode on CUDA: composed 1x1 heads (see composed_heads); False = layer by layer

    def _plain(self, name: str, x: Tensor) -> Tensor:
        """One of the bias-free / lateral 1x1 convs: native in eval mode on CUDA, else the module itself."""
        if not self.training and _native_convs(x):
            return self._packed[name](getattr(self, name), x)
        return getattr(self, name)(x)

    def _trunk(self, x: Tensor, lo: int, hi: int) -> Tensor:
        for i in range(lo, hi + 1):
            x = getattr(self, f"conv{i}")(x)
        return x

    def composed_heads(self) -> Dict[str, Tensor]:
        """The top-down path with its 1x1 convs composed.  Every op between the trunk and the three outputs is linear
        (1x1 convs, bilinear upsampling, additions) and 1x1 convs commute with the upsampling, so with
        W2 = output2, W3 = output3, (Wi1, bi1) = inner1, (Wi2, bi2) = inner2 (reference net.py:52-66):
            out2 = W2 top2            = up(W2 eighth) + (W2 Wi1) quarter + W2 bi1
            t    = W3 top2            = up(W3 eighth) + (W3 Wi1) quarter + W3 bi1
            out1 = W3 (up(top2) + Wi2 half + bi2) = up(t) + (W3 Wi2) half + W3 bi2
        and the 64-channel maps top2 (26 MB at 640x512 x 5 views) and top1 (105 MB, written once and read twice) never
        exist.  Products in fp64, rounded once.  Pure tensor algebra: CPU-testable."""
        f = lambda conv: conv.weight.detach().double().flatten(1)
        W2, W3, Wi1, Wi2 = f(self.output2), f(self.output3), f(self.inner1), f(self.inner2)
        bi1, bi2 = self.inner1.bias.detach().double(), self.inner2.bias.detach().double()
        as4 = lambda m: m.float().reshape(m.shape[0], m.shape[1], 1, 1).contiguous()
        return {"u_o": as4(W2), "u_t": as4(W3), "l2_o": as4(W2 @ Wi1), "l2_t": as4(W3 @ Wi1), "l1": as4(W3 @ Wi2),
                "c2_o": (W2 @ bi1).float(), "c2_t": (W3 @ bi1).float(), "c1": (W3 @ bi2).float()}

    def _fused_top_down(self, eighth: Tensor, quarter: Tensor, half: Tensor) -> Dict[int, Tensor]:
        """Eval mode on CUDA: six native launches (1x1 convs, the upsample+add fused into the lateral conv's epilogue)."""
        from . import ops

        srcs = [self.output2.weight, self.output3.weight, self.inner1.weight, self.inner1.bias, self.inner2.weight, self.inner2.bias]
        prec = ops.conv_precision()

        def make():
            h = self.composed_heads()
            packed = {k: ops.pack_conv_filter(v, prec) for k, v in h.items() if v.dim() == 4}
            packed.update({k: v.contiguous() for k, v in h.items() if v.dim() == 1})
            return packed

        w = self._composed_cache.get(srcs, make, key=prec)
        out: Dict[int, Tensor] = {3: self._plain("output1", eighth)}
        u_o = ops.conv2d_nhwc(eighth, w["u_o"], None, 32, 1)
        u_t = ops.conv2d_nhwc(eighth, w["u_t"], None, 16, 1)
        out[2] = ops.conv2d_nhwc(quarter, w["l2_o"], w["c2_o"], 32, 1, add_up2x=u_o)
        t = ops.conv2d_nhwc(quarter, w["l2_t"], w["c2_t"], 16, 1, add_up2x=u_t)
        out[1] = ops.conv2d_nhwc(half, w["l1"], w["c1"], 16, 1, add_up2x=t)
        return out

    def stem_weights(self):
        """BatchNorm-folded (w0, b0, w1, b1) of conv0 / conv1 as HOST tensors: K-S carries them in its kernel parameter block."""
        srcs = []
        for m in (self.conv0, self.conv1):
            srcs += [m.conv.weight, m.bn.weight, m.bn.bias, m.bn.running_mean, m.bn.running_var]

        def make():
            w0, b0 = _fold_bn(self.conv0.conv.weight, self.conv0.bn)
            w1, b1 = _fold_bn(self.conv1.conv.weight, self.conv1.bn)
            return tuple(t.detach().float().cpu().contiguous() for t in (w0, b0, w1, b1))

        return self._stem_cache.get(srcs, make)

    def _stem(self, x: Tensor) -> Tensor:
        """conv0 -> conv1.  Eval mode on CUDA in the fp32-accurate mode: ONE exact-fp32 launch reading the NCHW image planes in
        place (K-S, csrc/pm_stem.cu); otherwise the two layers one after the other."""
        from . import ops

        if (not self.training and _native_convs(x) and ops.STEM_FUSED and ops.conv_precision() == 3 and x.dim() == 4 and x.shape[1] == 3
                and x.dtype == torch.float32):
            return ops.conv_stem(x, *self.stem_weights())
        if _fast(x) and not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        return self._trunk(x, 0, 1)

    def forward(self, x: Tensor) -> Dict[int, Tensor]:
        half = self._trunk(self._stem(x), 2, 4)
        quarter = self._trunk(half, 5, 7)
        eighth = self._trunk(quarter, 8, 10)
        if not self.training and _native_convs(x) and self.fuse_top_down:
            return self._fused_top_down(eighth, quarter, half)
        out: Dict[int, Tensor] = {3: self._plain("output1", eighth)}
        top = self._top_down(eighth, "inner1", quarter)
        out[2] = self._plain("output2", top)
        top = self._top_down(top, "inner2", half)
        out[1] = self._plain("output3", top)
        return out

    def _top_down(self, coarse: Tensor, lateral_name: str, fine: Tensor) -> Tensor:
        """bilinear x2 upsample + lateral 1x1 conv (reference net.py:60-66).  On CUDA in eval mode the upsample, the
        add and the lateral conv's bias are ONE native launch (ATen's channels-last bilinear kernel was the single
        largest launch of the forward, the bias add another full pass over the largest tensor)."""
        lateral_conv = getattr(self, lateral_name)
        if _fast(coarse) and not self.training and not torch.is_grad_enabled():
            from . import ops

            if _native_convs(fine):
                lateral = self._packed[lateral_name](lateral_conv, fine, with_bias=False)
            else:
                lateral = F.conv2d(fine, lateral_conv.weight, None)
            return ops.upsample2x_add(coarse, lateral, lateral_conv.bias)
        return F.interpolate(coarse, scale_factor=2.0, mode="bilinear", align_corners=False) + lateral_conv(fine)


class Refinement(nn.Module):
    """Residual depth refinement from 1/2 to full resolution (reference models/net.py:73-122)."""

    def __init__(self) -> None:
        super().__init__()
        self.conv0 = _ConvBnReLU2d(3, 8)
        self.conv1 = _ConvBnReLU2d(1, 8)
        self.conv2 = _ConvBnReLU2d(8, 8)
        self.deconv = nn.ConvTranspose2d(8, 8, 3, padding=1, output_padding=1, stride=2, bias=False)
        self.bn = nn.BatchNorm2d(8)
        self.conv3 = _ConvBnReLU2d(16, 8)
        self.res = nn.Conv2d(8, 1, 3, padding=1, bias=False)
        self._cache = _FoldCache()
        self._deconv_frag = _FoldCache()
        self._host_cache = _FoldCache()
        self._res_packed = _PackedConv()

    def _native_tail(self, img: Tensor, d: Tensor) -> Tensor:
        """conv1 -> conv2 -> transposed conv (BatchNorm folded, ReLU) and conv0(img) written straight into the two
        halves of one 16-channel buffer (no torch.cat), -> conv3 -> res: six native launches."""
        from . import ops

        bn = self.bn
        srcs = [self.deconv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        prec = ops.conv_precision()

        def make():
            w, b = _fold_bn(self.deconv.weight, bn, out_dim=1)
            return ops.pack_conv_filter(w, prec, transposed=True), b.contiguous()

        frag, b = self._deconv_frag.get(srcs, make, key=prec)
        low = self.conv2.native(self.conv1.native(d))
        N, _, h, w = low.shape
        both = torch.empty((N, 16, 2 * h, 2 * w), dtype=torch.float32, device=low.device, memory_format=torch.channels_last)
        # ConvTranspose2d(k=3, stride=2, padding=1, output_padding=1) == stride-1 conv (pad 3-1-1 = 1) over the zero-stuffed input
        ops.conv2d_nhwc(low, frag, b, 8, 3, 1, 1, 1, relu=True, transposed2x=True, out=both, out_channel_offset=0)
        self.conv0.native(img, out=both, out_channel_offset=8)
        return self._res_packed(self.res, self.conv3.native(both))

    def _upsample(self, x: Tensor) -> Tensor:
        if self.training or not _fast(x):
            return F.relu(self.bn(self.deconv(x)), inplace=True)
        bn = self.bn
        srcs = [self.deconv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]
        w, b = self._cache.get(srcs, lambda: _fold_bn(self.deconv.weight, bn, out_dim=1))
        return F.relu_(F.conv_transpose2d(x, w, b, stride=2, padding=1, output_padding=1))

    def host_weights(self):
        """BatchNorm-folded weights of the six layers as HOST tensors, in the argument order of ops.refine_low (first four) and
        ops.refine_full (the rest): K-R carries them in its kernel parameter blocks."""
        srcs = [self.deconv.weight, self.res.weight, self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var]
        for m in (self.conv0, self.conv1, self.conv2, self.conv3):
            srcs += [m.conv.weight, m.bn.weight, m.bn.bias, m.bn.running_mean, m.bn.running_var]

        def make():
            host = lambda t: t.detach().float().cpu().contiguous()  # noqa: E731
            w1, b1 = _fold_bn(self.conv1.conv.weight, self.conv1.bn)
            w2, b2 = _fold_bn(self.conv2.conv.weight, self.conv2.bn)
            wd, bd = _fold_bn(self.deconv.weight, self.bn, out_dim=1)
            w0, b0 = _fold_bn(self.conv0.conv.weight, self.conv0.bn)
            w3, b3 = _fold_bn(self.conv3.conv.weight, self.conv3.bn)
            return tuple(host(t) for t in (w1, b1, w2, b2, wd, bd, w0, b0, w3, b3, self.res.weight))

        return self._host_cache.get(srcs, make)

    def _fused(self, img: Tensor, depth_half: Tensor, depth_min: Tensor, depth_max: Tensor) -> Tensor:
        """Eval mode on CUDA, fp32-accurate mode: the whole module in two exact-fp32 launches (K-R)."""
        from . import ops

        hw = self.host_weights()
        low = ops.refine_low(depth_half, depth_min, depth_max, *hw[:4])
        return ops.refine_full(low, img, depth_half, depth_min, depth_max, *hw[4:])

    def forward(self, img: Tensor, depth_half: Tensor, depth_min: Tensor, depth_max: Tensor) -> Tensor:
        from . import ops

        if (not self.training and _native_convs(img) and ops.REFINE_FUSED and ops.conv_precision() == 3 and img.dtype == torch.float32
                and img.shape[-2:] == (2 * depth_half.shape[-2], 2 * depth_half.shape[-1]) and self.res.bias is None):
            return self._fused(img, depth_half.float(), depth_min.float(), depth_max.float())
        B = depth_min.size(0)
        lo = depth_min.view(B, 1, 1, 1)
        span = (depth_max - depth_min).view(B, 1, 1, 1)
        d = (depth_half - lo) / span
        if _fast(img) and not self.training:
            img = img.contiguous(memory_format=torch.channels_last)
        if not self.training and _native_convs(img) and img.shape[-2:] == (2 * d.shape[-2], 2 * d.shape[-1]):
            res = self._native_tail(img, d)
        else:
            up = self._upsample(self.conv2(self.conv1(d)))
            res = self.res(self.conv3(torch.cat((up, self.conv0(img)), dim=1)))
        d = F.interpolate(d, scale_factor=2.0, mode="nearest") + res
        return d * span + lo


def _adjacent_views(tensors) -> bool:
    """True when the tensors are equally shaped contiguous views laid out back to back in ONE storage
    (e.g. slices of a stacked buffer), so that they can be re-viewed as one batch without a copy."""
    first = tensors[0]
    if not first.is_contiguous():
        return False
    store = first.untyped_storage().data_ptr()
    for i, t in enumerate(tensors):
        if (t.shape != first.shape or not t.is_contiguous() or t.untyped_storage().data_ptr() != store
                or t.storage_offset() != first.storage_offset() + i * first.numel()):
            return False
    return True


def _round_dims_to_8(images: List[Tensor], intrinsics: Tensor) -> Tuple[List[Tensor], Tensor, int, int]:
    """reference models/net.py:304-318 (mutates ``intrinsics`` in place like the reference)."""
    H0, W0 = images[0].shape[-2:]
    for i, im in enumerate(images):
        h, w = im.shape[-2:]
        nh, nw = int(round(h / 8)) * 8, int(round(w / 8)) * 8
        if (nh, nw) != (h, w):
            intrinsics[:, i, 0] *= nw / w
            intrinsics[:, i, 1] *= nh / h
            images[i] = F.interpolate(im, size=[nh, nw], mode="bilinear", align_corners=False)
    return images, intrinsics, H0, W0


class PatchmatchNet(nn.Module):
    """Coarse-to-fine cascade: features -> PatchMatch on stages 3, 2, 1 -> refinement.

    Constructor and ``forward`` mirror reference models/net.py:128-136 / :176-301;
    ``patchmatch_cls`` (extra, keyword-only) selects the stage implementation.
    """

    GROUPS = (4, 8, 8)  # net.py:158
    FEATURES = (16, 32, 64)  # net.py:153

    def __init__(
        self,
        patchmatch_interval_scale: List[float],
        propagation_range: List[int],
        patchmatch_iteration: List[int],
        patchmatch_num_sample: List[int],
        propagate_neighbors: List[int],
        evaluate_neighbors: List[int],
        *,
        patchmatch_cls: Type[nn.Module] = None,
    ) -> None:
        super().__init__()
        if patchmatch_cls is None:
            from .patchmatch import PatchMatch as patchmatch_cls  # the H100-native stage
        self.stages = 4
        self.feature = FeatureNet()
        self.patchmatch_num_sample = patchmatch_num_sample
        self.propagate_neighbors = propagate_neighbors
        self.evaluate_neighbors = evaluate_neighbors
        self.G = list(self.GROUPS)
        for i in range(self.stages - 1):
            setattr(
                self,
                f"patchmatch_{i + 1}",
                patchmatch_cls(
                    propagation_out_range=propagation_range[i],
                    patchmatch_iteration=patchmatch_iteration[i],
                    patchmatch_num_sample=patchmatch_num_sample[i],
                    patchmatch_interval_scale=patchmatch_interval_scale[i],
                    num_feature=self.FEATURES[i],
                    G=self.G[i],
                    propagate_neighbors=propagate_neighbors[i],
                    evaluate_neighbors=evaluate_neighbors[i],
                    stage=i + 1,
                ),
            )
        self.upsample_net = Refinement()
        self.register_buffer("_stage_scales", torch.tensor([0.125, 0.25, 0.5]).view(3, 1, 1, 1, 1), persistent=False)
        # eval mode: push all views through FeatureNet as one batch (set False to go view by view)
        self.stack_views = True

    def extract_features(self, images: List[Tensor]) -> List[Dict[int, Tensor]]:
        """One FeatureNet pass per view (reference net.py:203-208).  In eval mode the
        views are stacked into one batch (BatchNorm uses running statistics, so the
        per-sample result is unchanged and the launch count drops N-fold)."""
        if self.training or not self.stack_views or len({im.shape for im in images}) != 1:
            return [self.feature(im) for im in images]
        n, b = len(images), images[0].shape[0]
        first = images[0]
        if _adjacent_views(images):
            x = torch.as_strided(first, (n * b,) + tuple(first.shape[1:]), first.stride())  # views of one buffer: no copy
        else:
            x = torch.cat(images, dim=0)
        if _fast(x):  # the pyramid comes out channels-last, the layout the fused PatchMatch kernels read in place.  FeatureNet's
            # first layers read the NCHW planes themselves (K-S) or convert; only the reference view is needed channels-last
            # again, by Refinement's conv-family path; its fused form (K-R) reads the NCHW planes itself
            from . import ops

            if not (ops.REFINE_FUSED and ops.NATIVE_CONVS and ops.conv_precision() == 3):
                self._ref_image_cl = first.contiguous(memory_format=torch.channels_last)
        stacked = self.feature(x)
        return [{k: v[i * b:(i + 1) * b] for k, v in stacked.items()} for i in range(n)]

    def forward(
        self,
        images: List[Tensor],
        intrinsics: Tensor,
        extrinsics: Tensor,
        depth_min: Tensor,
        depth_max: Tensor,
    ) -> Tuple[Tensor, Tensor, Dict[int, List[Tensor]]]:
        assert len(images) == intrinsics.size(1), "Different number of images and intrinsic matrices"
        assert len(images) == extrinsics.size(1), "Different number of images and extrinsic matrices"
        images = list(images)
        images, intrinsics, H0, W0 = _round_dims_to_8(images, intrinsics)
        ref_image = images[0]
        Hr, Wr = ref_image.shape[-2:]

        self._ref_image_cl = None
        feats = self.extract_features(images)
        ref_feat, src_feats = feats[0], feats[1:]
        if self._ref_image_cl is not None:  # same values as ref_image, channels-last memory (eval fast path only)
            ref_image = self._ref_image_cl
            self._ref_image_cl = None
        # (when Refinement runs fused -- K-R reads the NCHW planes in place -- no channels-last copy was made)
        depth_min = depth_min.float()
        depth_max = depth_max.float()

        dev = intrinsics.device
        depth = torch.empty(0, device=dev)
        score = torch.empty(0, device=dev)
        view_weights = torch.empty(0, device=dev)
        per_stage: Dict[int, List[Tensor]] = {}

        all_proj = None
        if _fast(intrinsics):  # the three stages' projection matrices in one batch (5 launches instead of 15)
            K3 = intrinsics.unsqueeze(0).repeat(3, 1, 1, 1, 1)
            K3[:, :, :, :2] *= self._stage_scales
            all_proj = extrinsics.unsqueeze(0).repeat(3, 1, 1, 1, 1)
            all_proj[:, :, :, :3, :4] = torch.matmul(K3, extrinsics[:, :, :3, :4])
        scale = 0.125
        for stage in (3, 2, 1):
            if all_proj is not None:
                proj = all_proj[3 - stage]
            else:  # reference order of operations (net.py:226-231), kept bit-exact on the CPU
                K = intrinsics.clone()
                K[:, :, :2] *= scale
                proj = extrinsics.clone()
                proj[:, :, :3, :4] = torch.matmul(K, extrinsics[:, :, :3, :4])
            projs = torch.unbind(proj, 1)
            scale *= 2.0
            depths, score, view_weights = getattr(self, f"patchmatch_{stage}")(
                ref_feature=ref_feat[stage],
                src_features=[f[stage] for f in src_feats],
                ref_proj=projs[0],
                src_projs=projs[1:],
                depth_min=depth_min,
                depth_max=depth_max,
                depth=depth,
                view_weights=view_weights,
            )
            per_stage[stage] = depths
            depth = depths[-1].detach()
            if stage > 1:
                depth = F.interpolate(depth, scale_factor=2.0, mode="nearest")
                view_weights = F.interpolate(view_weights, scale_factor=2.0, mode="nearest")

        depth = self.upsample_net(ref_image, depth, depth_min, depth_max)
        if (Hr, Wr) != (H0, W0):
            depth = F.interpolate(depth, size=[H0, W0], mode="bilinear", align_corners=False)
        per_stage[0] = [depth]
        if self.training:
            return depth, torch.empty(0, device=dev), per_stage

        # photometric confidence (net.py:289-299): probability mass of the 4 hypotheses around the regressed index
        if _fast(score) and not torch.is_grad_enabled() and score.shape[1] == self.patchmatch_num_sample[0]:
            from . import ops

            return depth, ops.photometric_confidence(score, H0, W0), per_stage
        D = self.patchmatch_num_sample[0]
        mass4 = 4 * F.avg_pool3d(F.pad(score.unsqueeze(1), pad=(0, 0, 0, 0, 1, 2)), (4, 1, 1), stride=1, padding=0).squeeze(1)
        idx = torch.sum(score * torch.arange(D, device=score.device, dtype=torch.float).view(1, D, 1, 1), dim=1)
        idx = idx.unsqueeze(1).long().clamp(0, D - 1)
        conf = torch.gather(mass4, 1, idx)
        conf = F.interpolate(conf, size=[H0, W0], mode="nearest").squeeze(1)
        return depth, conf, per_stage


def patchmatchnet_loss(depth_patchmatch: Dict[int, List[Tensor]], depth_gt: List[Tensor], mask: List[Tensor]) -> Tensor:
    """Sum over the 4 pyramid levels and every PatchMatch iteration of the masked smooth-L1 depth error
    (reference models/net.py:321-342).  depth_gt / mask are per-level lists, finest first."""
    loss = 0
    for level in range(4):
        gt = depth_gt[level][mask[level]]
        for depth in depth_patchmatch[level]:
            loss = loss + F.smooth_l1_loss(depth[mask[level]], gt, reduction="mean")
    return loss


def load_reference_state(model: nn.Module, state: Dict[str, Tensor]) -> None:
    """Load a reference checkpoint's ``["model"]`` dict (keys carry the DataParallel
    ``module.`` prefix, reference eval.py:33-35) and insist every key matches."""
    clean = {(k[7:] if k.startswith("module.") else k): v for k, v in state.items()}
    missing, unexpected = model.load_state_dict(clean, strict=False)
    if missing or unexpected:
        raise RuntimeError(f"state dict mismatch: missing={missing} unexpected={unexpected}")
