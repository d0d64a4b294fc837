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

import os
from typing import Dict, List, Optional, Tuple, Type

import torch
import torch.nn as nn
import torch.nn.functional as F

Tensor = torch.Tensor


def _freeze_after_load(module, incompatible_keys) -> None:
    if not module.training and _freezing():
        module.freeze_script()


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


def ops_prefers(conv: nn.Conv2d) -> bool:
    from . import ops

    return ops.conv_prefers_native(conv.in_channels, conv.out_channels, conv.kernel_size[0])


# ---- TorchScript -------------------------------------------------------------------------------------------------------------
# A scripted network runs the eval-mode launch sequence of the eager one through `torch.ops.pmb200.*` (csrc/torch_binding.cpp).
# What eager decides per call (LIBRARY_FAST_PATH, ops.conv_precision(), ops.conv_form, ...) and the folded / packed weights it
# caches are frozen when the module goes to eval mode (eval(), or load_state_dict in eval mode):
# the call the reference makes right before torch.jit.script (train.py:52-53).  Frozen values are plain HOST tensors and Python
# scalars, never state-dict entries; the operators keep device copies of the host tensors (one upload per device).
# Native conv forms: 0 = the mma.sync kernel (conv2d_nhwc, fragment-ordered filter), 1 = the wgmma tap form, 2 = the wgmma
# halo-tile form (conv2d_tc5).  Layer modes: 0 = the reference op sequence, 1 = ATen's convolution on the folded weights, 2 = native.


def _freezing() -> bool:
    """False in a process that must not map the native libraries (PMB200_SKIP_TORCH_OPS=1, bench.py's reference arm): the
    freeze asks the library which conv forms it serves."""
    return os.environ.get("PMB200_SKIP_TORCH_OPS") != "1"


def _host(t: Tensor) -> Tensor:
    return t.detach().float().cpu()


def _script_conv(x: Tensor, form: int, filt: Tensor, bias: Optional[Tensor], cout: int, ks: int, stride: int, pad: int, dil: int,
                 relu: bool, precision: int, out: Optional[Tensor] = None, out_channel_offset: int = 0,
                 add_up2x: Optional[Tensor] = None, transposed2x: bool = False) -> Tensor:
    """A native conv in the scripted forward: ops.conv2d_nhwc (form 0) or ops.conv2d_tc5 (forms 1, 2), written into `out` at a
    channel offset when given, else into a new channels-last tensor."""
    H, W = x.size(2), x.size(3)
    if transposed2x:
        H, W = 2 * H, 2 * W
    if out is None:
        Ho = (H + 2 * pad - dil * (ks - 1) - 1) // stride + 1
        Wo = (W + 2 * pad - dil * (ks - 1) - 1) // stride + 1
        out = torch.empty([x.size(0), cout, Ho, Wo], dtype=torch.float32, device=x.device, memory_format=torch.channels_last)
    if form == 0:
        torch.ops.pmb200.conv2d_nhwc_out(x, filt, bias, cout, ks, stride, pad, dil, relu, precision, transposed2x, add_up2x, out,
                                         out_channel_offset)
    else:
        torch.ops.pmb200.conv2d_tc5_out(x, filt, bias, cout, ks, stride, pad, dil, relu, form == 2, out, out_channel_offset)
    return out


def _nonempty(t: Tensor) -> Optional[Tensor]:
    if t.numel() == 0:
        return None
    return t


class PackedConv:
    """The native form of one nn.Conv2d (ops.conv_form), its filter packed for that form (ops.pack_conv_filter_for) with an
    eval-mode BatchNorm folded in when given, and its bias; cached per form and precision until a source tensor is modified or
    moved.  The modules are passed at each call, so that module replicas sharing the object use their own weights."""

    def __init__(self) -> None:
        self._cache = _FoldCache()

    def packed(self, conv: nn.Conv2d, bn: Optional[nn.BatchNorm2d] = None) -> Tuple[int, Tensor, Optional[Tensor]]:
        """(form, filter image, bias or None)."""
        from . import ops

        form = ops.conv_form(conv.in_channels, conv.out_channels, conv.kernel_size[0], conv.stride[0])
        prec = ops.conv_precision()
        if bn is None:
            srcs = [conv.weight] + ([conv.bias] if conv.bias is not None else [])
        else:
            srcs = [conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        def make():
            w, b = (conv.weight, conv.bias) if bn is None else _fold_bn(conv.weight, bn)
            return ops.pack_conv_filter_for(w, form, prec), None if b is None else b.detach().clone()

        filt, bias = self._cache.get(srcs, make, key=(form, prec))
        return form, filt, bias

    def __call__(self, conv: nn.Conv2d, x: Tensor, bn: Optional[nn.BatchNorm2d] = None, relu: bool = False, with_bias: bool = True,
                 out: Optional[Tensor] = None, out_channel_offset: int = 0) -> Tensor:
        """The conv on the native kernel of its form (what _script_conv runs in the scripted forward)."""
        from . import ops

        form, filt, bias = self.packed(conv, bn)
        args = (x, filt, bias if with_bias else None, conv.out_channels, conv.kernel_size[0], conv.stride[0], conv.padding[0],
                conv.dilation[0])
        if form == 0:
            return ops.conv2d_nhwc(*args, relu=relu, out=out, out_channel_offset=out_channel_offset)
        return ops.conv2d_tc5(*args, relu=relu, out=out, out_channel_offset=out_channel_offset, halo=form == 2)


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
        self._cache = _FoldCache()  # folded weights for ATen's convolution
        self._packed = PackedConv()
        self._k, self._stride, self._pad, self._cout = k, stride, pad, cout
        # scripted forward, frozen by freeze_script (see "TorchScript" above)
        self._s_mode = 0
        self._s_fused_relu = _FUSED_CONV_RELU
        self._s_form = 0  # native form
        self._s_precision = 3
        self._s_native_w = torch.zeros(0)  # folded filter image for the native form, folded bias
        self._s_native_b = torch.zeros(0)
        self._s_lib_w = torch.zeros(0)  # folded channels-last filter and bias for ATen's convolution
        self._s_lib_b = torch.zeros(0)

    def freeze_script(self) -> None:
        """Freeze the layer's eval-mode decisions and folded weights for the scripted forward."""
        from . import ops

        self._s_mode = 0 if not LIBRARY_FAST_PATH else (2 if ops_prefers(self.conv) else 1)
        self._s_precision = ops.conv_precision()
        # Refinement's native tail calls the native form whatever the layer prefers
        self._s_form, frag, b = self._packed.packed(self.conv, self.bn)
        self._s_native_w, self._s_native_b = _host(frag), _host(b)
        if self._s_mode == 1:
            w, b = self.folded()
            self._s_lib_w, self._s_lib_b = _host(w), _host(b)

    def native_script(self, x: Tensor, out: Optional[Tensor] = None, out_channel_offset: int = 0) -> Tensor:
        return _script_conv(x, self._s_form, self._s_native_w, self._s_native_b, self._cout, self._k, self._stride, self._pad, 1, True,
                            self._s_precision, out, out_channel_offset)

    def _forward_script(self, x: Tensor) -> Tensor:
        if self._s_mode == 2:
            return self.native_script(x)
        if self._s_mode == 1:
            w = torch.ops.pmb200.device_copy(self._s_lib_w, x)
            b = torch.ops.pmb200.device_copy(self._s_lib_b, x)
            s, p = [self._stride, self._stride], [self._pad, self._pad]
            if self._s_fused_relu:
                return torch.cudnn_convolution_relu(x, w, b, s, p, [1, 1], 1)
            return F.relu_(F.conv2d(x, w, b, s, p, [1, 1]))
        return F.relu(self.bn(self.conv(x)), inplace=True)

    def native(self, x: Tensor, out: Tensor = None, out_channel_offset: int = 0) -> Tensor:
        return self._packed(self.conv, x, self.bn, relu=True, out=out, out_channel_offset=out_channel_offset)

    def folded(self):
        bn = self.bn
        srcs = [self.conv.weight, bn.weight, bn.bias, bn.running_mean, bn.running_var]

        def make():
            w, b = _fold_bn(self.conv.weight, bn)
            return w.contiguous(memory_format=torch.channels_last), b

        return self._cache.get(srcs, make)

    def forward(self, x: Tensor) -> Tensor:
        if torch.jit.is_scripting():
            return self._forward_script(x)
        return self._forward_eager(x)

    @torch.jit.unused
    def _forward_eager(self, x: Tensor) -> Tensor:
        if self.training or not _fast(x):
            return F.relu(self.bn(self.conv(x)), inplace=True)
        c = self.conv
        if ops_prefers(c):
            return self.native(x)
        w, b = self.folded()
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
        self._packed = {n: PackedConv() for n in ("output1", "inner1", "inner2", "output2", "output3")}
        self._composed_cache = _FoldCache()
        self._stem_cache = _FoldCache()
        self.fuse_top_down = True  # eval mode on CUDA: composed 1x1 heads (see composed_heads); False = layer by layer
        # scripted forward, frozen by freeze_script (see "TorchScript" above)
        self._s_fast = True
        self._s_stem_fused = False
        self._s_stem = [torch.zeros(0)] * 4  # stem_weights()
        self._s_top_down = 0  # 0 = the reference's, 1 = layer by layer (native lateral conv), 2 = composed heads
        self._s_precision = 3
        self._s_plain_form: Dict[str, int] = {}  # the plain 1x1 convs (_plain), by name: form, filter image, bias (empty: none)
        self._s_plain_w: Dict[str, Tensor] = {}
        self._s_plain_b: Dict[str, Tensor] = {}
        self._s_composed: Dict[str, Tensor] = {}  # composed_heads(), filters packed
        self.register_load_state_dict_post_hook(_freeze_after_load)

    def train(self, mode: bool = True):
        super().train(mode)
        if not mode and _freezing():
            self.freeze_script()
        return self

    def freeze_script(self) -> None:
        """Freeze the eval-mode decisions and folded weights of the scripted forward: the stem, each layer's conv form, the
        top-down path (following fuse_top_down) and its filters."""
        from . import ops

        for i in range(11):
            getattr(self, f"conv{i}").freeze_script()
        self._s_fast = LIBRARY_FAST_PATH
        self._s_precision = ops.conv_precision()
        self._s_stem_fused = self._s_fast and self._s_precision == 3
        self._s_stem = [_host(t) for t in self.stem_weights()] if self._s_stem_fused else [torch.zeros(0)] * 4
        self._s_top_down = 0 if not LIBRARY_FAST_PATH else (2 if self.fuse_top_down else 1)
        self._s_plain_form, self._s_plain_w, self._s_plain_b, self._s_composed = {}, {}, {}, {}
        if self._s_fast:
            for name, packed in self._packed.items():
                form, filt, bias = packed.packed(getattr(self, name))
                self._s_plain_form[name], self._s_plain_w[name] = form, _host(filt)
                self._s_plain_b[name] = torch.zeros(0) if bias is None else _host(bias)
        if self._s_top_down == 2:
            with torch.no_grad():
                for k, v in self.composed_heads().items():
                    self._s_composed[k] = _host(ops.pack_conv_filter(v, self._s_precision) if v.dim() == 4 else v)

    def _forward_script(self, x: Tensor) -> Dict[int, Tensor]:
        if self.training:
            raise RuntimeError("a scripted patchmatchnet_b200 network is inference-only; call eval() before torch.jit.script")
        if self._s_stem_fused and x.dim() == 4 and x.size(1) == 3 and x.dtype == torch.float32:
            y = torch.ops.pmb200.conv_stem(x, self._s_stem[0], self._s_stem[1], self._s_stem[2], self._s_stem[3])
        else:
            if self._s_fast and not x.is_contiguous(memory_format=torch.channels_last):
                x = x.contiguous(memory_format=torch.channels_last)
            y = self.conv1(self.conv0(x))
        half = self.conv4(self.conv3(self.conv2(y)))
        quarter = self.conv7(self.conv6(self.conv5(half)))
        eighth = self.conv10(self.conv9(self.conv8(quarter)))
        out: Dict[int, Tensor] = {3: self._plain_script("output1", eighth)}
        if self._s_top_down == 2:  # _fused_top_down
            w, p = self._s_composed, self._s_precision
            u_o = _script_conv(eighth, 0, w["u_o"], None, 32, 1, 1, 0, 1, False, p)
            u_t = _script_conv(eighth, 0, w["u_t"], None, 16, 1, 1, 0, 1, False, p)
            out[2] = _script_conv(quarter, 0, w["l2_o"], w["c2_o"], 32, 1, 1, 0, 1, False, p, add_up2x=u_o)
            t = _script_conv(quarter, 0, w["l2_t"], w["c2_t"], 16, 1, 1, 0, 1, False, p, add_up2x=u_t)
            out[1] = _script_conv(half, 0, w["l1"], w["c1"], 16, 1, 1, 0, 1, False, p, add_up2x=t)
            return out
        top = self._top_down_script(eighth, "inner1", quarter)
        out[2] = self._plain_script("output2", top)
        top = self._top_down_script(top, "inner2", half)
        out[1] = self._plain_script("output3", top)
        return out

    def _plain_script(self, name: str, x: Tensor) -> Tensor:
        if self._s_fast:
            cout = 64 if name == "output1" else (32 if name == "output2" else 16)
            return _script_conv(x, self._s_plain_form[name], self._s_plain_w[name], _nonempty(self._s_plain_b[name]), cout, 1, 1, 0, 1,
                                False, self._s_precision)
        if name == "output1":
            return self.output1(x)
        if name == "output2":
            return self.output2(x)
        return self.output3(x)

    def _top_down_script(self, coarse: Tensor, lateral_name: str, fine: Tensor) -> Tensor:
        if self._s_top_down == 0:
            lateral = self.inner1(fine) if lateral_name == "inner1" else self.inner2(fine)
            return F.interpolate(coarse, scale_factor=2.0, mode="bilinear", align_corners=False) + lateral
        lateral = _script_conv(fine, self._s_plain_form[lateral_name], self._s_plain_w[lateral_name], None, 64, 1, 1, 0, 1, False,
                               self._s_precision)
        bias = self.inner1.bias if lateral_name == "inner1" else self.inner2.bias
        return torch.ops.pmb200.upsample2x_add(coarse, lateral, bias)

    def _plain(self, name: str, x: Tensor) -> Tensor:
        """One of the bias-free / lateral 1x1 convs: native in eval mode on CUDA, else the module itself."""
        if not self.training and _fast(x):
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

        if (not self.training and _fast(x) and ops.conv_precision() == 3 and x.dim() == 4 and x.shape[1] == 3
                and x.dtype == torch.float32):
            return ops.conv_stem(x, *self.stem_weights())
        if _fast(x) and not x.is_contiguous(memory_format=torch.channels_last):
            x = x.contiguous(memory_format=torch.channels_last)
        return self._trunk(x, 0, 1)

    def forward(self, x: Tensor) -> Dict[int, Tensor]:
        if torch.jit.is_scripting():
            return self._forward_script(x)
        return self._forward_eager(x)

    @torch.jit.unused
    def _forward_eager(self, x: Tensor) -> Dict[int, Tensor]:
        half = self._trunk(self._stem(x), 2, 4)
        quarter = self._trunk(half, 5, 7)
        eighth = self._trunk(quarter, 8, 10)
        if not self.training and _fast(x) and self.fuse_top_down:
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
        if _fast(coarse) and not self.training:
            from . import ops

            lateral = self._packed[lateral_name](lateral_conv, fine, with_bias=False)
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
        self._deconv_frag = _FoldCache()
        self._host_cache = _FoldCache()
        self._res_packed = PackedConv()
        # scripted forward, frozen by freeze_script (see "TorchScript" above)
        self._s_fast = True
        self._s_fused = False
        self._s_host = [torch.zeros(0)] * 11  # host_weights() for K-R
        self._s_precision = 3
        self._s_deconv_w = torch.zeros(0)  # native tail: transposed conv (fragment order) and bias, residual conv form and filter
        self._s_deconv_b = torch.zeros(0)
        self._s_res_form = 0
        self._s_res_w = torch.zeros(0)
        self.register_load_state_dict_post_hook(_freeze_after_load)

    def train(self, mode: bool = True):
        super().train(mode)
        if not mode and _freezing():
            self.freeze_script()
        return self

    def freeze_script(self) -> None:
        """Freeze the eval-mode decisions and folded weights of the scripted forward: K-R, or the conv-family tail."""
        from . import ops

        for m in (self.conv0, self.conv1, self.conv2, self.conv3):
            m.freeze_script()
        self._s_fast = LIBRARY_FAST_PATH
        self._s_precision = ops.conv_precision()
        self._s_fused = self._s_fast and self._s_precision == 3 and self.res.bias is None
        self._s_host = [_host(t) for t in self.host_weights()] if self._s_fused else [torch.zeros(0)] * 11
        if self._s_fast:
            with torch.no_grad():
                w, b = _fold_bn(self.deconv.weight, self.bn, out_dim=1)
                self._s_deconv_w, self._s_deconv_b = _host(ops.pack_conv_filter(w, self._s_precision, transposed=True)), _host(b)
            self._s_res_form, filt, _ = self._res_packed.packed(self.res)
            self._s_res_w = _host(filt)

    def _forward_script(self, img: Tensor, depth_half: Tensor, depth_min: Tensor, depth_max: Tensor) -> Tensor:
        if self.training:
            raise RuntimeError("a scripted patchmatchnet_b200 network is inference-only; call eval() before torch.jit.script")
        if (self._s_fused and img.dtype == torch.float32 and img.size(-2) == 2 * depth_half.size(-2)
                and img.size(-1) == 2 * depth_half.size(-1)):
            hw = self._s_host
            dh, lo, hi = depth_half.float(), depth_min.float(), depth_max.float()
            low = torch.ops.pmb200.refine_low(dh, lo, hi, hw[0], hw[1], hw[2], hw[3])
            return torch.ops.pmb200.refine_full(low, img, dh, lo, hi, hw[4], hw[5], hw[6], hw[7], hw[8], hw[9], hw[10])
        B = depth_min.size(0)
        lo = depth_min.view(B, 1, 1, 1)
        span = (depth_max - depth_min).view(B, 1, 1, 1)
        d = (depth_half - lo) / span
        if self._s_fast:
            img = img.contiguous(memory_format=torch.channels_last)
        if self._s_fast and img.size(-2) == 2 * d.size(-2) and img.size(-1) == 2 * d.size(-1):  # _native_tail
            low = self.conv2.native_script(self.conv1.native_script(d))
            both = torch.empty([low.size(0), 16, 2 * low.size(2), 2 * low.size(3)], dtype=torch.float32, device=low.device,
                               memory_format=torch.channels_last)
            _script_conv(low, 0, self._s_deconv_w, self._s_deconv_b, 8, 3, 1, 1, 1, True, self._s_precision, both, 0,
                         transposed2x=True)
            self.conv0.native_script(img, both, 8)
            res = _script_conv(self.conv3.native_script(both), self._s_res_form, self._s_res_w, None, 1, 3, 1, 1, 1, False,
                               self._s_precision)
        else:  # the reference's layers; torch.cat needs the image at exactly twice the depth map's size
            up = F.relu(self.bn(self.deconv(self.conv2(self.conv1(d)))), inplace=True)
            res = self.res(self.conv3(torch.cat((up, self.conv0(img)), dim=1)))
        d = F.interpolate(d, scale_factor=2.0, mode="nearest") + res
        return d * span + lo

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
        if torch.jit.is_scripting():
            return self._forward_script(img, depth_half, depth_min, depth_max)
        return self._forward_eager(img, depth_half, depth_min, depth_max)

    @torch.jit.unused
    def _forward_eager(self, img: Tensor, depth_half: Tensor, depth_min: Tensor, depth_max: Tensor) -> Tensor:
        from . import ops

        fast = not self.training and _fast(img)
        if (fast and ops.conv_precision() == 3 and img.dtype == torch.float32
                and img.shape[-2:] == (2 * depth_half.shape[-2], 2 * depth_half.shape[-1]) and self.res.bias is None):
            return self._fused(img, depth_half.float(), depth_min.float(), depth_max.float())
        B = depth_min.size(0)
        lo = depth_min.view(B, 1, 1, 1)
        span = (depth_max - depth_min).view(B, 1, 1, 1)
        d = (depth_half - lo) / span
        if fast:
            img = img.contiguous(memory_format=torch.channels_last)
        if fast and img.shape[-2:] == (2 * d.shape[-2], 2 * d.shape[-1]):
            res = self._native_tail(img, d)
        else:  # the reference's layers; torch.cat needs the image at exactly twice the depth map's size
            up = F.relu(self.bn(self.deconv(self.conv2(self.conv1(d)))), inplace=True)
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
    # not part of a scripted network (a scripted module's state dict would list the buffer); it uses _s_stage_scales instead
    __jit_ignored_attributes__ = ["_stage_scales"]

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
        # scripted forward, frozen by freeze_script (see "TorchScript" above)
        self._s_fast = True
        self._s_ref_channels_last = False  # extract_features' channels-last copy of the reference image
        self._s_stage_scales = torch.tensor([0.125, 0.25, 0.5]).view(3, 1, 1, 1, 1)
        self.register_load_state_dict_post_hook(_freeze_after_load)

    def train(self, mode: bool = True):
        super().train(mode)
        if not mode and _freezing():
            self.freeze_script()
        return self

    def freeze_script(self) -> None:
        """Freeze the network-level eval-mode decisions of the scripted forward (FeatureNet, Refinement and the stages freeze
        their own)."""
        from . import ops

        self._s_fast = LIBRARY_FAST_PATH
        self._s_ref_channels_last = LIBRARY_FAST_PATH and ops.conv_precision() != 3

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
        from . import ops

        # the pyramid comes out channels-last, the layout the fused PatchMatch kernels read in place.  FeatureNet's first layers
        # read the NCHW planes themselves (K-S) or convert; only the reference view is needed channels-last again, by
        # Refinement's layer-by-layer path in the TF32 mode; its fused form (K-R) reads the NCHW planes itself
        if _fast(x) and ops.conv_precision() != 3:
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
        if torch.jit.is_scripting():
            return self._forward_script(images, intrinsics, extrinsics, depth_min, depth_max)
        return self._forward_eager(images, intrinsics, extrinsics, depth_min, depth_max)

    def _forward_script(
        self,
        images: List[Tensor],
        intrinsics: Tensor,
        extrinsics: Tensor,
        depth_min: Tensor,
        depth_max: Tensor,
    ) -> Tuple[Tensor, Tensor, Dict[int, List[Tensor]]]:
        """The eval-mode forward of `_forward_eager` in the TorchScript subset: the same launches under the decisions frozen at
        eval() time.  Views of one size are always concatenated into one batch (TorchScript cannot see whether they already
        share one buffer, which eager passes on without a copy).  Inference only, as scripting is in the reference."""
        if self.training:
            raise RuntimeError("a scripted patchmatchnet_b200 network is inference-only; call eval() before torch.jit.script")
        assert len(images) == intrinsics.size(1), "Different number of images and intrinsic matrices"
        assert len(images) == extrinsics.size(1), "Different number of images and extrinsic matrices"
        images = list(images)
        H0, W0 = images[0].size(-2), images[0].size(-1)
        for i in range(len(images)):  # _round_dims_to_8
            h, w = images[i].size(-2), images[i].size(-1)
            nh, nw = int(round(h / 8)) * 8, int(round(w / 8)) * 8
            if nh != h or nw != w:
                intrinsics[:, i, 0] *= nw / w
                intrinsics[:, i, 1] *= nh / h
                images[i] = F.interpolate(images[i], size=[nh, nw], mode="bilinear", align_corners=False)
        ref_image = images[0]
        Hr, Wr = ref_image.size(-2), ref_image.size(-1)

        same = True
        for im in images:
            if im.size() != images[0].size():
                same = False
        feats: List[Dict[int, Tensor]] = []
        if self.stack_views and same:  # extract_features
            b = images[0].size(0)
            x = torch.cat(images, dim=0)
            if self._s_ref_channels_last:
                ref_image = images[0].contiguous(memory_format=torch.channels_last)
            stacked = self.feature(x)
            for i in range(len(images)):
                feats.append({3: stacked[3][i * b:(i + 1) * b], 2: stacked[2][i * b:(i + 1) * b], 1: stacked[1][i * b:(i + 1) * b]})
        else:
            for im in images:
                feats.append(self.feature(im))
        depth_min = depth_min.float()
        depth_max = depth_max.float()

        dev = intrinsics.device
        depth = torch.empty(0, device=dev)
        score = torch.empty(0, device=dev)
        view_weights = torch.empty(0, device=dev)
        per_stage: Dict[int, List[Tensor]] = {}
        all_proj: Optional[Tensor] = None
        if self._s_fast:
            K3 = intrinsics.unsqueeze(0).repeat(3, 1, 1, 1, 1)
            K3[:, :, :, :2] *= torch.ops.pmb200.device_copy(self._s_stage_scales, K3)
            all_proj = extrinsics.unsqueeze(0).repeat(3, 1, 1, 1, 1)
            all_proj[:, :, :, :3, :4] = torch.matmul(K3, extrinsics[:, :, :3, :4])
        scale = 0.125
        for stage in [3, 2, 1]:
            if all_proj is not None:
                proj = all_proj[3 - stage]
            else:
                K = intrinsics.clone()
                K[:, :, :2] *= scale
                proj = extrinsics.clone()
                proj[:, :, :3, :4] = torch.matmul(K, extrinsics[:, :, :3, :4])
            projs = torch.unbind(proj, 1)
            scale *= 2.0
            src = [f[stage] for f in feats[1:]]
            if stage == 3:
                depths, score, view_weights = self.patchmatch_3(feats[0][3], src, projs[0], projs[1:], depth_min, depth_max, depth,
                                                                view_weights)
            elif stage == 2:
                depths, score, view_weights = self.patchmatch_2(feats[0][2], src, projs[0], projs[1:], depth_min, depth_max, depth,
                                                                view_weights)
            else:
                depths, score, view_weights = self.patchmatch_1(feats[0][1], src, projs[0], projs[1:], depth_min, depth_max, depth,
                                                                view_weights)
            per_stage[stage] = depths
            depth = depths[-1].detach()
            if stage > 1:
                depth = F.interpolate(depth, scale_factor=2.0, mode="nearest")
                view_weights = F.interpolate(view_weights, scale_factor=2.0, mode="nearest")

        depth = self.upsample_net(ref_image, depth, depth_min, depth_max)
        if Hr != H0 or Wr != W0:
            depth = F.interpolate(depth, size=[H0, W0], mode="bilinear", align_corners=False)
        per_stage[0] = [depth]
        D = self.patchmatch_num_sample[0]
        if self._s_fast and score.size(1) == D:
            return depth, torch.ops.pmb200.photometric_confidence(score, H0, W0), per_stage
        mass4 = 4 * F.avg_pool3d(F.pad(score.unsqueeze(1), pad=[0, 0, 0, 0, 1, 2]), (4, 1, 1), stride=1, padding=0).squeeze(1)
        idx = torch.sum(score * torch.arange(D, device=score.device, dtype=torch.float).view(1, D, 1, 1), dim=1)
        idx = idx.unsqueeze(1).long().clamp(0, D - 1)
        conf = torch.gather(mass4, 1, idx)
        conf = F.interpolate(conf, size=[H0, W0], mode="nearest").squeeze(1)
        return depth, conf, per_stage

    @torch.jit.unused
    def _forward_eager(
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
