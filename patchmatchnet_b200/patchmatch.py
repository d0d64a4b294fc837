"""H100-native ``PatchMatch``: drop-in for reference ``models/patchmatch.py:242-529``.

Same constructor, same ``forward`` signature and return triple, same parameter /
buffer names and shapes (the reference checkpoints load with every key matched),
same error behaviour (``assert`` on view/matrix count mismatch,
``NotImplementedError`` for neighbour counts the reference does not know).

What runs where (per PatchMatch iteration; DESIGN.md has the byte budgets):

    propa_conv / eval_conv, the three 1x1x1 MLP heads ... cuDNN (library ops, as the scope says)
    everything else ..................................... five hand-written sm_90a kernels
        K-C  init_propagate   hypothesis init + neighbour gather + sort          (a8, a9, a7)
        K-A  warp_corr        warp + bilinear gather + group correlation
                              + view-weighted aggregation, all views, one launch (a1, a2, a3)
        K-A' offset_corr      reference self-correlation at learned neighbours   (a11, a7)
        K-B  adaptive_eval    depth/feature weights + aggregation + softmax
                              + regression                                       (a10, a6, a5)
        relative_projection   src_proj . inv(ref_proj), once per stage, no host sync (a1 prologue)

There is no CPU or pure-PyTorch implementation of those kernels here: CPU tensors
raise.  (The CPU restatement lives in ``oracle/`` and is test infrastructure.)
"""
from __future__ import annotations

import weakref
from typing import Callable, List, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _native, ops
from .net import PackedConv

Tensor = torch.Tensor


_HEAD_CACHE: "weakref.WeakKeyDictionary" = weakref.WeakKeyDictionary()
_HEAD_FLOATS = 16 * 8 + 16 + 8 * 16 + 8 + 8 + 1  # sizeof(pmb200_mlp) / 4


def _refresh_after_load(module, incompatible_keys) -> None:
    if not module.training:
        module.refresh_script_heads()


def _offset_conv(conv: nn.Conv2d, packed: PackedConv, x: Tensor, native: bool) -> Tensor:
    """propa_conv / eval_conv (reference patchmatch.py:288-311, called at :486 / :498).  `native`: the conv's native form
    (its channels-last output is what the fused kernels consume in place), filter cached in `packed`."""
    if (not native or max(conv.in_channels, conv.out_channels) > 64
            or not ops.conv_prefers_native(conv.in_channels, conv.out_channels, conv.kernel_size[0])):
        return conv(x)
    return packed(conv, x)


def is_empty(x: Tensor) -> bool:
    """reference models/module.py:199-200: optional tensors are signalled by numel() == 0."""
    return x.numel() == 0


class _ConvBnReLU3d(nn.Module):
    """1x1x1 conv3d (no bias) + BatchNorm3d + ReLU; children ``conv`` / ``bn`` (reference module.py:43-72)."""

    def __init__(self, cin: int, cout: int) -> None:
        super().__init__()
        self.conv = nn.Conv3d(cin, cout, 1, stride=1, padding=0, bias=False)
        self.bn = nn.BatchNorm3d(cout)

    def forward(self, x: Tensor) -> Tensor:
        return F.relu(self.bn(self.conv(x)), inplace=True)


class _PointwiseHead(nn.Module):
    """G -> 16 -> 8 -> 1 per-voxel MLP shared by the three learned heads.  ``last`` names the final
    conv so the state-dict keys match the reference (``conv2`` in PixelwiseNet, ``similarity`` in
    SimilarityNet / FeatureWeightNet)."""

    def __init__(self, G: int, last: str) -> None:
        super().__init__()
        self.conv0 = _ConvBnReLU3d(G, 16)
        self.conv1 = _ConvBnReLU3d(16, 8)
        self._last = last
        setattr(self, last, nn.Conv3d(8, 1, 1, stride=1, padding=0))

    # forward lives in the subclasses with the last conv named literally, so that the module tree scripts
    # (TorchScript has no dynamic getattr): [N,G,D,H,W] -> [N,D,H,W]

    def folded_tensor(self) -> Tensor:
        """The same folded head as a flat CPU float32 tensor (the memory image of pmb200_mlp): what the
        `torch.ops.pmb200.*` operators take, because a TorchScript graph cannot hold a ctypes struct."""
        m = self.folded()
        return torch.frombuffer(bytearray(bytes(m)), dtype=torch.float32).clone()

    def folded(self) -> "_native.MlpStruct":
        """Eval-mode weights with BatchNorm folded into the convs, as the host struct the fused
        kernels take (pmb200_mlp).  Cached; recomputed when any parameter/buffer was modified.
        The fold needs one device->host copy, so the first call must happen outside graph capture
        (DepthEngine warms up before capturing)."""
        tensors = list(self.parameters()) + list(self.buffers())
        stamp = tuple((t.data_ptr(), t._version) for t in tensors)
        cached = _HEAD_CACHE.get(self)  # kept off the module: TorchScript would try to type a ctypes attribute
        if cached is not None and cached[0] == stamp:
            return cached[1]
        with torch.no_grad():
            def fold(block):
                w = block.conv.weight.double().flatten(1)  # [out,in]
                bn = block.bn
                scale = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
                return (w * scale[:, None]).float().cpu(), (bn.bias.double() - bn.running_mean.double() * scale).float().cpu()

            w0, b0 = fold(self.conv0)
            w1, b1 = fold(self.conv1)
            last = getattr(self, self._last)
            w2 = last.weight.detach().flatten().float().cpu()
            b2 = float(last.bias.detach().float().cpu())
        G = w0.shape[1]
        if G > 8 or w0.shape[0] != 16 or w1.shape != (8, 16):
            raise NotImplementedError("fused heads support G <= 8")
        m = _native.MlpStruct()
        pad = torch.zeros(16, 8)
        pad[:, :G] = w0
        m.w0[:] = pad.flatten().tolist()
        m.b0[:] = b0.tolist()
        m.w1[:] = w1.flatten().tolist()
        m.b1[:] = b1.tolist()
        m.w2[:] = w2.tolist()
        m.b2 = b2
        _HEAD_CACHE[self] = (stamp, m)
        return m


class PixelwiseNet(_PointwiseHead):
    """Pixel-wise view weight: max over hypotheses of sigmoid(MLP(similarity)); reference patchmatch.py:672-702."""

    def __init__(self, G: int) -> None:
        super().__init__(G, "conv2")

    def forward(self, x: Tensor) -> Tensor:
        y = self.conv2(self.conv1(self.conv0(x))).squeeze(1)
        return torch.max(torch.sigmoid(y), dim=1)[0].unsqueeze(1)


class SimilarityNet(_PointwiseHead):
    """Per-hypothesis score MLP; the neighbour aggregation that follows it in the reference
    (patchmatch.py:569-577) is part of kernel K-B."""

    def __init__(self, G: int) -> None:
        super().__init__(G, "similarity")

    def forward(self, x: Tensor) -> Tensor:
        return self.similarity(self.conv1(self.conv0(x))).squeeze(1)


class FeatureWeightNet(_PointwiseHead):
    """sigmoid(MLP(self-correlation)); the gather + correlation in front of it (reference
    patchmatch.py:613-622) is kernel K-A'."""

    def __init__(self, neighbors: int = 9, G: int = 8) -> None:
        super().__init__(G, "similarity")
        self.neighbors = neighbors
        self.G = G

    def forward(self, corr: Tensor) -> Tensor:
        return torch.sigmoid(self.similarity(self.conv1(self.conv0(corr))).squeeze(1))


class Evaluation(nn.Module):
    """Owner of the two evaluation heads (names as in reference patchmatch.py:132-143)."""

    def __init__(self, G: int = 8) -> None:
        super().__init__()
        self.G = G
        self.pixel_wise_net = PixelwiseNet(G)
        self.similarity_net = SimilarityNet(G)


class PatchMatch(nn.Module):
    """Learned PatchMatch on one pyramid level; see module docstring."""

    def __init__(
        self,
        propagation_out_range: int = 2,
        patchmatch_iteration: int = 2,
        patchmatch_num_sample: int = 16,
        patchmatch_interval_scale: float = 0.025,
        num_feature: int = 64,
        G: int = 8,
        propagate_neighbors: int = 16,
        evaluate_neighbors: int = 9,
        stage: int = 3,
    ) -> None:
        super().__init__()
        self.patchmatch_iteration = patchmatch_iteration
        self.patchmatch_interval_scale = patchmatch_interval_scale
        self.patchmatch_num_sample = patchmatch_num_sample
        self.propa_num_feature = num_feature
        self.G = G
        self.stage = stage
        self.dilation = propagation_out_range
        self.propagate_neighbors = propagate_neighbors
        self.evaluate_neighbors = evaluate_neighbors
        # Tests inject a shared U[0,1) draw here when comparing against an oracle on another device;
        # by default the draw is torch.rand on the compute device, exactly as reference patchmatch.py:61-63.
        self.rand_source = None  # Optional[Callable]
        # its counterpart in a scripted module (TorchScript cannot hold a callable): a fixed U[0,1) draw [B,48,H,W], empty = torch.rand
        self.rand_draw = torch.empty(0)
        # eval mode: apply the 1x1x1 heads in the kernels' epilogues (BatchNorm folded); set False to
        # run them as cuDNN ops on materialised similarity tensors (the training path always does)
        self.fuse_heads = True

        self.evaluation = Evaluation(G)
        # zero-initialised offset convs, always defined (reference patchmatch.py:286-311)
        self.propa_conv = nn.Conv2d(
            num_feature, max(2 * propagate_neighbors, 1), 3, stride=1,
            padding=self.dilation, dilation=self.dilation, bias=True,
        )
        self.eval_conv = nn.Conv2d(
            num_feature, 2 * evaluate_neighbors, 3, stride=1,
            padding=self.dilation, dilation=self.dilation, bias=True,
        )
        for conv in (self.propa_conv, self.eval_conv):
            nn.init.constant_(conv.weight, 0.0)
            nn.init.constant_(conv.bias, 0.0)
        self._propa_packed, self._eval_packed = PackedConv(), PackedConv()  # their native filters (eval mode)
        self.feature_weight_net = FeatureWeightNet(evaluate_neighbors, G)
        # Folded heads as plain CPU tensors for the TorchScript path (not buffers: the state dict must keep exactly
        # the reference's keys).  Refreshed on eval() / load_state_dict, i.e. before the reference scripts the model
        # (train.py:50-55: child_model.eval(); torch.jit.script(child_model)).
        self._head_fw = torch.zeros(_HEAD_FLOATS)
        self._head_pw = torch.zeros(_HEAD_FLOATS)
        self._head_sim = torch.zeros(_HEAD_FLOATS)
        # The offset convs' filters in tensor-core fragment order, and the conv precision (1 = TF32 operands, 3 = 3xTF32),
        # for the scripted forward: like everything in a scripted artefact they are frozen when it is made, i.e. the
        # precision is what torch.backends.cudnn.allow_tf32 selects at eval() / load_state_dict time.
        self._off_propa_frag = torch.zeros(1)
        self._off_eval_frag = torch.zeros(1)
        self._conv_precision = 3
        self._native_propa = False  # ops.conv_prefers_native(...) for the two offset convs, frozen likewise
        self._native_eval = False
        # which native form runs each offset conv, as ops.conv_form picks it for the eager path: 0 = the mma.sync kernel
        # (conv2d_nhwc, filter in fragment order), 1 = the wgmma tap form, 2 = the wgmma halo-tile form (conv2d_tc5)
        self._off_propa_form = 0
        self._off_eval_form = 0
        self.register_load_state_dict_post_hook(_refresh_after_load)

    # ------------------------------------------------------------------
    def refresh_script_heads(self) -> None:
        """Re-fold BatchNorm into the three heads for the scripted forward (call after changing weights in eval mode)."""
        if self.G <= 8:
            self._head_fw = self.feature_weight_net.folded_tensor()
            self._head_pw = self.evaluation.pixel_wise_net.folded_tensor()
            self._head_sim = self.evaluation.similarity_net.folded_tensor()
        self._conv_precision = ops.conv_precision()
        # the native conv takes 1..64 channels; wider layers (a valid reference configuration, e.g. num_feature=128)
        # stay with the library conv instead of failing in eval() (ADVICE r1)
        fits = lambda conv: max(conv.in_channels, conv.out_channels) <= 64
        self._native_propa = fits(self.propa_conv) and ops.conv_prefers_native(self.propa_conv.in_channels, self.propa_conv.out_channels, 3)
        self._native_eval = fits(self.eval_conv) and ops.conv_prefers_native(self.eval_conv.in_channels, self.eval_conv.out_channels, 3)
        self._off_propa_form, self._off_propa_frag = self._freeze_offset_conv(self.propa_conv, self._propa_packed, self._native_propa)
        self._off_eval_form, self._off_eval_frag = self._freeze_offset_conv(self.eval_conv, self._eval_packed, self._native_eval)

    def _freeze_offset_conv(self, conv: nn.Conv2d, packed: PackedConv, native: bool) -> Tuple[int, Tensor]:
        """(form, host filter image) of one offset conv for the scripted forward: the form `_offset_conv` takes in eager mode."""
        if not native:
            return 0, torch.zeros(1)
        form, filt, _ = packed.packed(conv)
        return form, filt.cpu()

    def train(self, mode: bool = True):
        super().train(mode)
        if not mode:
            self.refresh_script_heads()
        return self

    def _check_neighbour_counts(self) -> None:
        if self.propagate_neighbors not in (0, 4, 8, 16):
            raise NotImplementedError  # reference patchmatch.py:359-360
        if self.evaluate_neighbors not in (9, 17):
            raise NotImplementedError  # reference patchmatch.py:391-392

    def forward(
        self,
        ref_feature: Tensor,
        src_features: List[Tensor],
        ref_proj: Tensor,
        src_projs: List[Tensor],
        depth_min: Tensor,
        depth_max: Tensor,
        depth: Tensor,
        view_weights: Tensor,
    ) -> Tuple[List[Tensor], Tensor, Tensor]:
        if torch.jit.is_scripting():
            return self._forward_script(
                ref_feature, src_features, ref_proj, src_projs, depth_min, depth_max, depth, view_weights
            )
        else:
            return self._forward_eager(
                ref_feature, src_features, ref_proj, src_projs, depth_min, depth_max, depth, view_weights
            )

    def _forward_script(
        self,
        ref_feature: Tensor,
        src_features: List[Tensor],
        ref_proj: Tensor,
        src_projs: List[Tensor],
        depth_min: Tensor,
        depth_max: Tensor,
        depth: Tensor,
        view_weights: Tensor,
    ) -> Tuple[List[Tensor], Tensor, Tensor]:
        """The eval-mode cascade written in the TorchScript subset over `torch.ops.pmb200.*` (csrc/torch_binding.cpp):
        what runs inside a scripted model (reference train.py:53, eval.py:38).  Same kernels, same order as the fused
        branch of `_forward_eager`.  Inference only: scripting exports a deployment artefact in the reference too."""
        if self.training:
            raise RuntimeError("a scripted patchmatchnet_b200.PatchMatch is inference-only; call eval() before torch.jit.script")
        if self.propagate_neighbors != 0 and self.propagate_neighbors != 4 and self.propagate_neighbors != 8 and self.propagate_neighbors != 16:
            raise NotImplementedError
        if self.evaluate_neighbors != 9 and self.evaluate_neighbors != 17:
            raise NotImplementedError
        assert len(src_features) == len(
            src_projs
        ), "Patchmatch Evaluation: Different number of images and projection matrices"
        if view_weights.numel() != 0:
            assert (
                len(src_features) == view_weights.size(1)
            ), "Patchmatch Evaluation: Different number of images and view weights"
        B, H, W = ref_feature.size(0), ref_feature.size(2), ref_feature.size(3)
        Kp, Ke, iters = self.propagate_neighbors, self.evaluate_neighbors, self.patchmatch_iteration
        dmin = depth_min.reshape(B).float()
        dmax = depth_max.reshape(B).float()

        propa_off: Optional[Tensor] = None
        if Kp > 0 and not (self.stage == 1 and iters == 1):
            if self._native_propa:
                propa_off = self._script_offset_conv(ref_feature, self._off_propa_form, self._off_propa_frag, self.propa_conv.bias, 2 * Kp)
            else:
                propa_off = self.propa_conv(ref_feature)
        if self._native_eval:
            eval_off = self._script_offset_conv(ref_feature, self._off_eval_form, self._off_eval_frag, self.eval_conv.bias, 2 * Ke)
        else:
            eval_off = self.eval_conv(ref_feature)

        # the three layouts of _forward_eager: one pack; reference and uniform sources of another size apart; a ragged pack of
        # sources that differ from each other (CPU extents beside the flat data)
        same_size = True
        uniform = True
        for f in src_features:
            if f.size(0) != B or f.size(1) != ref_feature.size(1) or f.size(2) != H or f.size(3) != W:
                same_size = False
            if f.size() != src_features[0].size():
                uniform = False
        extents: Optional[Tensor] = None
        if same_size:
            pack = torch.ops.pmb200.pack_nhwc([ref_feature] + src_features)
            ref_nhwc = pack[0]
            src_nhwc = pack[1:]
        elif uniform:
            ref_nhwc = torch.ops.pmb200.pack_nhwc([ref_feature])[0]
            src_nhwc = torch.ops.pmb200.pack_nhwc(src_features)
        else:
            ref_nhwc = torch.ops.pmb200.pack_nhwc([ref_feature])[0]
            src_nhwc, extents = torch.ops.pmb200.pack_nhwc_views(src_features)
        rt = torch.ops.pmb200.relative_projection(ref_proj, src_projs)
        feature_weight = torch.ops.pmb200.offset_corr_weight(ref_nhwc, eval_off, self._head_fw, self.G, Ke, self.dilation)

        sample = depth
        vw = view_weights
        prob = torch.empty(0, device=ref_feature.device)
        outs: List[Tensor] = []
        for it in range(1, iters + 1):
            last_of_stage1 = self.stage == 1 and it == iters
            kp_now = 0
            if Kp > 0 and not last_of_stage1:
                kp_now = Kp
            if sample.numel() == 0:
                if self.rand_draw.numel() != 0:
                    seed = self.rand_draw.to(ref_feature.device)
                else:
                    seed = torch.rand([B, 48, H, W], device=ref_feature.device)
                mode, ns = 0, 48
            elif self.patchmatch_num_sample == 1:
                seed, mode, ns = sample, 2, 1
            else:
                seed, mode, ns = sample, 1, self.patchmatch_num_sample
            off_now: Optional[Tensor] = None
            if kp_now > 0:
                off_now = propa_off
            hyp, xs = torch.ops.pmb200.init_propagate(
                seed, off_now, dmin, dmax, mode, ns, kp_now, self.dilation, self.patchmatch_interval_scale
            )
            if vw.numel() == 0:
                if extents is None:
                    vw, sims = torch.ops.pmb200.warp_corr_view_weights(ref_nhwc, src_nhwc, rt, hyp, self._head_pw, self.G)
                else:
                    vw, sims = torch.ops.pmb200.warp_corr_view_weights_views(ref_nhwc, src_nhwc, extents, rt, hyp, self._head_pw, self.G)
                torch.ops.pmb200.aggregate_views_score_(sims, vw, self._head_sim, xs)
            elif extents is None:
                torch.ops.pmb200.warp_corr_score_(ref_nhwc, src_nhwc, rt, hyp, vw, self._head_sim, self.G, xs)
            else:
                torch.ops.pmb200.warp_corr_score_views_(ref_nhwc, src_nhwc, extents, rt, hyp, vw, self._head_sim, self.G, xs)
            new_depth, prob = torch.ops.pmb200.adaptive_eval(
                xs, hyp, eval_off, feature_weight, dmin, dmax, self.dilation, self.patchmatch_interval_scale, last_of_stage1
            )
            sample = new_depth.unsqueeze(1)
            outs.append(sample)
        return outs, prob, vw.detach()

    def _script_offset_conv(self, x: Tensor, form: int, frag: Tensor, bias: Optional[Tensor], cout: int) -> Tensor:
        """One offset conv in the form `refresh_script_heads` froze (what `_offset_conv` runs in eager mode)."""
        if form == 0:
            return torch.ops.pmb200.conv2d_nhwc(x, frag, bias, cout, 3, 1, self.dilation, self.dilation, False, self._conv_precision)
        return torch.ops.pmb200.conv2d_tc5(x, frag, bias, cout, 3, 1, self.dilation, self.dilation, False, form == 2)

    @torch.jit.unused
    def _forward_eager(
        self,
        ref_feature: Tensor,
        src_features: List[Tensor],
        ref_proj: Tensor,
        src_projs: List[Tensor],
        depth_min: Tensor,
        depth_max: Tensor,
        depth: Tensor,
        view_weights: Tensor,
    ) -> Tuple[List[Tensor], Tensor, Tensor]:
        self._check_neighbour_counts()
        assert len(src_features) == len(
            src_projs
        ), "Patchmatch Evaluation: Different number of images and projection matrices"
        if not is_empty(view_weights):
            assert (
                len(src_features) == view_weights.size()[1]
            ), "Patchmatch Evaluation: Different number of images and view weights"
        if not ops._on_device(ref_feature):
            raise RuntimeError(
                "patchmatchnet_b200.PatchMatch runs on CUDA (sm_90a) only; there is no CPU fallback "
                f"(got a tensor on {ref_feature.device})"
            )
        # autograd is needed when anything upstream or any parameter can receive a gradient
        need_grad = torch.is_grad_enabled() and (
            ref_feature.requires_grad
            or any(f.requires_grad for f in src_features)
            or any(p.requires_grad for p in self.parameters())
        )

        B, C, H, W = ref_feature.shape
        V = len(src_features)
        Kp, Ke = self.propagate_neighbors, self.evaluate_neighbors
        iters = self.patchmatch_iteration
        depth_min = depth_min.reshape(B).float()
        depth_max = depth_max.reshape(B).float()

        # learned 2-D offsets: native channels-last tensor-core conv (inference), cuDNN + autograd (training)
        native_conv = not torch.is_grad_enabled()
        propa_off: Optional[Tensor] = None
        if Kp > 0 and not (self.stage == 1 and iters == 1):
            propa_off = _offset_conv(self.propa_conv, self._propa_packed, ref_feature, native_conv)
        eval_off = _offset_conv(self.eval_conv, self._eval_packed, ref_feature, native_conv)

        # channels-last feature pack [1+V,B,H,W,C] (zero-copy if the producer already emitted it)
        same_size = all(f.shape == ref_feature.shape for f in src_features)
        src_shapes: Optional[Tuple[Tuple[int, int], ...]] = None  # training over a ragged source pack: each view's (H, W)
        if need_grad:
            from . import autograd as ag  # training configuration: native forward + native backward kernels

            if same_size:
                pack = ag.PackNHWC.apply(ref_feature, *src_features)
                ref_nhwc, src_nhwc = pack[0], pack[1:]
            elif any(f.shape != src_features[0].shape for f in src_features[1:]):
                # source views of different sizes: the flat data of a ragged pack travels through autograd, the
                # per-view sizes beside it (WarpCorrViews rebuilds the pack)
                ref_nhwc = ag.PackNHWC.apply(ref_feature)[0]
                src_nhwc = ag.PackNHWCViews.apply(*src_features)
                src_shapes = tuple(tuple(f.shape[2:]) for f in src_features)
            else:
                ref_nhwc = ag.PackNHWC.apply(ref_feature)[0]
                src_nhwc = ag.PackNHWC.apply(*src_features)
        elif same_size:
            pack = ops.pack_nhwc([ref_feature] + list(src_features))
            ref_nhwc, src_nhwc = pack[0], pack[1:]
        elif any(f.shape != src_features[0].shape for f in src_features[1:]):
            # source views of different sizes (several cameras, mixed orientations): a ragged pack, one extent per view
            ref_nhwc = ops.pack_nhwc([ref_feature])[0]
            src_nhwc = ops.pack_nhwc_views(list(src_features))
        else:
            ref_nhwc = ops.pack_nhwc([ref_feature])[0]
            src_nhwc = ops.pack_nhwc(list(src_features))
        with torch.no_grad():
            rt = ops.relative_projection(ref_proj, list(src_projs))

        # eval-mode fusion of the heads has no backward: it is used only when nothing needs a gradient
        fused = (not self.training) and (not need_grad) and self.fuse_heads and (C, self.G) in ops.FUSED_HEAD_SHAPES
        # feature weight of the evaluation neighbours, once per stage (reference patchmatch.py:475)
        if fused:
            feature_weight = ops.offset_corr_weight(ref_nhwc, eval_off, self.G, Ke, self.dilation, self.feature_weight_net.folded())
        elif need_grad:
            feature_weight = self.feature_weight_net(ag.OffsetCorr.apply(ref_nhwc.detach(), eval_off, self.G, Ke, self.dilation))
        else:
            feature_weight = self.feature_weight_net(ops.offset_corr(ref_nhwc, eval_off, self.G, Ke, self.dilation))

        sample = depth
        prob = torch.empty(0, device=ref_feature.device)
        outs: List[Tensor] = []
        for it in range(1, iters + 1):
            last_of_stage1 = self.stage == 1 and it == iters
            kp_now = Kp if (Kp > 0 and not last_of_stage1) else 0
            if is_empty(sample):
                draw = self.rand_source if self.rand_source is not None else torch.rand
                seed = draw(size=(B, 48, H, W), device=ref_feature.device)
                mode, ns = ops.MODE_RANDOM, 48
            elif self.patchmatch_num_sample == 1:
                seed, mode, ns = sample.detach(), ops.MODE_PASSTHROUGH, 1
            else:
                seed, mode, ns = sample.detach(), ops.MODE_PERTURB, self.patchmatch_num_sample
            xs = None
            if fused:  # (xnorm, score) interleaved: K-C writes .x, the K-A epilogue .y, K-B gathers both at once
                xs = ops.alloc_xs(B, ns + kp_now, H, W, ref_feature.device)
                hyp = ops.init_propagate(
                    seed, propa_off if kp_now > 0 else None, depth_min, depth_max,
                    mode, ns, kp_now, self.dilation, self.patchmatch_interval_scale, xs=xs,
                )
                xnorm = None
            elif need_grad and kp_now > 0:
                hyp, xnorm = ag.InitPropagate.apply(
                    seed, propa_off, depth_min, depth_max, mode, ns, kp_now, self.dilation, self.patchmatch_interval_scale
                )
            else:
                hyp, xnorm = ops.init_propagate(
                    seed, propa_off if kp_now > 0 else None, depth_min, depth_max,
                    mode, ns, kp_now, self.dilation, self.patchmatch_interval_scale, with_xnorm=True,
                )  # [B,D,H,W] hypotheses and their normalised inverse depth

            if fused:
                if is_empty(view_weights):
                    # first iteration on the coarsest stage: PixelwiseNet in the K-A epilogue; the per-view
                    # similarities are kept (L2-resident) and aggregated + scored by a light second kernel
                    view_weights, sims = ops.warp_corr_view_weights(
                        ref_nhwc, src_nhwc, rt, hyp, self.G, self.evaluation.pixel_wise_net.folded(), keep_sims=True
                    )
                    ops.aggregate_views_score(sims, view_weights, self.evaluation.similarity_net.folded(), xs=xs)
                else:
                    ops.warp_corr_score(
                        ref_nhwc, src_nhwc, rt, hyp, self.G, view_weights, self.evaluation.similarity_net.folded(), xs=xs
                    )
                score0 = None
            elif need_grad:
                if src_shapes is None:
                    warp_corr = lambda vw: ag.WarpCorr.apply(ref_nhwc, src_nhwc, rt, hyp, vw, self.G)
                else:
                    warp_corr = lambda vw: ag.WarpCorrViews.apply(ref_nhwc, src_nhwc, rt, hyp, vw, self.G, src_shapes)
                if is_empty(view_weights):
                    sims = warp_corr(None)  # [V,B,G,D,H,W]
                    if self.training:
                        view_weights = torch.cat([self.evaluation.pixel_wise_net(sims[v]) for v in range(V)], dim=1)
                    else:
                        vw = self.evaluation.pixel_wise_net(sims.reshape(V * B, self.G, hyp.shape[1], H, W))
                        view_weights = vw.view(V, B, H, W).permute(1, 0, 2, 3).contiguous()
                    score0 = self.evaluation.similarity_net(ag.AggregateViews.apply(sims, view_weights))
                else:
                    score0 = self.evaluation.similarity_net(warp_corr(view_weights))
            elif is_empty(view_weights):
                sims = ops.warp_corr(ref_nhwc, src_nhwc, rt, hyp, self.G)  # [V,B,G,D,H,W]
                if self.training:
                    vws = [self.evaluation.pixel_wise_net(sims[v]) for v in range(V)]
                    view_weights = torch.cat(vws, dim=1)
                else:  # BatchNorm uses running statistics: all views in one pass
                    D = hyp.shape[1]
                    vw = self.evaluation.pixel_wise_net(sims.view(V * B, self.G, D, H, W))  # [V*B,1,H,W]
                    view_weights = vw.view(V, B, H, W).permute(1, 0, 2, 3).contiguous()
                score0 = self.evaluation.similarity_net(ops.aggregate_views(sims, view_weights))  # [B,D,H,W]
            else:
                score0 = self.evaluation.similarity_net(ops.warp_corr(ref_nhwc, src_nhwc, rt, hyp, self.G, view_weights))
            if need_grad:
                new_depth, prob = ag.AdaptiveEval.apply(
                    score0, hyp, xnorm, eval_off, feature_weight, depth_min, depth_max,
                    self.dilation, self.patchmatch_interval_scale, last_of_stage1,
                )
            else:
                new_depth, prob = ops.adaptive_eval(
                    score0, hyp, eval_off, feature_weight, depth_min, depth_max,
                    self.dilation, self.patchmatch_interval_scale, last_of_stage1, xnorm=xnorm, xs=xs,
                )
            sample = new_depth.unsqueeze(1)
            outs.append(sample)
        return outs, prob, view_weights.detach()
