"""torch.autograd bridges for the native kernels (training configuration).

Forward = the same C-ABI launches the inference path uses; backward = the kernels in
``csrc/pm_backward.cu``.  Which inputs receive a gradient mirrors the reference graph
(SURVEY.md 3.4): the warp grid is built under ``no_grad`` (module.py:147), ``depth_weight`` and the
incoming depth are detached (patchmatch.py:74,85,503,506,669), ``FeatureWeightNet`` gets a detached
reference feature (patchmatch.py:475).  The 1x1x1 heads stay ordinary torch modules in training
(BatchNorm needs batch statistics), so their gradients come from torch's own autograd.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _native, ops

Tensor = torch.Tensor


def _ptr(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


class PackNHWC(torch.autograd.Function):
    """n NCHW maps -> one channels-last pack [n,B,H,W,C]; backward hands every map its slice, re-viewed as NCHW."""

    @staticmethod
    def forward(ctx, *maps: Tensor) -> Tensor:
        return ops.pack_nhwc([m.detach() for m in maps])

    @staticmethod
    def backward(ctx, g: Tensor):
        return tuple(g[i].permute(0, 3, 1, 2) for i in range(g.shape[0]))


class WarpCorr(torch.autograd.Function):
    """K-A.  Gradients: reference feature, source features."""

    @staticmethod
    def forward(ctx, ref_nhwc: Tensor, src_nhwc: Tensor, rt: Tensor, depth: Tensor, view_weights: Optional[Tensor], G: int):
        out = ops.warp_corr(ref_nhwc.detach(), src_nhwc.detach(), rt, depth.detach(), G,
                            None if view_weights is None else view_weights.detach())
        ctx.G = G
        ctx.has_w = view_weights is not None
        ctx.save_for_backward(ref_nhwc, src_nhwc, rt, depth, *( [view_weights] if view_weights is not None else []))
        return out

    @staticmethod
    def backward(ctx, g: Tensor):
        saved = ctx.saved_tensors
        ref, src, rt, depth = [t.detach().contiguous() for t in saved[:4]]
        vw = saved[4].detach().contiguous() if ctx.has_w else None
        g = g.contiguous()
        B, H, W, C = ref.shape
        V, _, Hs, Ws, _ = src.shape
        D = depth.shape[1]
        d_ref = torch.empty_like(ref)
        d_src = torch.empty_like(src)
        with ops._device_guard(ref):
            rc = _native.lib().pmb200_warp_corr_backward(
                ref.data_ptr(), src.data_ptr(), rt.data_ptr(), depth.data_ptr(), _ptr(vw), g.data_ptr(),
                d_ref.data_ptr(), d_src.data_ptr(), V, B, C, ctx.G, H, W, Hs, Ws, D, ops._stream(ref),
            )
        _native.check(rc, "warp_corr_backward")
        return d_ref, d_src, None, None, None, None


class PackNHWCViews(torch.autograd.Function):
    """n NCHW maps [B,C,H_v,W_v] -> the flat data of their ragged channels-last pack (ops.pack_nhwc_views; rebuild the pack
    with ops.ViewPack.from_shapes); backward hands every map its slice of the flat gradient, re-viewed as NCHW."""

    @staticmethod
    def forward(ctx, *maps: Tensor) -> Tensor:
        pack = ops.pack_nhwc_views([m.detach() for m in maps])
        ctx.slices = [(o, m.shape) for o, m in zip(pack.offsets, maps)]
        return pack.data

    @staticmethod
    def backward(ctx, g: Tensor):
        return tuple(g[o:o + s.numel()].view(s[0], s[2], s[3], s[1]).permute(0, 3, 1, 2) for o, s in ctx.slices)


class WarpCorrViews(torch.autograd.Function):
    """K-A over a ragged source pack: `src_flat` is the pack's data (PackNHWCViews), `shapes` the (H, W) of every source
    view.  Gradients: reference feature, the source pack."""

    @staticmethod
    def forward(ctx, ref_nhwc: Tensor, src_flat: Tensor, rt: Tensor, depth: Tensor, view_weights: Optional[Tensor], G: int,
                shapes: Tuple[Tuple[int, int], ...]):
        B, _, _, C = ref_nhwc.shape
        pack = ops.ViewPack.from_shapes(src_flat.detach(), shapes, B, C)
        out = ops.warp_corr(ref_nhwc.detach(), pack, rt, depth.detach(), G, None if view_weights is None else view_weights.detach())
        ctx.G, ctx.pack = G, pack
        ctx.has_w = view_weights is not None
        ctx.save_for_backward(ref_nhwc, rt, depth, *([view_weights] if view_weights is not None else []))
        return out

    @staticmethod
    def backward(ctx, g: Tensor):
        saved = ctx.saved_tensors
        ref, rt, depth = [t.detach().contiguous() for t in saved[:3]]
        vw = saved[3].detach().contiguous() if ctx.has_w else None
        pack = ctx.pack
        d_ref, d_src = warp_corr_views_backward(ref, pack, rt, depth, vw, g.contiguous(), ctx.G)
        return d_ref, d_src, None, None, None, None, None


def warp_corr_views_backward(ref: Tensor, pack: "ops.ViewPack", rt: Tensor, depth: Tensor, vw: Optional[Tensor], g: Tensor,
                             G: int) -> Tuple[Tensor, Tensor]:
    """pmb200_warp_corr_views_backward -> (d_ref [B,H,W,C], d_src: the flat gradient, laid out like pack.data)."""
    B, H, W, C = ref.shape
    V, D = len(pack), depth.shape[1]
    d_ref = torch.empty_like(ref)
    d_src = torch.empty_like(pack.data)
    with ops._device_guard(ref):
        rc = _native.lib().pmb200_warp_corr_views_backward(
            ref.data_ptr(), pack.data.data_ptr(), pack.extents, rt.data_ptr(), depth.data_ptr(), _ptr(vw), g.data_ptr(),
            d_ref.data_ptr(), d_src.data_ptr(), V, B, C, G, H, W, D, ops._stream(ref),
        )
    _native.check(rc, "warp_corr_views_backward")
    end = max(o + B * h * w * C for o, h, w in zip(pack.offsets, pack.heights, pack.widths))
    if end < d_src.numel():  # the alignment padding after the last view, which the entry point does not know about
        d_src[end:].zero_()
    return d_ref, d_src


class AggregateViews(torch.autograd.Function):
    """sum_v sims[v]*w_v / (1e-5 + sum_v w_v).  Gradients: similarities and view weights."""

    @staticmethod
    def forward(ctx, sims: Tensor, view_weights: Tensor):
        ctx.save_for_backward(sims, view_weights)
        return ops.aggregate_views(sims.detach(), view_weights.detach())

    @staticmethod
    def backward(ctx, g: Tensor):
        sims, vw = [t.detach().contiguous() for t in ctx.saved_tensors]
        g = g.contiguous()
        V, B, G, D, H, W = sims.shape
        d_sims = torch.empty_like(sims)
        d_vw = torch.empty_like(vw)
        with ops._device_guard(sims):
            rc = _native.lib().pmb200_aggregate_views_backward(
                sims.data_ptr(), vw.data_ptr(), g.data_ptr(), d_sims.data_ptr(), d_vw.data_ptr(), V, B, G, D, H, W,
                ops._stream(sims),
            )
        _native.check(rc, "aggregate_views_backward")
        return d_sims, d_vw


class OffsetCorr(torch.autograd.Function):
    """K-A'.  Gradient: the raw evaluation offsets (the reference feature is detached by the caller)."""

    @staticmethod
    def forward(ctx, ref_nhwc: Tensor, offsets: Tensor, G: int, K: int, dilation: int):
        ctx.cfg = (G, K, dilation)
        ctx.save_for_backward(ref_nhwc, offsets)
        return ops.offset_corr(ref_nhwc.detach(), offsets.detach(), G, K, dilation)

    @staticmethod
    def backward(ctx, g: Tensor):
        ref, off = [t.detach().contiguous() for t in ctx.saved_tensors]
        G, K, dilation = ctx.cfg
        g = g.contiguous()
        B, H, W, C = ref.shape
        d_off = torch.empty_like(off)
        with ops._device_guard(ref):
            rc = _native.lib().pmb200_offset_corr_backward(
                ref.data_ptr(), off.data_ptr(), g.data_ptr(), d_off.data_ptr(), B, C, G, H, W, K, dilation, ops._stream(ref)
            )
        _native.check(rc, "offset_corr_backward")
        return None, d_off, None, None, None


class InitPropagate(torch.autograd.Function):
    """K-C.  Gradient: the raw propagation offsets (through the positions of the neighbour gathers)."""

    @staticmethod
    def forward(ctx, seed: Tensor, offsets: Tensor, depth_min: Tensor, depth_max: Tensor, mode: int, Ns: int, Kp: int,
                dilation: int, interval_scale: float):
        hyp, xnorm = ops.init_propagate(seed.detach(), offsets.detach(), depth_min, depth_max, mode, Ns, Kp, dilation,
                                        interval_scale, with_xnorm=True)
        ctx.cfg = (mode, Ns, Kp, dilation, float(interval_scale))
        ctx.save_for_backward(seed, offsets, depth_min, depth_max)
        ctx.mark_non_differentiable(xnorm)
        return hyp, xnorm

    @staticmethod
    def backward(ctx, g_hyp: Tensor, _g_xnorm):
        seed, off, dmin, dmax = [t.detach().contiguous() for t in ctx.saved_tensors]
        mode, Ns, Kp, dilation, scale = ctx.cfg
        g = g_hyp.contiguous()
        B, _, H, W = seed.shape
        d_off = torch.empty_like(off)
        with ops._device_guard(seed):
            rc = _native.lib().pmb200_init_propagate_backward(
                seed.data_ptr(), off.data_ptr(), dmin.data_ptr(), dmax.data_ptr(), g.data_ptr(), d_off.data_ptr(),
                mode, B, H, W, Ns, Kp, dilation, scale, ops._stream(seed),
            )
        _native.check(rc, "init_propagate_backward")
        return None, d_off, None, None, None, None, None, None, None


class AdaptiveEval(torch.autograd.Function):
    """K-B.  Gradients: raw score, hypotheses (regression), raw evaluation offsets, feature weight."""

    @staticmethod
    def forward(ctx, score0: Tensor, hyp: Tensor, xnorm: Tensor, offsets: Tensor, feature_weight: Tensor,
                depth_min: Tensor, depth_max: Tensor, dilation: int, interval_scale: float, is_inverse: bool):
        depth, prob = ops.adaptive_eval(score0.detach(), hyp.detach(), offsets.detach(), feature_weight.detach(),
                                        depth_min, depth_max, dilation, interval_scale, is_inverse, xnorm=xnorm.detach())
        ctx.cfg = (dilation, float(interval_scale), bool(is_inverse))
        ctx.save_for_backward(score0, hyp, xnorm, offsets, feature_weight, depth_min, depth_max, prob)
        ctx.set_materialize_grads(False)
        return depth, prob

    @staticmethod
    def backward(ctx, g_depth: Optional[Tensor], g_prob: Optional[Tensor]):
        score0, hyp, xnorm, off, fw, dmin, dmax, prob = [t.detach().contiguous() for t in ctx.saved_tensors]
        dilation, scale, inverse = ctx.cfg
        if g_depth is None and g_prob is None:
            return (None,) * 10
        g_depth = None if g_depth is None else g_depth.contiguous()
        g_prob = None if g_prob is None else g_prob.contiguous()
        B, D, H, W = score0.shape
        K = fw.shape[1]
        d_score0 = torch.empty_like(score0)
        d_hyp = torch.empty_like(hyp)
        d_off = torch.empty_like(off)
        d_fw = torch.empty_like(fw)
        with ops._device_guard(score0):
            rc = _native.lib().pmb200_adaptive_eval_backward(
                score0.data_ptr(), hyp.data_ptr(), xnorm.data_ptr(), off.data_ptr(), fw.data_ptr(), dmin.data_ptr(),
                dmax.data_ptr(), prob.data_ptr(), _ptr(g_depth), _ptr(g_prob), d_score0.data_ptr(), d_hyp.data_ptr(),
                d_off.data_ptr(), d_fw.data_ptr(), B, D, H, W, K, dilation, scale, 1 if inverse else 0, ops._stream(score0),
            )
        _native.check(rc, "adaptive_eval_backward")
        return d_score0, d_hyp, None, d_off, d_fw, None, None, None, None, None


def loss_from_terms(terms: Tensor, levels) -> Tensor:
    """sum_m terms[m] / terms[n_maps + levels[m]] in float64 on the device, cast to float32 (nan for a level without masked
    pixels, as the reference's mean of an empty selection)."""
    n = len(levels)
    counts = terms[n + torch.tensor(list(levels), dtype=torch.int64).to(terms.device, non_blocking=True)]
    return (terms[:n] / counts).sum().float()


class DepthLoss(torch.autograd.Function):
    """patchmatchnet_loss (reference models/net.py:321-342) on the K-L kernels: loss = sum_m terms[m] / terms[n_maps + l_m],
    formed on the device in float64 and cast to float32 (no host synchronisation; a level without masked pixels gives nan,
    as the reference's mean of an empty selection does).  Gradients: the depth maps, in one launch.

        loss = DepthLoss.apply(levels, depth_gt, mask, all_reduce, scale, *maps)

    levels: the pyramid level of each map; depth_gt float32 [B,H,W], mask [B,H,W] at full resolution.  all_reduce: None, or a
    callable that sums the float64 terms across ranks in place before the loss is formed, so every rank holds the loss of the
    global batch; scale: the factor the backward applies (the world size when the parameter gradients are then averaged)."""

    @staticmethod
    def forward(ctx, levels, depth_gt: Tensor, mask: Tensor, all_reduce, scale: float, *maps: Tensor) -> Tensor:
        maps = [m.detach() for m in maps]
        terms = ops.depth_loss_terms(maps, levels, depth_gt, mask)
        if all_reduce is not None:
            all_reduce(terms)
        ctx.levels, ctx.scale = list(levels), float(scale)
        ctx.save_for_backward(depth_gt, mask, terms, *maps)
        return loss_from_terms(terms, levels)

    @staticmethod
    def backward(ctx, g: Tensor):
        gt, mask, terms, *maps = ctx.saved_tensors
        grads = ops.depth_loss_backward(maps, ctx.levels, gt, mask, terms, g.contiguous(), ctx.scale)
        return (None, None, None, None, None, *grads)
