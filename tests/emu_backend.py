"""Test-only CPU backend: runs the REAL host code of the package (ops wrappers, PatchMatch._forward_eager) on CPU tensors
against the CPU-emulated kernels (tests/warp_emu.h).  TEST INFRASTRUCTURE -- nothing under patchmatchnet_b200/ knows about it.

`install(monkeypatch, emu_lib, emu_conv_lib)` swaps three module hooks of patchmatchnet_b200.ops (`_on_device`,
`_device_guard`, `_stream`) and `_native.lib` for a facade whose `pmb200_*` attributes adapt the C-ABI argument lists to the
emulation harness entry points (which take the launch configuration explicitly instead of a stream).  The launch
configurations mirror the defaults of the launchers in csrc/pm_kernels.cu."""
import contextlib
import ctypes

from patchmatchnet_b200 import _native, ops


# launch configuration of the fourth-generation fused warp+correlation kernel under the emulator: 4 consumer warps (the
# launcher's default), a window slot of 96 texels (most boxes fit, some are clipped and take the global path) and 7
# persistent CTAs, so that every CTA walks several items through its rings
KA4_NW, KA4_CAP, KA4_GRID, KA4_STAGES = 4, 96, 7, 3


class EmulatedLibrary:
    def __init__(self, emu, emu_conv):
        self.emu, self.conv = emu, emu_conv
        self.calls = {}  # entry point -> number of calls (tests assert that the native path, not a torch op, ran)

    def __getattribute__(self, name):
        attr = object.__getattribute__(self, name)
        if name.startswith("pmb200_") and callable(attr):
            calls = object.__getattribute__(self, "calls")
            calls[name] = calls.get(name, 0) + 1
        return attr

    def pmb200_abi_version(self):
        return 1

    def pmb200_last_error(self):
        return b"emulated kernels"

    def pmb200_relative_projection(self, ref, ref_stride, arr, src_stride, V, B, out, stream):
        return self.emu.emu_relative_projection(ref, ref_stride, ctypes.cast(arr, ctypes.c_void_p), src_stride, V, B, out)

    def pmb200_pack_nhwc(self, arr, n, B, C, H, W, out, stream):
        return self.emu.emu_pack_nhwc(ctypes.cast(arr, ctypes.c_void_p), n, B, C, H, W, out)

    def pmb200_photometric_confidence(self, prob, out, B, D, h, w, H_out, W_out, stream):
        return self.emu.emu_photometric_confidence(prob, out, B, D, h, w, H_out, W_out)

    def pmb200_upsample2x_add_nhwc(self, x, y, bias, out, N, h, w, C, stream):
        return self.emu.emu_upsample2x_add_nhwc(x, y, bias, out, N, h, w, C)

    def _ka(self, epi, ref, src, rt, depth, vw, head, out, sims, stride, V, B, C, G, H, W, Hs, Ws, D):
        if (C, G) not in ((64, 8), (32, 8), (16, 4)):
            if epi > 1:
                return -2
            return self.emu.emu_warp_corr_generic(ref, src, rt, depth, vw, out, V, B, C, G, H, W, Hs, Ws, D)
        return self.emu.emu_warp_corr4(ref, src, rt, depth, vw, head, out, sims, stride, V, B, C, G, H, W, Hs, Ws, D, epi,
                                       KA4_NW, KA4_CAP, KA4_GRID, KA4_STAGES)

    def pmb200_warp_corr(self, ref, src, rt, depth, vw, out, V, B, C, G, H, W, Hs, Ws, D, stream):
        return self._ka(0 if vw is None else 1, ref, src, rt, depth, vw, None, out, None, 1, V, B, C, G, H, W, Hs, Ws, D)

    def pmb200_warp_corr_score(self, ref, src, rt, depth, vw, head, out, stride, V, B, C, G, H, W, Hs, Ws, D, stream):
        return self._ka(2, ref, src, rt, depth, vw, head, out, None, stride, V, B, C, G, H, W, Hs, Ws, D)

    def pmb200_warp_corr_view_weights(self, ref, src, rt, depth, head, out, sims, V, B, C, G, H, W, Hs, Ws, D, stream):
        ctypes.memset(out, 0, 4 * B * V * H * W)  # the launcher zero-fills the atomic-max target
        return self._ka(3, ref, src, rt, depth, None, head, out, sims, 1, V, B, C, G, H, W, Hs, Ws, D)

    def pmb200_aggregate_views(self, sims, vw, out, V, B, G, D, H, W, stream):
        return self.emu.emu_aggregate_views(sims, vw, out, V, B, G, D, H, W)

    def pmb200_aggregate_views_score(self, sims, vw, head, out, stride, V, B, G, D, H, W, stream):
        return self.emu.emu_aggregate_views_score(sims, vw, head, out, stride, V, B, G, D, H, W)

    def pmb200_offset_corr(self, ref, off, off_cl, out, B, C, G, H, W, K, dilation, stream):
        return self.emu.emu_offset_corr(ref, off, off_cl, None, out, B, C, G, H, W, K, dilation)

    def pmb200_offset_corr_weight(self, ref, off, off_cl, head, out, B, C, G, H, W, K, dilation, stream):
        return self.emu.emu_offset_corr(ref, off, off_cl, head, out, B, C, G, H, W, K, dilation)

    def pmb200_init_propagate(self, seed, off, off_cl, dmin, dmax, out, xn, xstride, mode, B, H, W, Ns, Kp, dilation, scale, stream):
        return self.emu.emu_init_propagate(seed, off, off_cl, dmin, dmax, out, xn, xstride, mode, B, H, W, Ns, Kp, dilation, scale)

    def pmb200_adaptive_eval(self, score0, depth, xnorm, xs, off, off_cl, fw, dmin, dmax, prob, depth_out, B, D, H, W, K, dilation,
                             scale, is_inverse, stream):
        return self.emu.emu_adaptive_eval(score0, depth, xnorm, xs, off, off_cl, fw, dmin, dmax, prob, depth_out, B, D, H, W, K,
                                          dilation, scale, is_inverse, 16, min(D, 16))

    # ---- backward kernels (training configuration; patchmatchnet_b200/autograd.py) ----
    def pmb200_warp_corr_backward(self, ref, src, rt, depth, vw, g, d_ref, d_src, V, B, C, G, H, W, Hs, Ws, D, stream):
        return self.emu.emu_warp_corr_backward(ref, src, rt, depth, vw, g, d_ref, d_src, V, B, C, G, H, W, Hs, Ws, D)

    def pmb200_aggregate_views_backward(self, sims, vw, g, d_sims, d_vw, V, B, G, D, H, W, stream):
        return self.emu.emu_aggregate_views_backward(sims, vw, g, d_sims, d_vw, V, B, G, D, H, W)

    def pmb200_offset_corr_backward(self, ref, off, g, d_off, B, C, G, H, W, K, dilation, stream):
        return self.emu.emu_offset_corr_backward(ref, off, g, d_off, B, C, G, H, W, K, dilation)

    def pmb200_init_propagate_backward(self, seed, off, dmin, dmax, g, d_off, mode, B, H, W, Ns, Kp, dilation, scale, stream):
        return self.emu.emu_init_propagate_backward(seed, off, dmin, dmax, g, d_off, mode, B, H, W, Ns, Kp, dilation, scale)

    def pmb200_adaptive_eval_backward(self, score0, hyp, xnorm, off, fw, dmin, dmax, prob, g_depth, g_prob, d_score0, d_hyp, d_off, d_fw,
                                      B, D, H, W, K, dilation, scale, inverse, stream):
        return self.emu.emu_adaptive_eval_backward(score0, hyp, xnorm, off, fw, dmin, dmax, prob, g_depth, g_prob, d_score0, d_hyp, d_off,
                                                   d_fw, B, D, H, W, K, dilation, scale, inverse)

    def pmb200_conv2d_tc5_supported(self, cin, cout, ks, stride):
        return 0  # wgmma has no emulation: the convs take the mma.sync kernel here, K-D5 is checked on the GPU only

    def pmb200_conv2d_filter_floats(self, cin, cout, ks, prec):
        return self.conv.emu_conv2d_filter_floats(cin, cout, ks, prec)

    def pmb200_conv2d_nhwc(self, *args):
        return self.conv.emu_conv2d_nhwc(*args)

    def pmb200_conv_stem(self, *args):
        return self.conv.emu_conv_stem(*args)

    def pmb200_refine_low(self, *args):
        return self.conv.emu_refine_low(*args)

    def pmb200_refine_full(self, *args):
        return self.conv.emu_refine_full(*args)


def install(monkeypatch, emu, emu_conv):
    facade = EmulatedLibrary(emu, emu_conv)
    monkeypatch.setattr(_native, "lib", lambda: facade)
    monkeypatch.setattr(_native, "check", lambda rc, what: (_ for _ in ()).throw(RuntimeError(f"{what}: emulated call returned {rc}")) if rc else None)
    monkeypatch.setattr(ops, "_on_device", lambda t: True)
    monkeypatch.setattr(ops, "_device_guard", lambda t: contextlib.nullcontext())
    monkeypatch.setattr(ops, "_stream", lambda t: None)
    return facade
