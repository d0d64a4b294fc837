"""Per-layer micro-benchmark of the native channels-last tensor-core conv (csrc/pm_conv.cu) against the cuDNN call it
replaces, at the sizes of one 640x512 1+4-view forward (5 stacked views through FeatureNet, 1 view through the rest).

    python tools/convbench.py > convbench.json

cold = L2 flushed before each launch (CUDA events on the launching stream), warm = 10 back-to-back launches.
GB/s = (input + output activation bytes) / cold time: the traffic a perfectly fused layer must move.
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops  # noqa: E402

dev = "cuda:0"
torch.backends.cudnn.benchmark = True
H, W = int(os.environ.get("CB_H", 512)), int(os.environ.get("CB_W", 640))
# name: (N, cin, cout, ks, stride, pad, dil, relu, h, w)
LAYERS = [
    ("feature.conv0", 5, 3, 8, 3, 1, 1, 1, True, H, W),
    ("feature.conv1", 5, 8, 8, 3, 1, 1, 1, True, H, W),
    ("feature.conv2", 5, 8, 16, 5, 2, 2, 1, True, H, W),
    ("feature.conv3/4", 5, 16, 16, 3, 1, 1, 1, True, H // 2, W // 2),
    ("feature.conv5", 5, 16, 32, 5, 2, 2, 1, True, H // 2, W // 2),
    ("feature.conv6/7", 5, 32, 32, 3, 1, 1, 1, True, H // 4, W // 4),
    ("feature.conv8", 5, 32, 64, 5, 2, 2, 1, True, H // 4, W // 4),
    ("feature.conv9/10", 5, 64, 64, 3, 1, 1, 1, True, H // 8, W // 8),
    ("feature.output1", 5, 64, 64, 1, 1, 0, 1, False, H // 8, W // 8),
    ("feature.inner1", 5, 32, 64, 1, 1, 0, 1, False, H // 4, W // 4),
    ("feature.output2", 5, 64, 32, 1, 1, 0, 1, False, H // 4, W // 4),
    ("feature.inner2", 5, 16, 64, 1, 1, 0, 1, False, H // 2, W // 2),
    ("feature.output3", 5, 64, 16, 1, 1, 0, 1, False, H // 2, W // 2),
    ("stage3.propa_conv", 1, 64, 32, 3, 1, 2, 2, False, H // 8, W // 8),
    ("stage3.eval_conv", 1, 64, 18, 3, 1, 2, 2, False, H // 8, W // 8),
    ("stage2.propa_conv", 1, 32, 16, 3, 1, 4, 4, False, H // 4, W // 4),
    ("stage2.eval_conv", 1, 32, 18, 3, 1, 4, 4, False, H // 4, W // 4),
    ("stage1.eval_conv", 1, 16, 18, 3, 1, 6, 6, False, H // 2, W // 2),
    ("refine.conv1", 1, 1, 8, 3, 1, 1, 1, True, H // 2, W // 2),
    ("refine.conv2", 1, 8, 8, 3, 1, 1, 1, True, H // 2, W // 2),
    ("refine.conv0", 1, 3, 8, 3, 1, 1, 1, True, H, W),
    ("refine.conv3", 1, 16, 8, 3, 1, 1, 1, True, H, W),
    ("refine.res", 1, 8, 1, 3, 1, 1, 1, False, H, W),
]
flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10):
    for _ in range(3):
        fn()
    cold = []
    for _ in range(iters):
        flush_buf.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        cold.append(a.elapsed_time(b) * 1e3)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(2_000_000)
    a.record()
    for _ in range(10):
        fn()
    b.record()
    b.synchronize()
    return sum(cold) / len(cold), min(cold), a.elapsed_time(b) * 1e2


rows = []
g = torch.Generator().manual_seed(0)
for (name, N, cin, cout, ks, S, pad, dil, relu, h, w) in LAYERS:
    x = torch.randn(N, cin, h, w, generator=g).to(dev).contiguous(memory_format=torch.channels_last)
    wt = (torch.randn(cout, cin, ks, ks, generator=g) / (cin * ks * ks) ** 0.5).to(dev)
    wcl = wt.contiguous(memory_format=torch.channels_last)
    b = torch.randn(cout, generator=g).to(dev)
    frags = {1: ops.pack_conv_filter(wt, 1), 3: ops.pack_conv_filter(wt, 3)}
    frag = frags[1]
    ho = (h + 2 * pad - dil * (ks - 1) - 1) // S + 1
    wo = (w + 2 * pad - dil * (ks - 1) - 1) // S + 1
    act_bytes = 4 * N * (h * w * cin + ho * wo * cout)
    flops = 2.0 * N * ho * wo * cout * cin * ks * ks
    row = {"layer": name, "shape": f"N{N} {cin}->{cout} k{ks} s{S} d{dil} {h}x{w}", "activation_mb": act_bytes / 1e6, "gflop": flops / 1e9}
    torch.backends.cudnn.allow_tf32 = True
    if relu and dil == 1:
        lib = lambda: torch.cudnn_convolution_relu(x, wcl, b, (S, S), (pad, pad), (dil, dil), 1)
    else:
        lib = lambda: F.conv2d(x, wcl, b, S, pad, dil)
    c, cmin, wm = timeit(lib)
    row["cudnn_tf32_us"] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
    best = None
    for prec in (1, 3):
        for mt in ((0, 1, 2, 4, -1) if prec == 1 else (0,)):
            fn = lambda: ops.conv2d_nhwc(x, frags[prec], b, cout, ks, S, pad, dil, relu=relu, precision=prec, rows_per_warp=mt)
            try:
                c, cmin, wm = timeit(fn)
            except Exception as e:  # noqa: BLE001
                row[f"native_p{prec}_mt{mt}_us"] = f"ERR {e}"
                continue
            row[f"native_p{prec}_mt{mt}_us"] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
            if prec == 1 and mt == 0:
                row["native_tf32_gbs"] = round(act_bytes / (c * 1e-6) / 1e9, 1)
                row["native_tf32_tflops"] = round(flops / (c * 1e-6) / 1e12, 2)
                row["speedup_vs_cudnn_cold"] = round(row["cudnn_tf32_us"]["cold"] / c, 2)
    if cin in (8, 16, 32, 64):  # K-D5: wgmma implicit GEMM, 3xTF32 (fp32-accurate) -- compare with native_p3
        try:
            f5 = ops.pack_conv_filter_tc5(wt)
            c, cmin, wm = timeit(lambda: ops.conv2d_tc5(x, f5, b, cout, ks, S, pad, dil, relu=relu))
            row["tc5_3xtf32_us"] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
            row["tc5_tflops_3x"] = round(3 * flops / (c * 1e-6) / 1e12, 1)
        except Exception as e:  # noqa: BLE001
            row["tc5_3xtf32_us"] = f"ERR {e}"
        if S == 1:  # K-D5h: halo tile once per output tile, taps as shifted descriptors
            try:
                f5h = ops.pack_conv_filter_tc5h(wt)
                c, cmin, wm = timeit(lambda: ops.conv2d_tc5(x, f5h, b, cout, ks, 1, pad, dil, relu=relu, halo=True))
                row["tc5h_3xtf32_us"] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
            except Exception as e:  # noqa: BLE001
                row["tc5h_3xtf32_us"] = f"ERR {e}"
    rows.append(row)
# K-S: conv0 -> conv1 fused (exact fp32) against the two K-D launches it replaces (3xTF32), same 5 x H x W input
x3 = torch.randn(5, 3, H, W, generator=g).to(dev)
w0, b0 = torch.randn(8, 3, 3, 3, generator=g) / 27 ** 0.5, torch.randn(8, generator=g)
w1, b1 = torch.randn(8, 8, 3, 3, generator=g) / 72 ** 0.5, torch.randn(8, generator=g)
stem_ab = {}
for ppt in (2, 4):  # output pixels per thread (LDCU : FFMA ratio 1 : 4 PPT in the conv1 phase)
    ops.set_tuning("stem_ppt", ppt)
    c, cmin, wm = timeit(lambda: ops.conv_stem(x3, w0, b0, w1, b1))
    stem_ab[f"ppt{ppt}"] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
ops.set_tuning("reset")
c, cmin, wm = timeit(lambda: ops.conv_stem(x3, w0, b0, w1, b1))
stem = {"pixels_per_thread_ab_us": stem_ab, "layer": "feature.conv0+conv1 fused (K-S)", "shape": f"N5 3->8->8 k3 {H}x{W}", "stem_us": {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)},
        "replaces_us_cold": sum(r["native_p3_mt0_us"]["cold"] for r in rows if r["layer"] in ("feature.conv0", "feature.conv1")),
        "gbs_in_plus_out": round(4 * 5 * H * W * (3 + 8) / (c * 1e-6) / 1e9, 1)}
# K-R: Refinement fused into two exact-fp32 launches against its conv-family path (the six native conv launches of
# Refinement._native_tail, without the elementwise depth tail), one view
from patchmatchnet_b200.net import Refinement  # noqa: E402

torch.backends.cudnn.allow_tf32 = False
ref_mod = Refinement().eval().to(dev)
rimg = torch.rand(1, 3, H, W, generator=g).to(dev)
rlo, rhi = torch.tensor([425.0], device=dev), torch.tensor([935.0], device=dev)
rdepth = 425.0 + 510.0 * torch.rand(1, 1, H // 2, W // 2, generator=g).to(dev)
refine = {"layer": "Refinement (K-R)", "shape": f"N1 {H}x{W}"}
rd = (rdepth - rlo) / (rhi - rlo)
rimg_cl = rimg.contiguous(memory_format=torch.channels_last)
with torch.no_grad():
    for key, fn in (("fused_us", lambda: ref_mod(rimg, rdepth, rlo, rhi)), ("conv_family_us", lambda: ref_mod._native_tail(rimg_cl, rd))):
        c, cmin, wm = timeit(fn)
        refine[key] = {"cold": round(c, 1), "cold_min": round(cmin, 1), "warm": round(wm, 1)}
torch.backends.cudnn.allow_tf32 = True
tot_lib = sum(r["cudnn_tf32_us"]["cold"] for r in rows)
tot_nat = sum(r["native_p1_mt0_us"]["cold"] for r in rows if isinstance(r.get("native_p1_mt0_us"), dict))
print(json.dumps({"gpu": torch.cuda.get_device_name(0), "size": [H, W], "sum_cold_us": {"cudnn_tf32": round(tot_lib, 1), "native_tf32": round(tot_nat, 1)},
                  "layers": rows, "stem": stem, "refinement": refine}, indent=1))
