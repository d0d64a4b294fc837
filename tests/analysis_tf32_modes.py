"""Which conv arithmetic keeps the 640x512 depth map within north_star's 1e-3 of the fp32 result?  (analysis script, CPU)

The tensor cores' TF32 path is emulated exactly enough for this question: operands reduced to 10 mantissa bits (by
truncation -- what the hardware does to raw fp32 bit patterns -- or by round-to-nearest), products and sums in fp32.
Every conv of the network (oracle port of the reference behind the repo's shell, CPU) goes through one of:
    fp32        untouched
    tf32_trunc  both operands truncated                      (library TF32 kernels fed raw fp32)
    tf32_native activations truncated, weights rounded       (pm_conv.cu precision 1)
    tf32_rna    both operands rounded to nearest
    2x_act      (a_hi + a_lo) . w_rna                        (activation split, weights rounded once)
    3x          a_hi.w_hi + a_hi.w_lo + a_lo.w_hi            (pm_conv.cu precision 3)
"native" layers = ops.conv_prefers_native's rule (memory-bound), "library" layers = the FLOP-bound ones.

    python tests/analysis_tf32_modes.py > tf32_modes.json
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402
from oracle import pm_oracle  # noqa: E402
from patchmatchnet_b200 import ops, synthetic  # noqa: E402
from tests import pm_cases  # noqa: E402

_conv2d, _convT = F.conv2d, F.conv_transpose2d


def trunc(x):
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def rna(x):
    return ops._tf32_round(x)


def conv_mode(fn, x, w, mode, *a, **k):
    if mode == "fp32":
        return fn(x, w, *a, **k)
    bias = a[0] if a else k.pop("bias", None)
    rest = a[1:]
    lin = lambda xx, ww: fn(xx, ww, None, *rest, **k)
    if mode == "tf32_trunc":
        y = lin(trunc(x), trunc(w))
    elif mode == "tf32_native":
        y = lin(trunc(x), rna(w))
    elif mode == "tf32_rna":
        y = lin(rna(x), rna(w))
    elif mode == "2x_act":
        xh = trunc(x)
        y = lin(xh, rna(w)) + lin(trunc(x - xh), rna(w))
    elif mode == "2x_act_rna":
        xh = rna(x)
        y = lin(xh, rna(w)) + lin(rna(x - xh), rna(w))
    elif mode == "3x":
        xh, wh = trunc(x), rna(w)
        y = lin(xh, wh) + lin(xh, rna(w - wh)) + lin(trunc(x - xh), wh)
    else:
        raise ValueError(mode)
    if bias is not None:
        y = y + bias.view(1, -1, 1, 1)
    return y


def run(policy):
    """policy(cin, cout, ks) -> mode"""
    def c2(x, w, *a, **k):
        return conv_mode(_conv2d, x, w, policy(w.shape[1], w.shape[0], w.shape[2]), *a, **k)

    def ct(x, w, *a, **k):
        return conv_mode(_convT, x, w, policy(w.shape[0], w.shape[1], w.shape[2]), *a, **k)

    F.conv2d, F.conv_transpose2d = c2, ct
    torch.conv2d_backup = None
    try:
        torch.manual_seed(0)
        with torch.no_grad():
            d, c, ps = NET([i.clone() for i in INP["images"]], INP["intrinsics"].clone(), INP["extrinsics"].clone(), INP["depth_min"], INP["depth_max"])
    finally:
        F.conv2d, F.conv_transpose2d = _conv2d, _convT
    return d, ps


H, W = int(os.environ.get("AH", 512)), int(os.environ.get("AW", 640))
NET, _ = bench.build_net(pm_oracle.PatchMatchOracle)
NET.stack_views = False
INP = synthetic.make_inputs(1, 5, H, W, seed=5)
g = torch.Generator().manual_seed(1234)
R48 = torch.rand(1, 48, H // 8, W // 8, generator=g)
NET.patchmatch_3.rand_source = lambda size, device: R48
native = lambda ci, co, ks: ks == 1 or ci * co * ks * ks <= 3200
base, base_ps = run(lambda ci, co, ks: "fp32")
rows = []
POLICIES = {
    "timed mode of round 1 (native: acts truncated; library: both truncated)": lambda ci, co, ks: "tf32_native" if native(ci, co, ks) else "tf32_trunc",
    "all tf32_native": lambda *a: "tf32_native",
    "all tf32_rna (operands rounded)": lambda *a: "tf32_rna",
    "native layers rounded, library layers truncated": lambda ci, co, ks: "tf32_rna" if native(ci, co, ks) else "tf32_trunc",
    "native 2x_act, library truncated": lambda ci, co, ks: "2x_act" if native(ci, co, ks) else "tf32_trunc",
    "native fp32, library truncated": lambda ci, co, ks: "fp32" if native(ci, co, ks) else "tf32_trunc",
    "native tf32_native, library fp32": lambda ci, co, ks: "tf32_native" if native(ci, co, ks) else "fp32",
    "all 2x_act": lambda *a: "2x_act",
    "all 2x_act_rna": lambda *a: "2x_act_rna",
    "all 3x": lambda *a: "3x",
}
for name, pol in POLICIES.items():
    d, ps = run(pol)
    row = {"policy": name, "depth_rel_l1": pm_cases.rel_l1(d, base),
           "stage_rel_l1": {s: pm_cases.rel_l1(ps[s][-1], base_ps[s][-1]) for s in (3, 2, 1)}}
    rows.append(row)
    print(json.dumps(row), file=sys.stderr)
print(json.dumps({"input": f"synthetic 1+4 views {W}x{H}, shipped checkpoint, oracle port on the CPU, seed 5", "bound": 1e-3, "rows": rows}, indent=1))
