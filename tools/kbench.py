"""Kernel micro-benchmark: capture the K-A / K-B / K-C launches of one real 640x512 forward (so the
hypotheses have the cascade's real clustering) and time each one in isolation -- L2 flushed, CUDA events --
for a sweep of kernel variants selected through environment variables (read per call by libpmb200.so).

    python tools/kbench.py > kbench.json
"""
import itertools
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from patchmatchnet_b200 import ops, synthetic  # noqa: E402

dev = "cuda:0"
torch.backends.cudnn.benchmark = True
torch.backends.cudnn.allow_tf32 = os.environ.get("PM_TF32", "0") == "1"  # default: the fp32-accurate mode bench.py times
H, W = int(os.environ.get("KB_H", 512)), int(os.environ.get("KB_W", 640))
BATCH = int(os.environ.get("KB_B", 1))
net, _ = bench.build_net()
net = net.to(dev)
inp = synthetic.make_inputs(BATCH, 5, H, W, seed=0)
args = lambda: ([i.to(dev) for i in inp["images"]], inp["intrinsics"].to(dev), inp["extrinsics"].to(dev), inp["depth_min"].to(dev), inp["depth_max"].to(dev))
names = ("warp_corr_score", "warp_corr_view_weights", "aggregate_views_score", "adaptive_eval", "init_propagate", "offset_corr_weight")
calls = []
origs = {n: getattr(ops, n) for n in names}
for n in names:
    def mk(n):
        def spy(*a, **k):
            calls.append((n, a, k))
            return origs[n](*a, **k)
        return spy
    setattr(ops, n, mk(n))
with torch.no_grad():
    for _ in range(2):
        calls.clear()
        torch.manual_seed(0)
        net(*args())
for n in names:
    setattr(ops, n, origs[n])
torch.cuda.synchronize()
flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, iters=12):
    """(cold mean us, cold min us, warm us): cold = L2 flushed before each launch; warm = 10 back-to-back launches."""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush_buf.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    torch.cuda._sleep(2_000_000)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10):
        fn()
    b.record()
    b.synchronize()
    return round(statistics.mean(ts), 2), round(min(ts), 2), round(a.elapsed_time(b) * 1e2, 2)


out = {"shape": f"{W}x{H} B{BATCH}", "rows": []}


def with_knobs(knobs, fn):
    ops.set_tuning("reset")
    for kk, vv in knobs.items():
        ops.set_tuning(kk, vv)
    try:
        return timeit(fn)
    finally:
        ops.set_tuning("reset")


# K-A: generation 4 (consumer warps x resident CTAs the ring is sized for) against generation 3 (rows per pass x pipeline)
ka_variants = ([dict(ka_gen=4, ka4_nw=nw, ka4_ctas=c, ka4_stages=st) for nw, c, st in
                ((4, 2, 2), (4, 2, 3), (4, 2, 4), (4, 3, 2), (4, 3, 3), (4, 4, 2), (8, 1, 4), (8, 2, 2), (8, 2, 3))]
               + [dict(ka_gen=3)] + [dict(ka_gen=3, ka3_dc=d, ka3_pipe=0) for d in (4, 8, 16)])
for (n, a, k) in calls:
    desc = n
    if n.startswith("warp_corr"):
        ref, src, depth = a[0], a[1], a[3]
        desc += f" C{ref.shape[3]} D{depth.shape[1]} {ref.shape[1]}x{ref.shape[2]} V{src.shape[0]}"
    elif n == "adaptive_eval":
        desc += f" D{a[1].shape[1]} {a[1].shape[2]}x{a[1].shape[3]}"
    elif n == "init_propagate":
        desc += f" Ns{a[5]} Kp{a[6]} {a[0].shape[2]}x{a[0].shape[3]}"
    elif n == "offset_corr_weight":
        desc += f" C{a[0].shape[3]} {a[0].shape[1]}x{a[0].shape[2]}"
    row = {"call": desc, "default_us": timeit(lambda: origs[n](*a, **k))}
    if n == "adaptive_eval" and os.environ.get("KB_SWEEP_EVAL", "1") == "1":
        for tp, dy in ((32, 8), (32, 4), (16, 16), (16, 8), (8, 32), (8, 16), (64, 4), (32, 2)):
            row[f"TP={tp},DY={dy}"] = with_knobs(dict(kb_tp=tp, kb_dy=dy), lambda: origs[n](*a, **k))
    if n in ("warp_corr_score", "warp_corr_view_weights") and os.environ.get("KB_SWEEP_KA", "1") == "1":
        for v in ka_variants:
            if n == "warp_corr_view_weights" and "ka3_dc" in v:
                v = {("ka3_dc_vw" if kk == "ka3_dc" else kk): vv for kk, vv in v.items()}
            tag = ",".join(f"{kk}={vv}" for kk, vv in v.items())
            row[tag] = with_knobs(v, lambda: origs[n](*a, **k))
    out["rows"].append(row)
print(json.dumps(out, indent=1))
