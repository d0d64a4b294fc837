"""Training on views of different sizes: what the ragged-pack backward costs, measured in one run.

    python tools/multisize_train_bench.py [--reps 30] [--steps 20] [--warmup 5] [--batch 2] --out multisize_train.json

(a) K-A backward per launch at the training shapes of a 640x512, 1 + 4 view batch (stage 3: C=64 at 80x64 with 32
    hypotheses; stage 2: C=32 at 160x128 with 16; stage 1: C=16 at 320x256 with 8), both modes: pmb200_warp_corr_backward
    on a stacked [V,B,Hs,Ws,C] pack and pmb200_warp_corr_views_backward on the SAME uniform data described as a ragged pack,
    alternated, CUDA events, median of --reps; with the largest difference of the two results (d_ref is expected
    bit-equal, d_src equal up to the order of its atomic adds).
(b) Train steps/s and peak memory, 1 + 4 views at 640x512, fp32-accurate: every view landscape (the uniform path) against
    two portrait 512x640 sources (the ragged path).  Forward, DepthLoss, backward and an Adam step on device batches; the
    step ends with the loss read back, as in the train command.
The GPU's name, power limit and maximum SM clock are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import _native, ops, reconstruct, synthetic, train  # noqa: E402
from patchmatchnet_b200 import autograd as ag  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def time_call(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop)


STAGES = [("stage3", 64, 8, 64, 80, 32), ("stage2", 32, 8, 128, 160, 16), ("stage1", 16, 4, 256, 320, 8)]


def backward_per_launch(reps, B=2, V=4):
    g = torch.Generator(device=DEV).manual_seed(0)
    out = []
    for name, C, G, H, W, D in STAGES:
        for weighted in (False, True):
            ref = torch.randn(B, H, W, C, device=DEV, generator=g)
            srcs = [torch.randn(B, C, H, W, device=DEV, generator=g) for _ in range(V)]
            Kc, Ec = synthetic.make_cameras(B, V + 1, H * 8, W * 8)
            ref_proj, src_projs = synthetic.stage_projections(Kc, Ec, 3)
            rt = ops.relative_projection(ref_proj.contiguous().to(DEV), [m.contiguous().to(DEV) for m in src_projs])
            depth = torch.sort(350.0 + 700.0 * torch.rand(B, D, H, W, device=DEV, generator=g), dim=1)[0].contiguous()
            vw = torch.rand(B, V, H, W, device=DEV, generator=g) if weighted else None
            gout = torch.randn((B, G, D, H, W) if weighted else (V, B, G, D, H, W), device=DEV, generator=g)
            uni, pack = ops.pack_nhwc(srcs), ops.pack_nhwc_views(srcs)
            d_ref_u, d_src_u = torch.empty_like(ref), torch.empty_like(uni)

            def uniform():
                rc = _native.lib().pmb200_warp_corr_backward(
                    ref.data_ptr(), uni.data_ptr(), rt.data_ptr(), depth.data_ptr(), None if vw is None else vw.data_ptr(),
                    gout.data_ptr(), d_ref_u.data_ptr(), d_src_u.data_ptr(), V, B, C, G, H, W, H, W, D, ops._stream(ref))
                _native.check(rc, "warp_corr_backward")

            res = {}

            def views():
                res["v"] = ag.warp_corr_views_backward(ref, pack, rt, depth, vw, gout, G)

            for _ in range(3):
                uniform()
                views()
            tu, tv = [], []
            for _ in range(reps):
                tu.append(time_call(uniform))
                tv.append(time_call(views))
            d_ref_v, d_src_v = res["v"]
            got = ops.ViewPack(d_src_v, pack.offsets, pack.heights, pack.widths, B, C)
            src_err = max(float((got.view(v) - d_src_u[v]).abs().max()) for v in range(V))
            out.append({"stage": name, "C": C, "G": G, "H": H, "W": W, "D": D, "B": B, "V": V, "weighted": weighted,
                        "uniform_ms": statistics.median(tu), "views_ms": statistics.median(tv),
                        "views_over_uniform": statistics.median(tv) / statistics.median(tu),
                        "d_ref_bit_equal": bool(torch.equal(d_ref_u, d_ref_v)), "d_src_max_abs_diff": src_err,
                        "d_src_scale": float(d_src_u.abs().max())})
    return out


def train_rate(sizes, steps, warmup, B):
    """steps/s and peak memory of the training step on one seeded device batch whose views have the given sizes"""
    dev = torch.device(DEV)
    g = torch.Generator().manual_seed(1)
    H, W = sizes[0]
    K, E = synthetic.make_cameras(B, len(sizes), H, W)
    for i, (h, w) in enumerate(sizes):
        K[:, i, 0, 2], K[:, i, 1, 2] = w / 2, h / 2
    gt = synthetic.DEPTH_MIN + (synthetic.DEPTH_MAX - synthetic.DEPTH_MIN) * torch.rand(B, H, W, generator=g)
    s = {"images": [torch.rand(B, 3, h, w, generator=g).to(dev) for h, w in sizes], "intrinsics": K.to(dev), "extrinsics": E.to(dev),
         "depth_min": torch.full((B,), synthetic.DEPTH_MIN, device=dev), "depth_max": torch.full((B,), synthetic.DEPTH_MAX, device=dev),
         "depth_gt": gt.to(dev), "mask": (torch.rand(B, H, W, generator=g) > 0.2).to(dev)}
    args = train.parse_args([])
    with reconstruct.precision(False):
        torch.manual_seed(1)
        net = train.build_network(args).to(dev).train()
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)

        def step():
            opt.zero_grad()
            loss, _ = train.forward_loss(net, s)
            loss.backward()
            opt.step()
            return float(loss)

        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    return {"sizes": [list(x) for x in sizes], "batch": B, "steps": steps, "warmup": warmup, "steps_per_s": steps / total,
            "ms_per_step": total / steps * 1e3, "peak_memory_gib": torch.cuda.max_memory_allocated() / 2 ** 30}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=2)
    ap.add_argument("--out", type=str, default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multisize_train_bench needs a CUDA device")
    torch.backends.cudnn.benchmark = True  # as the train command sets it
    L, P = (512, 640), (640, 512)
    res = {"card": card(), "backward_per_launch": backward_per_launch(a.reps),
           "train_uniform": train_rate([L] * 5, a.steps, a.warmup, a.batch),
           "train_two_portrait_sources": train_rate([L, L, P, L, P], a.steps, a.warmup, a.batch)}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
