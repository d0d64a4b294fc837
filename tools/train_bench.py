"""Training-side measurements, recorded with the card's name and power limit:

1. The per-step loss and metric work: this project's K-L kernels (autograd.DepthLoss forward + backward, ops.depth_metrics,
   one read of the scalars) against the reference's op sequence (create_stage_images, net.patchmatchnet_loss + backward,
   absolute_depth_error_metrics / threshold_metrics with boolean indexing per image and .item() per scalar), on the same
   seeded maps: B = 4, 640x512, the default six maps.  Wall time per step includes the host synchronisations; the CUDA-event
   time spans the same region.
2. The train command's step loop on a seeded converted-layout dataset: 640x512, 1+5 views, batch 4 (the reference's
   train.sh), warm-up then timed steps: samples/s, the share of the wall time spent waiting for the loader, peak memory;
   once fp32-accurate (the default) and once with --tf32.

    python tools/train_bench.py --out train_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import data_io, ops, train  # noqa: E402
from patchmatchnet_b200.autograd import DepthLoss  # noqa: E402
from patchmatchnet_b200.net import patchmatchnet_loss  # noqa: E402

LEVELS = [0, 1, 2, 2, 3, 3]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def loss_inputs(B, H, W, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    gt = 450.0 + 450.0 * torch.rand(B, H, W, generator=g)
    mask = (gt > 500.0) & (torch.rand(B, H, W, generator=g) > 0.1)
    maps = []
    for l in LEVELS:
        lv = gt[:, :: 1 << l, :: 1 << l][:, : H >> l, : W >> l].unsqueeze(1)
        maps.append(lv + 3.0 * torch.randn(lv.shape, generator=g))
    return gt.to(dev), mask.to(dev), [m.to(dev).requires_grad_(True) for m in maps]


def ours(gt, mask, maps):
    m8 = mask.view(torch.uint8)
    loss = DepthLoss.apply(LEVELS, gt, m8, None, 1.0, *maps)
    loss.backward()
    last = [maps[max(k for k, lv in enumerate(LEVELS) if lv == l)].detach() for l in range(4)]
    raw = ops.depth_metrics(last, gt, m8)
    abs_err = (raw[:, :4] / raw[:, 4:8]).mean(0)
    rates = train.threshold_rates(raw[:, 8:], raw[:, 4:5]).double().mean(0)
    return [float(loss.detach())] + torch.cat([abs_err, rates]).tolist()  # one read of the scalars


def reference(gt, mask, maps):
    gts = [gt.unsqueeze(1)] + [F.interpolate(gt.unsqueeze(1), scale_factor=0.5 ** l, mode="nearest") for l in (1, 2, 3)]
    mf = mask.unsqueeze(1).float()
    ms = [mf.bool()] + [F.interpolate(mf, scale_factor=0.5 ** l, mode="nearest").bool() for l in (1, 2, 3)]
    per = {l: [m for m, lv in zip(maps, LEVELS) if lv == l] for l in range(4)}
    loss = patchmatchnet_loss(per, gts, ms)
    loss.backward()
    out = [loss.item()]
    with torch.no_grad():
        for l in range(4):  # utils.py absolute_depth_error_metrics
            d, t, k = per[l][-1][:, 0], gts[l][:, 0], ms[l][:, 0]
            out.append(torch.stack([torch.mean((d[b][k[b]] - t[b][k[b]]).abs()) for b in range(d.shape[0])]).mean().item())
        for thr in (1, 2, 4, 8):  # utils.py threshold_metrics
            d, t, k = per[0][-1][:, 0], gts[0][:, 0], ms[0][:, 0]
            out.append(torch.stack([torch.mean((torch.abs(d[b][k[b]] - t[b][k[b]]).float() > float(thr)).float())
                                    for b in range(d.shape[0])]).mean().item())
    return out


def time_loss(fn, inputs, iters, warmup):
    gt, mask, maps = inputs
    for _ in range(warmup):
        fn(gt, mask, maps)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(iters):
        for m in maps:
            m.grad = None
        vals = fn(gt, mask, maps)
    e1.record()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3, e0.elapsed_time(e1) / iters, vals


def write_dataset(root, n_views, H, W, lights, seed=0):
    from PIL import Image

    rng = np.random.default_rng(seed)
    base = os.path.join(root, "scan1")
    for sub in ["cams", "depth_gt"] + [os.path.join("images", str(i)) for i in range(lights)]:
        os.makedirs(os.path.join(base, sub), exist_ok=True)
    with open(os.path.join(base, "pair.txt"), "w") as f:
        f.write(f"{n_views}\n")
        for r in range(n_views):
            src = [(r + k) % n_views for k in range(1, 6)]
            f.write(f"{r}\n5 " + " ".join(f"{s} {100.0 - k:.1f}" for k, s in enumerate(src)) + "\n")
    for v in range(n_views):
        E = np.eye(4)
        E[:3, 3] = [3.0 * v, 0.5 * v, 0.0]
        K = np.array([[800.0, 0, W / 2], [0, 800.0, H / 2], [0, 0, 1]])
        rows = ["extrinsic"] + [" ".join(f"{x:.9g}" for x in r) for r in E] + ["", "intrinsic"]
        rows += [" ".join(f"{x:.9g}" for x in r) for r in K] + ["", "425 935"]
        with open(os.path.join(base, "cams", "%08d_cam.txt" % v), "w") as f:
            f.write("\n".join(rows) + "\n")
        data_io.save_map(os.path.join(base, "depth_gt", "%08d.pfm" % v), rng.uniform(400, 900, (H, W)).astype(np.float32))
        for light in range(lights):
            Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(
                os.path.join(base, "images", str(light), "%08d.jpg" % v), quality=95)
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write("scan1\n")


def driver(steps, warmup, batch, workers, tf32):
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True  # as the train command sets it
    with tempfile.TemporaryDirectory() as tmp:
        write_dataset(tmp, n_views=25, H=512, W=640, lights=4)
        args = train.parse_args(["--input-folder", tmp, "--train-list", os.path.join(tmp, "list.txt"), "--test-list",
                                 os.path.join(tmp, "list.txt"), "--num-views", "5", "--num-light-idx", "4", "--batch-size", str(batch),
                                 "--num-workers", str(workers)])
        ds = train.MVSDataset(tmp, 5, args.image_max_dim, args.train_list, 4)
        loader = train.make_loader(ds, batch, True, workers, 1, 0, 1)
        sess = train.Session(dev, 0, 1, train.loss_levels(args.patchmatch_iteration))
        with train.precision(tf32):
            torch.manual_seed(1)
            net = train.build_network(args).to(dev).train()
            opt = torch.optim.Adam(net.parameters(), lr=1e-3)
            it = iter(loader)
            for _ in range(warmup):
                float(train.process_batch(net, next(it), sess, opt)[0])
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            wait = 0.0
            t0 = time.perf_counter()
            for _ in range(steps):
                w0 = time.perf_counter()
                sample = next(it)
                wait += time.perf_counter() - w0
                float(train.process_batch(net, sample, sess, opt)[0])  # the step's host synchronisation, as in the driver
            torch.cuda.synchronize()
            total = time.perf_counter() - t0
    return {"samples_per_s": steps * batch / total, "ms_per_step": total / steps * 1e3, "loader_wait_share": wait / total,
            "peak_memory_gib": torch.cuda.max_memory_allocated() / 2 ** 30, "steps": steps, "warmup": warmup, "batch": batch,
            "workers": workers, "views": "1+5", "size": "640x512", "tf32": tf32}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_bench needs a CUDA device")
    res = {"card": card()}
    inputs = loss_inputs(4, 512, 640, torch.device("cuda:0"))
    mine = time_loss(ours, inputs, a.iters, 5)
    ref = time_loss(reference, inputs, a.iters, 5)
    res["loss_metrics"] = {"ours_wall_ms": mine[0], "ours_event_ms": mine[1], "reference_wall_ms": ref[0], "reference_event_ms": ref[1],
                           "max_rel_diff_of_scalars": max(abs(x - y) / max(abs(y), 1e-30) for x, y in zip(mine[2], ref[2])),
                           "iters": a.iters, "shape": "B=4, 640x512, 6 maps"}
    res["driver"] = driver(a.steps, a.warmup, 4, a.workers, tf32=False)  # the command's default: fp32-accurate convolutions
    res["driver_tf32"] = driver(a.steps, a.warmup, 4, a.workers, tf32=True)  # --tf32, torch's default the reference ran with
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
