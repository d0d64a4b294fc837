"""Views of different sizes: what the per-view form costs, measured in one run.

    python tools/multisize_bench.py [--reps 30] [--scene-views 49] > multisize.json

(a) K-A per launch: the fused K-A launches of one real forward at the default bench.py shapes (640x512, 1 + 4 views) are
    captured, then each is timed through the uniform entry point (stacked [V,B,Hs,Ws,C] pack) and through the *_views entry
    point on the SAME uniform data described as a ragged pack, alternated, CUDA events, median of --reps.  Generation 3 is
    forced for both so that the difference is the per-view form itself.
(b) DepthEngine depth maps/s, 3 slots, CUDA graphs: a 1 + 4 request mixing 1600x1200 and 1200x1600 views beside a uniform
    1600x1200 request.
(c) reconstruct (--output-type both, DTU thresholds) on a seeded synthetic scene of --scene-views views at 1600x1200 where a
    third of the views are portrait: depth, fusion and end-to-end seconds, engines built and their set-up seconds.
The GPU's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops, reconstruct, synthetic  # noqa: E402
from patchmatchnet_b200.engine import DepthEngine  # noqa: E402
from patchmatchnet_b200.net import PatchmatchNet, load_reference_state  # noqa: E402
from tests import multisize_cases  # noqa: E402

DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = os.path.join(ROOT, "tests", "golden", "weights_000007.pt")


def build_net():
    net = PatchmatchNet(**synthetic.DEFAULT_NET_KWARGS)
    load_reference_state(net, torch.load(WEIGHTS, map_location="cpu"))
    return net.eval().to(DEV)


def time_call(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop)


def ka_per_launch(net, reps):
    """(a): every fused K-A launch of one 640x512 forward, uniform vs per-view entry point on the same data."""
    names = ("warp_corr_score", "warp_corr_view_weights")
    calls, origs = [], {n: getattr(ops, n) for n in names}
    for n in names:
        setattr(ops, n, (lambda n: lambda *a, **k: calls.append((n, a, k)) or origs[n](*a, **k))(n))
    inp = synthetic.make_inputs(1, 5, 512, 640, seed=0)
    try:
        with torch.no_grad():
            net([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV), inp["depth_min"].to(DEV),
                inp["depth_max"].to(DEV))
    finally:
        for n in names:
            setattr(ops, n, origs[n])
    torch.cuda.synchronize()
    ops.set_tuning("ka_gen", 3)
    rows = []
    try:
        for n, a, k in calls:
            ref, src = a[0], a[1].contiguous()
            V, B, Hs, Ws, C = src.shape
            n_view = B * Hs * Ws * C
            pack = ops.ViewPack(src.reshape(-1), [v * n_view for v in range(V)], [Hs] * V, [Ws] * V, B, C)
            k = {kk: vv for kk, vv in k.items() if kk != "xs"}
            uni = lambda: origs[n](ref, src, *a[2:], **k)
            per = lambda: origs[n](ref, pack, *a[2:], **k)
            for f in (uni, per):
                f()
            tu, tp = [], []
            for _ in range(reps):  # alternated
                tu.append(time_call(uni))
                tp.append(time_call(per))
            a_u, a_p = uni(), per()
            same = all(torch.equal(x, y) for x, y in zip(a_u if isinstance(a_u, tuple) else (a_u,), a_p if isinstance(a_p, tuple) else (a_p,)))
            rows.append({"entry": n, "C": C, "D": int(a[3].shape[1]), "H": int(ref.shape[1]), "W": int(ref.shape[2]),
                         "uniform_ms": statistics.median(tu), "views_ms": statistics.median(tp),
                         "ratio": statistics.median(tp) / statistics.median(tu), "bit_identical": same})
    finally:
        ops.set_tuning("reset")
    return rows


def engine_rate(net, sizes, reps):
    """(b): depth maps/s of one DepthEngine (3 slots, graphs) on repeated copies of one request of these view sizes."""
    inp = multisize_cases.make_net_inputs(sizes, seed=1)
    H, W = sizes[0]
    uniform = all(s == sizes[0] for s in sizes)
    t0 = time.perf_counter()
    eng = DepthEngine(net, 1, len(sizes), H, W, n_slots=3, view_sizes=None if uniform else sizes)
    args = ([i.to(DEV) for i in inp["images"]], inp["intrinsics"].to(DEV), inp["extrinsics"].to(DEV), inp["depth_min"].to(DEV),
            inp["depth_max"].to(DEV))
    for k in range(3):
        eng.set_device_inputs(k, *args)
    eng.prepare()
    setup = time.perf_counter() - t0
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(2):  # warm rounds
        start.record()
        eng.run_round(3, start, stop)
    torch.cuda.synchronize()
    rates = []
    for _ in range(reps):
        start.record()
        eng.run_round(3, start, stop)
        stop.synchronize()
        rates.append(3 * 1000.0 / start.elapsed_time(stop))
    del eng
    torch.cuda.synchronize()
    return {"sizes": sizes, "depth_maps_per_s": statistics.median(rates), "min": min(rates), "max": max(rates), "setup_seconds": setup}


def scene_run(views):
    """(c): reconstruct on a mixed-orientation 1600x1200 scene."""
    sizes = multisize_cases.mixed_sizes(views, 1200, 1600)
    with tempfile.TemporaryDirectory() as tmp:
        scene = os.path.join(tmp, "scene")
        multisize_cases.write_mixed_scene(scene, sizes, n_src=10)
        out = os.path.join(tmp, "out")
        cli = ["--input-folder", scene, "--output-folder", out, "--checkpoint-path", WEIGHTS, "--num-views", "4",
               "--geo-mask-thres", "3", "--photo-thres", "0.8"]
        stats = reconstruct.reconstruct(reconstruct.parse_args(cli), log=lambda *a: None)
    stats["portrait_views"] = sum(1 for s in sizes if s == (1600, 1200))
    return stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--scene-views", type=int, default=49)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("multisize_bench needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    net = build_net()
    ka = ka_per_launch(net, args.reps)
    L, P = (1200, 1600), (1600, 1200)
    eng = [engine_rate(net, [L] * 5, 10), engine_rate(net, [L, P, L, P, L], 10)]
    scene = scene_run(args.scene_views)
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit": smi, "ka_per_launch": ka,
                      "engine": eng, "reconstruct_mixed_scene": scene}))


if __name__ == "__main__":
    main()
