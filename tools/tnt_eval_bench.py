"""Tanks and Temples evaluation stages (csrc/pm_cloud.cu through tnt_eval) on synthetic clouds of T&T-like size.

    python tools/tnt_eval_bench.py [--rec 8000000] [--gt 6000000] [--tau 0.005] [--reps 3] > tnt_eval_bench.json

Clouds: tests/tnt_cases.surface scaled to a 20 m x 20 m patch (points at tens of metres from the origin, as in T&T), GT =
`--gt` samples, reconstruction = `--rec` noisy samples (0.3 tau) with 3 % outliers above the crop volume, started 2 tau off
the GT alignment.  Each stage is timed with the host clock around the call and a device synchronisation, after one warm-up
run of the whole evaluation, median of `--reps`: crop (both clouds), voxel down-sampling at tau / 2 (both clouds), the
three ICP rounds of tnt_eval.refine (each including its crops and down-sampling) and the two distance passes.  The device
name and power limit are printed beside the times."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import ops, tnt_eval  # noqa: E402
from tests import tnt_cases  # noqa: E402

SCALE = 10.0


def clouds(n_rec, n_gt, tau, seed=0):
    rng = np.random.RandomState(seed)
    o = tnt_cases.OFFSET
    gt = (tnt_cases.surface(rng, n_gt) - o) * SCALE + o
    rec = (tnt_cases.surface(rng, n_rec) - o) * SCALE + o + rng.normal(0, 0.3 * tau, (n_rec, 3))
    k = int(0.03 * n_rec)
    rec[:k, 2] += 3.0 * SCALE
    cv = tnt_cases.crop_volume()
    cv = dict(cv, polygon=(cv["polygon"] - o) * SCALE + o, axis_min=o[2] - 0.5 * SCALE, axis_max=o[2] + 0.5 * SCALE)
    init = np.eye(4)
    init[:3, 3] = [2 * tau, -tau, tau]
    return rec, gt, cv, init


def timed(fn, reps):
    ts, out = [], None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rec", type=int, default=8_000_000)
    ap.add_argument("--gt", type=int, default=6_000_000)
    ap.add_argument("--tau", type=float, default=0.005)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tnt_eval_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rec, gt, cv, init = clouds(args.rec, args.gt, args.tau)
    dev = "cuda:0"
    d_rec, d_gt = torch.as_tensor(rec, device=dev), torch.as_tensor(gt, device=dev)
    tau = args.tau
    tnt_eval.evaluate_scene(rec, gt, cv, init, tau, device=dev)  # warm-up of every stage

    stages = {}
    stages["crop_both"], (c_rec, c_gt) = timed(lambda: (tnt_eval.crop(d_rec, cv, init), tnt_eval.crop(d_gt, cv)), args.reps)
    stages["voxel_both_tau_half"], (v_rec, v_gt) = timed(
        lambda: (ops.voxel_downsample(c_rec, tau / 2), ops.voxel_downsample(c_gt, tau / 2)), args.reps)
    t = init
    rounds = []
    for name, method, voxel, dist in (("icp_round1", "voxel", tau, 80 * tau), ("icp_round2", "voxel", tau / 2, 20 * tau),
                                      ("icp_round3", "uniform", None, 2 * tau)):
        def one(t=t, method=method, voxel=voxel, dist=dist):
            s = tnt_eval._down(tnt_eval.crop(d_rec, cv, t), method, voxel)
            g = tnt_eval._down(tnt_eval.crop(d_gt, cv), method, voxel)
            return s.shape[0], g.shape[0], ops.icp(s, g, dist, max_iteration=20)
        stages[name], (ns, ng, r) = timed(one, args.reps)
        rounds.append({"n_source": ns, "n_target": ng, "iterations": r["iterations"], "fitness": r["fitness"]})
        t = r["transformation"] @ t
    s = ops.voxel_downsample(tnt_eval.crop(d_rec, cv, t), tau / 2)
    g = ops.voxel_downsample(tnt_eval.crop(d_gt, cv), tau / 2)
    allp = torch.cat([s, g])
    box = [(allp.min(0).values - 5 * tau).cpu().tolist(), (allp.max(0).values + 5 * tau).cpu().tolist()]
    stages["distances_both"], _ = timed(lambda: (ops.nearest_distance(g, s, box, 5 * tau), ops.nearest_distance(s, g, box, 5 * tau)),
                                        args.reps)
    stages["evaluate_scene_total"], res = timed(lambda: tnt_eval.evaluate_scene(rec, gt, cv, init, tau, device=dev), 1)
    print(json.dumps({
        "device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi,
        "clouds": {"rec": args.rec, "gt": args.gt, "tau": tau, "rec_cropped": int(c_rec.shape[0]), "gt_cropped": int(c_gt.shape[0]),
                   "rec_voxel_tau_half": int(v_rec.shape[0]), "gt_voxel_tau_half": int(v_gt.shape[0])},
        "seconds": stages, "rounds": rounds,
        "result": {k: res[k] for k in ("precision", "recall", "fscore", "fitness")},
        "note": "host clock around each stage with device synchronisation; evaluate_scene_total includes the host-to-device copies",
    }))


if __name__ == "__main__":
    main()
