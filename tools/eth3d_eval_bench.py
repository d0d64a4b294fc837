"""ETH3D evaluation stages (csrc/pm_scan.cu and csrc/pm_cloud.cu through eth3d_eval) on seeded synthetic scans of ETH3D-like
size.

    python tools/eth3d_eval_bench.py [--scans 4] [--scan-points 10000000] [--rec 10000000] [--reps 3] > eth3d_eval_bench.json

Scene: the room of tests/eth3d_cases.py (8 m x 6 m x 3 m with a pillar), ray-cast on the GPU from `--scans` scanner positions
on an angular grid of `--scan-points` rays each.  Reconstruction: `--rec` points, 96 % ground-truth samples with 3 mm noise,
2 % free-space outliers along the beams and 2 % points behind the walls.  Each stage is timed with the host clock around the
calls and a device synchronisation, after one warm-up run of the whole evaluation, median of `--reps`: the two distance
passes, the beam index builds (all scans), the beam pass (all scans, queries with d_acc above the smallest tolerance) and the
scoring of both clouds at the six default tolerances.  The device name and power limit are printed beside the times."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from patchmatchnet_b200 import _native, eth3d_eval, ops  # noqa: E402
from tests import eth3d_cases as ec  # noqa: E402

SCANNERS = [[1.6, 1.5, 1.5], [6.5, 1.4, 1.5], [1.7, 4.6, 1.4], [6.4, 4.8, 1.6]]


def ray_cast(o, d):
    """tests/eth3d_cases.ray_cast on the device."""
    room, pillar = (torch.as_tensor(b, device=d.device) for b in (ec.ROOM, ec.PILLAR))
    inv = 1.0 / d
    t_room = torch.maximum((room[0] - o) * inv, (room[1] - o) * inv).min(1).values
    t0, t1 = (pillar[0] - o) * inv, (pillar[1] - o) * inv
    near, far = torch.minimum(t0, t1).max(1).values, torch.maximum(t0, t1).min(1).values
    hit = (near <= far) & (near > 0)
    return torch.where(hit, torch.minimum(near, t_room), t_room)


def scene(n_scans, n_points, n_rec, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    n_el = int(math.sqrt(n_points / 2))
    n_az = n_points // n_el
    scans, gts = [], []
    for k in range(n_scans):
        o = torch.tensor(SCANNERS[k % len(SCANNERS)], dtype=torch.float64, device=dev)
        az = (torch.arange(n_az, device=dev, dtype=torch.float64) + torch.rand(1, generator=g, device=dev, dtype=torch.float64)) \
            * (2 * math.pi / n_az) - math.pi
        el = torch.linspace(-1.35, 1.45, n_el, device=dev, dtype=torch.float64)
        a, e = torch.meshgrid(az, el, indexing="ij")
        d = torch.stack([torch.cos(e) * torch.cos(a), torch.cos(e) * torch.sin(a), torch.sin(e)], -1).reshape(-1, 3)
        p = o + ray_cast(o, d)[:, None] * d
        m = np.eye(4)
        m[:3, 3] = SCANNERS[k % len(SCANNERS)]
        scans.append({"matrix": m, "points": (p - o).cpu().numpy()})  # local frame: identity rotation
        gts.append(p)
    gt = torch.cat(gts)
    n_out = n_rec // 50
    pick = torch.randint(gt.shape[0], (n_rec,), generator=g, device=dev)
    rec = gt[pick] + 0.003 * torch.randn(n_rec, 3, generator=g, device=dev, dtype=torch.float64)
    per = gts[0].shape[0]
    origins = torch.tensor([SCANNERS[int(i) // per % len(SCANNERS)] for i in range(0, gt.shape[0], per)], dtype=torch.float64,
                           device=dev)
    src = origins[pick[:n_out] // per]
    rec[:n_out] = src + torch.rand(n_out, 1, generator=g, device=dev, dtype=torch.float64) * 0.9 * (gt[pick[:n_out]] - src)
    rec[n_out:2 * n_out] = gt[pick[n_out:2 * n_out]] + (gt[pick[n_out:2 * n_out]] - src) * 0.3
    return scans, rec.cpu().numpy()


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
    ap.add_argument("--scans", type=int, default=4)
    ap.add_argument("--scan-points", type=int, default=10_000_000)
    ap.add_argument("--rec", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eth3d_eval_bench needs a CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    dev = "cuda:0"
    scans, rec = scene(args.scans, args.scan_points, args.rec, dev)
    taus = list(eth3d_eval.TOLERANCES)
    _, (d_rec, gt, d_acc, d_comp, observed) = eth3d_eval._evaluate(rec, scans, taus, eth3d_eval.BEAM_START_RADIUS,
                                                                   eth3d_eval.BEAM_DIVERGENCE_HALFANGLE_DEG, dev)  # warm-up
    cap = eth3d_eval.DISTANCE_CAP * max(taus)
    lo = torch.minimum(d_rec.amin(0), gt.amin(0)) - cap
    hi = torch.maximum(d_rec.amax(0), gt.amax(0)) + cap
    box = [lo.cpu().tolist(), hi.cpu().tolist()]
    stages = {}
    stages["distance_rec_to_gt"], _ = timed(lambda: ops.nearest_distance(gt, d_rec, box, cap), args.reps)
    stages["distance_gt_to_rec"], _ = timed(lambda: ops.nearest_distance(d_rec, gt, box, cap), args.reps)

    lib = _native.lib()
    sizes = [s["points"].shape[0] for s in scans]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    ws = [ops._workspace(lib.pmb200_beam_index_workspace_bytes(k), "beam_index_workspace_bytes", gt.device) for k in sizes]
    origins = [(ctypes.c_double * 3)(*s["matrix"][:3, 3].tolist()) for s in scans]
    stream = torch.cuda.current_stream().cuda_stream

    def build():
        for k, s in enumerate(scans):
            part = gt[offs[k]:offs[k + 1]]
            _native.check(lib.pmb200_beam_index(part.data_ptr(), sizes[k], origins[k], ws[k].data_ptr(), ws[k].numel(), stream),
                          "beam_index")

    mask = (d_acc > min(taus)).to(torch.uint8)
    tan_half = math.tan(math.radians(eth3d_eval.BEAM_DIVERGENCE_HALFANGLE_DEG))

    def beams():
        obs = torch.zeros(d_rec.shape[0], dtype=torch.uint8, device=dev)
        for k in range(len(scans)):
            _native.check(lib.pmb200_beam_observed(d_rec.data_ptr(), d_rec.shape[0], mask.data_ptr(), ws[k].data_ptr(), sizes[k],
                                                   origins[k], eth3d_eval.BEAM_START_RADIUS, tan_half, obs.data_ptr(), stream),
                          "beam_observed")
        return obs

    stages["beam_index_builds"], _ = timed(build, args.reps)
    stages["beam_pass"], obs = timed(beams, args.reps)
    assert torch.equal(obs, observed)
    stages["scores_six_tolerances"], _ = timed(
        lambda: [(ops.voxel_score(d_rec, d_acc, t, observed), ops.voxel_score(gt, d_comp, t)) for t in taus], args.reps)
    stages["evaluate_scene_total"], res = timed(lambda: eth3d_eval.evaluate_scene(rec, scans, taus, device=dev), 1)
    print(json.dumps({
        "device": torch.cuda.get_device_name(0), "nvidia_smi_name_power_limit_max_sm_clock": smi,
        "clouds": {"scans": len(scans), "scan_points": sizes, "gt": int(gt.shape[0]), "rec": int(d_rec.shape[0]),
                   "beam_queries": int(mask.sum()), "observed": int(observed.sum())},
        "seconds": stages,
        "result": [{k: t[k] for k in ("tolerance", "accuracy", "completeness", "f1", "inaccurate", "unobserved")}
                   for t in res["tolerances"]],
        "note": "host clock around each stage with device synchronisation; evaluate_scene_total includes the host-to-device copies",
    }))


if __name__ == "__main__":
    main()
