"""colmap_input on synthetic COLMAP models (tests/colmap_cases.py): model reading, host preparation, the GPU view scores and
depth ranges (csrc/pm_colmap.cu), and file writing, per phase.

    python tools/colmap_input_bench.py [--repeats 5] [--json out.json]

Two models: DTU-like (49 images, about 10k observations each) and large (1000 images, 1M points, track length 5: about 5M
observations).  The GPU phase is timed twice: a host clock around the whole phase (uploads, the count read-back, both
kernels, the copies back) ending in a device synchronise, and CUDA events around ops.view_scores and ops.depth_ranges alone.
Prints the card name and its power limit first, then one JSON line per model."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

from patchmatchnet_b200 import colmap_input as ci, ops  # noqa: E402
from tests import colmap_cases as cc  # noqa: E402

MODELS = {
    "dtu_like": dict(seed=49, n_images=49, n_points=49 * 10000 // 8, track=8, n_invalid=500, arc=1.2),
    "large": dict(seed=1000, n_images=1000, n_points=1000000, track=5, n_invalid=0, arc=2 * np.pi),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        power = out.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        power = "unknown"
    return name, power


def run(name, spec, repeats):
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        model = cc.make_model(**spec)
        sparse = os.path.join(tmp, "sparse")
        cc.write_bin(sparse, model)
        t0 = time.perf_counter()
        cams, images, points = ci.read_model(sparse)
        t1 = time.perf_counter()
        sm = ci.prepare(cams, images, points)
        t2 = time.perf_counter()
        phase, kern_s, kern_r = [], [], []
        for _ in range(repeats + 1):  # the first run warms up
            torch.cuda.synchronize()
            a = time.perf_counter()
            scores, ranges = ci.gpu_scores_and_ranges(sm, 5.0, 1.0, 10.0, dev)
            s_h, r_h = scores.cpu().numpy(), ranges.cpu().tolist()
            torch.cuda.synchronize()
            phase.append(time.perf_counter() - a)
            xyz, offs = torch.from_numpy(sm.xyz).to(dev), torch.from_numpy(sm.obs_offsets).to(dev)
            pts, ctr, ext = (torch.from_numpy(x).to(dev) for x in (sm.obs_points, sm.centers, sm.extrinsics))
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            s2 = ops.view_scores(xyz, offs, pts, ctr)
            ev[1].record()
            ops.depth_ranges(xyz, offs, pts, ext)
            ev[2].record()
            torch.cuda.synchronize()
            kern_s.append(ev[0].elapsed_time(ev[1]) / 1e3)
            kern_r.append(ev[1].elapsed_time(ev[2]) / 1e3)
            assert (s2.cpu().numpy() == s_h).all()  # deterministic
        t3 = time.perf_counter()
        ci.write_scene(tmp, sm, r_h, ci.select_views(s_h, -1))
        t4 = time.perf_counter()
    med = lambda v: float(np.median(v[1:]))  # noqa: E731
    return {"model": name, "images": len(images), "points": int(points.ids.size), "observations": int(sm.obs_points.size),
            "read_s": t1 - t0, "prepare_s": t2 - t1, "gpu_phase_s": med(phase), "view_scores_s": med(kern_s),
            "depth_ranges_s": med(kern_r), "write_s": t4 - t3, "repeats": repeats}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--models", nargs="+", default=list(MODELS), choices=list(MODELS))
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("colmap_input_bench needs a CUDA device")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    rows = []
    for m in args.models:
        r = run(m, MODELS[m], args.repeats)
        r.update(device=name, power_limit=power)
        print(json.dumps(r))
        rows.append(r)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
