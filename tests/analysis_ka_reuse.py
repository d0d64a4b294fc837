"""K-A gather statistics on the REAL hypotheses of a 640x512 cascade (analysis script, CPU only, not a test):

    python tests/analysis_ka_reuse.py > ka_gather_stats.json

For every K-A launch of one forward (hypotheses, projections captured from the oracle port of the reference running the
synthetic 1+4-view input with the shipped checkpoint) it reports, for the kernel's (pixels per warp, rows per pass):
  unique      share of (pixel, hypothesis, view) footprints that open a new source cell (consecutive-row comparison, as the
              kernel's phase 1 does) -- what the gather phase has to load;
  layers_mean / layers_max   mean over warp passes of the per-pixel unique-cell count and of its maximum over the warp's
              pixels: the gather loop runs `max` iterations while the average lane group needs `mean`;
  gather_efficiency = mean / max  -- the fraction of the gather loop's issue slots that do useful work.
Lives under tests/ because it drives the oracle (test infrastructure); the footprints come from the kernels' own
formula file compiled for the host (tests/hostmath.cpp)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402
from oracle import pm_oracle  # noqa: E402
from patchmatchnet_b200 import synthetic  # noqa: E402


def hostmath():
    src = os.path.join(REPO, "tests", "hostmath.cpp")
    out = os.path.join(REPO, "tests", "_hostmath.so")
    if not os.path.exists(out):
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out, "-x", "c++", src], check=True)
    return ctypes.CDLL(out)


def main():
    hm = hostmath()
    net, _ = bench.build_net(pm_oracle.PatchMatchOracle)
    inp = synthetic.make_inputs(1, 5, 512, 640, seed=0)
    calls = []
    orig = pm_oracle.homography_warp

    def spy(src_fea, src_proj, ref_proj, depth):
        calls.append((tuple(src_fea.shape), src_proj.clone(), ref_proj.clone(), depth.clone()))
        return orig(src_fea, src_proj, ref_proj, depth)

    pm_oracle.homography_warp = spy
    torch.manual_seed(0)
    with torch.no_grad():
        net(inp["images"], inp["intrinsics"].clone(), inp["extrinsics"], inp["depth_min"], inp["depth_max"])
    pm_oracle.homography_warp = orig

    # group the per-view calls of one evaluation into launches (same hypotheses tensor)
    launches = []
    for shp, sp, rp, d in calls:
        if launches and launches[-1]["depth"].shape == d.shape and torch.equal(launches[-1]["depth"], d):
            launches[-1]["src_projs"].append(sp)
        else:
            launches.append(dict(C=shp[1], depth=d, ref_proj=rp, src_projs=[sp]))
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    rows = []
    for L in launches:
        C, depth = L["C"], L["depth"]
        _, D, H, W = depth.shape
        ppw = 32 // (C // 8)
        dn = depth[0].reshape(-1).numpy().astype(np.float32).copy()
        keys = []
        for sp in L["src_projs"]:
            rel = sp[0].double() @ torch.linalg.inv(L["ref_proj"][0].double())
            rt = torch.cat([rel[:3, :3].reshape(9), rel[:3, 3]]).float().numpy().copy()
            w = np.zeros((D * H * W, 4), dtype=np.float32)
            key = np.zeros(D * H * W, dtype=np.int32)
            hm.hm_warp_cells(fp(rt), fp(dn), H, W, H, W, D, fp(w), ip(key))
            keys.append(key.reshape(D, H * W))
        keys = np.stack(keys)  # [V,D,HW]
        V = keys.shape[0]
        none = -2
        out = {"launch": f"C{C} D{D} {H}x{W} V{V}", "pixels_per_warp": ppw, "by_rows_per_pass": {}}
        for dc in (4, 8, 16, 32):
            if (ppw * dc) % 32 or dc > max(4, D):
                continue
            nch = (D + dc - 1) // dc
            pad = nch * dc - D
            k = np.concatenate([keys, np.full((V, pad, H * W), none, np.int32)], axis=1).reshape(V, nch, dc, H * W)
            prev = np.concatenate([np.full((V, nch, 1, H * W), none, np.int32), k[:, :, :-1]], axis=2)
            isnew = (k != none) & (k != prev)
            cg = isnew.sum(axis=2)  # [V,nch,HW] unique cells per (view, chunk, pixel)
            npx = H * W
            padpx = (-npx) % ppw
            cgp = np.concatenate([cg, np.zeros((V, nch, padpx), cg.dtype)], axis=2).reshape(V, nch, -1, ppw)
            mx = cgp.max(axis=3)
            live = (k != none).sum()
            out["by_rows_per_pass"][str(dc)] = {
                "unique": round(float(isnew.sum()) / max(1, int(live)), 4),
                "layers_mean": round(float(cgp.mean()), 3),
                "layers_max": round(float(mx.mean()), 3),
                "gather_efficiency": round(float(cgp.sum()) / max(1.0, float(mx.sum()) * ppw), 4),
            }
        rows.append(out)
    print(json.dumps({"input": "synthetic 1+4 views 640x512, shipped checkpoint, oracle port on the CPU", "launches": rows}, indent=1))


if __name__ == "__main__":
    main()
