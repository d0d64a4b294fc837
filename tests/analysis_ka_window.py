"""K-A gen-4 design aid (analysis script, CPU only, not a test): source-window statistics of reference-pixel tiles.

    python tests/analysis_ka_window.py > ka_window_stats.json

For every K-A launch of one 640x512 forward (hypotheses / projections captured from the oracle port running the synthetic
1+4-view input with the shipped checkpoint) and for several (tile, hypothesis rows per item) decompositions it reports,
per (tile, item, view): the bounding box of the bilinear taps in the source map (width / height percentiles), how many
footprints a fixed "wide" or "tall" window (the better of the two, centred on the box) would cover, the share of
footprints that open a new cell inside an item (consecutive-row comparison per pixel, as the kernel dedupes), and the
resulting staged bytes per launch.  Lives under tests/ because it drives the oracle (test infrastructure)."""
import ctypes
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402
from oracle import pm_oracle  # noqa: E402
from patchmatchnet_b200 import synthetic  # noqa: E402
from tests.analysis_ka_reuse import hostmath  # noqa: E402


def capture(height=512, width=640):
    net, _ = bench.build_net(pm_oracle.PatchMatchOracle)
    inp = synthetic.make_inputs(1, 5, height, width, seed=0)
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
    launches = []
    for shp, sp, rp, d in calls:
        if launches and launches[-1]["depth"].shape == d.shape and torch.equal(launches[-1]["depth"], d):
            launches[-1]["src_projs"].append(sp)
        else:
            launches.append(dict(C=shp[1], depth=d, ref_proj=rp, src_projs=[sp]))
    return launches


def main():
    hm = hostmath()
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    rows = []
    for L in capture():
        C, depth = L["C"], L["depth"]
        _, D, H, W = depth.shape
        dn = depth[0].reshape(-1).numpy().astype(np.float32).copy()
        keys = []
        for sp in L["src_projs"]:
            rel = sp[0].double() @ torch.linalg.inv(L["ref_proj"][0].double())
            rt = torch.cat([rel[:3, :3].reshape(9), rel[:3, 3]]).float().numpy().copy()
            w = np.zeros((D * H * W, 4), dtype=np.float32)
            key = np.zeros(D * H * W, dtype=np.int32)
            hm.hm_warp_cells(fp(rt), fp(dn), H, W, H, W, D, fp(w), ip(key))
            keys.append(key.reshape(D, H, W))
        keys = np.stack(keys)  # [V,D,H,W]
        V = keys.shape[0]
        none = keys == -2
        idx = keys & ((1 << 29) - 1)
        x0 = (idx % W).astype(np.int32)
        y0 = (idx // W).astype(np.int32)
        x1 = x0 + ((keys >> 29) & 1)
        y1 = y0 + ((keys >> 30) & 1)
        out = {"launch": f"C{C} D{D} {H}x{W} V{V}", "decompositions": {}}
        for (tw, th, dch) in ((8, 8, 8), (8, 8, 16), (8, 4, 16), (8, 4, 8), (16, 8, 8)):
            if dch > D and dch != 8:
                continue
            nty, ntx, ndc = (H + th - 1) // th, (W + tw - 1) // tw, (D + dch - 1) // dch
            bw, bh, newc, tot = [], [], 0, 0
            for v in range(V):
                for dc in range(ndc):
                    ds = slice(dc * dch, min(D, (dc + 1) * dch))
                    k = keys[v, ds]
                    prev = np.concatenate([np.full((1, H, W), -2, np.int32), k[:-1]], axis=0)
                    isnew = (k != -2) & (k != prev)
                    newc += int(isnew.sum())
                    tot += int((k != -2).sum())
                    big = 1 << 20
                    xa = np.where(none[v, ds], big, x0[v, ds]).min(axis=0)
                    xb = np.where(none[v, ds], -big, x1[v, ds]).max(axis=0)
                    ya = np.where(none[v, ds], big, y0[v, ds]).min(axis=0)
                    yb = np.where(none[v, ds], -big, y1[v, ds]).max(axis=0)
                    for ty in range(nty):
                        for tx in range(ntx):
                            s = (slice(ty * th, (ty + 1) * th), slice(tx * tw, (tx + 1) * tw))
                            a, b, c, d_ = xa[s].min(), xb[s].max(), ya[s].min(), yb[s].max()
                            if a > b:
                                continue
                            bw.append(b - a + 1)
                            bh.append(d_ - c + 1)
            bw, bh = np.array(bw), np.array(bh)
            area = bw * bh
            pct = lambda a: [int(np.percentile(a, q)) for q in (50, 90, 99, 100)]
            items = nty * ntx * ndc
            out["decompositions"][f"tile{tw}x{th}_d{dch}"] = {
                "items": items, "box_w_p50_90_99_max": pct(bw), "box_h_p50_90_99_max": pct(bh),
                "box_texels_p50_90_99_max": pct(area), "new_cell_share": round(newc / max(1, tot), 4),
                "staged_MB_exact_boxes": round(float(area.sum()) * C * 4 / 1e6, 1),
                "staged_MB_fixed_p99_box": round(float(np.percentile(area, 99)) * len(area) * C * 4 / 1e6, 1),
            }
        rows.append(out)
    print(json.dumps({"input": "synthetic 1+4 views 640x512, shipped checkpoint, oracle port on the CPU", "launches": rows}, indent=1))


if __name__ == "__main__":
    main()
