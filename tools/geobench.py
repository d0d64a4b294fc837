"""Geometric-consistency filtering (SURVEY.md 8f row f4): the one-launch kernel vs the reference algorithm on the host CPU.

    python tools/geobench.py > geobench.json

GPU: CUDA events on the launching stream, L2 flushed before each launch, depth maps resident; `e2e` additionally uploads
the (1 + V) depth maps + confidence from pinned host memory and downloads the three masks + averaged depth every call.
CPU: oracle/geo_oracle.py (bit-identical to eval.py:86-190 + :220-256) with cv2.remap when available, one pass.
Algorithmic bytes: 4*H*W*(1 + V + 1) read + H*W*(4 + 1 + 1 + 8) written."""
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import geo_oracle as go  # noqa: E402  (baseline leg only)
from patchmatchnet_b200 import ops  # noqa: E402
from tests import geo_cases  # noqa: E402

dev = "cuda:0"
flush_buf = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
try:
    import cv2

    remap = lambda s, x, y: cv2.remap(s, x, y, interpolation=cv2.INTER_LINEAR)
    remap_name = "cv2.remap"
except Exception:  # noqa: BLE001
    remap, remap_name = go.remap_linear, "numpy restatement of cv2.remap"
peak = 6581.6
try:
    peak = float(json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:  # noqa: BLE001
    pass
rows = []
for (H, W, V) in ((512, 640, 4), (1200, 1600, 10)):
    sc = geo_cases.make_scene(seed=1, H=H, W=W, n_src=V)
    cams = ops.compose_filter_cameras(sc["ref_K"], sc["ref_E"], sc["src_Ks"], sc["src_Es"]).to(dev)
    h_ref, h_conf = torch.from_numpy(sc["ref_depth"]).pin_memory(), torch.from_numpy(sc["confidence"]).pin_memory()
    h_src = torch.from_numpy(np.stack(sc["src_depths"])).pin_memory()
    d_ref, d_conf, d_src = h_ref.to(dev), h_conf.to(dev), h_src.to(dev)
    for _ in range(3):
        out = ops.geometric_filter(d_ref, d_conf, d_src, cams)
    ts = []
    for _ in range(10):
        flush_buf.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = ops.geometric_filter(d_ref, d_conf, d_src, cams)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    gpu_s = sum(ts) / len(ts)
    te = []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        o = ops.geometric_filter(h_ref.to(dev, non_blocking=True), h_conf.to(dev, non_blocking=True), h_src.to(dev, non_blocking=True), cams)
        host = [t.cpu() for t in o]
        torch.cuda.synchronize()
        te.append(time.perf_counter() - t0)
    t0 = time.perf_counter()
    want = go.fuse_reference_view(sc["ref_depth"], sc["ref_K"], sc["ref_E"], sc["src_depths"], sc["src_Ks"], sc["src_Es"], sc["confidence"], remap=remap)
    cpu_s = time.perf_counter() - t0
    got = [t.cpu().numpy() for t in out]
    alg = 4 * H * W * (2 + V) + H * W * 14
    rows.append({"shape": f"{W}x{H} ref + {V} src", "gpu_us": round(gpu_s * 1e6, 1), "gpu_us_min": round(min(ts) * 1e6, 1),
                 "algorithmic_mb": round(alg / 1e6, 2), "achieved_gbs": round(alg / gpu_s / 1e9, 1), "frac_of_hbm_peak": round(alg / gpu_s / 1e9 / peak, 3),
                 "ref_views_per_s_gpu": round(1 / gpu_s, 1), "e2e_ms_host_in_host_out": round(1e3 * min(te), 3),
                 "cpu_reference_s": round(cpu_s, 3), "cpu_remap": remap_name, "speedup_kernel": round(cpu_s / gpu_s, 1), "speedup_e2e": round(cpu_s / min(te), 1),
                 "mask_count_mismatch_px": int((got[1] != want[1]).sum()), "final_mask_mismatch_px": int((got[2] != want[2]).sum()),
                 "pixels": H * W})
print(json.dumps({"gpu": torch.cuda.get_device_name(0), "hbm_peak_gbs": peak, "cpu_threads": torch.get_num_threads(), "rows": rows}, indent=1))
