"""e2e (pinned host in -> pinned host out) through DepthEngine.infer_stream at several request counts, with the host-side
enqueue time of the loop measured separately: separates pipeline fill / drain, host-bound and GPU-bound regimes.

    python tools/e2e_probe.py
"""
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

torch.backends.cudnn.benchmark = True
torch.backends.cudnn.allow_tf32 = False
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
numa = bench.bind_to_gpu_numa_node(0)
net, _ = bench.build_net()
net = net.to(dev)
wl = bench.Workload(net, 1, 5, 512, 640, dev, 3, 0)
stream = torch.cuda.current_stream()
out = {"numa": numa, "rows": []}
for steps in (20, 20, 60, 200, 200):
    reqs = [wl.host_pinned] * steps
    torch.cuda.synchronize()
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    t0.record(stream)
    wl.eng.copy_stream.wait_event(t0)
    for sl in wl.eng._slots:
        sl["stream"].wait_event(t0)
    wl.eng.infer_stream(reqs)
    t1.record(stream)
    torch.cuda.synchronize()
    w1 = time.perf_counter()
    out["rows"].append({"requests": steps, "device_ms_per_request": t0.elapsed_time(t1) / steps, "wall_ms_per_request": 1e3 * (w1 - w0) / steps})
# host enqueue cost alone: GPU parked behind a long sleep so that nothing completes while the loop runs
torch.cuda._sleep(400_000_000)
w0 = time.perf_counter()
S = wl.eng.n_slots
reqs = [wl.host_pinned] * 12
# the loop of infer_stream without its final synchronize is not exposed; time the whole call minus the parked time instead
wl.eng.infer_stream(reqs)
w1 = time.perf_counter()
out["host_note"] = "last row: 12 requests enqueued behind a ~200 ms device sleep; wall = sleep + drain, see rows for the steady state"
out["parked_call_wall_ms"] = 1e3 * (w1 - w0)
print(json.dumps(out))
