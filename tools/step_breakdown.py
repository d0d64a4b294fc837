"""Where one step of the bench workload spends its device time: torch.profiler (CUDA activities) over one eager forward and
one CUDA-graph replay of a DepthEngine slot, 1 reference + 4 sources at 640x512, fp32-accurate mode (what bench.py times).

    python tools/step_breakdown.py --out DIR [--height 512 --width 640 --views 5 --warmup 3]

Writes DIR/step_breakdown.json: per kernel name the launch count, the summed device microseconds and the share of the
summed kernel time, for the eager forward and for the graph replay; plus the card name, power limit and maximum SM clock read
by nvidia-smi in the same run.  Kernels run one request at a time here (no concurrent slots), so the shares are of one
request's serial device time, not of the overlapped steady state bench.py measures.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from patchmatchnet_b200 import synthetic  # noqa: E402
from patchmatchnet_b200.engine import DepthEngine  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[torch.cuda.current_device()]
        return dict(zip(q.split(","), (v.strip() for v in line.split(","))))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "nvidia_smi_error": repr(e)[:200]}


def profiled(fn):
    """Device activities of one call of `fn` (synchronised before and after) -> per-kernel table."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    per = defaultdict(lambda: [0, 0.0])
    t0, t1 = float("inf"), 0.0
    for e in prof.events():
        if e.device_type != DeviceType.CUDA:
            continue
        per[e.name][0] += 1
        per[e.name][1] += e.time_range.elapsed_us()
        t0, t1 = min(t0, e.time_range.start), max(t1, e.time_range.end)
    total = sum(v[1] for v in per.values())
    rows = sorted(({"kernel": k, "launches": n, "device_us": round(us, 2), "share": round(us / total, 4) if total else 0.0}
                   for k, (n, us) in per.items()), key=lambda r: -r["device_us"])
    return {"kernel_us_total": round(total, 2), "span_us": round(t1 - t0, 2) if per else 0.0, "launches": sum(v[0] for v in per.values()),
            "kernels": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=640)
    ap.add_argument("--views", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_breakdown.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = False  # the fp32-accurate mode bench.py times
    torch.backends.cuda.matmul.allow_tf32 = False
    net, _ = bench.build_net()
    net = net.to(dev)
    inp = synthetic.make_inputs(1, a.views, a.height, a.width, seed=0)
    images = [i.to(dev) for i in inp["images"]]
    cams = (inp["intrinsics"].to(dev), inp["extrinsics"].to(dev), inp["depth_min"].to(dev), inp["depth_max"].to(dev))

    def eager():
        with torch.no_grad():
            net([im.clone() for im in images], cams[0].clone(), *cams[1:])

    for _ in range(a.warmup):
        eager()
    out = {"card": card(), "workload": {"batch": 1, "views": a.views, "height": a.height, "width": a.width, "mode": "fp32-accurate"},
           "eager_forward": profiled(eager)}

    eng = DepthEngine(net, 1, a.views, a.height, a.width, device=str(dev), use_graph=True, warmup=a.warmup, n_slots=1)
    eng.set_device_inputs(0, images, *cams)
    eng.prepare()
    stream = eng._slots[0]["stream"]

    def replay():
        with torch.cuda.stream(stream):
            eng.run_slot(0)

    for _ in range(a.warmup):
        replay()
    out["graph_replay"] = profiled(replay)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "step_breakdown.json"), "w") as f:
        json.dump(out, f, indent=1)
    for mode in ("eager_forward", "graph_replay"):
        r = out[mode]
        print(f"{mode}: {r['launches']} launches, {r['kernel_us_total']:.1f} us of kernels over a {r['span_us']:.1f} us span")
        for k in r["kernels"][:12]:
            print(f"  {k['share'] * 100:5.1f} %  {k['device_us']:9.1f} us  x{k['launches']:<3d} {k['kernel'][:110]}")
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
