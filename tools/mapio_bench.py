"""Host-side timing of the depth-map file I/O (SURVEY.md 8f row f5): native (libpmb200.so via patchmatchnet_b200.data_io)
against the unmodified reference functions (datasets/data_io.py of a reference checkout given with --reference) on the same arrays, in
the same tmpfs directory.  Host code only -- no GPU involved; prints one JSON object.

    python tools/mapio_bench.py [--height 1184 --width 1600 --repeat 5] [--reference <checkout>]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from patchmatchnet_b200 import data_io as dio  # noqa: E402


def best(fn, repeat):
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--height", type=int, default=1184)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--reference", default=None, help="checkout of the reference project to time against")
    args = ap.parse_args()
    ref = None
    if args.reference:
        sys.path.insert(0, os.path.abspath(args.reference))
        from datasets import data_io as ref  # noqa: E402
    rng = np.random.default_rng(0)
    arr = rng.uniform(425, 935, size=(args.height, args.width)).astype(np.float32)
    mb = arr.nbytes / 1e6
    out = {"map": f"{args.height}x{args.width} float32 ({mb:.2f} MB)", "host_cpus": os.cpu_count(), "repeat": args.repeat,
           "timing": "best of repeat, time.perf_counter, files in a tmpfs/tmp directory (page cache hot)", "rows": []}
    tmpdir = "/dev/shm" if os.path.isdir("/dev/shm") else None
    with tempfile.TemporaryDirectory(dir=tmpdir) as d:
        for ext in ("pfm", "bin"):
            p = os.path.join(d, f"m.{ext}")
            row = {"format": ext}
            row["native_save_ms"] = 1e3 * best(lambda: dio.save_map(p, arr), args.repeat)
            row["native_read_ms"] = 1e3 * best(lambda: dio.read_map(p), args.repeat)
            row["native_save_MBps"] = mb / (row["native_save_ms"] / 1e3)
            row["native_read_MBps"] = mb / (row["native_read_ms"] / 1e3)
            if ref is not None:
                row["reference_save_ms"] = 1e3 * best(lambda: ref.save_map(p, arr), max(1, args.repeat // 2))
                row["reference_read_ms"] = 1e3 * best(lambda: ref.read_map(p), max(1, args.repeat // 2))
                row["save_speedup"] = row["reference_save_ms"] / row["native_save_ms"]
                row["read_speedup"] = row["reference_read_ms"] / row["native_read_ms"]
            out["rows"].append(row)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
