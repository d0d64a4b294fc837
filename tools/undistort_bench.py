"""colmap_input --undistort, stage by stage: decode, pinned upload, border extents, warp, download and encode of one image,
each timed with CUDA events (device stages) or a host clock ending in a device synchronise (host stages); then the pipelined
path of the command (colmap_input.undistort_images) over a few copies of the same image.

    python tools/undistort_bench.py [--repeats 20] [--copies 8] [--json out.json]

Two cases: 6048 x 4032 THIN_PRISM_FISHEYE (the size of ETH3D's DSLR images) and 1920 x 1080 OPENCV, each from a JPEG source
(quality 95, 4:4:4) of a smooth synthetic texture.  The warp's bytes/s counts 3 bytes read and 3 written per target pixel.
Prints the card name and its power limit first, then one JSON line per case."""
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

CASES = {
    "eth3d_dslr_thin_prism": ci.Camera(1, "THIN_PRISM_FISHEYE", 6048, 4032, [3410.0, 3409.0, 3024.5, 2016.2, 0.0102, -0.0031, 0.0004,
                                                                           -0.0002, 0.0011, -0.0004, 0.0003, -0.0002]),
    "fullhd_opencv": ci.Camera(2, "OPENCV", 1920, 1080, [1400.0, 1398.0, 961.3, 538.9, -0.12, 0.045, 0.0007, -0.0004]),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        power = out.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        power = "unknown"
    return name, power


def texture(W, H):
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    chans = [np.sin(x / (37.0 + 9 * c)) * np.cos(y / (23.0 + 5 * c)) + 0.3 * np.sin((x + 2 * y) / 5.0 + c) for c in range(3)]
    return np.clip(127.5 + 90.0 * np.stack(chans, -1), 0, 255).astype(np.uint8)


def events_ms(fn, repeats):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()  # warm-up
    torch.cuda.synchronize()
    start.record()
    for _ in range(repeats):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / repeats


def host_ms(fn, repeats):
    fn()
    times = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    return float(np.median(times))


def run(name, cam, repeats, copies):
    from PIL import Image

    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "in", "images"))
        os.makedirs(os.path.join(tmp, "out", "images"))
        src_path = os.path.join(tmp, "in", "images", "src.jpg")
        Image.fromarray(texture(cam.width, cam.height)).save(src_path, format="JPEG", quality=95, subsampling=0)
        host_repeats = max(3, repeats // 4)

        decoded = {}

        def decode():
            decoded["img"], decoded["fmt"] = ci._decode_pinned(src_path)

        decode_ms = host_ms(decode, host_repeats)
        pinned = decoded["img"]
        dev_src = torch.empty(pinned.shape, dtype=torch.uint8, device=dev)
        upload_ms = events_ms(lambda: dev_src.copy_(pinned, non_blocking=True), repeats)
        extents_ms = events_ms(lambda: ops.undistort_extents([cam], dev), repeats)
        pin = ops.undistorted_camera(cam, ops.undistort_extents([cam], dev)[0].cpu().numpy())
        out = {}

        def warp():
            out["img"] = ops.undistort_image(dev_src, cam, pin)

        warp_ms = events_ms(warp, repeats)
        host_out = torch.empty(out["img"].shape, dtype=torch.uint8, pin_memory=True)
        download_ms = events_ms(lambda: host_out.copy_(out["img"], non_blocking=True), repeats)
        dst = os.path.join(tmp, "out", "images", "00000000.jpg")
        encode_ms = host_ms(lambda: ci._encode(host_out.numpy(), "JPEG", dst), host_repeats)

        # the command's pipelined path over `copies` images of this camera
        images = [ci.Image(k + 1, [1, 0, 0, 0], [0, 0, 0], cam.id, "src.jpg", np.zeros(0, np.int64)) for k in range(copies)]
        ci.undistort_images(os.path.join(tmp, "in"), os.path.join(tmp, "out"), images[:1], {cam.id: cam}, {cam.id: pin}, dev)
        torch.cuda.synchronize()
        t = time.perf_counter()
        ci.undistort_images(os.path.join(tmp, "in"), os.path.join(tmp, "out"), images, {cam.id: cam}, {cam.id: pin}, dev)
        torch.cuda.synchronize()
        pipeline_s = time.perf_counter() - t

    px = pin.width * pin.height
    stages = {"decode_ms": decode_ms, "upload_ms": upload_ms, "extents_ms": extents_ms, "warp_ms": warp_ms,
              "download_ms": download_ms, "encode_ms": encode_ms}
    return {
        "case": name, "model": cam.model, "source": [cam.width, cam.height], "target": [pin.width, pin.height], **stages,
        "warp_gbytes_per_s": 6 * px / (warp_ms * 1e-3) / 1e9,
        "stage_sum_ms": sum(stages.values()), "bounding_stage": max(stages, key=stages.get),
        "pipeline_images": copies, "pipeline_ms_per_image": pipeline_s * 1e3 / copies,
    }


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--copies", type=int, default=8)
    ap.add_argument("--json", type=str, default="")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("undistort_bench needs a CUDA device")
    name, power = card()
    print(f"card: {name}, power limit {power}")
    rows = [run(k, cam, args.repeats, args.copies) for k, cam in CASES.items()]
    for r in rows:
        print(json.dumps(r))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": name, "power_limit": power, "rows": rows}, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
