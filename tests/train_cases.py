"""Seeded inputs of the training tests (test and golden-generator infrastructure): a training tree in the converted layout
train reads, a raw DTU tree in the layout convert_dtu reads, and loss / metric tensors.  The same seed always writes the
same files, so tests regenerate exactly what tests/golden/make_train_golden.py gave the reference."""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import numpy as np

SCANS = ["scan1", "scan2"]
TREE_HW = (48, 64)
N_VIEWS = 4
LIGHTS = 2
LOSS_CASES = [(2, 64, 80), (1, 37, 53)]
LOSS_LEVELS = [0, 1, 2, 2, 3, 3]  # the default PatchMatch iterations (1, 2, 2)


def _pfm_bytes(data: np.ndarray) -> bytes:
    """A little-endian 'Pf' file of data [H,W] float32 (bottom row first), the bytes the reference's save_pfm writes."""
    h, w = data.shape
    return b"Pf\n" + f"{w} {h}\n".encode() + b"-1.000000\n" + np.flipud(data).astype("<f4").tobytes()


def _cam_text(E: np.ndarray, K: np.ndarray, depth_range: Tuple[float, float]) -> str:
    rows = ["extrinsic"] + [" ".join(f"{v:.9g}" for v in r) for r in E] + ["", "intrinsic"]
    rows += [" ".join(f"{v:.9g}" for v in r) for r in K] + ["", "%.9g %.9g" % depth_range]
    return "\n".join(rows) + "\n"


def _pair_text(n: int) -> str:
    lines = [str(n)]
    for r in range(n):
        src = [v for v in range(n) if v != r]
        lines += [str(r), " ".join([str(len(src))] + [f"{s} {100.0 - k:.1f}" for k, s in enumerate(src)])]
    return "\n".join(lines) + "\n"


def write_training_tree(root: str, seed: int = 7) -> None:
    """SCANS in the converted layout: pair.txt, cams/, images/<light>/%08d.jpg, depth_gt/%08d.pfm; part of every depth
    map lies below the depth range, so the masks are partial."""
    from PIL import Image

    rng = np.random.default_rng(seed)
    H, W = TREE_HW
    for scan in SCANS:
        base = os.path.join(root, scan)
        for sub in ["cams", "depth_gt"] + [os.path.join("images", str(i)) for i in range(LIGHTS)]:
            os.makedirs(os.path.join(base, sub), exist_ok=True)
        with open(os.path.join(base, "pair.txt"), "w") as f:
            f.write(_pair_text(N_VIEWS))
        for v in range(N_VIEWS):
            E = np.eye(4)
            E[:3, 3] = rng.uniform(-50, 50, 3)
            K = np.array([[rng.uniform(50, 80), 0, W / 2], [0, rng.uniform(50, 80), H / 2], [0, 0, 1]])
            with open(os.path.join(base, "cams", "%08d_cam.txt" % v), "w") as f:
                f.write(_cam_text(E, K, (450.0 + v, 900.5)))
            depth = rng.uniform(400.0, 950.0, (H, W)).astype(np.float32)
            with open(os.path.join(base, "depth_gt", "%08d.pfm" % v), "wb") as f:
                f.write(_pfm_bytes(depth))
            for light in range(LIGHTS):
                img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
                Image.fromarray(img).save(os.path.join(base, "images", str(light), "%08d.jpg" % v), quality=95)
    with open(os.path.join(root, "scans.txt"), "w") as f:
        f.write("\n".join(SCANS) + "\n")


RAW_HW = (1200, 1600)
RAW_VIEWS = [0, 3]


def write_raw_dtu_tree(root: str, seed: int = 11) -> str:
    """A raw DTU training tree (Cameras_1, Depths_raw, Rectified) with one scan of two views; -> the scan list path."""
    from PIL import Image

    rng = np.random.default_rng(seed)
    H, W = RAW_HW
    scan = "scan1"
    os.makedirs(os.path.join(root, "Cameras_1", "train"), exist_ok=True)
    os.makedirs(os.path.join(root, "Depths_raw", scan), exist_ok=True)
    os.makedirs(os.path.join(root, "Rectified", scan + "_train"), exist_ok=True)
    with open(os.path.join(root, "Cameras_1", "pair.txt"), "w") as f:
        f.write("2\n0\n1 3 100.0\n3\n1 0 100.0\n")
    for v in RAW_VIEWS:
        E = np.eye(4)
        E[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        E[:3, 3] = rng.uniform(-300, 300, 3)
        K = np.array([[rng.uniform(600, 700), 0, rng.uniform(150, 170)], [0, rng.uniform(600, 700), rng.uniform(110, 130)], [0, 0, 1]])
        with open(os.path.join(root, "Cameras_1", "train", "%08d_cam.txt" % v), "w") as f:
            f.write(_cam_text(E, K, (425.0, 2.5)))
        y, x = np.mgrid[0:H, 0:W].astype(np.float32)
        depth = (600.0 + 0.05 * x + 0.03 * y + rng.normal(0, 1.0, (H, W))).astype(np.float32)
        depth[rng.random((H, W)) < 0.2] = 0.0
        with open(os.path.join(root, "Depths_raw", scan, "depth_map_%04d.pfm" % v), "wb") as f:
            f.write(_pfm_bytes(depth))
        visual = (np.clip(depth / 1000.0, 0, 1) * 255).astype(np.uint8)
        visual[rng.random((H, W)) < 0.1] = 5  # 5 / 255 < 0.04 < 15 / 255: some pixels fall below the mask threshold
        Image.fromarray(visual).save(os.path.join(root, "Depths_raw", scan, "depth_visual_%04d.png" % v))
        for light in range(7):
            img = rng.integers(0, 256, (512, 640, 3), dtype=np.uint8)
            Image.fromarray(img).save(os.path.join(root, "Rectified", scan + "_train", "rect_%03d_%d_r5000.png" % (v + 1, light)))
    path = os.path.join(root, "scans.txt")
    with open(path, "w") as f:
        f.write(scan + "\n")
    return path


def loss_case(B: int, H: int, W: int, seed: int) -> Dict[str, object]:
    """float64 ground truth [B,1,H,W], mask [B,1,H,W] bool, and the maps of LOSS_LEVELS ([B,1,H>>l,W>>l]) as the ground
    truth of their level plus errors both below and above 1 in magnitude."""
    rng = np.random.default_rng(seed)
    gt = rng.uniform(450.0, 900.0, (B, 1, H, W))
    mask = (gt > 500.0) & (rng.random((B, 1, H, W)) > 0.2)
    maps: List[np.ndarray] = []
    for l in LOSS_LEVELS:
        g = gt[..., : (H >> l) << l: 1 << l, : (W >> l) << l: 1 << l]
        scale = np.where(rng.random(g.shape) < 0.5, 0.4, 6.0)
        maps.append(g + rng.normal(0.0, 1.0, g.shape) * scale)
    return {"gt": gt, "mask": mask, "maps": maps}
