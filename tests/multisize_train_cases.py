"""Seeded training requests whose views differ in size (test infrastructure), shared by
tests/golden/make_multisize_train_golden.py (which ran the reference on them) and the tests that compare against its fixture,
tests/golden/multisize_train_case.pt.

    B = 1   multisize_cases.make_net_inputs: the 1 + 4 view request of the inference fixture (three sizes after rounding)
    B = 2   the same view sizes, two samples per view that agree view by view (what one batch of such data holds)

Each case also carries per-level ground truth and masks for patchmatchnet_loss and the stage-3 random draw (rand48)."""
from __future__ import annotations

import os
import zlib
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from patchmatchnet_b200 import synthetic
from tests import multisize_cases

B2_SEED = 43


def make_batch2_inputs(sizes=multisize_cases.NET_SIZES, seed: int = B2_SEED) -> Dict[str, object]:
    """multisize_cases.make_net_inputs with two samples per view: images [2,3,H_v,W_v], the two samples' cameras differ."""
    g = torch.Generator().manual_seed(seed)
    images = [torch.rand(2, 3, h, w, generator=g) for h, w in sizes]
    H, W = sizes[0]
    K, E = synthetic.make_cameras(2, len(sizes), H, W)
    for i, (h, w) in enumerate(sizes):
        K[:, i, 0, 2] = w / 2
        K[:, i, 1, 2] = h / 2
    state = torch.get_rng_state()
    torch.manual_seed(seed + 1000)
    rand48 = torch.rand(size=(2, 48, H // 8, W // 8))
    torch.set_rng_state(state)
    return {"images": images, "intrinsics": K, "extrinsics": E, "depth_min": torch.full((2,), synthetic.DEPTH_MIN),
            "depth_max": torch.full((2,), synthetic.DEPTH_MAX), "rand48": rand48}


def make_case(B: int) -> Dict[str, object]:
    """inputs (+ "seed": what torch.manual_seed gets right before the forward, so that the reference's stage-3 torch.rand
    draws rand48) and per-level "gts" [B,1,H>>l,W>>l] / "masks" (bool) for patchmatchnet_loss."""
    if B == 1:
        inp, seed = multisize_cases.make_net_inputs(), multisize_cases.NET_SEED + 1000
    elif B == 2:
        inp, seed = make_batch2_inputs(), B2_SEED + 1000
    else:
        raise ValueError(B)
    H, W = multisize_cases.NET_SIZES[0]
    g = torch.Generator().manual_seed(7 + B)
    gts: List[torch.Tensor] = []
    masks: List[torch.Tensor] = []
    for lvl in range(4):
        h, w = H >> lvl, W >> lvl
        gts.append(synthetic.DEPTH_MIN + (synthetic.DEPTH_MAX - synthetic.DEPTH_MIN) * torch.rand(B, 1, h, w, generator=g))
        masks.append(torch.rand(B, 1, h, w, generator=g) > 0.2)
    return dict(inp, seed=seed, gts=gts, masks=masks)


# ---- how the fixture stores gradients ---------------------------------------------------------------------------------------
# Gradients are compared with a bound, not bit for bit: CPU convolution backward kernels sum in an order that depends on the
# machine (vector width, threads), so even the reference's own gradients differ in the last bits from one CPU to another.
# Each gradient is stored quantised per tensor to 12 bits of its largest magnitude (error at most half a step, 2^-12 of that
# magnitude) and zlib-compressed; float32 for both cases would take about 1.8 MB.
Q_STEPS = 2047


def pack_grads(grads: Dict[str, Optional[torch.Tensor]]) -> Dict[str, object]:
    """{"names": every parameter name, "shapes": [shape or None (no gradient)], "scales": float64 [n], "blob": uint8 tensor of
    the zlib-compressed int16 values of every gradient, back to back in name order}"""
    names, shapes, scales, parts = list(grads), [], [], []
    for g in grads.values():
        if g is None:
            shapes.append(None)
            scales.append(0.0)
            continue
        a = g.detach().cpu().double().numpy()
        scale = float(np.abs(a).max()) or 1.0
        shapes.append(tuple(a.shape))
        scales.append(scale)
        parts.append(np.round(a / scale * Q_STEPS).astype(np.int16).ravel())
    blob = zlib.compress(np.concatenate(parts).tobytes(), 9)
    return {"names": names, "shapes": shapes, "scales": torch.tensor(scales, dtype=torch.float64),
            "blob": torch.frombuffer(bytearray(blob), dtype=torch.uint8)}


def unpack_grads(packed) -> Dict[str, Optional[Tuple[torch.Tensor, float]]]:
    """{name: None or (float64 gradient, scale)}: each stored value lies within half_step(scale) of the reference's; scale is
    the reference tensor's largest magnitude"""
    q = np.frombuffer(zlib.decompress(packed["blob"].numpy().tobytes()), dtype=np.int16)
    out: Dict[str, Optional[Tuple[torch.Tensor, float]]] = {}
    pos = 0
    for name, shape, scale in zip(packed["names"], packed["shapes"], packed["scales"].tolist()):
        if shape is None:
            out[name] = None
            continue
        n = int(np.prod(shape))
        out[name] = (torch.from_numpy(q[pos:pos + n].astype(np.float64) * (scale / Q_STEPS)).reshape(shape), scale)
        pos += n
    return out


def half_step(scale: float) -> float:
    return 0.5 * scale / Q_STEPS


# ---- a small ETH3D-style training tree for convert_eth3d ------------------------------------------------------------------

ETH3D_SCANS = ["courtyard", "pipes"]


def write_raw_eth3d_tree(root: str) -> str:
    """Per scan: cams/index2prefix.txt (ids not in file order, names with "_undistorted" and sub-folders), cams/pair.txt,
    cams/%08d_cam.txt, images/<name>.png (views of different sizes) and depths/<name without _undistorted>.pfm with zeros
    where ETH3D has no ground truth.  -> the scan list's path."""
    from PIL import Image

    from patchmatchnet_b200 import data_io

    rng = np.random.default_rng(11)
    for s, scan in enumerate(ETH3D_SCANS):
        ids = [3, 0, 1] if s == 0 else [0, 2]
        names = {v: "dslr_images_undistorted/DSC_{:04d}.JPG".format(100 * s + v).replace(".JPG", ".png") for v in ids}
        cam_dir = os.path.join(root, scan, "cams")
        os.makedirs(cam_dir, exist_ok=True)
        with open(os.path.join(cam_dir, "index2prefix.txt"), "w") as f:
            f.write("{}\n".format(len(ids)))
            for v in ids:
                f.write("{} {}\n".format(v, names[v]))
        with open(os.path.join(cam_dir, "pair.txt"), "w") as f:
            f.write("{}\n".format(len(ids)))
            for v in ids:
                others = [u for u in ids if u != v]
                f.write("{}\n{} {}\n".format(v, len(others), " ".join("{} {:.3f}".format(u, 10.0 - u) for u in others)))
        for k, v in enumerate(ids):
            h, w = (24, 32) if (v + s) % 2 == 0 else (32, 24)
            with open(os.path.join(cam_dir, "{:0>8}_cam.txt".format(v)), "w") as f:
                f.write("extrinsic\n1 0 0 {0}\n0 1 0 0\n0 0 1 0\n0 0 0 1\n\nintrinsic\n30 0 {1}\n0 30 {2}\n0 0 1\n\n1.5 9.5\n"
                        .format(0.1 * v, w / 2, h / 2))
            img = os.path.join(root, scan, "images", names[v])
            os.makedirs(os.path.dirname(img), exist_ok=True)
            Image.fromarray(rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)).save(img)
            depth = rng.uniform(2.0, 9.0, size=(h, w)).astype(np.float32)
            depth[rng.uniform(size=(h, w)) < 0.3] = 0.0
            dpath = os.path.join(root, scan, "depths", os.path.splitext(names[v].replace("_undistorted", ""))[0] + ".pfm")
            os.makedirs(os.path.dirname(dpath), exist_ok=True)
            data_io.save_pfm(dpath, depth)
    scan_list = os.path.join(root, "scans.txt")
    with open(scan_list, "w") as f:
        f.write("\n".join(ETH3D_SCANS) + "\n")
    return scan_list
