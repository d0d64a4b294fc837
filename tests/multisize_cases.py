"""Seeded requests whose views differ in size (test infrastructure): a 1 + 4 view network request and a geometric-filter
scene.  Shared by tests/golden/make_multisize_golden.py (which ran the reference on them) and the tests that compare against
its fixture, tests/golden/multisize_case.pt."""
from __future__ import annotations

import math
import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from patchmatchnet_b200 import synthetic
from tests import geo_cases

# reference, a same-size source, a portrait source, a source that is not a multiple of 8 (adjust_image_dims rescales it to
# 64 x 80) and a smaller landscape source: three distinct sizes after rounding
NET_SIZES: List[Tuple[int, int]] = [(64, 80), (64, 80), (80, 64), (60, 76), (48, 72)]
NET_SEED = 41

GEO_REF_HW = (96, 128)
GEO_SRC_HW: List[Tuple[int, int]] = [(96, 128), (128, 96), (72, 100), (120, 160)]


def make_net_inputs(sizes=NET_SIZES, seed: int = NET_SEED) -> Dict[str, object]:
    """images [1,3,H_v,W_v] U[0,1) per view; cameras of synthetic.make_cameras with each view's principal point at the centre of
    its own image; depth range; rand48, the stage-3 draw of the reference's torch.rand stream seeded with seed + 1000."""
    g = torch.Generator().manual_seed(seed)
    images = [torch.rand(1, 3, h, w, generator=g) for h, w in sizes]
    H, W = sizes[0]
    K, E = synthetic.make_cameras(1, len(sizes), H, W)
    for i, (h, w) in enumerate(sizes):
        K[0, i, 0, 2] = w / 2
        K[0, i, 1, 2] = h / 2
    state = torch.get_rng_state()
    torch.manual_seed(seed + 1000)
    rand48 = torch.rand(size=(1, 48, H // 8, W // 8))
    torch.set_rng_state(state)
    return {"images": images, "intrinsics": K, "extrinsics": E, "depth_min": torch.full((1,), synthetic.DEPTH_MIN),
            "depth_max": torch.full((1,), synthetic.DEPTH_MAX), "rand48": rand48}


def make_geo_scene(seed: int = 0) -> Dict[str, object]:
    """geo_cases.make_scene with a size per source view: the plane rendered into each source camera at that camera's own
    size (principal point at its centre), then corrupted the same way."""
    rng = np.random.default_rng(seed)
    H, W = GEO_REF_HW
    n = np.array([0.12, -0.08, 1.0])
    n = n / np.linalg.norm(n)
    d0 = 600.0
    cams, sizes = [], [GEO_REF_HW] + GEO_SRC_HW
    for i, (h, w) in enumerate(sizes):
        E = np.eye(4, dtype=np.float64)
        if i:
            sgn = 1.0 if i % 2 else -1.0
            E[:3, :3] = geo_cases._rot_y(math.radians(2.0 * i) * sgn) @ geo_cases._rot_x(math.radians(0.7 * i))
            E[:3, 3] = [40.0 * sgn * i, -15.0 * (i % 3), 5.0 * i]
        f = 1.2 * W  # one focal length in pixels of the reference's size: views differ in extent, not in scale
        K = np.array([[f, 0, w / 2 + 1.5 * i], [0, f, h / 2], [0, 0, 1]], dtype=np.float32)
        cams.append((K, E.astype(np.float32)))
    depths = [geo_cases.plane_depth(k, e, h, w, n, d0) for (k, e), (h, w) in zip(cams, sizes)]
    for i in range(1, len(sizes)):
        h, w = sizes[i]
        for _ in range(3):
            y0, x0 = int(rng.integers(0, h - 16)), int(rng.integers(0, w - 24))
            depths[i][y0:y0 + 16, x0:x0 + 24] *= np.float32(1.0 + rng.choice([-1, 1]) * rng.uniform(0.005, 0.05))
        depths[i] += rng.normal(0, 0.05, size=(h, w)).astype(np.float32)
    depths[0][H // 3: H // 3 + 6, :] *= np.float32(1.03)
    conf = rng.uniform(0.5, 1.0, size=(H, W)).astype(np.float32)
    return dict(ref_depth=depths[0], ref_K=cams[0][0], ref_E=cams[0][1], src_depths=depths[1:],
                src_Ks=[c[0] for c in cams[1:]], src_Es=[c[1] for c in cams[1:]], confidence=conf)


def mixed_sizes(n_views: int, H: int, W: int, portrait_every: int = 3) -> List[Tuple[int, int]]:
    """(H, W) per view: landscape H x W, every `portrait_every`-th view (1, 4, 7, ...) portrait W x H."""
    return [(W, H) if i % portrait_every == 1 else (H, W) for i in range(n_views)]


def write_mixed_scene(root: str, sizes: Sequence[Tuple[int, int]], n_src: int, quality: int = 95) -> Dict[str, object]:
    """tests/scene_cases.write_scene with a size per view: the plane scene's cameras with one focal length in pixels and each
    view's principal point at the centre of its own image.  -> {"cams", "pairs"}."""
    from PIL import Image

    from tests import scene_cases

    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    os.makedirs(os.path.join(root, "cams"), exist_ok=True)
    H0, W0 = sizes[0]
    cams = []
    for i, ((K, E), (h, w)) in enumerate(zip(scene_cases.cameras(len(sizes), H0, W0), sizes)):
        K = K.copy()
        K[0, 2], K[1, 2] = w / 2 + 1.5 * i, h / 2
        cams.append((K, E))
    pairs = scene_cases.all_pairs(len(sizes), n_src)
    with open(os.path.join(root, "pair.txt"), "w") as f:
        f.write(scene_cases.pair_text(pairs))
    for v, ((K, E), (h, w)) in enumerate(zip(cams, sizes)):
        with open(os.path.join(root, "cams", "%08d_cam.txt" % v), "w") as f:
            f.write(scene_cases.cam_text(K, E))
        Image.fromarray(scene_cases.texture(K, E, h, w)).save(os.path.join(root, "images", "%08d.jpg" % v), quality=quality)
    return {"cams": cams, "pairs": pairs}
