"""Seeded synthetic Tanks and Temples scenes, written in the T&T file layouts (test infrastructure).

GT: samples of a curved surface about 2 m across, placed at T&T-like coordinates (tens of metres from the origin).  The
reconstruction: fresh samples of the same surface with Gaussian noise of 0.3 tau, missing a strip of it, plus outliers
outside the crop volume, all expressed in a reconstruction frame related to the GT frame by a known similarity S (rec ->
GT).  The cameras: a ring of centres around the surface; the scene folder's cams/ hold them in the reconstruction frame, and
the COLMAP SfM log holds them in an SfM frame that _trans.txt maps onto the GT frame.  Every coordinate is float32
representable, so the PLY files (float32) carry the points exactly."""
from __future__ import annotations

import json
import os

import numpy as np
import torch

from patchmatchnet_b200 import data_io

OFFSET = np.array([31.0, -17.0, 6.0])


def rotation(axis, angle) -> np.ndarray:
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    k = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * k + (1 - np.cos(angle)) * k @ k


def similarity(scale, axis, angle, t) -> np.ndarray:
    m = np.eye(4)
    m[:3, :3] = scale * rotation(axis, angle)
    m[:3, 3] = t
    return m


def apply(m, p) -> np.ndarray:
    return np.asarray(p, np.float64) @ m[:3, :3].T + m[:3, 3]


def f32(p) -> np.ndarray:
    return np.asarray(p, np.float64).astype(np.float32).astype(np.float64)


def surface(rng, n) -> np.ndarray:
    x, y = rng.uniform(-1.0, 1.0, n), rng.uniform(-1.0, 1.0, n)
    z = 0.25 * np.sin(2.0 * x) * np.cos(1.5 * y) + 0.1 * x * y
    return np.stack([x, y, z], axis=1) + OFFSET


def crop_volume():
    """A hexagon in x-y (orthogonal axis Z) that cuts the surface's corners off, and z bounds around it."""
    ang = np.arange(6) * (np.pi / 3) + 0.2
    poly = np.stack([OFFSET[0] + 0.9 * np.cos(ang), OFFSET[1] + 0.9 * np.sin(ang), np.full(6, OFFSET[2])], axis=1)
    return {"orthogonal_axis": 2, "axis_min": OFFSET[2] - 0.5, "axis_max": OFFSET[2] + 0.5, "polygon": f32(poly)}


def make_scene(seed: int, n_gt: int = 60000, n_rec: int = 50000, tau: float = 0.02, n_cams: int = 40, outliers: float = 0.03):
    rng = np.random.RandomState(seed)
    gt = f32(surface(rng, n_gt))
    rec_gt = surface(rng, n_rec)
    rec_gt = rec_gt[~((rec_gt[:, 0] - OFFSET[0] > 0.2) & (rec_gt[:, 0] - OFFSET[0] < 0.35))]  # a strip the reconstruction missed
    rec_gt = rec_gt + rng.normal(0.0, 0.3 * tau, rec_gt.shape)
    k = int(outliers * len(rec_gt))
    far = rng.uniform(-1, 1, (k, 3)) * 0.4 + OFFSET + np.array([0.0, 0.0, 1.2])  # above axis_max: outside the crop
    rec_gt = np.concatenate([rec_gt, far])
    s = similarity(1.7, [0.3, -0.5, 0.8], 0.6, [-3.0, 2.0, 0.5])  # rec -> GT
    rec = f32(apply(np.linalg.inv(s), rec_gt))
    ang = np.linspace(0, 2 * np.pi, n_cams, endpoint=False)
    centres_gt = np.stack([OFFSET[0] + 2.5 * np.cos(ang), OFFSET[1] + 2.5 * np.sin(ang), OFFSET[2] + 1.0 + 0.3 * np.sin(3 * ang)], 1)
    trans = similarity(0.8, [0.1, 0.9, -0.2], -0.4, [4.0, -1.0, 2.0])  # SfM -> GT
    log = np.zeros((n_cams, 4, 4))
    centres_sfm = apply(np.linalg.inv(trans), centres_gt)
    for i in range(n_cams):
        log[i] = similarity(1.0, rng.normal(size=3), rng.uniform(0, 3), centres_sfm[i])  # camera-to-world, rotation arbitrary
    extr = np.zeros((n_cams, 4, 4))
    centres_rec = apply(np.linalg.inv(s), centres_gt)
    for i in range(n_cams):
        r = rotation(rng.normal(size=3), rng.uniform(0, 3))
        extr[i] = np.eye(4)
        extr[i, :3, :3] = r
        extr[i, :3, 3] = -r @ centres_rec[i]
    return {"gt": gt, "rec": rec, "crop": crop_volume(), "S": s, "trans": trans, "log": log, "extrinsics": extr, "tau": tau}


def _save_points(path, pts):
    xyz = np.asarray(pts, np.float32).reshape(-1, 3)
    body = np.concatenate([xyz.view(np.uint8).reshape(-1, 12), np.full((len(xyz), 3), 128, np.uint8)], axis=1)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    data_io.save_ply(path, torch.from_numpy(np.ascontiguousarray(body)))


def write_tree(root: str, scenes, **kw):
    """root/gt/<Scene>/{<Scene>.ply, .json, _trans.txt, _COLMAP_SfM.log}, root/outputs/<Scene>/fused.ply and
    root/scenes/<Scene>/cams/%08d_cam.txt.  -> {scene: make_scene(...)}."""
    out = {}
    for k, scene in enumerate(scenes):
        c = make_scene(100 + k, **kw)
        g = os.path.join(root, "gt", scene)
        os.makedirs(g, exist_ok=True)
        _save_points(os.path.join(g, f"{scene}.ply"), c["gt"])
        cv = c["crop"]
        with open(os.path.join(g, f"{scene}.json"), "w") as f:
            json.dump({"axis_max": cv["axis_max"], "axis_min": cv["axis_min"], "bounding_polygon": cv["polygon"].tolist(),
                       "class_name": "SelectionPolygonVolume", "orthogonal_axis": "XYZ"[cv["orthogonal_axis"]],
                       "version_major": 1, "version_minor": 0}, f, indent=1)
        np.savetxt(os.path.join(g, f"{scene}_trans.txt"), c["trans"], fmt="%.17g")
        with open(os.path.join(g, f"{scene}_COLMAP_SfM.log"), "w") as f:
            for i, m in enumerate(c["log"]):
                f.write(f"{i} {i} 0\n" + "".join(" ".join(f"{v:.17g}" for v in row) + "\n" for row in m))
        _save_points(os.path.join(root, "outputs", scene, "fused.ply"), c["rec"])
        cams = os.path.join(root, "scenes", scene, "cams")
        os.makedirs(cams, exist_ok=True)
        for i, e in enumerate(c["extrinsics"]):
            with open(os.path.join(cams, "%08d_cam.txt" % i), "w") as f:
                f.write("extrinsic\n" + "".join(" ".join(f"{v:.9g}" for v in row) + "\n" for row in e))
                f.write("\nintrinsic\n500 0 320\n0 500 240\n0 0 1\n\n1.0 5.0\n")
        out[scene] = c
    return out
