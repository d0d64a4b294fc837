"""Synthetic DTU-like evaluation inputs, generated from a seed (no DTU data is needed or stored).

A "scan" is a smooth height-field surface over a square of side `side` mm: the STL cloud samples it, the fused cloud samples
it again with Gaussian noise plus a fraction of outliers spread over the box; the observation mask is the set of voxels
within 10 mm of the STL points (as DTU's ObsMask{scan}_10 is) and the plane cuts the scan near its base.  All coordinates
are float32-representable, because PLY files store float32."""
from __future__ import annotations

import os

import numpy as np


def height(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    return 20.0 * np.sin(x / 30.0) * np.cos(y / 45.0) + 0.002 * x * y


def surface(rng: np.random.RandomState, n: int, side: float, offset=(0.0, 0.0, 600.0)) -> np.ndarray:
    x = rng.uniform(-side / 2, side / 2, n)
    y = rng.uniform(-side / 2, side / 2, n)
    p = np.stack([x, y, height(x, y)], axis=1) + np.asarray(offset)
    return p.astype(np.float32).astype(np.float64)


def make_scan(seed: int, n_stl: int = 20000, n_data: int = 40000, side: float = 200.0, noise: float = 0.4,
              outlier_frac: float = 0.01, res: float = 4.0):
    rng = np.random.RandomState(seed)
    stl = surface(rng, n_stl, side)
    data = surface(rng, n_data, side) + rng.normal(0.0, noise, (n_data, 3))
    n_out = int(round(outlier_frac * n_data))
    lo = stl.min(axis=0) - 40.0
    hi = stl.max(axis=0) + 40.0
    data[:n_out] = rng.uniform(lo - 40.0, hi + 40.0, (n_out, 3))  # some fall outside BB and its blocks on purpose
    data = data[rng.permutation(n_data)].astype(np.float32).astype(np.float64)
    return {"data": data, "stl": stl, **scan_truth(stl, lo, hi, res)}


def scan_truth(stl: np.ndarray, lo: np.ndarray, hi: np.ndarray, res: float):
    """bb = [lo, hi], the observation mask (voxels of `res` within 10 mm of an STL point, per axis) and the plane near the
    base of the STL cloud -> {"obs_mask", "bb", "res", "plane"}."""
    bb = np.stack([lo, hi]).astype(np.float64)
    dims = np.ceil((hi - lo) / res).astype(int) + 1
    mask = np.zeros(dims, dtype=bool)
    vox = np.unique(np.floor((stl - lo) / res).astype(int), axis=0)
    r = int(np.ceil(10.0 / res))
    for dx in range(-r, r + 1):
        for dy in range(-r, r + 1):
            for dz in range(-r, r + 1):
                v = np.clip(vox + [dx, dy, dz], 0, dims - 1)
                mask[v[:, 0], v[:, 1], v[:, 2]] = True
    z0 = float(np.percentile(stl[:, 2], 10))
    plane = np.array([0.05, 0.0, 1.0, -z0], dtype=np.float64)  # above: 0.05 x + z > z0
    return {"obs_mask": mask, "bb": bb, "res": float(res), "plane": plane}


def ply_bytes(points: np.ndarray, colours: bool = True) -> bytes:
    """Binary little-endian PLY with float x, y, z (+ uchar red, green, blue): the layout of the project's save_ply."""
    n = points.shape[0]
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("red", "u1"), ("green", "u1"), ("blue", "u1")] if colours else [])
    rec = np.zeros(n, dtype=props)
    for a, k in enumerate("xyz"):
        rec[k] = points[:, a]
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n
    header += "".join("property %s %s\n" % ("float" if t == "<f4" else "uchar", k) for k, t in props) + "end_header\n"
    return header.encode("ascii") + rec.tobytes()


def write_mvs_tree(root: str, outputs: str, scans, seed: int = 0, **kw):
    """DTU's `MVS Data` layout (Points/stl/stl%03d_total.ply, ObsMask/ObsMask{scan}_10.mat, ObsMask/Plane{scan}.mat) under
    `root`, and each scan's fused cloud at outputs/scan{scan}/fused.ply.  -> {scan: make_scan(...) dict}."""
    from scipy.io import savemat

    cases = {}
    os.makedirs(os.path.join(root, "Points", "stl"), exist_ok=True)
    os.makedirs(os.path.join(root, "ObsMask"), exist_ok=True)
    for scan in scans:
        c = make_scan(seed + scan, **kw)
        cases[scan] = c
        with open(os.path.join(root, "Points", "stl", "stl%03d_total.ply" % scan), "wb") as f:
            f.write(ply_bytes(c["stl"], colours=False))
        savemat(os.path.join(root, "ObsMask", f"ObsMask{scan}_10.mat"),
                {"ObsMask": c["obs_mask"], "BB": c["bb"], "Res": c["res"]})
        savemat(os.path.join(root, "ObsMask", f"Plane{scan}.mat"), {"P": c["plane"].reshape(4, 1)})
        os.makedirs(os.path.join(outputs, f"scan{scan}"), exist_ok=True)
        with open(os.path.join(outputs, f"scan{scan}", "fused.ply"), "wb") as f:
            f.write(ply_bytes(c["data"]))
    return cases
