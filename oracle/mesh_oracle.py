"""Oracle of the TSDF mesher (include/patchmatch_b200.h "Meshes"; beyond the reference, which has no mesher): allocation,
integration and marching cubes restated in numpy float64.  The triangle table is read from the text of
patchmatchnet_b200/csrc/pm_mesh_math.cuh; the tests check it with invariants of their own.  Never imported by the product.
"""
from __future__ import annotations

import os
import re

import numpy as np

_HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "patchmatchnet_b200", "csrc",
                       "pm_mesh_math.cuh")
KEY_BIAS = 1 << 20
VOXEL_LIMIT = 1 << 23
# corner c at offset (x, y, z); edges as (lower corner offset, axis)
CORNERS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)], dtype=np.int64)
EDGE_OFFSET = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (0, 0, 1), (0, 0, 0),
                        (1, 0, 0), (1, 1, 0), (0, 1, 0)], dtype=np.int64)
EDGE_AXIS = np.array([0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2], dtype=np.int64)
UNIT = np.eye(3, dtype=np.int64)


def read_table(path: str = _HEADER) -> np.ndarray:
    """kTriTable of the header -> int8 [256,16] (edge triples, -1 after the last)."""
    text = open(path).read()
    body = text[text.index("kTriTable[256][kTableWidth] = {") :]
    body = body[body.index("{") + 1 : body.index("};")]
    rows = re.findall(r"\{([^{}]*)\}", body)
    tab = np.array([[int(v) for v in r.split(",") if v.strip()] for r in rows], dtype=np.int8)
    assert tab.shape == (256, 16), tab.shape
    return tab


def block_key(b: np.ndarray) -> np.ndarray:
    """[..., 3] int block coordinates -> uint64 keys."""
    b = b.astype(np.int64) + KEY_BIAS
    return (b[..., 2].astype(np.uint64) << np.uint64(42)) | (b[..., 1].astype(np.uint64) << np.uint64(21)) | b[..., 0].astype(np.uint64)


def key_blocks(keys: np.ndarray) -> np.ndarray:
    k = keys.astype(np.uint64)
    m = np.uint64((1 << 21) - 1)
    return np.stack([(k & m), (k >> np.uint64(21)) & m, (k >> np.uint64(42)) & m], -1).astype(np.int64) - KEY_BIAS


def allocate(points: np.ndarray, s: float, trunc: int) -> np.ndarray:
    """Sorted unique uint64 keys of the blocks the cubes [p - tau, p + tau] meet; ValueError when a voxel index does not fit."""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    tau = trunc * s
    lo, hi = np.floor((p - tau) / s), np.floor((p + tau) / s)
    if not (np.all(lo >= -VOXEL_LIMIT) and np.all(hi < VOXEL_LIMIT)):
        raise ValueError("a seed point's voxel index does not fit")
    lo, hi = lo.astype(np.int64) >> 3, hi.astype(np.int64) >> 3
    keys = [block_key(np.stack([np.where(c & 1, hi[:, 0], lo[:, 0]), np.where(c & 2, hi[:, 1], lo[:, 1]),
                                np.where(c & 4, hi[:, 2], lo[:, 2])], -1)) for c in range(8)]
    return np.unique(np.concatenate(keys)) if len(p) else np.zeros(0, np.uint64)


def voxel_coords(keys: np.ndarray) -> np.ndarray:
    """[n_blocks * 512, 3] int64 voxel indices in the volume's order (block, then x fastest)."""
    b = key_blocks(keys)
    v = np.arange(512)
    local = np.stack([v & 7, (v >> 3) & 7, v >> 6], -1)
    return (8 * b[:, None, :] + local[None]).reshape(-1, 3)


def integrate(keys, s: float, trunc: int, depths, images, Ks, Es):
    """-> (tsdf float32, weight float32, colour uint8 [.,3]) per voxel of the volume's order."""
    tau = trunc * s
    X = (voxel_coords(keys).astype(np.float64) + 0.5) * s
    n = np.zeros(len(X), np.int64)
    F = np.zeros(len(X))
    C = np.zeros((len(X), 3))
    for d, img, K, E in zip(depths, images, Ks, Es):
        d = np.asarray(d, np.float32)
        img = np.asarray(img, np.float32)
        K = np.asarray(K, np.float32).astype(np.float64)
        Rt = np.asarray(E, np.float32).astype(np.float64)[:3]
        H, W = d.shape
        xc = ((Rt[0, 0] * X[:, 0] + Rt[0, 1] * X[:, 1]) + Rt[0, 2] * X[:, 2]) + Rt[0, 3]
        yc = ((Rt[1, 0] * X[:, 0] + Rt[1, 1] * X[:, 1]) + Rt[1, 2] * X[:, 2]) + Rt[1, 3]
        zc = ((Rt[2, 0] * X[:, 0] + Rt[2, 1] * X[:, 1]) + Rt[2, 2] * X[:, 2]) + Rt[2, 3]
        front = zc > 0
        zs = np.where(front, zc, 1.0)
        with np.errstate(invalid="ignore", over="ignore"):
            u = ((K[0, 0] * xc + K[0, 1] * yc) + K[0, 2] * zc) / zs
            v = ((K[1, 0] * xc + K[1, 1] * yc) + K[1, 2] * zc) / zs
            fx, fy = np.floor(u + 0.5), np.floor(v + 0.5)
        ok = front & (fx >= 0) & (fx < W) & (fy >= 0) & (fy < H)
        px, py = np.where(ok, fx, 0).astype(np.int64), np.where(ok, fy, 0).astype(np.int64)
        dv = d[py, px].astype(np.float64)
        ok &= np.isfinite(dv) & (dv > 0)
        sdf = dv - zc
        ok &= ~(sdf < -tau)
        n += ok
        F += np.where(ok, np.minimum(1.0, sdf / tau), 0.0)
        C += np.where(ok[:, None], img[:, py, px].T.astype(np.float64), 0.0)
    nn = np.maximum(n, 1)
    tsdf = np.where(n > 0, F / nn, 1.0).astype(np.float32)
    colour = np.where(n[:, None] > 0, np.clip(np.rint(255.0 * (C / nn[:, None])), 0, 255), 0).astype(np.uint8)
    return tsdf, n.astype(np.float32), colour


def marching_cubes(keys, s: float, tsdf, weight, colour, min_weight: int = 1, table=None):
    """Marching cubes over a volume in the layout integrate returns (colour [.,3] or [.,4]) -> (positions float32 [nv,3],
    colours uint8 [nv,3], faces int32 [nf,3]) in the documented order."""
    tab = read_table() if table is None else table
    keys = np.asarray(keys, np.uint64)
    coords = voxel_coords(keys)
    tsdf = np.asarray(tsdf, np.float32)
    valid = np.asarray(weight) >= min_weight
    colour = np.asarray(colour)[:, :3]

    def lookup(c):
        """voxel indices of coordinates [m,3] -> global index or -1"""
        k = block_key(c >> 3)
        pos = np.searchsorted(keys, k)
        posc = np.minimum(pos, len(keys) - 1)
        hit = (pos < len(keys)) & (keys[posc] == k)
        local = (c[:, 0] & 7) + 8 * (c[:, 1] & 7) + 64 * (c[:, 2] & 7)
        return np.where(hit, posc * 512 + local, -1)

    G = len(coords)
    corner_idx = np.stack([lookup(coords + CORNERS[c]) for c in range(8)], -1)  # [G,8]
    corner_valid = (corner_idx >= 0) & valid[np.maximum(corner_idx, 0)]
    cube_ok = corner_valid.all(1)
    neg = tsdf[np.maximum(corner_idx, 0)] < 0
    case = (neg * (1 << np.arange(8))).sum(1)
    meshed = cube_ok & (case != 0) & (case != 255)
    meshed_ext = np.append(meshed, False)  # index -1 -> False

    # owned edges: (voxel, axis), sign change between two valid voxels, one of the four cubes meshed
    owned = np.zeros((G, 3), bool)
    other = np.zeros((G, 3), np.int64)
    for k in range(3):
        b = lookup(coords + UNIT[k])
        other[:, k] = b
        ok = valid & (b >= 0)
        ok &= valid[np.maximum(b, 0)]
        ok &= (tsdf < 0) != (tsdf[np.maximum(b, 0)] < 0)
        j, l = [a for a in range(3) if a != k]
        any_meshed = np.zeros(G, bool)
        for dj in (0, 1):
            for dl in (0, 1):
                any_meshed |= meshed_ext[lookup(coords - dj * UNIT[j] - dl * UNIT[l])]
        owned[:, k] = ok & any_meshed
    vid = np.full((G, 3), -1, np.int64)
    flat = owned.ravel()
    vid.ravel()[flat] = np.arange(int(flat.sum()))
    a_idx, axis = np.nonzero(owned)
    b_idx = other[a_idx, axis]
    Xa = (coords[a_idx].astype(np.float64) + 0.5) * s
    Xb = (coords[b_idx].astype(np.float64) + 0.5) * s
    ta, tb = tsdf[a_idx].astype(np.float64), tsdf[b_idx].astype(np.float64)
    t = ta / (ta - tb)
    pos = (Xa + t[:, None] * (Xb - Xa)).astype(np.float32)
    ca, cb = colour[a_idx].astype(np.float64), colour[b_idx].astype(np.float64)
    col = np.clip(np.rint(ca + t[:, None] * (cb - ca)), 0, 255).astype(np.uint8)

    cubes = np.nonzero(meshed)[0]
    rows = tab[case[cubes]].astype(np.int64)  # [m,16]
    faces = []
    per_cube = []
    for q in range(5):
        e = rows[:, 3 * q : 3 * q + 3]
        has = e[:, 0] >= 0
        ee = np.maximum(e, 0)
        vox = lookup((coords[cubes][:, None, :] + EDGE_OFFSET[ee]).reshape(-1, 3)).reshape(-1, 3)
        f = vid[vox, EDGE_AXIS[ee]]
        per_cube.append(np.where(has[:, None], f, -2))
    tri = np.stack(per_cube, 1).reshape(-1, 3)  # cube-major, then table order
    faces = tri[tri[:, 0] != -2]
    assert (faces >= 0).all(), "a meshed cube refers to an edge without a vertex"
    return pos, col, faces.astype(np.int32)


def mesh(points, depths, images, Ks, Es, s: float, trunc: int = 3, min_weight: int = 1):
    """Allocation, integration and marching cubes -> (positions, colours, faces, keys, (tsdf, weight, colour))."""
    keys = allocate(points, s, trunc)
    vol = integrate(keys, s, trunc, depths, images, Ks, Es)
    pos, col, faces = marching_cubes(keys, s, *vol, min_weight=min_weight)
    return pos, col, faces, keys, vol
