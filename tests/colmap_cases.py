"""Seeded synthetic COLMAP sparse models, written in the .bin and .txt forms (test and benchmark infrastructure).

A model is a dict of arrays:
    cameras   [(camera_id, model_name, width, height, params)]
    images    [(image_id, qvec (4,), tvec (3,), camera_id, name, point3d_ids int64 [n2d])]   (file order; -1 = no 3D point)
    point_ids uint64 [P], xyz float64 [P,3], rgb uint8 [P,3], error float64 [P]
Cameras sit on a ring around the origin looking at it; points fill a ball in the middle; each point is observed by a run of
nearby cameras (its track)."""
from __future__ import annotations

import os
import struct
from typing import Dict, List

import numpy as np

MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4, "OPENCV_FISHEYE": 5, "FULL_OPENCV": 6,
             "FOV": 7, "SIMPLE_RADIAL_FISHEYE": 8, "RADIAL_FISHEYE": 9, "THIN_PRISM_FISHEYE": 10}


def look_at_quaternion(center: np.ndarray, target: np.ndarray) -> np.ndarray:
    """(qw, qx, qy, qz), qw >= 0, of the world -> camera rotation of a camera at `center` whose +z axis looks at `target`."""
    z = target - center
    z = z / np.linalg.norm(z)
    x = np.cross([0.0, 1.0, 0.0], z)
    x = x / np.linalg.norm(x)
    y = np.cross(z, x)
    r = np.stack([x, y, z])  # rows: camera axes in world coordinates
    return rotation_to_quaternion(r)


def rotation_to_quaternion(r: np.ndarray) -> np.ndarray:
    t = np.trace(r)
    if t > 0:
        s = 2.0 * np.sqrt(1.0 + t)
        q = [0.25 * s, (r[2, 1] - r[1, 2]) / s, (r[0, 2] - r[2, 0]) / s, (r[1, 0] - r[0, 1]) / s]
    else:
        i = int(np.argmax(np.diag(r)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = 2.0 * np.sqrt(1.0 + r[i, i] - r[j, j] - r[k, k])
        q = [0.0] * 4
        q[0] = (r[k, j] - r[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (r[j, i] + r[i, j]) / s
        q[1 + k] = (r[k, i] + r[i, k]) / s
    q = np.array(q)
    q = q / np.linalg.norm(q)
    return -q if q[0] < 0 else q


def make_model(seed: int, n_images: int, n_points: int, track: int = 5, n_invalid: int = 0, radius: float = 10.0,
               point_radius: float = 3.0, id_base: int = 1, cameras=None, image_ids=None, n_global: int = 0,
               arc: float = 2 * np.pi) -> Dict[str, object]:
    """Tracks of `track` cameras (consecutive on the ring, wrapping), 2D points in shuffled order plus `n_invalid` entries of -1
    per image.  The last `n_global` points are seen by every image.  `cameras`: a list of (id, model, w, h, params) assigned to
    the images in turn (default: one PINHOLE)."""
    rng = np.random.default_rng(seed)
    cameras = cameras or [(1, "PINHOLE", 640, 480, [500.0, 510.0, 320.0, 240.0])]
    ang = arc * np.arange(n_images) / n_images  # cameras spread over `arc` radians of the ring
    centers = np.stack([radius * np.cos(ang), 0.3 * radius * np.sin(3 * ang), radius * np.sin(ang)], axis=1)
    xyz = rng.normal(0, point_radius / 2, (n_points, 3))
    start = rng.integers(0, n_images, n_points)
    members = (start[:, None] + np.arange(min(track, n_images))[None, :]) % n_images  # [P, track]
    img_of = members.ravel()
    pt_of = np.repeat(np.arange(n_points), members.shape[1])
    if n_global:
        xyz = np.concatenate([xyz, rng.normal(0, point_radius / 2, (n_global, 3))])
        img_of = np.concatenate([img_of, np.tile(np.arange(n_images), n_global)])
        pt_of = np.concatenate([pt_of, np.repeat(np.arange(n_points, n_points + n_global), n_images)])
        n_points += n_global
    order = np.lexsort((rng.random(img_of.size), img_of))  # group by image, shuffled within
    img_sorted, pt_sorted = img_of[order], pt_of[order]
    bounds = np.searchsorted(img_sorted, np.arange(n_images + 1))
    point_ids = (np.uint64(id_base) + np.arange(n_points, dtype=np.uint64) * np.uint64(3)).astype(np.uint64)
    images = []
    ids = image_ids if image_ids is not None else list(range(1, n_images + 1))
    for i in range(n_images):
        c = centers[i]
        q = look_at_quaternion(c, np.zeros(3))
        r = quaternion_matrix(q)
        t = -r @ c
        obs = point_ids[pt_sorted[bounds[i]:bounds[i + 1]]].astype(np.int64)
        if n_invalid:
            obs = np.insert(obs, rng.integers(0, obs.size + 1, n_invalid), -1)
        cam = cameras[i % len(cameras)]
        images.append((int(ids[i]), q, t, cam[0], "img_%04d.png" % i, obs))
    return {"cameras": cameras, "images": images, "point_ids": point_ids, "xyz": xyz,
            "rgb": rng.integers(0, 256, (n_points, 3)).astype(np.uint8), "error": rng.uniform(0, 2, n_points)}


def quaternion_matrix(q) -> np.ndarray:
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _tracks(model) -> List[np.ndarray]:
    """Per point: (image_id, point2d_idx) int32 pairs, from the images' observation lists."""
    pid = model["point_ids"]
    order = np.argsort(pid)
    img_col, idx_col, pt_col = [], [], []
    for im in model["images"]:
        obs = im[5]
        valid = np.nonzero(obs != -1)[0]
        at = np.minimum(np.searchsorted(pid[order], obs[valid].astype(np.uint64)), pid.size - 1)
        known = pid[order][at] == obs[valid].astype(np.uint64)  # an ID missing from the points (a broken model) has no track
        valid, pos = valid[known], order[at[known]]
        img_col.append(np.full(valid.size, im[0], np.int64))
        idx_col.append(valid)
        pt_col.append(pos)
    img_col, idx_col, pt_col = (np.concatenate(a) if a else np.zeros(0, np.int64) for a in (img_col, idx_col, pt_col))
    srt = np.argsort(pt_col, kind="stable")
    bounds = np.searchsorted(pt_col[srt], np.arange(pid.size + 1))
    pairs = np.stack([img_col[srt], idx_col[srt]], axis=1).astype(np.int32)
    return [pairs[bounds[k]:bounds[k + 1]] for k in range(pid.size)], bounds


def write_bin(path: str, model) -> None:
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model["cameras"])))
        for cid, name, w, h, params in model["cameras"]:
            f.write(struct.pack("<iiQQ", cid, MODEL_IDS[name], w, h) + struct.pack("<%dd" % len(params), *params))
    rng = np.random.default_rng(1)
    with open(os.path.join(path, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model["images"])))
        for iid, q, t, cid, name, obs in model["images"]:
            f.write(struct.pack("<idddddddi", iid, *q, *t, cid) + name.encode() + b"\x00" + struct.pack("<Q", obs.size))
            rec = np.empty(obs.size, dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
            rec["x"], rec["y"], rec["id"] = rng.uniform(0, 640, obs.size), rng.uniform(0, 480, obs.size), obs
            f.write(rec.tobytes())
    tracks, bounds = _tracks(model)
    n = model["point_ids"].size
    lengths = np.diff(bounds)
    head = np.empty(n, dtype=np.dtype([("id", "<u8"), ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("r", "u1"), ("g", "u1"),
                                        ("b", "u1"), ("e", "<f8"), ("n", "<u8")]))
    head["id"] = model["point_ids"]
    head["x"], head["y"], head["z"] = model["xyz"].T
    head["r"], head["g"], head["b"] = model["rgb"].T
    head["e"], head["n"] = model["error"], lengths
    body = np.concatenate(tracks).view(np.uint8).ravel() if n else np.zeros(0, np.uint8)
    is_head = np.repeat(np.tile([True, False], n), np.stack([np.full(n, 51), 8 * lengths], axis=1).ravel())
    out = np.empty(is_head.size, dtype=np.uint8)
    out[is_head] = head.view(np.uint8).ravel()
    out[~is_head] = body
    with open(os.path.join(path, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", n))
        f.write(out.tobytes())


def write_txt(path: str, model) -> None:
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        for cid, name, w, h, params in model["cameras"]:
            f.write("%d %s %d %d %s\n" % (cid, name, w, h, " ".join(repr(float(p)) for p in params)))
    rng = np.random.default_rng(1)
    with open(os.path.join(path, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n")
        for iid, q, t, cid, name, obs in model["images"]:
            f.write("%d %s %s %d %s\n" % (iid, " ".join(repr(float(v)) for v in q), " ".join(repr(float(v)) for v in t), cid, name))
            f.write(" ".join("%r %r %d" % (float(x), float(y), p) for x, y, p in zip(rng.uniform(0, 640, obs.size), rng.uniform(0, 480, obs.size), obs)) + "\n")
    tracks, _ = _tracks(model)
    with open(os.path.join(path, "points3D.txt"), "w") as f:
        f.write("# 3D point list with one line of data per point:\n")
        for k in range(model["point_ids"].size):
            x, y, z = model["xyz"][k]
            r, g, b = model["rgb"][k]
            tr = " ".join("%d %d" % (a, c) for a, c in tracks[k])
            f.write("%d %r %r %r %d %d %d %r %s\n" % (int(model["point_ids"][k]), float(x), float(y), float(z), r, g, b, float(model["error"][k]), tr))


def write_images(folder: str, model, size=(8, 6)) -> None:
    """Tiny distinct PNG files under folder/images/<name> for every image of the model."""
    from PIL import Image

    os.makedirs(os.path.join(folder, "images"), exist_ok=True)
    for k, im in enumerate(model["images"]):
        arr = np.full((size[1], size[0], 3), k % 256, dtype=np.uint8)
        Image.fromarray(arr).save(os.path.join(folder, "images", im[4]))


def dense_obs(model) -> List[np.ndarray]:
    """Per image: dense point indices (into the model's point arrays) of its valid observations, in order."""
    pid = model["point_ids"]
    order = np.argsort(pid)
    out = []
    for im in model["images"]:
        obs = im[5][im[5] != -1].astype(np.uint64)
        out.append(order[np.searchsorted(pid[order], obs)])
    return out
