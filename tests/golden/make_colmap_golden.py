"""Generate tests/golden/colmap_io.npz: a small COLMAP sparse model (in the .bin and .txt forms), what the UNMODIFIED
reference's readers return for it, the cams/* and pair.txt its colmap_input.py writes from it, and what its colmap_output.py
writes for a scene folder with small depth / confidence maps in the .pfm and in the .bin form.  The input files are stored as
bytes next to the results, so the tests read exactly the files the reference read.

The model: 12 images in non-sorted ID order, cameras 1 / 3 / 7 (PINHOLE, SIMPLE_RADIAL, OPENCV), point IDs above 2^32 with
gaps, -1 entries, one duplicated observation, points seen by every image (every pair of views shares one, so only the view
itself scores 0), and every triangulation angle >= 0.5 degrees.  The generator checks that distinct scores of a row differ by
more than 1e-9 relative and that no printed %f value is within 1e-9 of a rounding boundary, so byte equality is a fair test.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet):
    python tests/golden/make_colmap_golden.py <path to the reference checkout>"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "colmap_io.npz")
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REPO)
sys.path.insert(1, REF)
import colmap_input as ref_in  # noqa: E402  (the reference's module: its command is under __main__)
from datasets import data_io as ref_io  # noqa: E402

from oracle import colmap_oracle as co  # noqa: E402
from patchmatchnet_b200 import colmap_input as ci  # noqa: E402
from tests import colmap_cases as cc  # noqa: E402

CAMERAS = [(1, "PINHOLE", 64, 48, [50.5, 51.25, 32.0, 24.0]), (3, "SIMPLE_RADIAL", 80, 60, [61.0, 40.0, 30.0, 0.0125]),
           (7, "OPENCV", 72, 54, [55.0, 56.5, 36.0, 27.0, 0.01, -0.002, 0.001, 0.0005])]
IMAGE_IDS = [5, 2, 9, 1, 12, 7, 3, 11, 4, 8, 10, 6]


def fixture(seed):
    m = cc.make_model(seed, 12, 150, track=4, n_invalid=2, id_base=2 ** 32 + 5, cameras=CAMERAS, image_ids=IMAGE_IDS, n_global=3,
                      arc=1.2)
    iid, q, t, cid, name, obs = m["images"][4]
    valid = obs[obs != -1]
    m["images"][4] = (iid, q, t, cid, name, np.insert(obs, 3, valid[-1]))  # one point listed twice in image 4
    return m


def fair(m):
    """The fixture's checks (see the module docstring)."""
    sm = ci.prepare(*model_of(m))
    obs = [sm.obs_points[sm.obs_offsets[i]:sm.obs_offsets[i + 1]] for i in range(len(m["images"]))]
    scores = co.view_scores(sm.centers, obs, sm.xyz)
    ranges = co.depth_ranges(sm.extrinsics, obs, sm.xyz)
    n = scores.shape[0]
    for i in range(n):
        for j in range(n):
            if i != j and not scores[i, j] > 0:
                return False
            x = np.asarray(sm.xyz[obs[i]])
            if i < j:
                a, b = sm.centers[i] - x, sm.centers[j] - x
                cos = (a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)
                shared = np.isin(obs[i], obs[j])
                if (np.degrees(np.arccos(np.clip(cos[shared], -1, 1))) < 0.5).any():
                    return False
        row = np.sort(scores[i])
        if (np.diff(row) <= 1e-9 * np.abs(row[1:])).any():
            return False
    values = list(scores.ravel()) + [v for r in ranges for v in r]
    frac = np.array([abs(v) * 1e6 % 1.0 for v in values])
    return not (np.abs(frac - 0.5) < 1e-3).any()


def model_of(m):
    with tempfile.TemporaryDirectory() as d:
        cc.write_bin(d, m)
        return ci.read_model(d)


seed = 1
while not fair(fixture(seed)):
    seed += 1
model = fixture(seed)
print("fixture seed", seed)

files, want = {}, {}
with tempfile.TemporaryDirectory() as tmp:
    scene = os.path.join(tmp, "colmap")
    cc.write_bin(os.path.join(scene, "sparse"), model)
    cc.write_txt(os.path.join(tmp, "txt"), model)
    cc.write_images(scene, model)
    for ext, d in ((".bin", os.path.join(scene, "sparse")), (".txt", os.path.join(tmp, "txt"))):
        for name in ("cameras", "images", "points3D"):
            files[f"sparse{ext}/{name}"] = np.fromfile(os.path.join(d, name + ext), dtype=np.uint8)
        cams, ims, pts = ref_in.read_model(d, ext)
        k = "read" + ext
        want[f"{k}.cam_ids"] = np.array(list(cams), dtype=np.int64)
        want[f"{k}.cam_models"] = np.array([c.model for c in cams.values()])
        want[f"{k}.cam_wh"] = np.array([[c.width, c.height] for c in cams.values()], dtype=np.int64)
        want[f"{k}.cam_params"] = np.array([v for c in cams.values() for v in c.params], dtype=np.float64)
        want[f"{k}.image_ids"] = np.array([im.id for im in ims], dtype=np.int64)
        want[f"{k}.image_qt"] = np.array([list(im.qvec) + list(im.tvec) for im in ims], dtype=np.float64)
        want[f"{k}.image_cam"] = np.array([im.camera_id for im in ims], dtype=np.int64)
        want[f"{k}.image_names"] = np.array([im.name for im in ims])
        want[f"{k}.image_nobs"] = np.array([len(im.point3d_ids) for im in ims], dtype=np.int64)
        want[f"{k}.image_obs"] = np.array([p for im in ims for p in im.point3d_ids], dtype=np.int64)
        want[f"{k}.point_ids"] = np.array(list(pts), dtype=np.uint64)
        want[f"{k}.point_xyz"] = np.array([p.xyz for p in pts.values()], dtype=np.float64)
        want[f"{k}.point_rgb"] = np.array([p.rgb for p in pts.values()], dtype=np.int64)
        want[f"{k}.point_error"] = np.array([p.error for p in pts.values()], dtype=np.float64)
    for im in model["images"]:
        files["images/" + im[4]] = np.fromfile(os.path.join(scene, "images", im[4]), dtype=np.uint8)

    # the reference's command, unmodified, on the .bin model
    subprocess.run([sys.executable, os.path.join(REF, "colmap_input.py"), "--input_folder", scene], check=True, cwd=REF,
                   stdout=subprocess.DEVNULL)
    for i in range(len(model["images"])):
        want[f"input.cams/{i:08d}_cam.txt"] = np.fromfile(os.path.join(scene, "cams", f"{i:08d}_cam.txt"), dtype=np.uint8)
    want["input.pair.txt"] = np.fromfile(os.path.join(scene, "pair.txt"), dtype=np.uint8)

    # colmap_output.py on a scene folder made of that output (cams, pair.txt, images/%08d.jpg) plus small maps
    rng = np.random.default_rng(seed)
    n = len(model["images"])
    for fmt in (".pfm", ".bin"):
        src = os.path.join(tmp, "out_scene" + fmt)
        os.makedirs(os.path.join(src, "images"))
        os.makedirs(os.path.join(src, "cams"))
        os.makedirs(os.path.join(src, "depth_est"))
        os.makedirs(os.path.join(src, "confidence"))
        for i in range(n):
            for sub, name in (("images", f"{i:08d}.jpg"), ("cams", f"{i:08d}_cam.txt")):
                with open(os.path.join(scene, sub, name), "rb") as a, open(os.path.join(src, sub, name), "wb") as b:
                    b.write(a.read())
            h, w = 6 + i % 3, 8
            ref_io.save_map(os.path.join(src, "depth_est", f"{i:08d}{fmt}"), rng.uniform(400, 900, (h, w)).astype(np.float32))
            ref_io.save_map(os.path.join(src, "confidence", f"{i:08d}{fmt}"), rng.uniform(0, 1, (h, w)).astype(np.float32))
        with open(os.path.join(scene, "pair.txt"), "rb") as a, open(os.path.join(src, "pair.txt"), "wb") as b:
            b.write(a.read())
        for sub in ("depth_est", "confidence"):
            for name in sorted(os.listdir(os.path.join(src, sub))):
                files[f"output{fmt}/{sub}/{name}"] = np.fromfile(os.path.join(src, sub, name), dtype=np.uint8)
        ws = os.path.join(tmp, "ws" + fmt)
        os.makedirs(ws)
        subprocess.run([sys.executable, os.path.join(REF, "colmap_output.py"), "--input_folder", src, "--output_folder", ws],
                       check=True, cwd=REF, stdout=subprocess.DEVNULL)
        for root, _, names in os.walk(ws):
            for name in names:
                rel = os.path.relpath(os.path.join(root, name), ws)
                if not rel.startswith("images"):
                    want[f"output{fmt}.{rel}"] = np.fromfile(os.path.join(root, name), dtype=np.uint8)

np.savez_compressed(OUT, **{"file." + k: v for k, v in files.items()}, **{"want." + k: v for k, v in want.items()})
print("wrote", OUT, len(files), "files,", len(want), "expected arrays")
