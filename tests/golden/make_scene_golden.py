"""Generate tests/golden/scene_io.npz: small scene inputs (cam files, a pair file, a JPEG and a PNG) and what the UNMODIFIED
reference's readers return for them -- read_cam_file, read_pair_file, read_image (datasets/data_io.py) -- plus the scaled
intrinsics, camera matrices and depth range its MVSDataset (datasets/mvs.py) builds for every request of a scene made of those
files.  The input files are stored as bytes next to the results, so the tests read exactly the files the reference read.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet):
    python tests/golden/make_scene_golden.py <path to the reference checkout>"""
import io
import os
import sys
import tempfile

import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "scene_io.npz")
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
sys.path.insert(0, os.path.abspath(sys.argv[1]))
from datasets import data_io as ref  # noqa: E402
from datasets.mvs import MVSDataset  # noqa: E402

rng = np.random.default_rng(20261015)


def cam_text(E, K, depth_line, trailing=""):
    rows = ["extrinsic"] + [" ".join(f"{v:.9g}" for v in r) for r in E] + ["", "intrinsic"]
    rows += [" ".join(f"{v:.9g}" for v in r) for r in K]
    if depth_line is not None:
        rows += ["", depth_line]
    return "\n".join(rows) + "\n" + trailing


def random_cam(i):
    a = 0.05 * i
    E = np.eye(4)
    E[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    E[:3, 3] = rng.uniform(-300, 300, 3)
    K = np.array([[rng.uniform(300, 3000), 0, rng.uniform(20, 40)], [0, rng.uniform(300, 3000), rng.uniform(15, 30)], [0, 0, 1]])
    return E, K


cams = {}
E, K = random_cam(0)
cams["cam_depth"] = cam_text(E, K, "425.123456 933.8")
E, K = random_cam(1)
cams["cam_nodepth"] = "\n".join(cam_text(E, K, None).split("\n")[:10]) + "\n"  # 10 lines: no line 11 / 12
E, K = random_cam(2)
text = cam_text(E, K, "4.25e+02 2.5E0 192 9.3380e2   ", trailing="\n  \n")  # exponents, trailing blanks and blank lines
text = text.replace("\n", "  \n", 3)  # trailing blanks on the first rows as well
cams["cam_exp_trailing"] = text.replace(f"{K[0][0]:.9g}", f"{K[0][0]:.6e}")
E, K = random_cam(3)
cams["cam_blank_depth_line"] = cam_text(E, K, None) + "\n\n"  # 12 lines, the 12th empty

pair = "5\n0\n3 1 10.5 2 3.25 3 1.0\n1\n0\n2\n4 0 1.0 1 2.0 3 0.5 4 0.25\n3\n2 2 7.0 0 1e3\n4\n1 3 2.0\n"


def smooth_image(h, w, c):
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([np.sin(x / (3.0 + k) + y / (5.0 + k)) for k in range(c)], axis=-1)
    return np.clip(127.5 + 90.0 * base + rng.normal(0, 20, (h, w, c)), 0, 255).astype(np.uint8)


def encode(arr, fmt):
    buf = io.BytesIO()
    Image.fromarray(arr).save(buf, format=fmt, **({"quality": 90} if fmt == "JPEG" else {}))
    return np.frombuffer(buf.getvalue(), dtype=np.uint8)


files = {k: np.frombuffer(v.encode("ascii"), dtype=np.uint8) for k, v in cams.items()}
files["pair"] = np.frombuffer(pair.encode("ascii"), dtype=np.uint8)
files["jpg"] = encode(smooth_image(48, 64, 3), "JPEG")
files["png"] = encode(smooth_image(30, 50, 3), "PNG")
MAX_DIMS = (-1, 100, 40)

expected = {}
with tempfile.TemporaryDirectory() as tmp:
    paths = {}
    for name, data in files.items():
        paths[name] = os.path.join(tmp, name + {"jpg": ".jpg", "png": ".png"}.get(name, ".txt"))
        with open(paths[name], "wb") as f:
            f.write(data.tobytes())
    for name in cams:
        k, e, d = ref.read_cam_file(paths[name])
        expected[f"{name}.intrinsics"], expected[f"{name}.extrinsics"], expected[f"{name}.depth_params"] = k, e, d
    pairs = ref.read_pair_file(paths["pair"])
    expected["pair.refs"] = np.array([r for r, _ in pairs], dtype=np.int64)
    expected["pair.srcs"] = np.array([len(s) for _, s in pairs], dtype=np.int64)
    expected["pair.flat"] = np.array([v for _, s in pairs for v in s], dtype=np.int64)
    for kind in ("jpg", "png"):
        for md in MAX_DIMS:
            img, oh, ow = ref.read_image(paths[kind], md)
            expected[f"{kind}.{md}.image"] = img
            expected[f"{kind}.{md}.original_hw"] = np.array([oh, ow], dtype=np.int64)

    # a scene: views 0..4 with the JPEG as every image, the cam files above (all with a depth range) and the pair file
    scene = os.path.join(tmp, "scene")
    os.makedirs(os.path.join(scene, "images"))
    os.makedirs(os.path.join(scene, "cams"))
    with open(os.path.join(scene, "pair.txt"), "w") as f:
        f.write(pair)
    scene_cams = []
    for v in range(5):
        E, K = random_cam(10 + v)
        t = cam_text(E, K, f"{400 + 10 * v} {900 + 5 * v}.5")
        scene_cams.append(np.frombuffer(t.encode("ascii"), dtype=np.uint8))
        with open(os.path.join(scene, "cams", f"{v:08d}_cam.txt"), "w") as f:
            f.write(t)
        with open(os.path.join(scene, "images", f"{v:08d}.jpg"), "wb") as f:
            f.write(files["jpg"].tobytes())
    for i, t in enumerate(scene_cams):
        files[f"scene_cam{i}"] = t
    for md in MAX_DIMS:
        ds = MVSDataset(scene, num_views=2, max_dim=md)
        for j in range(len(ds)):
            s = ds[j]
            expected[f"scene.{md}.{j}.intrinsics"] = s["intrinsics"]
            expected[f"scene.{md}.{j}.extrinsics"] = s["extrinsics"]
            expected[f"scene.{md}.{j}.depth_range"] = np.array([s["depth_min"], s["depth_max"]], dtype=np.float32)
            expected[f"scene.{md}.{j}.filename"] = np.array(s["filename"])

np.savez_compressed(OUT, **{"file." + k: v for k, v in files.items()}, **{"want." + k: v for k, v in expected.items()})
print("wrote", OUT, len(files), "files,", len(expected), "expected arrays")
