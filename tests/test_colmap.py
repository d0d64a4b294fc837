"""COLMAP interop without a GPU: the sparse-model readers, host math, the CPU oracle's scene files and colmap_output against
the reference's recorded results (tests/golden/colmap_io.npz, made by tests/golden/make_colmap_golden.py), error cases, the
command line, and the argument checks of the pm_colmap C ABI."""
import ctypes
import os

import numpy as np
import pytest

from oracle import colmap_oracle as co
from patchmatchnet_b200 import _native, colmap_input as ci, colmap_output as cout
from tests import colmap_cases as cc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "colmap_io.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def write_files(golden, root, prefix, sub_map):
    """Write the stored files whose key starts with `prefix` under root, mapping the first path part through sub_map."""
    for k, v in golden.items():
        if not k.startswith("file." + prefix):
            continue
        rel = k[len("file."):]
        head, _, rest = rel.partition("/")
        path = os.path.join(root, sub_map.get(head, head), rest)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        v.tofile(path)


def colmap_folder(golden, root, form=".bin"):
    os.makedirs(os.path.join(root, "sparse"), exist_ok=True)
    for name in ("cameras", "images", "points3D"):
        golden[f"file.sparse{form}/{name}"].tofile(os.path.join(root, "sparse", name + form))
    write_files(golden, root, "images/", {})
    return root


def want_text(golden, key):
    return golden["want." + key].tobytes()


# ---- readers ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("form", [".bin", ".txt"])
def test_readers_match_the_reference(golden, tmp_path, form):
    root = colmap_folder(golden, str(tmp_path), form)
    assert ci.model_ext(os.path.join(root, "sparse")) == form
    cams, ims, pts = ci.read_model(os.path.join(root, "sparse"))
    k = "want.read" + form
    assert list(cams) == golden[k + ".cam_ids"].tolist()
    assert [c.id for c in cams.values()] == list(cams)
    assert [c.model for c in cams.values()] == golden[k + ".cam_models"].tolist()
    assert [[c.width, c.height] for c in cams.values()] == golden[k + ".cam_wh"].tolist()
    assert np.array([v for c in cams.values() for v in c.params]).tobytes() == golden[k + ".cam_params"].tobytes()
    assert [im.id for im in ims] == golden[k + ".image_ids"].tolist()
    assert np.array([list(im.qvec) + list(im.tvec) for im in ims]).tobytes() == golden[k + ".image_qt"].tobytes()
    assert [im.camera_id for im in ims] == golden[k + ".image_cam"].tolist()
    assert [im.name for im in ims] == golden[k + ".image_names"].tolist()
    assert [im.point3d_ids.size for im in ims] == golden[k + ".image_nobs"].tolist()
    assert np.concatenate([im.point3d_ids for im in ims]).tolist() == golden[k + ".image_obs"].tolist()
    assert pts.ids.dtype == np.uint64 and pts.ids.tolist() == golden[k + ".point_ids"].tolist()
    assert pts.xyz.tobytes() == golden[k + ".point_xyz"].tobytes()
    assert pts.rgb.tolist() == golden[k + ".point_rgb"].tolist()
    assert pts.error.tobytes() == golden[k + ".point_error"].tobytes()
    assert int(pts.ids.min()) > 2 ** 32 and len(set(im.id for im in ims)) == len(ims)
    assert [im.id for im in ims] != sorted(im.id for im in ims)


def test_bin_is_preferred_over_txt(golden, tmp_path):
    colmap_folder(golden, str(tmp_path), ".txt")
    root = colmap_folder(golden, str(tmp_path), ".bin")
    assert ci.model_ext(os.path.join(root, "sparse")) == ".bin"


# ---- the scene files: oracle vs the reference's recorded command output --------------------------------------------------------

def oracle_scene(root, out, num_src=-1):
    cams, ims, pts = ci.read_model(os.path.join(root, "sparse"))
    sm = ci.prepare(cams, ims, pts)
    obs = [sm.obs_points[sm.obs_offsets[i]:sm.obs_offsets[i + 1]] for i in range(len(ims))]
    scores = co.view_scores(sm.centers, obs, sm.xyz)
    ranges = co.depth_ranges(sm.extrinsics, obs, sm.xyz)
    ci.write_scene(out, sm, ranges, ci.select_views(scores, num_src))
    return sm, scores, ranges


def test_oracle_scene_files_equal_the_references(golden, tmp_path):
    root = colmap_folder(golden, str(tmp_path / "in"))
    out = str(tmp_path / "out")
    sm, scores, _ = oracle_scene(root, out)
    n = len(sm.intrinsics)
    for i in range(n):
        with open(os.path.join(out, "cams", f"{i:08d}_cam.txt"), "rb") as f:
            assert f.read() == want_text(golden, f"input.cams/{i:08d}_cam.txt"), i
    with open(os.path.join(out, "pair.txt"), "rb") as f:
        assert f.read() == want_text(golden, "input.pair.txt")
    assert (np.count_nonzero(scores, axis=1) == n - 1).all()  # every pair shares a point: only the self entry is 0


def test_num_src_images_truncates_rows(golden, tmp_path):
    root = colmap_folder(golden, str(tmp_path / "in"))
    out = str(tmp_path / "out")
    oracle_scene(root, out, num_src=3)
    lines = open(os.path.join(out, "pair.txt")).read().split("\n")
    assert lines[0] == "12" and lines[2].split()[0] == "3" and len(lines[2].split()) == 7


def test_duplicates_count_in_obs_i_but_once_in_obs_j():
    xyz = np.array([[0.0, 0.0, 0.0], [1.0, 0.5, 0.0]])
    centers = np.array([[0.0, 0.0, -10.0], [1.5, 0.0, -10.0]])
    one = co.view_scores(centers, [[0, 1], [0, 1]], xyz)
    dup_i = co.view_scores(centers, [[0, 0, 1], [0, 1]], xyz)
    dup_j = co.view_scores(centers, [[0, 1], [0, 0, 1]], xyz)
    term0 = co.view_scores(centers, [[0], [0]], xyz)[0, 1]
    assert dup_i[0, 1] == pytest.approx(one[0, 1] + term0, rel=1e-15)
    assert dup_j[0, 1] == one[0, 1] and one[0, 0] == 0.0


def test_tie_order_is_descending_index():
    scores = np.array([[0.0, 1.0, 0.0, 1.0, 0.0], [1.0, 0, 0, 0, 0], [0, 0, 0, 0, 0], [1.0, 0, 0, 0, 0], [0, 0, 0, 0, 0]])
    assert [k for k, _ in ci.select_views(scores, -1)[0]] == [3, 1, 4, 2, 0]
    assert [k for k, _ in ci.select_views(scores, 2)[2]] == [4, 3]


# ---- host math ------------------------------------------------------------------------------------------------------------------

ALL_MODELS = {
    "SIMPLE_PINHOLE": [100.0, 30.0, 20.0], "PINHOLE": [100.0, 110.0, 30.0, 20.0], "SIMPLE_RADIAL": [100.0, 30.0, 20.0, 0.1],
    "SIMPLE_RADIAL_FISHEYE": [100.0, 30.0, 20.0, 0.1], "RADIAL": [100.0, 30.0, 20.0, 0.1, 0.2],
    "RADIAL_FISHEYE": [100.0, 30.0, 20.0, 0.1, 0.2], "OPENCV": [100.0, 110.0, 30.0, 20.0, 0.1, 0.2, 0.3, 0.4],
    "OPENCV_FISHEYE": [100.0, 110.0, 30.0, 20.0, 0.1, 0.2, 0.3, 0.4],
    "FULL_OPENCV": [100.0, 110.0, 30.0, 20.0] + [0.1] * 8, "FOV": [100.0, 110.0, 30.0, 20.0, 0.5],
    "THIN_PRISM_FISHEYE": [100.0, 110.0, 30.0, 20.0] + [0.1] * 8,
}


def test_intrinsics_of_all_models():
    assert set(ALL_MODELS) == set(ci.PARAM_TYPE) == {name for name, _ in ci.CAMERA_MODELS.values()}
    for model, params in ALL_MODELS.items():
        assert len(params) == dict(ci.CAMERA_MODELS.values())[model]
        k = ci.intrinsic_matrix(ci.Camera(1, model, 64, 48, params))
        fy = params[0] if len(ALL_MODELS[model]) in (3, 4, 5) and "fx" not in ci.PARAM_TYPE[model] else params[1]
        cx, cy = (params[1], params[2]) if "f" in ci.PARAM_TYPE[model] else (params[2], params[3])
        assert k.dtype == np.float64 and k.tolist() == [[params[0], 0, cx], [0, fy, cy], [0, 0, 1]], model
        assert ci.has_distortion(ci.Camera(1, model, 64, 48, params)) == (model not in ("SIMPLE_PINHOLE", "PINHOLE")), model
    assert not ci.has_distortion(ci.Camera(1, "OPENCV", 64, 48, [1.0, 1.0, 0.5, 0.5, 0.0, 0.0, 0.0, 0.0]))


def test_quaternion_to_rotation():
    r = ci.quaternion_to_rotation_matrix([np.cos(np.pi / 4), 0.0, 0.0, np.sin(np.pi / 4)])
    np.testing.assert_allclose(r, [[0, -1, 0], [1, 0, 0], [0, 0, 1]], atol=1e-15)
    rng = np.random.default_rng(0)
    for _ in range(20):
        q = rng.normal(size=4)
        q /= np.linalg.norm(q)
        r = ci.quaternion_to_rotation_matrix(list(q))
        np.testing.assert_allclose(r, cc.quaternion_matrix(q), atol=1e-15)
        np.testing.assert_allclose(r @ r.T, np.eye(3), atol=1e-14)
        np.testing.assert_allclose(cout.rotation_matrix_to_quaternion(r), q if q[0] >= 0 else -q, atol=1e-12)
    e = ci.extrinsic_matrix(ci.Image(1, [1.0, 0, 0, 0], [1.0, 2.0, 3.0], 1, "a", np.zeros(0, np.int64)))
    assert e.tolist() == [[1, 0, 0, 1], [0, 1, 0, 2], [0, 0, 1, 3], [0, 0, 0, 1]]
    assert ci.camera_center(e).tolist() == [-1.0, -2.0, -3.0]


# ---- errors -----------------------------------------------------------------------------------------------------------------

def small_model():
    return cc.make_model(0, 4, 30, track=3, n_invalid=1)


def test_missing_point_id_is_a_value_error(tmp_path):
    m = small_model()
    iid, q, t, cid, name, obs = m["images"][2]
    m["images"][2] = (iid, q, t, cid, name, np.append(obs, 999999))
    cc.write_txt(str(tmp_path), m)
    with pytest.raises(ValueError, match=r"image 2 \(img_0002.png\) observes point 999999"):
        ci.prepare(*ci.read_model(str(tmp_path)))


def test_image_without_observations_is_a_value_error(tmp_path):
    m = small_model()
    iid, q, t, cid, name, obs = m["images"][1]
    m["images"][1] = (iid, q, t, cid, name, np.array([-1, -1], dtype=np.int64))
    cc.write_bin(str(tmp_path), m)
    with pytest.raises(ValueError, match=r"image 1 \(img_0001.png\) has no valid observation"):
        ci.prepare(*ci.read_model(str(tmp_path)))


def test_missing_model(tmp_path):
    with pytest.raises(FileNotFoundError, match="no COLMAP model"):
        ci.read_model(str(tmp_path))
    (tmp_path / "cameras.bin").write_bytes(b"")
    with pytest.raises(FileNotFoundError):
        ci.read_model(str(tmp_path))


# ---- command line -------------------------------------------------------------------------------------------------------------

def test_input_parser_defaults_and_messages(tmp_path):
    a = ci.parse_args([])
    assert (a.input_folder, a.output_folder, a.num_src_images, a.theta0, a.sigma1, a.sigma2) == (None, "", -1, 5, 1, 10)
    assert not hasattr(a, "convert_format")
    with pytest.raises(Exception, match="^Invalid input folder$"):
        ci.check_args(ci.parse_args(["--input-folder", str(tmp_path / "nope")]))
    with pytest.raises(Exception, match="^Invalid output folder$"):
        ci.check_args(ci.parse_args(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path / "nope")]))
    a = ci.parse_args(["--input-folder", str(tmp_path)])
    ci.check_args(a)
    assert a.output_folder == str(tmp_path)


def test_input_without_cuda_raises_before_any_output(golden, tmp_path, monkeypatch):
    import torch

    root = colmap_folder(golden, str(tmp_path))
    before = sorted(os.listdir(root))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="needs a CUDA device"):
        ci.main(["--input-folder", root])
    assert sorted(os.listdir(root)) == before


def test_output_parser_defaults_and_messages(tmp_path):
    a = cout.parse_args([])
    assert (a.input_folder, a.results_folder, a.output_folder) == (None, "", "")
    with pytest.raises(Exception, match="^Invalid input folder$"):
        cout.check_args(cout.parse_args(["--input-folder", str(tmp_path / "nope")]))
    with pytest.raises(Exception, match="^Invalid results folder$"):
        cout.check_args(cout.parse_args(["--input-folder", str(tmp_path), "--results-folder", str(tmp_path / "nope")]))
    with pytest.raises(Exception, match="^Invalid output folder$"):
        cout.check_args(cout.parse_args(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path / "nope")]))


# ---- colmap_output against the reference's files ------------------------------------------------------------------------------

def _image_lines(text):
    """images.txt data lines -> {id: (fields without the quaternion, quaternion floats)}."""
    out = {}
    for line in text.split("\n"):
        if line and not line.startswith("#"):
            f = line.split()
            out[f[0]] = (f[5:], [float(v) for v in f[1:5]])
    return out


@pytest.mark.parametrize("fmt", [".pfm", ".bin"])
def test_colmap_output_matches_the_reference(golden, tmp_path, fmt):
    scene = str(tmp_path / "scene")
    write_files(golden, scene, "output" + fmt + "/", {})
    inner = os.path.join(scene, "output" + fmt)
    for sub in ("images", "cams"):
        os.makedirs(os.path.join(inner, sub))
    for i in range(12):
        want_cam = want_text(golden, f"input.cams/{i:08d}_cam.txt")
        with open(os.path.join(inner, "cams", f"{i:08d}_cam.txt"), "wb") as f:
            f.write(want_cam)
        golden[f"file.images/img_{i:04d}.png"].tofile(os.path.join(inner, "images", f"{i:08d}.jpg"))
    with open(os.path.join(inner, "pair.txt"), "wb") as f:
        f.write(want_text(golden, "input.pair.txt"))
    ws = str(tmp_path / "ws")
    os.makedirs(ws)
    assert cout.main(["--input-folder", inner, "--output-folder", ws]) == 0
    prefix = "want.output" + fmt + "."
    wanted = {k[len(prefix):]: v.tobytes() for k, v in golden.items() if k.startswith(prefix)}
    got_files = set()
    for root, _, names in os.walk(ws):
        for name in names:
            rel = os.path.relpath(os.path.join(root, name), ws)
            if not rel.startswith("images"):
                got_files.add(rel)
    assert got_files == set(wanted)
    for rel, want in wanted.items():
        got = open(os.path.join(ws, rel), "rb").read()
        if rel == os.path.join("sparse", "cameras.txt"):
            g, w = got.decode().split("\n"), want.decode().split("\n")
            assert g[:3] == w[:3] and set(g[3:]) == set(w[3:])
        elif rel == os.path.join("sparse", "images.txt"):
            g, w = _image_lines(got.decode()), _image_lines(want.decode())
            assert got.decode().split("\n")[:4] == want.decode().split("\n")[:4] and g.keys() == w.keys()
            for key in w:
                assert g[key][0] == w[key][0]
                np.testing.assert_allclose(g[key][1], w[key][1], rtol=0, atol=1e-12)
        else:
            assert got == want, rel
    for i in range(12):
        assert os.path.isfile(os.path.join(ws, "images", f"{i:08d}.jpg"))
    for sub in ("consistency_graphs", "normal_maps"):
        assert os.path.isdir(os.path.join(ws, "stereo", sub))


# ---- C ABI argument checks (no CUDA call is made) -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    _native.build_library()
    return _native.lib()


def test_colmap_abi_rejects_bad_arguments(lib):
    one = ctypes.c_void_p(16)  # never dereferenced: validation fails first
    assert lib.pmb200_view_scores_count(None, one, 4, 10, one, one, 1 << 20, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores_count(one, one, 0, 10, one, one, 1 << 20, None) == -1
    assert b"n_images" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores_count(one, one, 65536, 10, one, one, 1 << 20, None) == -1
    assert lib.pmb200_view_scores_count(one, one, 4, 1 << 31, one, one, 1 << 20, None) == -1
    assert b"n_obs" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores(one, 5, one, one, one, 4, 10, 1 << 31, 5.0, 1.0, 10.0, one, one, 1 << 20, None) == -1
    assert b"2^31" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores(one, 5, one, one, one, 4, 10, 3, 5.0, 0.0, 10.0, one, one, 1 << 20, None) == -1
    assert b"sigma" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores(one, 5, one, one, one, 4, 10, 3, float("nan"), 1.0, 10.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_view_scores(one, 5, one, one, None, 4, 10, 3, 5.0, 1.0, 10.0, one, one, 1 << 20, None) == -1
    assert lib.pmb200_view_scores(one, -1, one, one, one, 4, 10, 3, 5.0, 1.0, 10.0, one, one, 1 << 20, None) == -1
    assert b"n_points" in lib.pmb200_last_error()
    assert lib.pmb200_view_scores_workspace_bytes(4, 10, 1 << 31) == -1
    assert lib.pmb200_view_scores_workspace_bytes(70000, 10, 0) == -1
    assert lib.pmb200_depth_ranges(one, 5, one, one, None, 4, 10, one, one, 1 << 20, None) == -1
    assert b"null pointer" in lib.pmb200_last_error()
    assert lib.pmb200_depth_ranges(one, 5, one, one, one, 65536, 10, one, one, 1 << 20, None) == -1
    assert lib.pmb200_depth_ranges_workspace_bytes(4, -1) == -1
