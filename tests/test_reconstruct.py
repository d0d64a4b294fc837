"""Scene input readers and the reconstruct command's host side (no GPU).

The readers (data_io.read_cam_file, read_pair_file, read_image, scale_intrinsics) reproduce tests/golden/scene_io.npz bit for
bit: the reference's own readers and its MVSDataset on the stored input files (written by tests/golden/make_scene_golden.py)."""
import os
import re

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import data_io, reconstruct
from tests import scene_cases

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scene_io.npz")
MAX_DIMS = (-1, 100, 40)


@pytest.fixture(scope="module")
def golden():
    z = np.load(GOLDEN)
    return {k: z[k] for k in z.files}


@pytest.fixture()
def files(golden, tmp_path):
    out = {}
    for key, data in golden.items():
        if key.startswith("file."):
            name = key[5:]
            out[name] = str(tmp_path / (name + {"jpg": ".jpg", "png": ".png"}.get(name, ".txt")))
            with open(out[name], "wb") as f:
                f.write(data.tobytes())
    return out


def _same(got, want):
    got = np.asarray(got)
    return got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want)


def test_read_cam_file_matches_the_reference(golden, files):
    names = [k[5:] for k in golden if k.startswith("file.cam_")]
    assert len(names) == 4
    for name in names:
        k, e, d = data_io.read_cam_file(files[name])
        assert _same(k, golden[f"want.{name}.intrinsics"]) and _same(e, golden[f"want.{name}.extrinsics"]), name
        assert _same(d, golden[f"want.{name}.depth_params"]), name
    assert golden["want.cam_nodepth.depth_params"].dtype == np.float64 and golden["want.cam_nodepth.depth_params"].size == 0
    assert golden["want.cam_exp_trailing.depth_params"].size == 4


def test_read_pair_file_matches_the_reference(golden, files):
    pairs = data_io.read_pair_file(files["pair"])
    assert [r for r, _ in pairs] == golden["want.pair.refs"].tolist()  # the zero-source entry (view 1) is dropped
    assert [len(s) for _, s in pairs] == golden["want.pair.srcs"].tolist()
    assert [v for _, s in pairs for v in s] == golden["want.pair.flat"].tolist()
    assert 1 not in [r for r, _ in pairs]


@pytest.mark.parametrize("kind", ["jpg", "png"])
@pytest.mark.parametrize("max_dim", MAX_DIMS)
def test_read_image_matches_the_reference(golden, files, kind, max_dim):
    img, h, w = data_io.read_image(files[kind], max_dim)
    assert _same(img, golden[f"want.{kind}.{max_dim}.image"])
    assert [h, w] == golden[f"want.{kind}.{max_dim}.original_hw"].tolist()
    if max_dim == 40:
        assert max(img.shape[:2]) < max(h, w)  # the cv2.resize branch


@pytest.mark.parametrize("max_dim", MAX_DIMS)
def test_scene_requests_and_scaled_intrinsics_match_the_reference_dataset(golden, files, tmp_path, max_dim):
    """MVSDataset(num_views=2, max_dim) on a scene of these files: request order, views, scaled intrinsics, depth range."""
    scene = tmp_path / "scene"
    (scene / "images").mkdir(parents=True)
    (scene / "cams").mkdir()
    (scene / "pair.txt").write_bytes(golden["file.pair"].tobytes())
    for v in range(5):
        (scene / "images" / f"{v:08d}.jpg").write_bytes(golden["file.jpg"].tobytes())
        (scene / "cams" / f"{v:08d}_cam.txt").write_bytes(golden[f"file.scene_cam{v}"].tobytes())
    requests = reconstruct.scan_requests(data_io.read_pair_file(str(scene / "pair.txt")), 2)
    assert len(requests) == sum(1 for k in golden if k.startswith(f"want.scene.{max_dim}.") and k.endswith(".intrinsics"))
    for j, views in enumerate(requests):
        ks, es = [], []
        for v in views:
            img, oh, ow = data_io.read_image(str(scene / "images" / f"{v:08d}.jpg"), max_dim)
            k, e, d = data_io.read_cam_file(str(scene / "cams" / f"{v:08d}_cam.txt"))
            ks.append(data_io.scale_intrinsics(k, img.shape[:2], oh, ow))
            es.append(e)
            if v == views[0]:
                assert _same(d[:2], golden[f"want.scene.{max_dim}.{j}.depth_range"])
        assert _same(np.stack(ks), golden[f"want.scene.{max_dim}.{j}.intrinsics"]), j
        assert _same(np.stack(es), golden[f"want.scene.{max_dim}.{j}.extrinsics"]), j
        assert str(golden[f"want.scene.{max_dim}.{j}.filename"]) == "{}/%08d{}" % views[0]


def test_scale_intrinsics_returns_a_scaled_float32_copy():
    k = np.array([[1000.0, 0, 320], [0, 1000, 256], [0, 0, 1]], dtype=np.float32)
    s = data_io.scale_intrinsics(k, (256, 320), 512, 640)
    assert s.dtype == np.float32 and s is not k and k[0, 0] == 1000.0
    assert s[0].tolist() == [500.0, 0.0, 160.0] and s[1].tolist() == [0.0, 500.0, 128.0] and s[2].tolist() == [0, 0, 1]


def test_save_image_semantics(tmp_path):
    from PIL import Image

    mask = np.array([[True, False], [False, True]])
    data_io.save_image(str(tmp_path / "m.png"), mask)
    assert np.array(Image.open(tmp_path / "m.png")).tolist() == [[255, 0], [0, 255]]
    data_io.save_image(str(tmp_path / "f.png"), np.array([[0.0, 0.5], [0.999, 1.0]], dtype=np.float32))
    assert np.array(Image.open(tmp_path / "f.png")).tolist() == [[0, 127], [254, 255]]


def test_parser_defaults_are_eval_py_defaults():
    a = reconstruct.parse_args([])
    assert (a.input_folder, a.output_folder, a.checkpoint_path) == (None, "", None)
    assert (a.file_format, a.input_type, a.output_type) == (".pfm", "params", "both")
    assert (a.num_views, a.image_max_dim, a.scan_list) == (20, -1, "")
    assert a.patchmatch_interval_scale == [0.005, 0.0125, 0.025] and a.patchmatch_range == [6, 4, 2]
    assert a.patchmatch_iteration == [1, 2, 2] and a.patchmatch_num_sample == [8, 8, 16]
    assert a.propagate_neighbors == [0, 8, 16] and a.evaluate_neighbors == [9, 9, 9]
    assert (a.geo_pixel_thres, a.geo_depth_thres, a.geo_mask_thres, a.photo_thres) == (1.0, 0.01, 5, 0.5)
    assert (a.seed, a.tf32) == (0, False)
    for dropped in ("--batch-size", "--display", "--num-light-idx", "--batch_size", "--num_light_idx"):
        with pytest.raises(SystemExit):
            reconstruct.parse_args([dropped, "1"])


def test_invalid_arguments_raise_eval_py_messages(tmp_path):
    ckpt = tmp_path / "w.pt"
    ckpt.write_bytes(b"x")
    missing = str(tmp_path / "nowhere")
    with pytest.raises(Exception, match=re.escape(f"Invalid input folder: {missing}")):
        reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", missing, "--checkpoint-path", str(ckpt)]))
    with pytest.raises(Exception, match=re.escape("Invalid input folder: None")):
        reconstruct.reconstruct(reconstruct.parse_args(["--checkpoint-path", str(ckpt)]))
    with pytest.raises(Exception, match=re.escape("Invalid checkpoint file: None")):
        reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", str(tmp_path)]))
    bad = str(tmp_path / "scans.txt")
    with pytest.raises(Exception, match=re.escape(f"Invalid scan list file: {bad}")):
        reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", str(tmp_path), "--checkpoint-path", str(ckpt),
                                                        "--scan-list", bad]))


def test_scene_enumeration(tmp_path):
    root = tmp_path / "data"
    pairs_a = [(0, [1, 2, 3, 4]), (2, [3, 0]), (1, [0, 4, 2])]
    pairs_b = [(3, [2]), (0, [1, 2, 3])]
    for scan, pairs in (("scan1", pairs_a), ("scan4", pairs_b)):
        (root / scan).mkdir(parents=True)
        (root / scan / "pair.txt").write_text(scene_cases.pair_text(pairs))
    (tmp_path / "list.txt").write_text("scan4\nscan1\n")
    assert reconstruct.list_scans("") == [""]
    scans = reconstruct.list_scans(str(tmp_path / "list.txt"))
    assert scans == ["scan4", "scan1"]
    pairs = data_io.read_pair_file(str(root / "scan1" / "pair.txt"))
    assert pairs == pairs_a
    assert reconstruct.scan_requests(pairs, 2) == [[0, 1, 2], [2, 3, 0], [1, 0, 4]]
    assert reconstruct.scan_requests(pairs, 20) == [[0, 1, 2, 3, 4], [2, 3, 0], [1, 0, 4, 2]]
    assert reconstruct.scan_views(pairs, 1, fusion=False) == [0, 1, 2, 3]  # view 4 only appears beyond the cut
    assert reconstruct.scan_views(pairs, 1, fusion=True) == [0, 1, 2, 3, 4]  # the filter takes every listed source
    assert reconstruct.scan_requests(data_io.read_pair_file(str(root / "scan4" / "pair.txt")), 2) == [[3, 2], [0, 1, 2]]


def test_no_cuda_raises_before_any_output(tmp_path, monkeypatch):
    scene = tmp_path / "scene"
    scene_cases.write_scene(str(scene), 3, 16, 24, 2)
    ckpt = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
    out = tmp_path / "out"
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    before = sorted(p for p in scene.rglob("*"))
    with pytest.raises(RuntimeError, match="CUDA"):
        reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", str(scene), "--output-folder", str(out),
                                                        "--checkpoint-path", ckpt]))
    assert not out.exists()
    with pytest.raises(RuntimeError, match="CUDA"):  # output folder defaulting to the input folder: nothing added there
        reconstruct.reconstruct(reconstruct.parse_args(["--input-folder", str(scene), "--checkpoint-path", ckpt]))
    assert sorted(p for p in scene.rglob("*")) == before
