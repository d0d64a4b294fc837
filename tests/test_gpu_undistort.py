"""Undistortion on the GPU (csrc/pm_undistort.cu through ops) against tests/undistort_oracle.py: border extents, the
undistorted camera and the warp for every camera model, one full-size ETH3D DSLR image, and the colmap_input --undistort
command, down to the geometry of a reconstruction from distorted views.

The warp agrees with the oracle bit for bit, except for the models that use atan or tan, where CUDA's and libm's results
differ in the last bit: there at most 1e-5 of the pixels may differ, by 1."""
import os

import numpy as np
import pytest

from patchmatchnet_b200 import colmap_input as ci, data_io, ops, reconstruct
from tests import colmap_cases as cc, scene_cases
from tests import undistort_oracle as uo
from tests.test_gpu_colmap import WEIGHTS, _plane_model
from tests.test_undistort import ALL, IDS, H0, W0, camera

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scaled(model, params, W, H):
    """The parameters of a W0 x H0 case for a W x H camera (pinhole part scaled)."""
    p = list(params)
    sx, sy = W / W0, H / H0
    if model in uo.SINGLE_FOCAL:
        p[0:3] = [p[0] * sx, p[1] * sx, p[2] * sy]
    else:
        p[0:4] = [p[0] * sx, p[1] * sy, p[2] * sx, p[3] * sy]
    return p


def _gpu_warp(cam, pin, src):
    import torch

    return ops.undistort_image(torch.from_numpy(src).to(DEV), cam, pin).cpu().numpy()


def _compare(model, got, want):
    diff = np.abs(got.astype(np.int16) - want.astype(np.int16)).max(axis=2)
    if model in uo.USES_ATAN:
        assert diff.max() <= 1 and (diff > 0).sum() <= int(1e-5 * diff.size), ((diff > 0).sum(), diff.size)
    else:
        assert got.tobytes() == want.tobytes(), (diff > 0).sum()


def test_extents_and_cameras_match_the_oracle():
    cams = [camera(m, p, cam_id=k + 1) for k, (m, p) in enumerate(ALL)]
    got = ops.undistort_extents(cams, DEV).cpu().numpy()  # every case in one launch
    assert got.shape == (len(cams), 8)
    for k, (cam, name) in enumerate(zip(cams, IDS)):
        want = uo.extents(cam.model, cam.params, W0, H0)
        np.testing.assert_allclose(got[k], want, rtol=0, atol=1e-9, err_msg=name)
        for b in (0.0, 0.3, 1.0):
            pin = ops.undistorted_camera(cam, got[k], b)
            w, h, kp = uo.undistorted_camera(cam.model, cam.params, W0, H0, want, b)
            assert (pin.model, pin.width, pin.height) == ("PINHOLE", w, h), name
            np.testing.assert_allclose(pin.params, kp, rtol=1e-12, atol=0, err_msg=name)


@pytest.mark.parametrize("size", [(61, 47), (640, 480)])
@pytest.mark.parametrize("model,params", ALL, ids=IDS)
def test_warp_matches_the_oracle(model, params, size):
    W, H = size
    cam = camera(model, _scaled(model, params, W, H), W, H)
    src = np.random.default_rng(W + len(params)).integers(0, 256, (H, W, 3)).astype(np.uint8)
    for b in (0.0, 1.0):
        pin = ops.undistorted_camera(cam, ops.undistort_extents([cam], DEV)[0].cpu().numpy(), b)
        got = _gpu_warp(cam, pin, src)
        want = uo.undistort_image(model, cam.params, src, pin.params, pin.width, pin.height)
        _compare(model, got, want)
        assert (got > 0).any()


def test_eth3d_dslr_size_thin_prism_fisheye():
    W, H = 6048, 4032
    params = [3410.0, 3409.0, 3024.5, 2016.2, 0.0102, -0.0031, 0.0004, -0.0002, 0.0011, -0.0004, 0.0003, -0.0002]
    cam = camera("THIN_PRISM_FISHEYE", params, W, H)
    y, x = np.mgrid[0:H, 0:W]
    src = np.stack([(x * 7 + y * 3) % 256, (x // 5 + y * 11) % 256, (x * y) % 251], -1).astype(np.uint8)
    pin = ops.undistorted_camera(cam, ops.undistort_extents([cam], DEV)[0].cpu().numpy(), 0.0)
    w, h, kp = uo.undistorted_camera(cam.model, params, W, H, uo.extents(cam.model, params, W, H), 0.0)
    assert (pin.width, pin.height) == (w, h)
    np.testing.assert_allclose(pin.params, kp, rtol=1e-12, atol=0)
    _compare("THIN_PRISM_FISHEYE", _gpu_warp(cam, pin, src), uo.undistort_image(cam.model, params, src, pin.params, w, h))


# ---- the command ----------------------------------------------------------------------------------------------------------

W1, H1 = 96, 72
TWO_CAMERAS = [(1, "SIMPLE_RADIAL", W1, H1, [80.0, 48.5, 35.5, -0.08]),
               (2, "OPENCV", W1, H1, [82.0, 81.0, 47.0, 36.5, 0.05, -0.02, 0.001, -0.0015])]


def _write_model(root, cameras, n_images=6, seed=3, size=(W1, H1), mode="RGB", fmt="png"):
    from PIL import Image

    m = cc.make_model(seed, n_images, 300, track=4, cameras=cameras)
    m["images"] = [(iid, q, t, cid, name.replace(".png", "." + fmt), obs) for iid, q, t, cid, name, obs in m["images"]]
    cc.write_bin(os.path.join(root, "sparse"), m)
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    rng = np.random.default_rng(seed)
    for im in m["images"]:
        arr = rng.integers(0, 256, (size[1], size[0], 3)).astype(np.uint8)
        Image.fromarray(arr).convert(mode).save(os.path.join(root, "images", im[4]))
    return m


def _run(src, out, *extra):
    os.makedirs(out, exist_ok=True)
    assert ci.main(["--input-folder", src, "--output-folder", out, *extra]) == 0


def _files(root):
    out = {}
    for d, _, names in os.walk(root):
        for n in names:
            p = os.path.join(d, n)
            out[os.path.relpath(p, root)] = open(p, "rb").read()
    return out


def test_command_undistorts_a_two_camera_model(tmp_path):
    from PIL import Image

    src = str(tmp_path / "in")
    m = _write_model(src, TWO_CAMERAS)
    plain, und, again = (str(tmp_path / n) for n in ("plain", "und", "again"))
    _run(src, plain)
    _run(src, und, "--undistort")
    _run(src, again, "--undistort")
    assert _files(und) == _files(again)
    a, b = _files(plain), _files(und)
    assert a.keys() == b.keys() and a["pair.txt"] == b["pair.txt"]
    cams = {c[0]: ci.Camera(*c) for c in TWO_CAMERAS}
    pins = {c.id: ops.undistorted_camera(c, ops.undistort_extents([c], DEV)[0].cpu().numpy()) for c in cams.values()}
    for i, im in enumerate(m["images"]):
        cam, pin = cams[im[3]], pins[im[3]]
        name = f"cams/{i:08d}_cam.txt"
        lines_a, lines_b = a[name].decode().split("\n"), b[name].decode().split("\n")
        assert lines_a[:6] == lines_b[:6] and lines_a[-2:] == lines_b[-2:]  # extrinsics and the depth range
        k = [float(v) for v in " ".join(lines_b[7:10]).split()]
        assert k == [pin.params[0], 0.0, pin.params[2], 0.0, pin.params[1], pin.params[3], 0.0, 0.0, 1.0]
        with Image.open(os.path.join(und, "images", f"{i:08d}.jpg")) as f:
            assert f.format == "PNG"
            got = np.asarray(f)
        source = np.asarray(Image.open(os.path.join(src, "images", im[4])))
        assert got.tobytes() == _gpu_warp(cam, pin, source).tobytes()
        assert got.shape == (pin.height, pin.width, 3)


def test_command_writes_jpeg_for_jpeg_sources(tmp_path):
    from PIL import Image, JpegImagePlugin

    src = str(tmp_path / "in")
    _write_model(src, TWO_CAMERAS[:1], n_images=3, fmt="jpg")
    out = str(tmp_path / "out")
    _run(src, out, "--undistort")
    for i in range(3):
        with Image.open(os.path.join(out, "images", f"{i:08d}.jpg")) as f:
            assert f.format == "JPEG" and f.mode == "RGB"
            assert JpegImagePlugin.get_sampling(f) == 0  # 4:4:4: no chroma subsampling


def test_pinhole_model_is_unchanged_by_undistort(tmp_path):
    src = str(tmp_path / "in")
    _write_model(src, [(1, "PINHOLE", W1, H1, [80.0, 81.0, 48.0, 36.0]), (2, "SIMPLE_RADIAL", W1, H1, [80.0, 48.0, 36.0, 0.0])])
    plain, und = str(tmp_path / "plain"), str(tmp_path / "und")
    _run(src, plain)
    _run(src, und, "--undistort")
    assert _files(plain) == _files(und)


@pytest.mark.parametrize("case", ["size", "mode", "blank", "scale"])
def test_invalid_input_raises_before_any_output(tmp_path, case, monkeypatch):
    src = str(tmp_path / "in")
    if case == "size":
        _write_model(src, TWO_CAMERAS, size=(W1 + 1, H1))
        match = r"image 0 \(img_0000.png\) is 97 x 72, but its camera 1 is 96 x 72"
    elif case == "mode":
        _write_model(src, TWO_CAMERAS, mode="L")
        match = r"image 0 \(img_0000.png\) is L, not RGB"
    else:
        _write_model(src, TWO_CAMERAS)
        match = "blank-pixels" if case == "blank" else r"camera 1 \(SIMPLE_RADIAL\).*not finite"
    if case == "scale":  # every border point of camera 1 without a solution
        real = ops.undistort_extents
        monkeypatch.setattr(ops, "undistort_extents", lambda cams, dev: real(cams, dev).fill_(float("nan")))
    out = str(tmp_path / "out")
    os.makedirs(out)
    extra = ["--blank-pixels", "1.5"] if case == "blank" else []
    with pytest.raises(ValueError, match=match):
        ci.main(["--input-folder", src, "--output-folder", out, "--undistort", *extra])
    assert os.listdir(out) == []


# ---- geometry end to end --------------------------------------------------------------------------------------------------

DISTORTION = [-0.3, 0.05, 0.001, -0.0008]   # OPENCV k1, k2, p1, p2: up to 9 px at the corners
# median distance of the fused points to the plane, scene units (depth ~600); measured on an H100: 14.45 from the undistorted
# views, 15.85 from the distorted ones read as pinhole views
PLANE_BOUND = 15.0


def _render_distorted(model, params, E, H, W):
    """uint8 [H,W,3]: the plane's texture through a distorted camera, one ray per pixel centre (x + 0.5, y + 0.5) from
    the oracle's ImageToWorld, the colour function of scene_cases.texture."""
    xs, ys = np.meshgrid(np.arange(W) + 0.5, np.arange(H) + 0.5)
    u, v = uo.image_to_world(model, params, xs.ravel(), ys.ravel())
    rays = np.stack([u, v, np.ones_like(u)])
    R, t = E[:3, :3].astype(np.float64), E[:3, 3].astype(np.float64)
    n, d0 = scene_cases.PLANE_N, scene_cases.PLANE_D0
    z = (d0 + n @ (R.T @ t)) / (n @ (R.T @ rays))
    world = R.T @ (rays * z - t[:, None])
    x, y = world[0].reshape(H, W), world[1].reshape(H, W)
    chans = [np.sin(x / (2.1 + c)) * np.cos(y / (2.7 + 0.5 * c)) + 0.5 * np.sin((x + 2 * y) / 0.9 + c) for c in range(3)]
    return np.clip(127.5 + 80.0 * np.stack(chans, axis=-1), 0, 255).astype(np.uint8)


def test_reconstruction_from_distorted_views(tmp_path):
    from PIL import Image

    n_views, (H, W) = 6, (128, 160)
    model, cams = _plane_model(n_views, H, W, 3000, seed=4)
    colmap = tmp_path / "colmap"
    (colmap / "images").mkdir(parents=True)
    cameras = []
    for i, (k, e) in enumerate(cams):
        params = [float(k[0, 0]), float(k[1, 1]), float(k[0, 2]), float(k[1, 2])] + DISTORTION
        cameras.append((i + 1, "OPENCV", W, H, params))
        Image.fromarray(_render_distorted("OPENCV", params, e, H, W)).save(str(colmap / "images" / ("view_%02d.png" % i)))
    model["cameras"] = cameras
    cc.write_bin(str(colmap / "sparse"), model)
    median = {}
    for name, extra in (("und", ["--undistort"]), ("plain", [])):
        scene, results = tmp_path / ("scene_" + name), tmp_path / ("results_" + name)
        scene.mkdir()
        _run(str(colmap), str(scene), "--num-src-images", str(n_views - 2), *extra)
        reconstruct.reconstruct(reconstruct.parse_args([
            "--input-folder", str(scene), "--output-folder", str(results), "--checkpoint-path", WEIGHTS, "--num-views", "2",
            "--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]),
            log=lambda *a: None)
        pts = data_io.read_ply_points(str(results / "fused.ply")).astype(np.float64)
        assert len(pts) > 1000, (name, len(pts))
        median[name] = float(np.median(np.abs(pts @ scene_cases.PLANE_N - scene_cases.PLANE_D0)))
    print(f"median distance to the plane: undistorted {median['und']:.4f}, distorted {median['plain']:.4f}")
    assert median["und"] < PLANE_BOUND and median["und"] < median["plain"], median
