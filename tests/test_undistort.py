"""Undistortion on the CPU: the camera models and the warp of csrc/pm_camera_math.cuh (built for the host from
tests/host_camera.cpp) against tests/undistort_oracle.py and against OpenCV, the scale of ops.undistorted_camera on a case
worked by hand, the C ABI's argument checks, and the --undistort options of colmap_input."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from patchmatchnet_b200 import _native, colmap_input as ci, ops
from tests import undistort_oracle as uo

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p
MODEL_ID = {name: k for k, (name, _) in ci.CAMERA_MODELS.items()}

# (model, mild parameters, strong parameters) of 640 x 480 cameras; FOV also has a case in its small-omega branch
CASES = [
    ("SIMPLE_PINHOLE", [500.0, 320.0, 240.0], [800.0, 300.5, 250.25]),
    ("PINHOLE", [500.0, 510.0, 320.0, 240.0], [450.0, 520.0, 330.0, 235.0]),
    ("SIMPLE_RADIAL", [500.0, 320.0, 240.0, 0.05], [450.0, 318.0, 242.0, -0.12]),
    ("RADIAL", [500.0, 320.0, 240.0, 0.03, -0.01], [450.0, 321.0, 238.0, -0.3, 0.1]),
    ("OPENCV", [500.0, 505.0, 320.0, 240.0, 0.02, -0.01, 0.001, -0.0005], [450.0, 455.0, 322.0, 237.0, -0.28, 0.07, 0.002, -0.001]),
    ("OPENCV_FISHEYE", [500.0, 505.0, 320.0, 240.0, 0.01, -0.005, 0.001, -0.0002], [400.0, 402.0, 318.0, 243.0, 0.1, -0.05, 0.02, -0.005]),
    ("FULL_OPENCV", [500.0, 505.0, 320.0, 240.0, 0.02, -0.01, 0.001, -0.0005, 0.001, 0.01, -0.005, 0.001],
     [450.0, 455.0, 322.0, 237.0, -0.15, 0.03, 0.002, -0.001, -0.002, 0.05, -0.01, 0.002]),
    ("FOV", [500.0, 505.0, 320.0, 240.0, 0.3], [400.0, 405.0, 321.0, 239.0, 1.0]),
    ("FOV", [500.0, 505.0, 320.0, 240.0, 0.005], [500.0, 505.0, 320.0, 240.0, 0.009]),
    ("SIMPLE_RADIAL_FISHEYE", [500.0, 320.0, 240.0, 0.02], [420.0, 322.0, 238.0, -0.1]),
    ("RADIAL_FISHEYE", [500.0, 320.0, 240.0, 0.02, -0.005], [420.0, 322.0, 238.0, -0.1, 0.02]),
    ("THIN_PRISM_FISHEYE", [500.0, 505.0, 320.0, 240.0, 0.01, -0.005, 0.0005, -0.0003, 0.001, -0.0005, 0.0008, -0.0006],
     [420.0, 425.0, 318.0, 243.0, 0.08, -0.03, 0.002, -0.001, 0.01, -0.002, 0.003, -0.002]),
]
ALL = [(m, p) for m, a, b in CASES for p in (a, b)]
IDS = [f"{m}-{'mild' if k % 2 == 0 else 'strong'}{'-small' if m == 'FOV' and p[4] < 0.01 else ''}" for k, (m, p) in enumerate(ALL)]
W0, H0 = 640, 480


def camera(model, params, W=W0, H=H0, cam_id=1):
    return ci.Camera(cam_id, model, W, H, list(params))


def _p(a):
    return a.ctypes.data_as(P)


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


@pytest.fixture(scope="module")
def hostcam(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostcam") / "_hostcam.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_camera.cpp")], check=True)
    lib = ctypes.CDLL(out)
    for name in ("hc_world_to_image", "hc_image_to_world"):
        getattr(lib, name).argtypes = [ctypes.c_int, P, ctypes.c_longlong, P, P, P, P]
    lib.hc_border_points.argtypes = [ctypes.c_int, P, ctypes.c_int, ctypes.c_int, P, P]
    lib.hc_undistort_image.argtypes = [ctypes.c_int, P, ctypes.c_int, ctypes.c_int, P, P, ctypes.c_int, ctypes.c_int, P]
    return lib


def _host_map(lib, name, model, params, a, b):
    p = _d(list(params) + [0.0] * (12 - len(params)))
    a, b = _d(a).ravel(), _d(b).ravel()
    x, y = np.empty_like(a), np.empty_like(a)
    getattr(lib, name)(MODEL_ID[model], _p(p), a.size, _p(a), _p(b), _p(x), _p(y))
    return x, y


def host_undistort(lib, model, params, src, kp, out_w, out_h):
    p = _d(list(params) + [0.0] * (12 - len(params)))
    src = np.ascontiguousarray(src, dtype=np.uint8)
    out = np.empty((out_h, out_w, 3), np.uint8)
    lib.hc_undistort_image(MODEL_ID[model], _p(p), src.shape[1], src.shape[0], _p(src), _p(_d(kp)), out_w, out_h, _p(out))
    return out


def _normalised_grid(params, model, n=41, margin=1.0):
    """Normalised points whose pinhole projections cover the image and a margin around it."""
    fx, fy, cx, cy = uo.pinhole_part(model, params)
    xs, ys = np.meshgrid(np.linspace(-margin * 0.1 * W0, W0 * (1 + 0.1 * margin), n), np.linspace(-0.1 * H0, 1.1 * H0, n))
    return (xs.ravel() - cx) / fx, (ys.ravel() - cy) / fy


def test_model_table_matches_colmap_input():
    assert {m for m, _, _ in CASES} == set(ci.PARAM_TYPE)
    for m, a, b in CASES:
        assert len(a) == len(b) == len(ci.PARAM_TYPE[m])


@pytest.mark.parametrize("model,params", ALL, ids=IDS)
def test_world_to_image_matches_the_oracle(hostcam, model, params):
    u, v = _normalised_grid(params, model)
    u = np.concatenate([u, [0.0, 1e-17, -3e-9]])
    v = np.concatenate([v, [0.0, 0.0, 2e-9]])
    got = _host_map(hostcam, "hc_world_to_image", model, params, u, v)
    want = uo.world_to_image(model, params, u, v)
    for g, w in zip(got, want):
        np.testing.assert_allclose(g, w, rtol=1e-12, atol=0)
        assert (g == w).all()  # the same operations in the same order


def _project_cv2(K, dist, u, v):
    import cv2

    pts = np.stack([u, v, np.ones_like(u)], 1).reshape(-1, 1, 3)
    out, _ = cv2.projectPoints(pts, np.zeros(3), np.zeros(3), K, np.asarray(dist, dtype=np.float64))
    return out.reshape(-1, 2)


@pytest.mark.parametrize("which", [0, 1])
def test_opencv_models_agree_with_opencv(hostcam, which):
    import cv2

    for model, dist_of in (("OPENCV", lambda p: p[4:8]), ("FULL_OPENCV", lambda p: p[4:12])):
        params = [c for c in CASES if c[0] == model][0][1 + which]
        K = np.array([[params[0], 0, params[2]], [0, params[1], params[3]], [0, 0, 1.0]])
        u, v = _normalised_grid(params, model, n=21)
        got = np.stack(_host_map(hostcam, "hc_world_to_image", model, params, u, v), 1)
        np.testing.assert_allclose(got, _project_cv2(K, dist_of(params), u, v), rtol=0, atol=1e-9)
    params = [c for c in CASES if c[0] == "OPENCV_FISHEYE"][0][1 + which]
    K = np.array([[params[0], 0, params[2]], [0, params[1], params[3]], [0, 0, 1.0]])
    u, v = _normalised_grid(params, "OPENCV_FISHEYE", n=21)
    want = cv2.fisheye.distortPoints(np.stack([u, v], 1).reshape(-1, 1, 2), K, np.asarray(params[4:8])).reshape(-1, 2)
    got = np.stack(_host_map(hostcam, "hc_world_to_image", "OPENCV_FISHEYE", params, u, v), 1)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-9)


@pytest.mark.parametrize("model,params", ALL, ids=IDS)
def test_image_to_world_round_trip(hostcam, model, params):
    xs, ys = np.meshgrid(np.linspace(0.0, W0, 33), np.linspace(0.0, H0, 25))
    xs, ys = np.append(xs.ravel(), uo.pinhole_part(model, params)[2]), np.append(ys.ravel(), uo.pinhole_part(model, params)[3])
    u, v = _host_map(hostcam, "hc_image_to_world", model, params, xs, ys)
    assert np.isfinite(u).all() and np.isfinite(v).all()
    x, y = _host_map(hostcam, "hc_world_to_image", model, params, u, v)
    assert np.abs(x - xs).max() < 1e-9 and np.abs(y - ys).max() < 1e-9
    ou, ov = uo.image_to_world(model, params, xs, ys)
    np.testing.assert_allclose(u, ou, rtol=0, atol=1e-12)
    np.testing.assert_allclose(v, ov, rtol=0, atol=1e-12)


@pytest.mark.parametrize("model,params", ALL, ids=IDS)
def test_border_points_match_the_oracle(hostcam, model, params):
    W, H = 61, 47
    p = _d(list(params) + [0.0] * (12 - len(params)))
    n = 2 * H + 2 * W
    mapped, side = np.empty(n), np.empty(n, np.int32)
    hostcam.hc_border_points(MODEL_ID[model], _p(p), W, H, _p(mapped), _p(side))
    px, py, want_side = uo.border_points(W, H)
    fx, fy, cx, cy = uo.pinhole_part(model, params)
    u, v = uo.image_to_world(model, params, px, py)
    assert (side == want_side).all()
    np.testing.assert_allclose(mapped, np.where(want_side < 2, fx * u + cx, fy * v + cy), rtol=0, atol=1e-9)


def _image(seed, H, W):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (H, W, 3)).astype(np.uint8)


@pytest.mark.parametrize("model,params", ALL, ids=IDS)
def test_undistort_pixel_matches_the_oracle_bit_for_bit(hostcam, model, params):
    # odd sizes; the camera scaled to them, the target pinhole a little wider and shifted so that some pixels fall outside
    for (W, H), seed in (((61, 47), 0), ((33, 21), 1)):
        p = list(params)
        s = W / W0
        fx, fy, cx, cy = uo.pinhole_part(model, p)
        if model in uo.SINGLE_FOCAL:
            p[0:3] = [fx * s, cx * s, cy * s]
        else:
            p[0:4] = [fx * s, fy * s, cx * s, cy * s]
        src = _image(seed, H, W)
        fx, fy, cx, cy = uo.pinhole_part(model, p)
        for kp, ow, oh in (([fx, fy, cx, cy], W, H), ([fx * 0.9, fy * 1.1, cx + 1.3, cy - 0.7], W + 4, H - 3)):
            got = host_undistort(hostcam, model, p, src, kp, ow, oh)
            want = uo.undistort_image(model, p, src, kp, ow, oh)
            assert got.tobytes() == want.tobytes()
            assert (got > 0).any()


def test_undistort_pixel_edges_and_rounding(hostcam):
    # PINHOLE onto itself: the identity, including the last row and column (clamped neighbours)
    src = _image(3, 9, 11)
    kp = [8.0, 4.0, 5.5, 4.5]  # powers of two: the ray and its projection are exact
    assert host_undistort(hostcam, "PINHOLE", kp, src, kp, 11, 9).tobytes() == src.tobytes()
    # half a pixel to the right: each output is the mean of two neighbours, rounded half away from zero
    src = np.zeros((1, 3, 3), np.uint8)
    src[0, :, 0] = [0, 1, 3]
    out = host_undistort(hostcam, "PINHOLE", [1.0, 1.0, 1.5, 0.5], src, [1.0, 1.0, 1.0, 0.5], 3, 1)
    assert out[0, :, 0].tolist() == [1, 2, 0]  # 0.5 -> 1, 2.0 -> 2, the last one is outside [0, W - 1]


def test_scale_on_a_case_worked_by_hand():
    # W = 100, cx = 50: left extents (-10, 5), right extents (90, 110); H = 80, cy = 40: top (0, 0), bottom (80, 80)
    cam = camera("SIMPLE_RADIAL", [100.0, 50.0, 40.0, 0.1], 100, 80, cam_id=7)
    ext = [-10.0, 5.0, 90.0, 110.0, 0.0, 0.0, 80.0, 80.0]
    # x: min_sx = min(50 / 60, 49.5 / 60) = 0.825, max_sx = max(50 / 45, 49.5 / 40) = 1.2375
    #    b = 0: sx = 1 / 1.2375 = 0.80808..., W' = int(80.80...) = 80, cx' = 50 * 80 / 100 = 40
    # y: min_sy = min(40 / 40, 39.5 / 40) = 0.9875, max_sy = max(1, 0.9875) = 1; sy = 1, H' = 80, cy' = 40
    got = ops.undistorted_camera(cam, ext, 0.0)
    assert (got.id, got.model, got.width, got.height) == (7, "PINHOLE", 80, 80)
    assert got.params == [100.0, 100.0, 40.0, 40.0]
    # b = 1: sx = 1 / 0.825 = 1.2121..., W' = 121, cx' = 60.5; sy = 1 / 0.9875 = 1.0126..., H' = 81, cy' = 40.5
    got = ops.undistorted_camera(cam, ext, 1.0)
    assert (got.width, got.height) == (121, 81) and got.params == [100.0, 100.0, 60.5, 40.5]
    assert uo.undistorted_camera("SIMPLE_RADIAL", cam.params, 100, 80, ext, 1.0) == (121, 81, [100.0, 100.0, 60.5, 40.5])
    # clamped to [0.2, 2]
    assert ops.undistorted_camera(cam, [45.0, 45.0, 55.0, 55.0, 0.0, 0.0, 80.0, 80.0], 0.0).width == 20  # sx = 0.1
    assert ops.undistorted_camera(cam, [-100.0, -100.0, 200.0, 200.0, 0.0, 0.0, 80.0, 80.0], 0.0).width == 200  # sx = 3
    with pytest.raises(ValueError, match=r"camera 7 \(SIMPLE_RADIAL\).*not finite"):
        ops.undistorted_camera(cam, [np.nan] * 8, 0.0)
    with pytest.raises(ValueError, match="blank_pixels"):
        ops.undistorted_camera(cam, ext, 1.5)


def _rejects(rc):
    assert rc == -1
    return _native.lib().pmb200_last_error().decode()


def test_abi_rejects_bad_arguments():
    lib = _native.lib()
    dummy = ctypes.c_void_p(16)
    good = ops._camera_struct(camera("OPENCV", CASES[4][1]))
    kp = (ctypes.c_double * 4)(500.0, 500.0, 320.0, 240.0)

    def cams(**kw):
        c = ops._camera_struct(camera("OPENCV", CASES[4][1]))
        for k, v in kw.items():
            if k == "p0":
                c.params[0] = v
            elif k == "p5":
                c.params[5] = v
            else:
                setattr(c, k, v)
        return c

    for bad, what in ((cams(model=11), "model"), (cams(model=-1), "model"), (cams(width=0), "width"), (cams(height=1 << 21), "width"),
                      (cams(p0=0.0), "focal"), (cams(p5=float("nan")), "finite"), (cams(p5=float("inf")), "finite")):
        assert what in _rejects(lib.pmb200_undistort_image(dummy, ctypes.byref(bad), kp, 10, 10, dummy, None))
        assert what in _rejects(lib.pmb200_undistort_extents(ctypes.byref(bad), 1, dummy, dummy, None))
    assert "null" in _rejects(lib.pmb200_undistort_image(None, ctypes.byref(good), kp, 10, 10, dummy, None))
    assert "null" in _rejects(lib.pmb200_undistort_extents(ctypes.byref(good), 1, None, dummy, None))
    assert "n_cameras" in _rejects(lib.pmb200_undistort_extents(ctypes.byref(good), 0, dummy, dummy, None))
    for w, h in ((0, 10), (10, 0), (1 << 21, 10)):
        assert "out_width" in _rejects(lib.pmb200_undistort_image(dummy, ctypes.byref(good), kp, w, h, dummy, None))
    for bad_kp in ((0.0, 500.0, 320.0, 240.0), (500.0, 500.0, float("nan"), 240.0)):
        assert "pinhole" in _rejects(lib.pmb200_undistort_image(dummy, ctypes.byref(good), (ctypes.c_double * 4)(*bad_kp), 10, 10,
                                                                dummy, None))


def test_ops_reject_bad_cameras_and_cpu_tensors():
    import torch

    with pytest.raises(ValueError, match="unknown model"):
        ops._camera_struct(camera("FISHEYE9", [1.0]))
    with pytest.raises(ValueError, match="has 8 parameters"):
        ops._camera_struct(camera("OPENCV", [500.0, 500.0, 320.0, 240.0]))
    cam = camera("OPENCV", CASES[4][1])
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.undistort_image(torch.zeros((H0, W0, 3), dtype=torch.uint8), cam, camera("PINHOLE", [500.0, 500.0, 320.0, 240.0]))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.undistort_extents([cam], "cpu")


def test_input_parser_undistort_options():
    a = ci.parse_args([])
    assert (a.undistort, a.blank_pixels) == (False, 0.0)
    a = ci.parse_args(["--undistort", "--blank-pixels", "0.25"])
    assert (a.undistort, a.blank_pixels) == (True, 0.25)
