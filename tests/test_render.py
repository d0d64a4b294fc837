"""The renderer without a GPU: the oracle's hand cases (coverage, fill rule, occlusion, ties, splat clipping, near plane and
the 2^22 bound), data_io.read_ply, the orbit and Open3D cameras, and the command's argument checks."""
import json
import os

import numpy as np
import pytest
import torch

from patchmatchnet_b200 import data_io, render
from tests import render_cases as rc
from tests import render_oracle as ro

IDENT = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0]], np.float64)  # u = x / z


def _mesh_frags(xyz, faces, W, H, near=1e-3, P=IDENT):
    P32, _ = ro.camera(P)
    return ro.mesh_zbuffer(ro.project_vertices(P32, np.asarray(xyz, np.float32), W, H, near), faces, W, H, count=True)


def _tri(pts2d, z=1.0):
    return np.array([[x * z, y * z, z] for x, y in pts2d], np.float32)


def test_single_triangle_covers_its_pixels_with_the_top_left_rule():
    # right triangle (0,0) (4,0) (0,4): the top edge y = 0 and the left edge x = 0 are in, the hypotenuse x + y = 4 is out
    zbuf, frags = _mesh_frags(_tri([(0, 0), (4, 0), (0, 4)]), [[0, 1, 2]], 8, 8)
    want = np.zeros((8, 8), np.int64)
    for y in range(8):
        for x in range(8):
            want[y, x] = x + y < 4
    assert (frags == want).all()
    # the opposite winding covers the same pixels
    _, frags2 = _mesh_frags(_tri([(0, 0), (0, 4), (4, 0)]), [[0, 1, 2]], 8, 8)
    assert (frags2 == want).all()


def test_shared_edge_and_fan_cover_every_pixel_once():
    # a quad split along its diagonal through pixel centres, and along the other diagonal
    quad = _tri([(0.0, 0.0), (9.0, 0.0), (9.0, 7.0), (0.0, 7.0)])
    for faces in ([[0, 1, 2], [0, 2, 3]], [[0, 1, 3], [1, 2, 3]]):
        _, frags = _mesh_frags(quad, faces, 12, 10)
        inner = frags[:7, :9]  # the half-open quad [0, 9) x [0, 7) under the top-left rule
        assert (inner == 1).all(), inner
        assert frags.sum() == 9 * 7
    # a fan whose centre is a pixel centre, covering the frame: every pixel exactly once
    xyz, faces, P = rc.fan(64, 48)
    _, frags = _mesh_frags(xyz, faces, 64, 48, P=P)
    assert (frags == 1).all(), np.argwhere(frags != 1)[:5]
    # ... and a random fan centre off the pixel grid
    xyz, faces, P = rc.fan(64, 48, k=17, centre=(31.37, 20.5))
    assert (_mesh_frags(xyz, faces, 64, 48, P=P)[1] == 1).all()


def test_occlusion_and_equal_depth_tie():
    near_tri, far_tri = _tri([(-10, -10), (30, -10), (-10, 30)], 2.0), _tri([(-10, -10), (30, -10), (-10, 30)], 3.0)
    xyz = np.concatenate([far_tri, near_tri])
    rgb = np.array([[255, 0, 0]] * 3 + [[0, 0, 255]] * 3, np.uint8)
    img, depth = ro.render_mesh(xyz, rgb, [[0, 1, 2], [3, 4, 5]], IDENT, 8, 8, 1e-3)
    assert (img[..., 2] == 255).all() and (img[..., 0] == 0).all() and np.allclose(depth, 2.0, rtol=1e-6, atol=0)
    # the same triangle twice: the lower face index wins the exact tie, whatever the order
    img, _ = ro.render_mesh(np.concatenate([near_tri, near_tri]), rgb, [[3, 4, 5], [0, 1, 2]], IDENT, 8, 8, 1e-3)
    assert (img[..., 2] == 255).all()
    # points: the same point twice, the lower index wins
    pts = np.array([[2, 2, 1], [2, 2, 1]], np.float32)
    img, depth = ro.render_points(pts, np.array([[9, 9, 9], [200, 200, 200]], np.uint8), None, IDENT, 5, 5, 1e-3)
    assert tuple(img[2, 2]) == (9, 9, 9) and depth[2, 2] == 1.0
    # a nearer point with a larger index still wins
    pts = np.array([[2, 2, 1], [1.5, 1.5, 0.75]], np.float32)
    img, depth = ro.render_points(pts, np.array([[9, 9, 9], [200, 200, 200]], np.uint8), None, IDENT, 5, 5, 1e-3)
    assert tuple(img[2, 2]) == (200, 200, 200) and depth[2, 2] == 0.75


def test_point_splats_are_clipped_at_the_border():
    pts = np.array([[0, 0, 1], [5.4, 3.6, 1], [-2, 1, 1]], np.float32)  # (5.4, 3.6) rounds to (5, 4)
    img, depth = ro.render_points(pts, None, None, IDENT, 6, 5, 1e-3, point_size=3, background=(0, 0, 0))
    cov = depth > 0
    want = np.zeros((5, 6), bool)
    want[0:2, 0:2] = True      # around (0, 0)
    want[3:5, 4:6] = True      # around (5, 4)
    assert (cov == want).all(), cov.astype(int)
    assert (img[cov] == 160).all() and (img[~cov] == 0).all()
    # rint is half to even: u = 2.5 -> 2, 3.5 -> 4
    img, depth = ro.render_points(np.array([[2.5, 0, 1], [3.5, 2, 1]], np.float32), None, None, IDENT, 6, 3, 1e-3)
    assert depth[0, 2] == 1 and depth[2, 4] == 1 and (depth > 0).sum() == 2


def test_near_plane_and_the_2_22_bound():
    pts = np.array([[0, 0, 0.5], [1, 1, 1e-4], [2, 2, -1], [3, 3, 0.001]], np.float32)
    depth = ro.render_points(pts, None, None, IDENT, 4, 4, 1e-3)[1]
    assert depth[0, 0] == 0.5 and depth[1, 1] == 0 and depth[2, 2] == 0 and depth[3, 3] == 0  # z <= near is skipped
    big = _tri([(0, 0), (8, 0), (0, 8)])
    for v, z in ((2, 1e-3), (2, -1.0)):
        t = big.copy()
        t[v, 2] = z
        assert _mesh_frags(t, [[0, 1, 2]], 8, 8)[1].sum() == 0  # a vertex at or behind near drops the face
    t = big.copy()
    t[1, 0] = 2.0 ** 22
    assert _mesh_frags(t, [[0, 1, 2]], 8, 8)[1].sum() > 0  # |u| = 2^22 is still rasterised
    t[1, 0] = np.nextafter(np.float32(2.0 ** 22), np.float32(np.inf))
    assert _mesh_frags(t, [[0, 1, 2]], 8, 8)[1].sum() == 0  # beyond it the face is dropped
    # zero area and out-of-range indices are skipped
    assert _mesh_frags(_tri([(0, 0), (4, 4), (8, 8)]), [[0, 1, 2]], 8, 8)[1].sum() == 0
    assert _mesh_frags(big, [[0, 1, 3]], 8, 8)[1].sum() == 0


def test_shading_and_perspective_colours():
    # a point facing the camera is unshaded; tilted 60 degrees it gets 0.25 + 0.75 * 0.5
    pts = np.array([[0, 0, 2]], np.float32)
    n = np.array([[0, np.sin(np.pi / 3), np.cos(np.pi / 3)]], np.float32)
    img, _ = ro.render_points(pts, np.array([[200, 100, 40]], np.uint8), n, IDENT, 1, 1, 1e-3, shade=True)
    f = 0.25 + 0.75 * 0.5
    assert np.abs(img[0, 0].astype(float) - np.array([200, 100, 40]) * f).max() <= 1
    img, _ = ro.render_points(pts, np.array([[200, 100, 40]], np.uint8), None, IDENT, 1, 1, 1e-3, shade=True)
    assert tuple(img[0, 0]) == (200, 100, 40)  # no normals: unshaded
    # a mesh with one colour everywhere keeps it; flat shading of a face facing the camera keeps it too (|n.l| ~ 1 at the
    # centre of a small frame)
    tri = _tri([(-20, -20), (60, -20), (-20, 60)], 4.0)
    img, _ = ro.render_mesh(tri, np.full((3, 3), 90, np.uint8), [[0, 1, 2]], IDENT, 3, 3, 1e-3)
    assert (img == 90).all()


def test_camera_rounding_matches_ops():
    from patchmatchnet_b200 import ops

    P = rc.pinhole() @ np.diag([1.0, 1.0, 1.0, 1.0])
    p32, c32 = ops.render_camera_arrays(P)
    q32, d32 = ro.camera(P)
    assert (p32 == q32.ravel()).all() and (c32 == d32).all()
    with pytest.raises(ValueError):
        ops.render_camera_arrays(np.zeros((3, 4)))
    with pytest.raises(ValueError):
        ops.render_camera_arrays(np.full((3, 4), np.nan))


# ---- read_ply -------------------------------------------------------------------------------------------------------------


def _write_binary(path, header_props, rows, faces=None, count_t="uchar", index_t="int"):
    names = [n for n, _ in header_props]
    h = "ply\nformat binary_little_endian 1.0\ncomment test\nelement vertex %d\n" % len(rows)
    h += "".join("property %s %s\n" % (t, n) for n, t in header_props)
    if faces is not None:
        h += "element face %d\nproperty list %s %s vertex_indices\n" % (len(faces), count_t, index_t)
    h += "end_header\n"
    np_t = {"float": "<f4", "double": "<f8", "uchar": "u1", "int": "<i4", "uint": "<u4"}
    dt = np.dtype([(n, np_t[t]) for n, t in header_props])
    body = np.array([tuple(r) for r in rows], dtype=dt).tobytes()
    if faces is not None:
        fdt = np.dtype([("n", np_t[count_t]), ("v", np_t[index_t], (len(faces[0]),))])
        body += np.array([(len(f), f) for f in faces], dtype=fdt).tobytes()
    with open(path, "wb") as f:
        f.write(h.encode() + body)


XYZ = [("x", "float"), ("y", "float"), ("z", "float")]
RGB = [("red", "uchar"), ("green", "uchar"), ("blue", "uchar")]
NRM = [("nx", "float"), ("ny", "float"), ("nz", "float")]


def test_read_ply_binary_with_and_without_colours_and_normals(tmp_path):
    p = str(tmp_path / "a.ply")
    _write_binary(p, XYZ, [(1, 2, 3), (4, 5, 6)])
    xyz, rgb, nrm, faces = data_io.read_ply(p)
    assert xyz.dtype == np.float32 and (xyz == [[1, 2, 3], [4, 5, 6]]).all() and rgb is None and nrm is None and faces is None
    _write_binary(p, XYZ + NRM + RGB + [("quality", "float")], [(1, 2, 3, 0, 0, 1, 10, 20, 30, 0.5)])
    xyz, rgb, nrm, faces = data_io.read_ply(p)
    assert rgb.dtype == np.uint8 and (rgb == [[10, 20, 30]]).all() and (nrm == [[0, 0, 1]]).all() and faces is None


@pytest.mark.parametrize("count_t,index_t", [("uchar", "int"), ("int", "int"), ("uchar", "uint"), ("uint", "uint")])
def test_read_ply_faces_with_list_counts(tmp_path, count_t, index_t):
    p = str(tmp_path / "m.ply")
    _write_binary(p, XYZ + RGB, [(0, 0, 1, 1, 2, 3), (1, 0, 1, 4, 5, 6), (0, 1, 1, 7, 8, 9)], faces=[[0, 1, 2], [2, 1, 0]],
                  count_t=count_t, index_t=index_t)
    xyz, rgb, nrm, faces = data_io.read_ply(p)
    assert faces.dtype == np.int32 and (faces == [[0, 1, 2], [2, 1, 0]]).all() and rgb.shape == (3, 3)


def test_read_ply_rejects_quads_bad_indices_and_malformed_files(tmp_path):
    p = str(tmp_path / "q.ply")
    _write_binary(p, XYZ, [(0, 0, 1)] * 4, faces=[[0, 1, 2, 3]])
    with pytest.raises(ValueError, match="triangle"):
        data_io.read_ply(p)
    _write_binary(p, XYZ, [(0, 0, 1)] * 3, faces=[[0, 1, 3]])
    with pytest.raises(ValueError, match="outside"):
        data_io.read_ply(p)
    _write_binary(p, XYZ, [(0, 0, 1)] * 3, faces=[[0, 1, -1]])
    with pytest.raises(ValueError, match="outside"):
        data_io.read_ply(p)
    for text in (b"nope\n", b"ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nend_header\n",
                 b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\n",
                 b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\nend_header\n1 2\n",
                 b"ply\nformat ascii 1.0\nelement vertex 1\nproperty half x\nend_header\n1\n",
                 b"ply\nformat ascii 1.0\nelement face 1\nproperty list uchar int vertex_indices\nelement vertex 0\n"
                 b"property float x\nproperty float y\nproperty float z\nend_header\n3 0 0 0\n",
                 b"ply\nformat binary_little_endian 1.0\nelement vertex 2\nproperty float x\nproperty float y\nproperty float z\n"
                 b"end_header\n" + b"\0" * 12):
        with open(p, "wb") as f:
            f.write(text)
        with pytest.raises(ValueError):
            data_io.read_ply(p)


def test_read_ply_ascii_and_double(tmp_path):
    p = str(tmp_path / "a.ply")
    with open(p, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 3\nproperty double x\nproperty double y\nproperty double z\n"
                "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face 1\nproperty list uchar int vertex_index\n"
                "end_header\n0.1 0 1 1 2 3\n1 0 1 4 5 6\n0 1 1 7 8 9\n3 0 1 2\n")
    xyz, rgb, nrm, faces = data_io.read_ply(p)
    assert xyz.dtype == np.float32 and xyz[0, 0] == np.float32(0.1)  # narrowed from double
    assert (rgb[2] == [7, 8, 9]).all() and (faces == [[0, 1, 2]]).all()
    with open(p, "w") as f:
        f.write("ply\nformat ascii 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\nelement face 1\n"
                "property list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n1 1 0\n0 1 0\n4 0 1 2 3\n")
    with pytest.raises(ValueError, match="triangle"):
        data_io.read_ply(p)
    # a double-precision binary cloud, as ground-truth scans are stored
    _write_binary(p, [("x", "double"), ("y", "double"), ("z", "double")], [(1 / 3, 2.0, 1e10)])
    xyz = data_io.read_ply(p)[0]
    assert xyz.dtype == np.float32 and (xyz == np.array([[1 / 3, 2.0, 1e10]], np.float32)).all()


def test_read_ply_round_trips_save_ply(tmp_path):
    rng = np.random.default_rng(1)
    pos = rng.normal(size=(50, 3)).astype(np.float32)
    col = rng.integers(0, 256, (50, 3), dtype=np.uint8)
    nrm = rng.normal(size=(50, 3)).astype(np.float32)
    plain = torch.from_numpy(np.concatenate([pos.view(np.uint8).reshape(50, 12), col], 1))
    oriented = torch.from_numpy(np.concatenate([pos.view(np.uint8).reshape(50, 12), nrm.view(np.uint8).reshape(50, 12), col], 1))
    faces = torch.from_numpy(rng.integers(0, 50, (30, 3)).astype(np.int32))
    for body, fc in ((plain, None), (oriented, None), (plain, faces)):
        p = str(tmp_path / "r.ply")
        data_io.save_ply(p, body, fc)
        xyz, rgb, n, f = data_io.read_ply(p)
        assert (xyz == pos).all() and (rgb == col).all()
        assert (n is None) == (body.shape[1] == 15) and (n is None or (n == nrm).all())
        assert (f is None) == (fc is None) and (f is None or (f == fc.numpy()).all())
        assert (data_io.read_ply_points(p) == pos.astype(np.float64)).all()


# ---- cameras and arguments ------------------------------------------------------------------------------------------------


def test_orbit_cameras_look_at_the_centre_fit_the_sphere_and_honour_up():
    centre, radius, W, H = np.array([1.0, -2.0, 3.0]), 2.5, 320, 200
    up = np.array([0.0, 0.0, 1.0])
    cams = render.orbit_cameras(centre, radius, 6, 25.0, up, W, H)
    assert len(cams) == 6
    sphere = centre + radius * rc_unit_sphere(2000)
    for P in cams:
        K = render.orbit_intrinsics(W, H)
        RT = np.linalg.solve(K, P)  # [R | t]
        C = render.camera_centre(P)
        u = P @ np.append(centre, 1.0)
        assert np.allclose(u[:2] / u[2], [(W - 1) / 2, (H - 1) / 2])  # the centre projects to the frame's centre
        q = P @ np.vstack([sphere.T, np.ones(len(sphere))])
        uv = q[:2] / q[2]
        assert (q[2] > 0).all() and (uv[0] >= -0.5).all() and (uv[0] <= W - 0.5).all() and (uv[1] >= -0.5).all() and (uv[1] <= H - 0.5).all()
        assert uv[1].min() < 0.5 or uv[0].min() < 0.5  # and it fills the frame (tangent to the tighter side)
        assert np.dot(-RT[1, :3], up) > 0  # image-up points along up
        d = (C - centre) / np.linalg.norm(C - centre)
        assert np.isclose(np.degrees(np.arcsin(np.dot(d, up))), 25.0)  # the elevation
    centres = np.array([render.camera_centre(P) for P in cams])
    assert np.allclose(np.linalg.norm(centres - centre, axis=1), np.linalg.norm(centres[0] - centre))


def rc_unit_sphere(n):
    v = np.random.default_rng(0).normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def test_percentile_box_ignores_outliers():
    rng = np.random.default_rng(0)
    pts = rng.uniform(-1, 1, (1000, 3)).astype(np.float32)
    pts[:5] = 1e6
    lo, hi = render.percentile_box(torch.from_numpy(pts))
    assert (hi < 1.0 + 1e-6).all() and (lo > -1.0 - 1e-6).all() and (hi - lo > 1.8).all()


def test_open3d_viewpoint_reader(tmp_path):
    K = np.array([[500.0, 0, 319.5], [0, 510.0, 239.5], [0, 0, 1]])
    E = np.eye(4)
    E[:3, :3] = [[0, -1, 0], [1, 0, 0], [0, 0, 1]]
    E[:3, 3] = [0.1, 0.2, 3.0]
    doc = {"class_name": "PinholeCameraParameters", "extrinsic": E.ravel(order="F").tolist(),
           "intrinsic": {"height": 480, "intrinsic_matrix": K.ravel(order="F").tolist(), "width": 640},
           "version_major": 1, "version_minor": 0}
    p = str(tmp_path / "vp.json")
    with open(p, "w") as f:
        json.dump(doc, f)
    P, w, h = render.read_viewpoint(p)
    assert (w, h) == (640, 480) and np.allclose(P, K @ E[:3])
    with open(p, "w") as f:
        json.dump({"intrinsic": {}}, f)
    with pytest.raises(ValueError):
        render.read_viewpoint(p)


def test_view_camera_scales_intrinsics_like_reconstruct(tmp_path):
    from tests import scene_cases

    sc = scene_cases.write_scene(str(tmp_path), 2, 60, 80, n_src=1)
    P, w, h = render.view_camera(str(tmp_path), 1, 40)
    K, E = sc["cams"][1]
    assert (w, h) == (40, 30)
    Ks = data_io.scale_intrinsics(K, (30, 40), 60, 80)
    assert np.allclose(P, Ks.astype(np.float64) @ E.astype(np.float64)[:3])
    up = render.scene_up(str(tmp_path))
    assert np.isclose(np.linalg.norm(up), 1.0) and up[1] < -0.9  # the cameras' image-up is about -Y


def test_argument_errors(tmp_path):
    ply = str(tmp_path / "c.ply")
    _write_binary(ply, XYZ, [(0, 0, 1)])
    bad = [[], ["--views", "0"], ["--orbit", "-1"], ["--viewpoint", str(tmp_path / "none.json")], ["--orbit", "2", "--point-size", "2"],
           ["--orbit", "2", "--point-size", "17"], ["--orbit", "2", "--width", "0"], ["--orbit", "2", "--background", "0", "0", "256"],
           ["--orbit", "2", "--up", "0", "0", "0"], ["--orbit", "2", "--near", "0"]]
    for extra in bad:
        with pytest.raises(ValueError):
            render.check_args(render.parse_args(["--ply", ply] + extra))
    with pytest.raises(ValueError):
        render.check_args(render.parse_args(["--ply", str(tmp_path / "missing.ply"), "--orbit", "1"]))
    render.check_args(render.parse_args(["--ply", ply, "--orbit", "3"]))
