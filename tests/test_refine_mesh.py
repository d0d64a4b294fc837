"""The mesh refinement without a GPU: the oracle's analytic vertex gradient against central differences of its own energy
(plane and sphere, visibility and windows frozen), the host build of pm_refine_mesh_math.cuh (tests/host_refine_mesh.cpp)
against oracle/refine_oracle.py formula by formula, the argument checks of the refine command and of reconstruct
--mesh-refine, and the level arithmetic (refine_mesh_bytes needs a device to size its sort: tests/test_gpu_refine_mesh.py)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import refine_oracle as rfo, texture_oracle as to
from patchmatchnet_b200 import data_io, ops, reconstruct, refine
from tests import refine_cases as rc

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = ctypes.c_void_p


# ---- the gradient is the energy's gradient --------------------------------------------------------------------------------

def _fd_case(name):
    if name == "plane":
        xyz, faces, images, Ks, Es = rc.plane_case()
        pairs = [(1, 0), (1, 2), (0, 1)]
    else:
        images, Ks, Es = rc.sphere_views(n_views=14, H=60, W=80)
        sel = [0] + [j for _, j in rc.sphere_pairs(Es, 2)[:2]]  # view 0 and its two nearest
        images, Ks, Es = [images[k] for k in sel], [Ks[k] for k in sel], [Es[k] for k in sel]
        xyz, faces = rc.icosphere(3)
        xyz = rc.radial_noise(xyz, 0.01, seed=3)
        pairs = [(0, 1), (0, 2), (1, 0)]
    return xyz, faces.astype(np.int64), images, Ks, Es, pairs


@pytest.mark.parametrize("name", ["plane", "sphere"])
def test_gradient_equals_central_differences(name):
    """dE/dx of the oracle (float64, no fixed point) against (E(x + h e) - E(x - h e)) / 2h for the vertices with the
    largest gradients, coverage, validity and counted windows frozen at x.  Relative tolerance 1e-4 on each vertex's
    gradient vector."""
    xyz, faces, images, Ks, Es, pairs = _fd_case(name)
    vl = rfo.views(Ks, Es, images, 1, to.box_centre(xyz))[0]
    frozen = rfo.freeze(xyz, faces, vl, pairs)
    x = xyz.astype(np.float64)
    E0, G = rfo.frozen_energy_and_gradient(x, faces, vl, pairs, frozen)
    assert E0 > 0 and sum(int(u.sum()) for _, u in frozen) > 100
    mag = np.linalg.norm(G, axis=1)
    top = np.argsort(-mag)[:12]
    assert mag[top[-1]] > 0
    h = 1e-6 * rfo.box_diagonal(xyz)
    worst = 0.0
    for v in top:
        fd = np.zeros(3)
        for c in range(3):
            xp, xm = x.copy(), x.copy()
            xp[v, c] += h
            xm[v, c] -= h
            fd[c] = (rfo.frozen_energy_and_gradient(xp, faces, vl, pairs, frozen)[0] -
                     rfo.frozen_energy_and_gradient(xm, faces, vl, pairs, frozen)[0]) / (2 * h)
        worst = max(worst, np.linalg.norm(fd - G[v]) / np.linalg.norm(G[v]))
    print(f"[{name}] E = {E0:.4f}, worst relative gradient error over {len(top)} vertices: {worst:.2e}")
    assert worst < 1e-4


# ---- the host build of pm_refine_mesh_math.cuh --------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def hostrm(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("hostrm") / "_hostrm.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-o", out,
                    os.path.join(REPO, "tests", "host_refine_mesh.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.hr_grey.argtypes = [P, ctypes.c_int, P]
    lib.hr_box.argtypes = [P, ctypes.c_int, P]
    lib.hr_hits.argtypes = [P, P, P, P, ctypes.c_int] + [P] * 9
    lib.hr_samples.argtypes = [P, ctypes.c_int, ctypes.c_int, P, P, P, P, ctypes.c_int, P]
    lib.hr_windows.argtypes = [P, P, ctypes.c_int, P, P]
    lib.hr_contributions.argtypes = [P] * 5 + [ctypes.c_int, ctypes.c_double, ctypes.c_double, P]
    lib.hr_steps.argtypes = [P] * 4 + [ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_double, P]
    return lib


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64 if a.dtype == np.float64 else np.uint32)


def test_host_grey_and_levels_equal_the_oracle(hostrm):
    rng = np.random.default_rng(1)
    img = rng.uniform(0, 1, (3, 37, 53)).astype(np.float32)
    g = np.zeros(37 * 53, np.float32)
    hostrm.hr_grey(img.ctypes.data, 37 * 53, g.ctypes.data)
    want = rfo.grey_levels(img, 3)
    assert np.array_equal(_bits(g), _bits(want[0].ravel()))
    q = np.ascontiguousarray(np.stack([want[0][0:36:2, 0:52:2], want[0][0:36:2, 1:52:2], want[0][1:36:2, 0:52:2],
                                       want[0][1:36:2, 1:52:2]], -1).reshape(-1, 4))
    b = np.zeros(len(q), np.float32)
    hostrm.hr_box(q.ctypes.data, len(q), b.ctypes.data)
    assert np.array_equal(_bits(b), _bits(want[1].ravel())) and want[2].shape == (9, 13)


def test_host_hits_samples_and_windows_equal_the_oracle(hostrm):
    rng = np.random.default_rng(2)
    images, Ks, Es = rc.sphere_views(n_views=14, H=60, W=80)
    j = rc.sphere_pairs(Es, 1)[0][1]
    xyz, faces = rc.icosphere(3)
    vi, vj = rfo.views([Ks[0], Ks[j]], [Es[0], Es[j]], [images[0], images[j]], 1, to.box_centre(xyz))[0]
    zi, zj = rfo.zbuffer(xyz, faces.astype(np.int64), vi), rfo.zbuffer(xyz, faces.astype(np.int64), vj)
    px = rfo.pair_pixels(xyz, faces.astype(np.int64), vi, vj, zi, zj)
    idx = np.flatnonzero(zi != np.uint64(0xFFFFFFFFFFFFFFFF))
    f = (zi[idx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    n = len(idx)
    xy = np.ascontiguousarray(np.stack([idx % vi["W"], idx // vi["W"]], 1).astype(np.float64))
    tri = np.ascontiguousarray(xyz[faces[f]].reshape(n, 9))
    C = np.zeros(3)
    ok = np.zeros(n, np.int32)
    r, X, beta = np.zeros((n, 3)), np.zeros((n, 3)), np.zeros((n, 3))
    t, nr = np.zeros(n), np.zeros(n)
    obl = np.zeros(n, np.int32)
    Cj = np.ascontiguousarray(vj["C"])
    hostrm.hr_hits(np.ascontiguousarray(vi["K"]).ctypes.data, np.ascontiguousarray(vi["Rt"]).ctypes.data, xy.ctypes.data, tri.ctypes.data,
                   n, Cj.ctypes.data, C.ctypes.data, ok.ctypes.data, r.ctypes.data, t.ctypes.data, nr.ctypes.data, X.ctypes.data,
                   beta.ctypes.data, obl.ctypes.data)
    assert np.array_equal(_bits(C), _bits(vi["C"]))
    rw = rfo.rays(vi, xy[:, 0], xy[:, 1])
    assert np.array_equal(_bits(r), _bits(rw))
    wok, _, wnr, wt, wX, wbeta = rfo.hits(xyz, faces.astype(np.int64), f, vi["C"], rw)
    assert np.array_equal(ok.astype(bool), wok) and wok.mean() > 0.9
    for got, want in ((t, wt), (nr, wnr), (X, wX), (beta, wbeta)):
        assert np.array_equal(_bits(got[wok]), _bits(want[wok]))
    wobl = wok & rfo.oblique_ok(rfo.cross(xyz[faces[f, 1]].astype(np.float64) - xyz[faces[f, 0]], xyz[faces[f, 2]].astype(np.float64)
                                          - xyz[faces[f, 0]]), wnr, rw, wX, vj["C"])
    assert np.array_equal(obl.astype(bool), wobl) and 0.2 < wobl.mean() < wok.mean()
    # samples at random points and at the image's last row and column
    m = 4000
    W, H = vj["W"], vj["H"]
    uv = np.ascontiguousarray(np.stack([rng.uniform(0, W - 1, m), rng.uniform(0, H - 1, m)], 1))
    uv[:10, 0] = W - 1
    uv[10:20, 1] = H - 1
    q = np.ascontiguousarray(np.stack([uv[:, 0], uv[:, 1], rng.uniform(1, 5, m)], 1))
    rr = np.ascontiguousarray(rng.normal(size=(m, 3)))
    out = np.zeros((m, 4))
    g = np.ascontiguousarray(vj["grey"])
    hostrm.hr_samples(g.ctypes.data, W, H, uv.ctypes.data, np.ascontiguousarray(vj["P"]).ctypes.data, q.ctypes.data, rr.ctypes.data, m,
                      out.ctypes.data)
    b, du, dv = rfo.bilinear(g, uv[:, 0], uv[:, 1])
    for k, want in enumerate((b, du, dv, rfo.db_dt(vj["P"], q[:, 0], q[:, 1], q[:, 2], rr, du, dv))):
        assert np.array_equal(_bits(out[:, k].copy()), _bits(want))
    # windows: the oracle's own sums at its valid pixels, plus thresholds
    use, E, c = rfo.windows(px)
    cnt = np.zeros(px["valid"].shape, np.int64)
    S = [np.zeros(px["valid"].shape) for _ in range(5)]
    for dy, dx in rfo.OFFSETS:
        mm = rfo._shifted(px["valid"], dy, dx, False)
        a_, b_ = np.where(mm, rfo._shifted(px["a"], dy, dx, 0.0), 0.0), np.where(mm, rfo._shifted(px["b"], dy, dx, 0.0), 0.0)
        cnt += mm
        for k, term in enumerate((a_, b_, a_ * a_, b_ * b_, a_ * b_)):
            S[k] = np.where(mm, S[k] + term, S[k])
    sel = np.flatnonzero(px["valid"].ravel())
    cn = np.ascontiguousarray(cnt.ravel()[sel].astype(np.int32))
    Ss = np.ascontiguousarray(np.stack([s.ravel()[sel] for s in S], 1))
    wok2 = np.zeros(len(sel), np.int32)
    wout = np.zeros((len(sel), 4))
    hostrm.hr_windows(cn.ctypes.data, Ss.ctypes.data, len(sel), wok2.ctypes.data, wout.ctypes.data)
    assert np.array_equal(wok2.astype(bool), use.ravel()[sel]) and 0.2 < wok2.mean() < 1.0
    u = wok2.astype(bool)
    assert np.array_equal(_bits(wout[u, 0].copy()), _bits(E.ravel()[sel][u]))
    for k in range(3):
        assert np.array_equal(_bits(wout[u, 1 + k].copy()), _bits(c[k].ravel()[sel][u]))


def test_host_contributions_and_steps_equal_the_oracle(hostrm):
    rng = np.random.default_rng(4)
    m = 3000
    g = rng.normal(size=m) * 10
    nrm = np.ascontiguousarray(rng.normal(size=(m, 3)))
    nr = -rng.uniform(0.1, 2, m)
    t = rng.uniform(1, 5, m)
    beta = rng.dirichlet([1, 1, 1], m)
    out = np.zeros((m, 3, 5), np.int64)
    f, L = 170.0, 2.7
    hostrm.hr_contributions(g.ctypes.data, nrm.ctypes.data, nr.ctypes.data, t.ctypes.data, np.ascontiguousarray(beta).ctypes.data, m, f, L,
                            out.ctypes.data)
    px = {"face": np.arange(m), "beta": beta, "nr": nr, "n": nrm, "t": t}
    faces = np.arange(3 * m).reshape(m, 3)
    want = rfo.scatter(px, g, np.ones(m, bool), faces, f, L, 3 * m)
    assert np.array_equal(out.reshape(3 * m, 5), want)
    acc = np.ascontiguousarray(np.concatenate([rng.integers(-2 ** 40, 2 ** 40, (m, 3)), rng.integers(0, 2 ** 36, (m, 2))], 1))
    acc[:5, 3] = 0
    un = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    x = rng.normal(size=(m, 3)).astype(np.float32)
    u2 = np.ascontiguousarray(rng.normal(size=(m, 3)) * 1e-3)
    got = np.zeros((m, 3), np.float32)
    hostrm.hr_steps(acc.ctypes.data, np.ascontiguousarray(un).ctypes.data, x.ctypes.data, u2.ctypes.data, m, 0.5, 0.3, L, got.ctypes.data)
    assert np.array_equal(_bits(got), _bits(rfo.step_positions(x, acc, un, u2, 0.5, 0.3, L)))


# ---- commands and memory --------------------------------------------------------------------------------------------------

def test_refine_command_checks(tmp_path):
    from tests import scene_cases

    scene = tmp_path / "scene"
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    mesh = str(tmp_path / "m.ply")
    data_io.save_ply(mesh, torch.zeros((3, 15), dtype=torch.uint8), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    out = str(tmp_path / "o" / "r.ply")
    base = ["--ply", mesh, "--input-folder", str(scene), "--output", out]
    with pytest.raises(ValueError, match="does not exist"):
        refine.main(base)
    os.makedirs(tmp_path / "o")
    with pytest.raises(ValueError, match="no such file"):
        refine.main(["--ply", str(tmp_path / "missing.ply"), "--input-folder", str(scene), "--output", out])
    with pytest.raises(ValueError, match="view 99"):
        refine.main(base + ["--views", "0", "99"])
    for bad, msg in ((["--neighbours", "0"], "neighbours"), (["--iterations", "-1"], "iterations"), (["--levels", "0"], "levels"),
                     (["--levels", "17"], "levels"), (["--smoothness", "-1"], "smoothness"), (["--smoothness", "inf"], "smoothness")):
        with pytest.raises(ValueError, match=msg):
            refine.main(base + bad)
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError, match="pair.txt"):
        refine.main(["--ply", mesh, "--input-folder", str(tmp_path / "empty"), "--output", out])
    assert refine.check_args(refine.build_parser().parse_args(base)) == [0, 1, 2]
    assert os.listdir(tmp_path / "o") == []


def test_scene_pairs_restrict_to_the_views_used(tmp_path):
    p = tmp_path / "pair.txt"
    p.write_text("3\n0\n3 2 1.0 5 1.0 1 1.0\n2\n2 0 1.0 1 1.0\n5\n1 2 1.0\n")
    assert refine.scene_pairs(str(p), [0, 2, 5], 4) == [(0, 1), (0, 2), (1, 0), (2, 1)]
    assert refine.scene_pairs(str(p), [0, 2], 1) == [(0, 1), (1, 0)]


def test_reconstruct_refine_option(tmp_path):
    from tests import scene_cases

    assert "mesh_refine" not in vars(reconstruct.parse_args([]))
    assert reconstruct.mesh_options(reconstruct.parse_args(["--mesh", "--mesh-refine"])).mesh_refine
    assert not reconstruct.mesh_options(reconstruct.parse_args(["--mesh"])).mesh_refine
    scene, out = tmp_path / "scene", tmp_path / "out"
    out.mkdir()
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    ckpt = tmp_path / "model.pt"
    ckpt.write_bytes(b"")
    base = ["--input-folder", str(scene), "--output-folder", str(out), "--checkpoint-path", str(ckpt), "--output-type", "fusion"]
    with pytest.raises(ValueError, match="--mesh-refine needs --mesh"):
        reconstruct.main(base + ["--mesh-refine"])
    with pytest.raises(ValueError, match="needs --mesh"):
        reconstruct.main(base + ["--mesh-refine", "--mesh-texture"])
    # a pair.txt whose sources are not among its reference views leaves no pair: refused before anything is written
    (scene / "pair.txt").write_text("2\n0\n1 7 1.0\n1\n1 8 1.0\n")
    with pytest.raises(ValueError, match="no pair to refine against"):
        reconstruct.main(base + ["--mesh", "--mesh-refine"])
    assert os.listdir(out) == []


def test_refine_command_refuses_views_without_a_pair(tmp_path):
    from tests import scene_cases

    scene = tmp_path / "scene"
    scene_cases.write_scene(str(scene), 3, 24, 32, n_src=2)
    mesh = str(tmp_path / "m.ply")
    data_io.save_ply(mesh, torch.zeros((3, 15), dtype=torch.uint8), torch.tensor([[0, 1, 2]], dtype=torch.int32))
    out = tmp_path / "o"
    out.mkdir()
    with pytest.raises(ValueError, match="only smoothing"):
        refine.main(["--ply", mesh, "--input-folder", str(scene), "--output", str(out / "r.ply"), "--views", "1"])
    assert os.listdir(out) == []


def test_refine_mesh_rejects_bad_arguments_before_any_launch():
    with pytest.raises(ValueError, match="CUDA"):
        ops.refine_mesh(torch.zeros((3, 3)), torch.zeros((1, 3), dtype=torch.int32), [torch.zeros((3, 4, 4))], [np.eye(3)],
                        [np.eye(4)], [])


def test_refine_level_arithmetic():
    assert ops.refine_level_sizes((1080, 1920), 3) == [(1080, 1920), (540, 960), (270, 480)]
    assert ops.refine_level_sizes((7, 5), 3) == [(7, 5), (3, 2), (1, 1)]
    K = np.array([[100.0, 0.5, 63.5], [0, 90.0, 47.5], [0, 0, 1]])
    for a, b in zip(ops.refine_level_intrinsics(K, 3), rfo.level_K(K, 3)):
        assert np.array_equal(a, b)
    assert ops.refine_level_intrinsics(K, 2)[1].tolist() == [[50.0, 0.25, 31.5], [0, 45.0, 23.5], [0, 0, 1]]


# ---- the C ABI's rejections ---------------------------------------------------------------------------------------------

def _rejects(rc):
    from patchmatchnet_b200 import _native

    assert rc == -1, rc
    return _native.lib().pmb200_last_error().decode()


def _abi_views(n_views=2, levels=1, W=64, H=48):
    """A valid level-major view table for 48 x 64 views (identity rotations, cameras 3 apart along x)."""
    eye = np.eye(4)
    Es = []
    for v in range(n_views):
        E = eye.copy()
        E[0, 3] = -3.0 * v
        Es.append(E)
    K = np.array([[50.0, 0, 31.5], [0, 50.0, 23.5], [0, 0, 1]])
    table, grey = ops.refine_view_table([K] * n_views, Es, [(H, W)] * n_views, levels, [0.0, 0.0, 5.0])
    return table, grey


def test_abi_rejects_bad_arguments():
    """Every EINVAL of pmb200_refine_mesh and its workspace query that comes before the device is touched (the workspace
    check needs the CUB sort's size from a device: tests/test_gpu_refine_mesh.py)."""
    import ctypes as C

    from patchmatchnet_b200 import _native

    lib = _native.lib()
    d = C.c_void_p(16)
    table, grey = _abi_views()
    pairs = (C.c_int * 4)(0, 1, 1, 0)
    stats = (C.c_double * 6)()

    def call(xyz=d, nv=3, faces=d, nf=1, g=d, gf=grey, views=None, n_views=2, levels=1, pr=pairs, n_pairs=2, iterations=1, alpha=0.3,
             lam=0.4, L=1.0, st=stats, ws=d):
        return lib.pmb200_refine_mesh(xyz, nv, faces, nf, g, gf, C.addressof(views or table), n_views, levels, pr, n_pairs, iterations,
                                      alpha, lam, L, None, st, ws, 1 << 40, None)

    assert "null" in _rejects(call(xyz=None))
    assert "null" in _rejects(call(faces=None))
    assert "null" in _rejects(call(g=None))
    assert "null" in _rejects(call(pr=None))
    assert "null" in _rejects(call(st=None))
    assert "null" in _rejects(call(ws=None))
    assert "2^31" in _rejects(call(nv=-1))
    assert "2^31" in _rejects(call(nv=1 << 31))
    assert "2^29" in _rejects(call(nf=1 << 29))
    assert "levels" in _rejects(call(levels=0))
    assert "levels" in _rejects(call(levels=17))
    assert "levels" in _rejects(call(n_views=0))
    assert "grey" in _rejects(call(gf=grey - 1))  # an image outside the grey buffer
    assert "does not exist" in _rejects(lib.pmb200_refine_mesh(d, 3, d, 1, d, grey, C.addressof(table), 2, 1, (C.c_int * 2)(0, 2), 1, 1,
                                                               0.3, 0.4, 1.0, None, stats, d, 1 << 40, None))
    assert "does not exist" in _rejects(call(pr=(C.c_int * 2)(-1, 0), n_pairs=1))
    assert "itself" in _rejects(call(pr=(C.c_int * 2)(1, 1), n_pairs=1))
    assert "n_pairs" in _rejects(call(n_pairs=-1))
    assert "iterations" in _rejects(call(iterations=-1))
    assert "alpha" in _rejects(call(alpha=float("nan")))
    assert "alpha" in _rejects(call(alpha=-0.1))
    assert "smoothness" in _rejects(call(lam=float("inf")))
    assert "unit length" in _rejects(call(L=0.0))
    assert "unit length" in _rejects(call(L=float("inf")))
    for field, k, bad in (("P", 3, float("inf")), ("K", 0, float("nan")), ("K", 0, 0.0), ("Rt", 5, float("nan")), ("near_z", None, 0.0)):
        t2, _ = _abi_views()
        if k is None:
            setattr(t2[1], field, bad)
        else:
            getattr(t2[1], field)[k] = bad
        assert "finite cameras" in _rejects(call(views=t2)), field
        assert _rejects(lib.pmb200_refine_mesh_workspace_bytes(3, 1, C.addressof(t2), 2))
    t3, g3 = _abi_views(levels=2)
    t3[3].width = 33  # level 1 of view 1 is not half of its level 0
    assert "half" in _rejects(call(views=t3, levels=2, gf=g3))
    t4, _ = _abi_views()
    t4[0].width = 16385
    assert "16384" in _rejects(call(views=t4))
    assert _rejects(lib.pmb200_refine_mesh_workspace_bytes(-1, 0, C.addressof(table), 2))
    assert _rejects(lib.pmb200_refine_mesh_workspace_bytes(3, 1, None, 2))
    assert _rejects(lib.pmb200_refine_mesh_pyramid(None, 64, 48, 1, d, None))
    assert "levels" in _rejects(lib.pmb200_refine_mesh_pyramid(d, 64, 48, 7, d, None))  # 48 >> 6 == 0


def test_refine_mesh_bytes_python_terms():
    """The part of refine_mesh_bytes outside the native workspace: 4 bytes per pixel of every level's grey image and 52 per
    vertex (the refined positions and the int64 sums)."""
    sizes = [(1080, 1920)] * 3 + [(1201, 1601)]
    assert ops.refine_mesh_extra_bytes(1000, sizes, 1) == 4 * (3 * 1080 * 1920 + 1201 * 1601) + 52 * 1000
    assert ops.refine_mesh_extra_bytes(1000, sizes, 3) - ops.refine_mesh_extra_bytes(1000, sizes, 1) == \
        4 * (3 * (540 * 960 + 270 * 480) + 600 * 800 + 300 * 400)
    assert ops.refine_mesh_extra_bytes(0, [(1, 1)], 1) == 4
