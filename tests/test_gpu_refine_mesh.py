"""The mesh refinement on the GPU: one iteration's per-vertex sums and new positions equal oracle/refine_oracle.py bit for bit
(the albedo sphere, the plane, views of different sizes, two levels), reruns are bit-identical, the default schedule
converges on an analytic sphere, vertices no pixel reaches move by smoothing alone, reconstruct --mesh-refine and the refine
command end to end, and the tnt and eth3d scene-size rows simplified to 1 % within refine_mesh_bytes."""
import os

import numpy as np
import pytest
import torch

from oracle import refine_oracle as rfo, texture_oracle as to
from patchmatchnet_b200 import data_io, ops, reconstruct, refine
from tests import refine_cases as rc, scene_cases
from tests.test_gpu_mesh_at_scene_sizes import build_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
THRES = ["--geo-pixel-thres", "4", "--geo-depth-thres", "0.05", "--geo-mask-thres", "1", "--photo-thres", "0.05"]
FOOTPRINT = 2.2 / 170  # pixel footprint at the front of the sphere for mesh_cases.sphere_scene's cameras


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _case(name):
    if name == "plane":
        xyz, faces, images, Ks, Es = rc.plane_case(H=96, W=128, n=24)
        xyz = xyz.copy()
        xyz[:, 2] += (0.05 * np.sin(3 * xyz[:, 0]) * np.cos(2 * xyz[:, 1])).astype(np.float32)
        return xyz, faces, images, Ks, Es, [(1, 0), (1, 2), (0, 1), (2, 1)]
    sizes = [(120, 160), (160, 120), (90, 200)] if name == "sizes" else None
    images, Ks, Es = rc.sphere_views(n_views=8 if sizes else 14, sizes=sizes)
    xyz, faces = rc.icosphere(4)
    return rc.radial_noise(xyz, 2 * FOOTPRINT, seed=1), faces, images, Ks, Es, rc.sphere_pairs(Es, 3)


def _gpu(xyz, faces, images, Ks, Es, pairs, **kw):
    out, st = ops.refine_mesh(_d(xyz), _d(faces), [_d(i) for i in images], Ks, Es, pairs, with_sums=True, **kw)
    return out.cpu().numpy(), st["sums"].cpu().numpy(), st


@pytest.mark.parametrize("name,levels", [("sphere", 1), ("plane", 1), ("sizes", 1), ("sphere", 2)])
def test_one_iteration_equals_the_oracle(name, levels):
    xyz, faces, images, Ks, Es, pairs = _case(name)
    got, sums, st = _gpu(xyz, faces, images, Ks, Es, pairs, iterations=1, levels=levels)
    want, stats, acc = rfo.refine(xyz, faces.astype(np.int64), images, Ks, Es, pairs, 1, levels, ops.REFINE_ALPHA, ops.REFINE_SMOOTHNESS)
    reached = int((acc[:, 3] > 0).sum())
    print(f"[{name}, {levels} levels] {len(faces)} faces: {reached} of {len(xyz)} vertices reached, energy {st['energy']}, "
          f"windows {st['windows']}")
    assert reached > 0.3 * len(xyz)
    assert np.array_equal(sums, acc)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert st["windows"] == [n for _, n in stats]
    assert st["energy"] == [e for e, _ in stats]
    assert not np.array_equal(got, xyz)


def test_reruns_are_bit_identical():
    xyz, faces, images, Ks, Es, pairs = _case("sphere")
    a = _gpu(xyz, faces, images, Ks, Es, pairs, iterations=2)
    b = _gpu(xyz, faces, images, Ks, Es, pairs, iterations=2)
    assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])
    assert a[2]["energy"] == b[2]["energy"]


def test_default_schedule_converges_on_the_sphere():
    """An icosphere with 2.7-pixel edges displaced radially by a smooth field of up to 2 pixel footprints, refined with the
    defaults against 14 views carrying a 10-pixel-period albedo: the RMS radial error at least halves, the maximum error
    does not grow, and the energy of the last iteration is below the first's.  The true sphere stays within 0.1 footprint
    RMS."""
    images, Ks, Es = rc.sphere_views()
    pairs = rc.sphere_pairs(Es, ops.REFINE_NEIGHBOURS)
    x0, faces = rc.icosphere(5)
    noisy = rc.radial_noise(x0, 2 * FOOTPRINT, seed=0)
    out, _, st = _gpu(noisy, faces, images, Ks, Es, pairs)
    e0, e1 = rc.radial_error(noisy) / FOOTPRINT, rc.radial_error(out) / FOOTPRINT
    rms0, rms1 = float(np.sqrt((e0 ** 2).mean())), float(np.sqrt((e1 ** 2).mean()))
    print(f"[convergence] RMS {rms0:.3f} -> {rms1:.3f} footprints, max {np.abs(e0).max():.3f} -> {np.abs(e1).max():.3f}; energy per "
          f"iteration {[round(e, 1) for e in st['energy']]}; {st['seconds']:.3f} s")
    assert rms1 <= 0.5 * rms0
    assert np.abs(e1).max() <= np.abs(e0).max()
    assert st["energy"][-1] < st["energy"][0]
    true, _, st = _gpu(x0, faces, images, Ks, Es, pairs)
    et = rc.radial_error(true) / FOOTPRINT
    print(f"[true sphere] RMS {np.sqrt((et ** 2).mean()):.3f}, max {np.abs(et).max():.3f} footprints")
    assert np.sqrt((et ** 2).mean()) <= 0.1


def test_unreached_vertices_move_by_smoothing_alone():
    xyz, faces, images, Ks, Es, pairs = _case("sphere")
    far = np.array([[50, 50, 50], [51, 50, 50], [50, 51, 50], [50.5, 50.5, 51]], np.float32)
    x = np.concatenate([xyz, far])
    n = len(xyz)
    f = np.concatenate([faces, np.array([[n, n + 1, n + 2], [n, n + 2, n + 3]], np.int32)])
    xd, fd = _d(x), _d(f)
    x_keep, f_keep = xd.clone(), fd.clone()
    out, st = ops.refine_mesh(xd, fd, [_d(i) for i in images], Ks, Es, pairs, iterations=1, with_sums=True)
    assert torch.equal(xd, x_keep) and torch.equal(fd, f_keep)
    sums = st["sums"].cpu().numpy()
    assert (sums[n:] == 0).all()
    want = rfo.update(x, f.astype(np.int64), np.zeros((len(x), 5), np.int64), ops.REFINE_ALPHA, ops.REFINE_SMOOTHNESS,
                      rfo.box_diagonal(x))
    got = out.cpu().numpy()
    assert np.array_equal(got[n:].view(np.uint32), want[n:].view(np.uint32))
    assert not np.array_equal(got[n:], x[n:])  # the lone quad is smoothed


def test_refine_mesh_bytes_arithmetic():
    sizes = [(1080, 1920)] * 10 + [(1200, 1600)]
    b1 = ops.refine_mesh_bytes(100_000, 200_000, sizes, 1)
    b2 = ops.refine_mesh_bytes(100_000, 200_000, sizes, 2)
    assert b2 - b1 == 4 * sum((h // 2) * (w // 2) for h, w in sizes)
    all_pix = sum(h * w for h, w in sizes)
    low = 8 * all_pix + 46 * 1080 * 1920 + 4 * all_pix + 52 * 100_000 + 112 * 100_000 + 52 * 200_000
    assert low <= b1 < low + 64 * 200_000 + 2 ** 26


# ---- end to end ---------------------------------------------------------------------------------------------------------------

def _files(d):
    out = {}
    for sub, _, names in os.walk(d):
        for n in names:
            out[os.path.relpath(os.path.join(sub, n), d)] = open(os.path.join(sub, n), "rb").read()
    return out


def test_reconstruct_mesh_refine_and_the_command(tmp_path):
    scene = str(tmp_path / "scene")
    scene_cases.write_scene(scene, 6, 128, 160, n_src=5)
    common = ["--input-folder", scene, "--checkpoint-path", WEIGHTS, "--num-views", "3", *THRES, "--mesh", "--mesh-target-faces", "2000"]
    run = lambda out, *extra: reconstruct.reconstruct(reconstruct.parse_args(common + ["--output-folder", str(tmp_path / out), *extra]),
                                                      log=lambda *a: None)
    plain_stats = run("plain", "--mesh-texture")
    stats = run("ref", "--mesh-texture", "--mesh-refine")
    plain, ref = _files(str(tmp_path / "plain")), _files(str(tmp_path / "ref"))
    assert sorted(set(ref) - set(plain)) == ["mesh_refined.ply"]
    for name in plain:
        if not name.startswith("mesh_textured"):
            assert ref[name] == plain[name], name
    assert ref["mesh_textured.obj"] != plain["mesh_textured.obj"]  # the refined mesh is the one textured
    assert not any(k.startswith("refine") for k in plain_stats)
    assert stats["refine_seconds"] > 0 and stats["refine_energy_last"] < stats["refine_energy_first"]
    xr, cr, _, fr = data_io.read_ply(str(tmp_path / "ref" / "mesh_refined.ply"))
    xs, cs, _, fs = data_io.read_ply(str(tmp_path / "ref" / "mesh_simplified.ply"))
    assert np.array_equal(fr, fs) and np.array_equal(cr, cs) and xr.shape == xs.shape and not np.array_equal(xr, xs)
    refs = [r for r, _ in data_io.read_pair_file(os.path.join(scene, "pair.txt"))]
    out = str(tmp_path / "cli" / "mesh_refined.ply")
    os.makedirs(os.path.dirname(out))
    refine.main(["--ply", str(tmp_path / "ref" / "mesh_simplified.ply"), "--input-folder", scene, "--views", *map(str, refs),
                 "--output", out])
    assert open(out, "rb").read() == ref["mesh_refined.ply"]


# ---- at scene sizes -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["tnt", "eth3d"])
def test_scene_size_row_at_one_percent(name):
    row = build_scene(name, DEV)
    verts, faces = ops.tsdf_mesh(row["seeds"], row["depths"], row["images"], row["Ks"], row["Es"], row["s"])
    xyz, rgb = verts[:, :12].contiguous().view(torch.float32), verts[:, 12:].contiguous()
    body, sfaces, _ = ops.simplify_mesh(xyz, rgb, faces, faces.shape[0] // 100)
    del verts, faces, xyz, rgb
    images, Ks, Es = row["images"], row["Ks"], row["Es"]
    del row
    sx = body[:, :12].contiguous().view(torch.float32)
    V = len(images)
    pairs = rc.sphere_pairs(Es, ops.REFINE_NEIGHBOURS)  # each view and its 4 nearest by camera centre
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out, st = ops.refine_mesh(sx, sfaces, images, Ks, Es, pairs, iterations=1)
    torch.cuda.synchronize()
    used = torch.cuda.max_memory_allocated() - base
    budget = ops.refine_mesh_bytes(sx.shape[0], sfaces.shape[0], [tuple(i.shape[1:]) for i in images], ops.REFINE_LEVELS)
    print(f"[{name} 1 %] {sfaces.shape[0]} faces, {V} views, {len(pairs)} pairs: {st['seconds']:.3f} s (z-buffers "
          f"{st['zbuffer_seconds']:.3f}, pixels {st['pixel_seconds']:.3f}, update {st['update_seconds']:.4f}), windows {st['windows']}; "
          f"peak {used / 2 ** 20:.1f} MiB of {budget / 2 ** 20:.1f} MiB")
    assert used <= budget
    # the rows carry mesh_cases' smooth colour, so whether any window passes the variance threshold says nothing here
    assert st["pixel_pairs"] > 0 and torch.isfinite(out).all()
