"""The reconstruct command on the GPU: fusion against the CPU oracle (oracle/geo_oracle.py), depth maps against a direct
DepthEngine run, `both` against `depth` then `fusion`, TorchScript checkpoints, and the chain into dtu_eval.

Fixtures are generated from seeds in this file (tests/scene_cases.py).  Mask bounds are test_geo's: a pixel within rounding
of a threshold may flip (the kernel's float64 dot products are fused multiply-adds, BLAS's are not), at most 1e-4 of the
pixels per mask."""
import json
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import geo_oracle as go
from patchmatchnet_b200 import data_io, dtu_eval, ops, reconstruct
from patchmatchnet_b200.engine import DepthEngine
from tests import dtu_cases, scene_cases
from tests.test_geo import _check_body

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WEIGHTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights_000007.pt")
DTU_THRES = ["--geo-pixel-thres", "1", "--geo-depth-thres", "0.01", "--geo-mask-thres", "3", "--photo-thres", "0.8"]
N_VIEWS = 6
FUSION_HW = (96, 128)
DEPTH_HW = (128, 160)


def _run(*argv):
    return reconstruct.reconstruct(reconstruct.parse_args([str(a) for a in argv]), log=lambda *a: None)


def _fusion_tree(root, out_dir=None):
    sc = scene_cases.write_scene(str(root), N_VIEWS, *FUSION_HW, n_src=N_VIEWS - 1)
    scene_cases.write_fusion_maps(str(out_dir or root), sc["cams"], *FUSION_HW, seed=7)
    return sc


def _mask(path):
    m = np.array(Image.open(path))
    assert m.dtype == np.uint8 and set(np.unique(m)) <= {0, 255}
    return m == 255


def _cam(scene, v, max_dim=-1):
    img, oh, ow = data_io.read_image(os.path.join(scene, "images", f"{v:08d}.jpg"), max_dim)
    k, e, d = data_io.read_cam_file(os.path.join(scene, "cams", f"{v:08d}_cam.txt"))
    return img, data_io.scale_intrinsics(k, img.shape[:2], oh, ow), e, d


def _ply(path):
    raw = open(path, "rb").read()
    head, _, body = raw.partition(b"end_header\n")
    return head + b"end_header\n", np.frombuffer(body, dtype=np.uint8).reshape(-1, 15)


def _flips_ok(got, want):
    return (got != want).sum() <= max(1, int(1e-4 * want.size))


def test_fusion_matches_the_oracle(tmp_path):
    scene = str(tmp_path / "scene")
    sc = _fusion_tree(scene)
    _run("--input-folder", scene, "--checkpoint-path", WEIGHTS, "--output-type", "fusion", *DTU_THRES)
    header, records = _ply(os.path.join(scene, "fused.ply"))
    assert header == (b"ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\n"
                      b"property float z\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n" % len(records))
    offset, frac = 0, {"photo": [], "geo": [], "final": []}
    for ref, srcs in sc["pairs"]:
        read = lambda kind, v: data_io.read_map(os.path.join(scene, kind, f"{v:08d}.pfm"))[..., 0]
        img, K, E, _ = _cam(scene, ref)
        cams = [_cam(scene, s) for s in srcs]
        ref_depth, conf = read("depth_est", ref), read("confidence", ref)
        src_depths = [read("depth_est", s) for s in srcs]
        with np.errstate(divide="ignore", invalid="ignore"):
            photo, msum, final, _ = go.fuse_reference_view(ref_depth, K, E, src_depths, [c[1] for c in cams], [c[2] for c in cams],
                                                           conf, 1.0, 0.01, 0.8, 3)
        got = {k: _mask(os.path.join(scene, "mask", f"{ref:08d}_{k}.png")) for k in ("photo", "geo", "final")}
        assert np.array_equal(got["photo"], photo)
        assert _flips_ok(got["geo"], msum >= 3) and _flips_ok(got["final"], final)
        for k in frac:
            frac[k].append(got[k].mean())
        # the records of this view: the oracle's back-projection of the command's own final mask and averaged depth
        filt = ops.geometric_filter(torch.from_numpy(ref_depth).to(DEV), torch.from_numpy(conf).to(DEV),
                                    torch.from_numpy(np.stack(src_depths)).to(DEV),
                                    ops.compose_filter_cameras(K, E, [c[1] for c in cams], [c[2] for c in cams]), 1.0, 0.01, 0.8, 3)
        assert np.array_equal(filt[2].cpu().numpy(), got["final"])
        want_v, want_c = go.fuse_points(got["final"], filt[3].cpu().numpy(), img, K, E)
        n = int(got["final"].sum())
        _check_body(records[offset:offset + n], want_v, want_c)
        offset += n
    assert offset == len(records) > 0
    for k, v in frac.items():  # both outcomes are exercised
        assert 0.05 < np.mean(v) < 0.95, (k, v)


@pytest.fixture(scope="module")
def depth_tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("depth_scene"))
    scene_cases.write_scene(root, N_VIEWS, *DEPTH_HW, n_src=N_VIEWS - 1)
    return root


def _direct_engine(scene, seed=0, n_slots=3):
    """The same decoded requests through a DepthEngine built alike: every slot filled with the first request for warm-up and
    capture, then request j on slot j % n_slots, one after another."""
    args = reconstruct.parse_args(["--checkpoint-path", WEIGHTS])
    requests = reconstruct.scan_requests(data_io.read_pair_file(os.path.join(scene, "pair.txt")), args.num_views)
    decoded = {v: _cam(scene, v) for v in range(N_VIEWS)}

    def inputs(views):
        images = [torch.from_numpy(decoded[v][0].transpose(2, 0, 1).copy()).to(DEV) for v in views]
        K = torch.from_numpy(np.stack([decoded[v][1] for v in views])).unsqueeze(0).to(DEV)
        E = torch.from_numpy(np.stack([decoded[v][2] for v in views])).unsqueeze(0).to(DEV)
        d = decoded[views[0]][3]
        return images, K, E, torch.tensor(d[:1], device=DEV), torch.tensor(d[1:2], device=DEV)

    out = {}
    with reconstruct.precision(False), torch.no_grad():
        net = reconstruct.load_network(args).to(DEV)
        eng = DepthEngine(net, 1, len(requests[0]), *DEPTH_HW, device=DEV, n_slots=n_slots, seed=seed)
        for k in range(n_slots):
            eng.set_device_inputs(k, *inputs(requests[0]))
        torch.cuda.synchronize()
        eng.prepare()
        for j, views in enumerate(requests):
            eng.set_device_inputs(j % n_slots, *inputs(views))
            depth, conf = eng.run_slot(j % n_slots)
            out[views[0]] = (depth[0, 0].cpu().numpy().copy(), conf[0].cpu().numpy().copy())
    return out


def _maps(out_dir, fmt):
    return {v: (data_io.read_map(os.path.join(out_dir, "depth_est", f"{v:08d}{fmt}")),
                data_io.read_map(os.path.join(out_dir, "confidence", f"{v:08d}{fmt}"))) for v in range(N_VIEWS)}


def _files(out_dir, sub):
    d = os.path.join(out_dir, sub)
    return {n: open(os.path.join(d, n), "rb").read() for n in sorted(os.listdir(d))}


@pytest.mark.parametrize("fmt", [".pfm", ".bin"])
def test_depth_maps_equal_a_direct_engine_run(depth_tree, tmp_path, fmt):
    args = ["--input-folder", depth_tree, "--checkpoint-path", WEIGHTS, "--output-type", "depth", "--file-format", fmt]
    stats = _run(*args, "--output-folder", tmp_path / "a")
    _run(*args, "--output-folder", tmp_path / "b")
    assert stats["depth_maps"] == N_VIEWS and not os.path.exists(tmp_path / "a" / "fused.ply")
    for sub in ("depth_est", "confidence"):
        a, b = _files(str(tmp_path / "a"), sub), _files(str(tmp_path / "b"), sub)
        assert sorted(a) == [f"{v:08d}{fmt}" for v in range(N_VIEWS)] and a == b  # a second run writes the same bytes
    got = _maps(str(tmp_path / "a"), fmt)
    want = _direct_engine(depth_tree)
    for v in range(N_VIEWS):
        assert got[v][0].shape == (*DEPTH_HW, 1) and got[v][1].shape == (*DEPTH_HW, 1)
        assert np.array_equal(got[v][0][..., 0], want[v][0]) and np.array_equal(got[v][1][..., 0], want[v][1]), v
    depth = np.stack([got[v][0] for v in range(N_VIEWS)])
    assert np.isfinite(depth).all() and (depth > 0).all()


def test_both_equals_depth_then_fusion(depth_tree, tmp_path):
    common = ["--input-folder", depth_tree, "--checkpoint-path", WEIGHTS, *DTU_THRES]
    _run(*common, "--output-folder", tmp_path / "both", "--output-type", "both")
    _run(*common, "--output-folder", tmp_path / "split", "--output-type", "depth")
    _run(*common, "--output-folder", tmp_path / "split", "--output-type", "fusion")
    for sub in ("depth_est", "confidence", "mask"):
        a, b = _files(str(tmp_path / "both"), sub), _files(str(tmp_path / "split"), sub)
        assert len(a) == (3 if sub == "mask" else 1) * N_VIEWS and a == b, sub
    a = open(tmp_path / "both" / "fused.ply", "rb").read()
    assert a == open(tmp_path / "split" / "fused.ply", "rb").read()
    assert len(_ply(str(tmp_path / "both" / "fused.ply"))[1]) > 0


def _scripted_stand_in(state):
    """A TorchScript archive whose state dict equals `state`: a tree of modules holding the tensors under the same keys (the
    native PatchmatchNet calls ctypes, which TorchScript cannot compile)."""

    class Holder(torch.nn.Module):
        def forward(self, x: torch.Tensor) -> torch.Tensor:
            return x

    root = Holder()
    for key, value in state.items():
        *path, leaf = key.split(".")
        mod = root
        for name in path:
            if name not in mod._modules:
                mod.add_module(name, Holder())
            mod = mod._modules[name]
        mod.register_buffer(leaf, value.clone())
    return torch.jit.script(root)


def test_module_checkpoint_gives_the_params_maps(depth_tree, tmp_path):
    state = torch.load(WEIGHTS, map_location="cpu")
    archive = str(tmp_path / "module.pt")
    _scripted_stand_in(state).save(archive)
    assert sorted(torch.jit.load(archive).state_dict()) == sorted(state)
    common = ["--input-folder", depth_tree, "--output-type", "depth"]
    _run(*common, "--checkpoint-path", WEIGHTS, "--output-folder", tmp_path / "params")
    _run(*common, "--checkpoint-path", archive, "--input-type", "module", "--output-folder", tmp_path / "module")
    for sub in ("depth_est", "confidence"):
        assert _files(str(tmp_path / "params"), sub) == _files(str(tmp_path / "module"), sub)


def test_chain_into_dtu_eval(tmp_path):
    data, outputs = tmp_path / "data", tmp_path / "outputs"
    _fusion_tree(data / "scan1", outputs / "scan1")
    (tmp_path / "scans.txt").write_text("scan1\n")
    stats = _run("--input-folder", data, "--output-folder", outputs, "--scan-list", tmp_path / "scans.txt",
                 "--checkpoint-path", WEIGHTS, "--output-type", "fusion", *DTU_THRES)
    assert stats["points"] > 0
    # ground truth around the fused cloud: STL = every other point, jittered; observed within 10 mm; plane below everything
    from scipy.io import savemat

    pts = data_io.read_ply_points(str(outputs / "scan1" / "fused.ply"))
    rng = np.random.RandomState(3)
    stl = (pts[::2] + rng.normal(0, 0.2, (len(pts[::2]), 3))).astype(np.float32).astype(np.float64)
    root = tmp_path / "MVS Data"
    (root / "Points" / "stl").mkdir(parents=True)
    (root / "ObsMask").mkdir()
    (root / "Points" / "stl" / "stl001_total.ply").write_bytes(dtu_cases.ply_bytes(stl, colours=False))
    res, lo, hi = 4.0, stl.min(0) - 20.0, stl.max(0) + 20.0
    dims = np.ceil((hi - lo) / res).astype(int) + 1
    mask = np.zeros(dims, dtype=bool)
    vox = np.floor((stl - lo) / res).astype(int)
    for dx in range(-3, 4):
        for dy in range(-3, 4):
            for dz in range(-3, 4):
                v = np.clip(vox + [dx, dy, dz], 0, dims - 1)
                mask[v[:, 0], v[:, 1], v[:, 2]] = True
    savemat(str(root / "ObsMask" / "ObsMask1_10.mat"), {"ObsMask": mask, "BB": np.stack([lo, hi]), "Res": res})
    savemat(str(root / "ObsMask" / "Plane1.mat"), {"P": np.array([[0.0], [0.0], [1.0], [-(stl[:, 2].min() - 10.0)]])})
    out = str(tmp_path / "dtu.json")
    assert dtu_eval.main(["--data-path", str(root), "--outputs", str(outputs), "--scans", "1", "--json", out]) == 0
    final = json.load(open(out))["final"]
    assert math.isfinite(final["acc"]) and math.isfinite(final["comp"])
