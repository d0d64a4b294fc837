"""GPU tests of training: the K-L loss and metric kernels against the oracle and the reference's op sequence, reruns, the
sharded loss, a driver step's gradients, the command end to end on a seeded plane-scene training set, and overfitting."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import train_oracle
from patchmatchnet_b200 import data_io, ops, reconstruct, train
from patchmatchnet_b200.autograd import DepthLoss
from patchmatchnet_b200.net import patchmatchnet_loss
from tests import scene_cases, train_cases
from tests.geo_cases import plane_depth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LEVELS = train_cases.LOSS_LEVELS


def _case(B, H, W, seed):
    c = train_cases.loss_case(B, H, W, seed)
    gt = c["gt"].astype(np.float32)[:, 0]
    maps = [m.astype(np.float32) for m in c["maps"]]
    mask = c["mask"][:, 0]
    return gt, mask, maps


def _dev(gt, mask, maps):
    return (torch.from_numpy(gt).to(DEV), torch.from_numpy(mask.astype(np.uint8)).to(DEV), [torch.from_numpy(m).to(DEV) for m in maps])


def _reference_loss(maps, gt, mask):
    """create_stage_images + patchmatchnet_loss as train.py:145-147 run them."""
    g = [gt.unsqueeze(1)] + [F.interpolate(gt.unsqueeze(1), scale_factor=0.5 ** l, mode="nearest") for l in (1, 2, 3)]
    m = mask.unsqueeze(1).float()
    ms = [m.bool()] + [F.interpolate(m, scale_factor=0.5 ** l, mode="nearest").bool() for l in (1, 2, 3)]
    per_level = {l: [x for x, lv in zip(maps, LEVELS) if lv == l] for l in range(4)}
    return patchmatchnet_loss(per_level, g, ms)


@pytest.mark.parametrize("shape", [(1, 64, 80), (3, 37, 53), (2, 512, 640)])
def test_terms_match_the_oracle(shape):
    gt, mask, maps = _case(*shape, seed=sum(shape))
    want = train_oracle.loss_terms(maps, LEVELS, gt, mask, elem=np.float32)
    g, m, ms = _dev(gt, mask, maps)
    terms = ops.depth_loss_terms(ms, LEVELS, g, m).cpu().numpy()
    n = len(LEVELS)
    assert np.array_equal(terms[n:], want[n:])  # exact counts
    np.testing.assert_allclose(terms[:n], want[:n], rtol=1e-12, atol=0)


def test_empty_level_gives_nan():
    gt, mask, maps = _case(2, 64, 80, seed=3)
    mask[:, ::8, ::8] = False  # every level-3 pixel is masked out; the other levels keep some
    g, m, ms = _dev(gt, mask, maps)
    terms = ops.depth_loss_terms(ms, LEVELS, g, m)
    assert float(terms[len(LEVELS) + 3]) == 0 and float(terms[len(LEVELS)]) > 0
    loss = DepthLoss.apply(LEVELS, g, m, None, 1.0, *ms)
    assert torch.isnan(loss) and torch.isnan(_reference_loss(ms, g, m.bool()))


@pytest.mark.parametrize("shape", [(2, 64, 80), (3, 37, 53), (2, 512, 640)])
def test_loss_and_gradients_match_the_reference_ops(shape):
    gt, mask, maps = _case(*shape, seed=11 + shape[0])
    g, m, ms = _dev(gt, mask, maps)
    a = [x.clone().requires_grad_(True) for x in ms]
    b = [x.clone().requires_grad_(True) for x in ms]
    mine = DepthLoss.apply(LEVELS, g, m, None, 1.0, *a)
    ref = _reference_loss(b, g, m.bool())
    assert mine.dtype == torch.float32
    assert abs(float(mine.detach()) - float(ref.detach())) <= 1e-6 * abs(float(ref.detach()))
    (3.0 * mine).backward()
    (3.0 * ref).backward()
    for x, y in zip(a, b):
        torch.testing.assert_close(x.grad, y.grad, rtol=1e-6, atol=1e-6 * float(y.grad.abs().max()))


def test_reruns_are_bit_identical():
    gt, mask, maps = _case(2, 512, 640, seed=5)
    g, m, ms = _dev(gt, mask, maps)
    t0 = ops.depth_loss_terms(ms, LEVELS, g, m)
    g0 = ops.depth_loss_backward(ms, LEVELS, g, m, t0, torch.ones((), device=DEV), 1.0)
    last = [ms[max(k for k, lv in enumerate(LEVELS) if lv == l)] for l in range(4)]
    r0 = ops.depth_metrics(last, g, m)
    for _ in range(3):
        t1 = ops.depth_loss_terms(ms, LEVELS, g, m)
        assert torch.equal(t0, t1)
        for x, y in zip(g0, ops.depth_loss_backward(ms, LEVELS, g, m, t1, torch.ones((), device=DEV), 1.0)):
            assert torch.equal(x, y)
        assert torch.equal(r0, ops.depth_metrics(last, g, m))


@pytest.mark.parametrize("shape", [(2, 64, 80), (3, 37, 53), (4, 512, 640)])
def test_metrics_match_the_reference_formulas(shape):
    gt, mask, maps = _case(*shape, seed=21)
    g, m, ms = _dev(gt, mask, maps)
    last = [ms[max(k for k, lv in enumerate(LEVELS) if lv == l)] for l in range(4)]
    raw = ops.depth_metrics(last, g, m)
    gts = [g] + [F.interpolate(g.unsqueeze(1), scale_factor=0.5 ** l, mode="nearest")[:, 0] for l in (1, 2, 3)]
    mks = [m.bool()] + [F.interpolate(m.unsqueeze(1).float(), scale_factor=0.5 ** l, mode="nearest")[:, 0].bool() for l in (1, 2, 3)]
    for b in range(shape[0]):
        for l in range(4):
            d, t, k = last[l][b, 0], gts[l][b], mks[l][b]
            assert float(raw[b, 4 + l]) == float(k.sum())
            want = float(torch.mean((d[k] - t[k]).abs()))  # utils.py:220-221
            assert abs(float(raw[b, l] / raw[b, 4 + l]) - want) <= 1e-6 * want
        for j, thr in enumerate(train.THRESHOLDS):
            d, t, k = last[0][b, 0], gts[0][b], mks[0][b]
            want = torch.mean((torch.abs(d[k] - t[k]).float() > float(thr)).float())  # utils.py:203-206
            got = train.threshold_rates(raw[b, 8 + j], raw[b, 4])
            assert got.dtype == torch.float32 and torch.equal(got, want), (b, thr, float(got), float(want))


def test_two_shards_give_the_full_batch_loss():
    gt, mask, maps = _case(4, 64, 80, seed=9)
    g, m, ms = _dev(gt, mask, maps)
    full = [x.clone().requires_grad_(True) for x in ms]
    loss = DepthLoss.apply(LEVELS, g, m, None, 1.0, *full)
    loss.backward()
    # two ranks of two images each: terms summed before the loss is formed, backward scaled by the world size, then averaged
    halves = [[x[s].clone().requires_grad_(True) for x in ms] for s in (slice(0, 2), slice(2, 4))]
    local = [ops.depth_loss_terms(h, LEVELS, g[s], m[s]) for h, s in zip(halves, (slice(0, 2), slice(2, 4)))]
    total = local[0] + local[1]
    for h, s in zip(halves, (slice(0, 2), slice(2, 4))):
        shard_loss = DepthLoss.apply(LEVELS, g[s], m[s], lambda t: t.copy_(total), 2.0, *h)
        assert abs(float(shard_loss) - float(loss)) <= 1e-12 * abs(float(loss))
        shard_loss.backward()
    for k, x in enumerate(full):
        merged = torch.cat([halves[0][k].grad, halves[1][k].grad]) / 2.0
        torch.testing.assert_close(merged, x.grad, rtol=1e-6, atol=1e-6 * float(x.grad.abs().max()))


# ---- the driver ---------------------------------------------------------------------------------------------------------

H, W = 128, 160


def _write_plane_training_set(root, scans=("scan1", "scan2"), n_views=4, lights=2):
    from PIL import Image

    cams = scene_cases.cameras(n_views, H, W)
    for scan in scans:
        base = os.path.join(root, scan)
        for sub in ["cams", "depth_gt"] + [os.path.join("images", str(i)) for i in range(lights)]:
            os.makedirs(os.path.join(base, sub), exist_ok=True)
        with open(os.path.join(base, "pair.txt"), "w") as f:
            f.write(scene_cases.pair_text(scene_cases.all_pairs(n_views, 2)))
        for v, (K, E) in enumerate(cams):
            with open(os.path.join(base, "cams", "%08d_cam.txt" % v), "w") as f:
                f.write(scene_cases.cam_text(K, E))
            depth = plane_depth(K, E, H, W, scene_cases.PLANE_N, scene_cases.PLANE_D0).astype(np.float32)
            depth[: H // 8] = 0.0  # a strip without ground truth: the masks are partial
            data_io.save_map(os.path.join(base, "depth_gt", "%08d.pfm" % v), depth)
            tex = scene_cases.texture(K, E, H, W)
            for light in range(lights):
                img = np.clip(tex.astype(np.int32) + 10 * light, 0, 255).astype(np.uint8)
                Image.fromarray(img).save(os.path.join(base, "images", str(light), "%08d.jpg" % v), quality=95)
    with open(os.path.join(root, "train.txt"), "w") as f:
        f.write("\n".join(scans) + "\n")
    with open(os.path.join(root, "val.txt"), "w") as f:
        f.write(scans[0] + "\n")
    return cams


@pytest.fixture(scope="module")
def plane_set(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("plane_train"))
    _write_plane_training_set(root)
    return root


def _batch(root, idx):
    ds = train.MVSDataset(root, num_views=2, max_dim=-1, scan_list=os.path.join(root, "train.txt"), num_light_idx=2)
    return train.collate([ds[i] for i in idx])


def _net():
    torch.manual_seed(1)
    return train.build_network(train.parse_args([])).to(DEV).train()


@pytest.fixture
def fp32_accurate():
    with reconstruct.precision(False):
        yield


def test_driver_step_gradients_match_the_reference_loss(plane_set, fp32_accurate):
    sample = _batch(plane_set, [0, 5])
    net = _net()
    sess = train.Session(DEV, 0, 1, train.loss_levels([1, 2, 2]))
    opt = torch.optim.SGD(net.parameters(), lr=0.0)
    torch.cuda.manual_seed(3)
    loss, _ = train.process_batch(net, sample, sess, opt)
    mine = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
    net.zero_grad(set_to_none=True)
    s = train.to_device(sample, DEV)
    torch.cuda.manual_seed(3)
    _, _, per_stage = net(list(s["images"]), s["intrinsics"], s["extrinsics"], s["depth_min"], s["depth_max"])
    gt = s["depth_gt"].unsqueeze(1)
    gts = [gt] + [F.interpolate(gt, scale_factor=0.5 ** l, mode="nearest") for l in (1, 2, 3)]
    mf = s["mask"].unsqueeze(1).float()
    masks = [mf.bool()] + [F.interpolate(mf, scale_factor=0.5 ** l, mode="nearest").bool() for l in (1, 2, 3)]
    ref = patchmatchnet_loss(per_stage, gts, masks)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert len(mine) > 100
    # a tensor whose true gradient is zero (the bias in front of a softmax) carries only rounding noise, so the tolerance has a
    # floor at 1e-8 of the network's largest gradient
    floor = 1e-8 * max(float(p.grad.abs().max()) for p in net.parameters() if p.grad is not None)
    for n, p in net.named_parameters():
        if n not in mine:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0
            continue
        g = p.grad
        tol = max(1e-4 * float(g.abs().max()), floor)
        assert float((mine[n] - g).abs().max()) <= tol, n


def _args(root, out, *extra):
    return train.parse_args(["--input-folder", root, "--output-folder", out, "--train-list", os.path.join(root, "train.txt"),
                             "--test-list", os.path.join(root, "val.txt"), "--num-views", "2", "--num-light-idx", "2",
                             "--batch-size", "2", "--summary-freq", "2", "--num-workers", "2", "--image-max-dim", "-1", *extra])


def test_command_end_to_end(plane_set, tmp_path, capsys):
    out = str(tmp_path / "run")
    res = train.run(_args(plane_set, out, "--epochs", "2"))
    assert res["start_epoch"] == 0
    files = sorted(os.listdir(out))
    assert files == ["module_000000.pt", "module_000001.pt", "params_000000.ckpt", "params_000001.ckpt", "train_log.jsonl"]
    ck = torch.load(os.path.join(out, "params_000001.ckpt"), map_location="cpu")
    assert ck["epoch"] == 1 and all(k.startswith("module.") for k in ck["model"])
    steps_per_epoch = 16 // 2
    assert {int(v["step"]) for v in ck["optimizer"]["state"].values()} == {2 * steps_per_epoch}
    lines = [json.loads(l) for l in open(os.path.join(out, "train_log.jsonl"))]
    tags = {l["tag"] for l in lines}
    for mode in ("train", "test", "full_test"):
        for t in train.SCALAR_TAGS:
            assert f"{mode}/{t}" in tags
    assert all(np.isfinite(l["value"]) for l in lines)
    # the exported module carries the checkpoint's weights
    module = torch.jit.load(os.path.join(out, "module_000001.pt"), map_location="cpu").state_dict()
    assert sorted(module) == sorted(k[7:] for k in ck["model"])
    for k, v in module.items():
        assert torch.equal(v, ck["model"]["module." + k]), k
    # --resume continues at the next epoch from the stored optimizer state
    res = train.run(_args(plane_set, out, "--epochs", "3", "--resume"))
    assert res["start_epoch"] == 2
    ck2 = torch.load(os.path.join(out, "params_000002.ckpt"), map_location="cpu")
    assert ck2["epoch"] == 2 and {int(v["step"]) for v in ck2["optimizer"]["state"].values()} == {3 * steps_per_epoch}
    # --mode test validates one checkpoint
    capsys.readouterr()
    res = train.run(_args(plane_set, out, "--mode", "test", "--checkpoint-path", os.path.join(out, "params_000001.ckpt")))
    assert "final" in capsys.readouterr().out and set(res["final"]) == set(train.SCALAR_TAGS)
    assert all(np.isfinite(v) for v in res["final"].values())
    # reconstruct reads the exported module as it reads the checkpoint
    scene = str(tmp_path / "scene")
    scene_cases.write_scene(scene, 3, H, W, n_src=2)
    common = ["--input-folder", scene, "--output-type", "depth", "--num-views", "2"]
    reconstruct.reconstruct(reconstruct.parse_args(common + ["--checkpoint-path", os.path.join(out, "params_000001.ckpt"),
                                                            "--output-folder", str(tmp_path / "p")]), log=lambda *a: None)
    reconstruct.reconstruct(reconstruct.parse_args(common + ["--checkpoint-path", os.path.join(out, "module_000001.pt"), "--input-type",
                                                            "module", "--output-folder", str(tmp_path / "m")]), log=lambda *a: None)
    for v in range(3):
        for sub in ("depth_est", "confidence"):
            a = open(tmp_path / "p" / sub / ("%08d.pfm" % v), "rb").read()
            assert a == open(tmp_path / "m" / sub / ("%08d.pfm" % v), "rb").read()


def test_overfitting_one_sample_lowers_the_loss(plane_set, fp32_accurate):
    sample = _batch(plane_set, [1, 6])
    net = _net()
    sess = train.Session(DEV, 0, 1, train.loss_levels([1, 2, 2]))
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    losses = []
    for step in range(40):
        torch.cuda.manual_seed(step)
        loss, _ = train.process_batch(net, sample, sess, opt)
        losses.append(float(loss))
    assert np.isfinite(losses).all()
    assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
