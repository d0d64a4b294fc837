"""CPU tests of training: the oracle against the reference's loss, gradients and metrics (tests/golden/train_io.npz), the
dataset, parser, learning-rate schedule, checkpoint keys, find_latest_checkpoint, the batch sampler, the two-rank loss-term
combination, the ABI's argument checks and convert_dtu's bytes."""
import ctypes
import hashlib
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import train_oracle
from patchmatchnet_b200 import _native, convert_dtu, train
from tests import train_cases

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_io.npz"))


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300)))


@pytest.mark.parametrize("c", range(len(train_cases.LOSS_CASES)))
def test_oracle_equals_reference_loss_gradients_and_metrics(c):
    B, H, W = train_cases.LOSS_CASES[c]
    case = train_cases.loss_case(B, H, W, seed=100 + c)
    loss, grads = train_oracle.loss_and_grads(case["maps"], train_cases.LOSS_LEVELS, case["gt"], case["mask"])
    assert _rel(loss, GOLDEN[f"loss_{c}"]) <= 1e-12
    for k, g in enumerate(grads):
        want = GOLDEN[f"loss_{c}_grad_{k}"]
        assert g.shape == want.shape
        np.testing.assert_allclose(g, want, rtol=1e-12, atol=1e-300)
    per_level = {l: case["maps"][max(k for k, lv in enumerate(train_cases.LOSS_LEVELS) if lv == l)] for l in range(4)}
    got = train_oracle.metrics(per_level, case["gt"], case["mask"])
    for b in range(B):
        for l in range(4):
            assert _rel(got[f"depth-error-stage-{l}"][b], GOLDEN[f"metric_{c}_{b}_abs_{l}"]) <= 1e-12
        for t in (1, 2, 4, 8):
            assert got[f"threshold-{t}mm-error"][b] == GOLDEN[f"metric_{c}_{b}_thr_{t}"]  # bit for bit (float32)


def test_oracle_float32_terms_stay_close_to_float64():
    case = train_cases.loss_case(2, 64, 80, seed=100)
    t64 = train_oracle.loss_terms(case["maps"], train_cases.LOSS_LEVELS, case["gt"], case["mask"])
    t32 = train_oracle.loss_terms([m.astype(np.float32) for m in case["maps"]], train_cases.LOSS_LEVELS, case["gt"].astype(np.float32),
                                  case["mask"], elem=np.float32)
    assert np.array_equal(t64[6:], t32[6:]) and _rel(t32[:6], t64[:6]) < 1e-4


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("train_tree"))
    train_cases.write_training_tree(root)
    return root


def test_dataset_equals_reference_samples(tree):
    ds = train.MVSDataset(tree, num_views=2, max_dim=-1, scan_list=os.path.join(tree, "scans.txt"), num_light_idx=2)
    assert len(ds) == int(GOLDEN["ds_full_len"])
    assert [f"{s}|{l}|{r}|{','.join(map(str, src))}" for s, l, r, src in ds.metas] == list(GOLDEN["ds_full_metas"])
    for i in range(len(ds)):
        s = ds[i]
        assert np.array_equal(np.stack(s["images"]), GOLDEN[f"ds_full_{i}_images"])
        for k in ("intrinsics", "extrinsics", "depth_gt", "mask"):
            got, want = np.asarray(s[k]), GOLDEN[f"ds_full_{i}_{k}"]
            assert got.dtype == want.dtype and np.array_equal(got, want), (i, k)
        assert np.array_equal(np.array([s["depth_min"], s["depth_max"]]), GOLDEN[f"ds_full_{i}_range"])
        assert s["filename"] == str(GOLDEN[f"ds_full_{i}_filename"])


def test_dataset_rescaled_ground_truth_keeps_its_channel(tree):
    """The reference fails on a max_dim that rescales depth_gt (cv2.resize drops the channel axis before its transpose);
    here the sample carries the rescaled map as [1,h,w] and its mask."""
    assert "axes don't match" in str(GOLDEN["ds_scaled_0_error"])
    ds = train.MVSDataset(tree, num_views=2, max_dim=40, scan_list=os.path.join(tree, "scans.txt"), num_light_idx=2)
    s = ds[0]
    assert s["images"][0].shape == (3, 30, 40) and s["depth_gt"].shape == (1, 30, 40)
    assert np.array_equal(s["mask"], s["depth_gt"] >= s["depth_min"])
    full = train.MVSDataset(tree, num_views=2, max_dim=-1, scan_list=os.path.join(tree, "scans.txt"), num_light_idx=2)[0]
    assert np.allclose(s["intrinsics"][:, :2], full["intrinsics"][:, :2] * (40 / 64))


def test_dataset_missing_ground_truth_names_the_path(tree, tmp_path):
    import shutil

    root = str(tmp_path / "t")
    shutil.copytree(tree, root)
    gone = os.path.join(root, "scan2", "depth_gt", "00000001.pfm")
    os.remove(gone)
    ds = train.MVSDataset(root, num_views=2, scan_list=os.path.join(root, "scans.txt"), num_light_idx=2)
    assert ds.metas[9][0] == "scan2" and ds.metas[9][2] == 1
    with pytest.raises(FileNotFoundError, match=gone):
        ds[9]


def test_parser_defaults_and_errors(tmp_path):
    a = train.parse_args([])
    assert (a.mode, a.output_folder, a.checkpoint_path, a.num_views, a.image_max_dim, a.num_light_idx, a.batch_size) == \
        ("train", "", "", 5, 640, -1, 12)
    assert (a.resume, a.epochs, a.learning_rate, a.lr_epochs, a.weight_decay, a.summary_freq, a.save_freq, a.rand_seed) == \
        (False, 16, 0.001, "10,12,14:2", 0.0, 20, 1, 1)
    assert a.patchmatch_interval_scale == [0.005, 0.0125, 0.025] and a.propagation_range == [6, 4, 2]
    assert a.patchmatch_iteration == [1, 2, 2] and a.patchmatch_num_sample == [8, 8, 16]
    assert a.propagate_neighbors == [0, 8, 16] and a.evaluate_neighbors == [9, 9, 9]
    assert a.tf32 is False and a.num_workers == 8
    with pytest.raises(Exception, match="Invalid input folder: nowhere"):
        train.check_args(train.parse_args(["--input-folder", "nowhere"]))
    (tmp_path / "l.txt").write_text("scan1\n")
    with pytest.raises(Exception, match="Invalid training scan list file: x.txt"):
        train.check_args(train.parse_args(["--input-folder", str(tmp_path), "--train-list", "x.txt"]))
    with pytest.raises(Exception, match="Invalid validation scan list file: y.txt"):
        train.check_args(train.parse_args(["--input-folder", str(tmp_path), "--train-list", str(tmp_path / "l.txt"), "--test-list", "y.txt"]))
    a = train.parse_args(["--input-folder", str(tmp_path), "--train-list", str(tmp_path / "l.txt"), "--test-list", str(tmp_path / "l.txt")])
    train.check_args(a)
    assert a.output_folder == str(tmp_path)


def _lrs(start: int, opt_state=None, epochs: int = 16):
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=1e-3)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    sched = train.make_scheduler(opt, "10,12,14:2", start)
    out = {}
    for e in range(start, epochs):
        sched.step()
        out[e] = opt.param_groups[0]["lr"]
        if e == 9:
            saved = opt.state_dict()
    return out, (saved if start <= 9 else None)


def test_learning_rate_schedule_fresh_and_resumed():
    fresh, at9 = _lrs(0)
    for e in range(16):
        assert fresh[e] == pytest.approx(1e-3 * 0.5 ** sum(m <= e + 1 for m in (10, 12, 14)), rel=1e-12)
    assert fresh[9] == pytest.approx(5e-4) and fresh[10] == pytest.approx(5e-4)
    resumed, _ = _lrs(10, at9)  # resuming at a milestone epoch decays once more, as the reference does
    assert resumed[10] == pytest.approx(2.5e-4)
    for e in range(10, 16):
        assert resumed[e] == pytest.approx(fresh[e] / 2)
    p = torch.nn.Parameter(torch.zeros(1))
    opt = torch.optim.Adam([p], lr=1e-3)
    sched = train.make_scheduler(opt, "10,12,14:2", 0)
    for e in range(11):
        sched.step()
    resumed11, _ = _lrs(11, opt.state_dict())
    for e in range(11, 16):
        assert resumed11[e] == pytest.approx(fresh[e])


def test_checkpoint_keys_follow_the_reference():
    net = train.build_network(train.parse_args([]))
    names = [n for n, _ in net.named_parameters()]
    assert names == list(GOLDEN["param_names"])
    assert [",".join(map(str, p.shape)) for _, p in net.named_parameters()] == list(GOLDEN["param_shapes"])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    state = train.checkpoint_state(net, opt, 3)
    assert list(state["model"]) == list(GOLDEN["state_keys"]) and all(k.startswith("module.") for k in state["model"])
    assert state["epoch"] == 3 and len(state["optimizer"]["param_groups"][0]["params"]) == len(names)


def test_find_latest_checkpoint_matches_reference(tmp_path):
    k = 0
    while f"latest_{k}" in GOLDEN.files:
        d = tmp_path / str(k)
        d.mkdir()
        for n in GOLDEN[f"latest_{k}_listing"]:
            if n:
                (d / str(n)).write_text("")
        got = train.find_latest_checkpoint(str(d))
        assert os.path.basename(got) == str(GOLDEN[f"latest_{k}"])
        k += 1
    assert k == 4


@pytest.mark.parametrize("n,B,world", [(17, 4, 1), (17, 4, 2), (16, 5, 3), (9, 8, 8), (3, 4, 2)])
def test_batch_sampler_partitions_global_batches(n, B, world):
    for shuffle in (True, False):
        samplers = [train.GlobalBatchSampler(n, B, shuffle=shuffle, drop_last=shuffle, seed=5, rank=r, world=world) for r in range(world)]
        for epoch in (0, 1):
            for s in samplers:
                s.set_epoch(epoch)
            per_rank = [list(s) for s in samplers]
            globals_ = samplers[0].global_batches()
            assert all(s.global_batches() == globals_ for s in samplers)  # every rank draws the same permutation
            assert all(len(p) == len(samplers[0]) == len(globals_) for p in per_rank)
            for j, batch in enumerate(globals_):
                assert sum((p[j] for p in per_rank), []) == batch  # rank slices, in order, make the global batch
                sizes = [len(p[j]) for p in per_rank]
                assert max(sizes) - min(sizes) <= 1
            flat = sum(globals_, [])
            assert len(set(flat)) == len(flat) and (shuffle or flat == list(range(n)))
        if shuffle:
            assert len(samplers[0]) == n // B


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _terms_worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from patchmatchnet_b200.autograd import loss_from_terms

        sess = train.Session(torch.device("cpu"), rank, world, train_cases.LOSS_LEVELS)
        n = len(sess.loss_levels)
        # stand-in term buffers (the loss kernels fill the real ones): the two shards' sums add up to the global batch's
        full = torch.tensor([3.0, 5.0, 7.0, 11.0, 13.0, 17.0, 40.0, 10.0, 4.0, 2.0], dtype=torch.float64)
        share = torch.tensor([1.0, 2.0, 3.0, 4.0, 5.0, 6.0, 15.0, 3.0, 1.0, 1.0], dtype=torch.float64)
        terms = share.clone() if rank == 0 else full - share
        sess.all_reduce(terms)
        loss = loss_from_terms(terms, sess.loss_levels)
        want = sum(float(full[m] / full[n + l]) for m, l in enumerate(sess.loss_levels))
        ok = loss.dtype == torch.float32 and abs(float(loss) - want) <= 1e-6 * want
        # a rank with an empty share of a small last validation batch contributes zeros to both collectives
        if rank == 1:
            empty_loss, scalars = train.process_batch(None, None, sess)
            extra = scalars[1:].tolist()
        else:
            t = full.clone()
            sess.all_reduce(t)
            sums = torch.tensor([2.0] * 8 + [4.0], dtype=torch.float64)
            sess.all_reduce(sums)
            empty_loss, extra = loss_from_terms(t, sess.loss_levels), (sums[:8] / sums[8]).tolist()
        q.put((rank, ok, float(empty_loss), extra))
    except Exception as e:  # pragma: no cover
        q.put((rank, repr(e), None, None))
    finally:
        dist.destroy_process_group()


def test_two_rank_loss_terms_combine_to_the_global_loss():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_terms_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=180) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert [r[1] for r in res] == [True, True], res
    assert res[0][2] == res[1][2] and res[0][3] == res[1][3] == [0.5] * 8  # both ranks hold the same global-batch values


def _lib():
    _native.build_library()
    return _native.lib()


def test_abi_argument_checks():
    lib = _lib()
    lv = (ctypes.c_int * 17)(*([0] * 17))
    assert lib.pmb200_depth_loss_workspace_bytes(lv, 6, 2, 64, 80) > 0
    assert lib.pmb200_depth_loss_workspace_bytes(lv, 0, 2, 64, 80) == -1
    assert lib.pmb200_depth_loss_workspace_bytes(lv, 17, 2, 64, 80) == -1
    for B, H, W in ((0, 64, 80), (2, 0, 80), (2, 64, -1)):
        assert lib.pmb200_depth_loss_workspace_bytes(lv, 6, B, H, W) == -1
    bad = (ctypes.c_int * 2)(0, 4)
    assert lib.pmb200_depth_loss_workspace_bytes(bad, 2, 1, 64, 80) == -1
    bad = (ctypes.c_int * 2)(-1, 0)
    assert lib.pmb200_depth_loss_workspace_bytes(bad, 2, 1, 64, 80) == -1
    assert lib.pmb200_depth_loss_workspace_bytes(None, 2, 1, 64, 80) == -1
    fake = 1 << 20  # never dereferenced: every call below is rejected before a launch
    ptrs, keep = _native.pointer_array([fake] * 2)
    lv2 = (ctypes.c_int * 2)(0, 1)
    need = lib.pmb200_depth_loss_workspace_bytes(lv2, 2, 1, 64, 80)
    assert lib.pmb200_depth_loss(ptrs, lv2, 2, fake, fake, 1, 64, 80, fake, fake, need - 8, None) == -1  # workspace too small
    assert lib.pmb200_depth_loss(ptrs, lv2, 2, None, fake, 1, 64, 80, fake, fake, need, None) == -1
    assert lib.pmb200_depth_loss(ptrs, lv2, 2, fake, fake, 1, 64, 80, None, fake, need, None) == -1
    assert lib.pmb200_depth_loss(None, lv2, 2, fake, fake, 1, 64, 80, fake, fake, need, None) == -1
    nulls, keep2 = _native.pointer_array([fake, 0])
    assert lib.pmb200_depth_loss(nulls, lv2, 2, fake, fake, 1, 64, 80, fake, fake, need, None) == -1
    assert lib.pmb200_depth_loss_backward(ptrs, lv2, 2, fake, fake, 1, 64, 80, fake, fake, 1.0, nulls, None) == -1
    assert lib.pmb200_depth_loss_backward(ptrs, lv2, 0, fake, fake, 1, 64, 80, fake, fake, 1.0, ptrs, None) == -1
    assert lib.pmb200_depth_loss_backward(ptrs, lv2, 2, fake, fake, 1, 64, 80, None, fake, 1.0, ptrs, None) == -1
    m4, keep4 = _native.pointer_array([fake] * 4)
    thr = (ctypes.c_float * 9)(*([1.0] * 9))
    assert lib.pmb200_depth_metrics(m4, fake, fake, 1, 64, 80, thr, 9, fake, None) == -1
    assert lib.pmb200_depth_metrics(m4, fake, fake, 0, 64, 80, thr, 4, fake, None) == -1
    assert lib.pmb200_depth_metrics(m4, fake, None, 1, 64, 80, thr, 4, fake, None) == -1
    m4n, keep5 = _native.pointer_array([fake, fake, 0, fake])
    assert lib.pmb200_depth_metrics(m4n, fake, fake, 1, 64, 80, thr, 4, fake, None) == -1
    assert "depth_metrics" in lib.pmb200_last_error().decode()


def test_ops_reject_cpu_tensors():
    from patchmatchnet_b200 import ops

    gt = torch.ones(1, 16, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.depth_loss_terms([gt], [0], gt, torch.ones(1, 16, 16, dtype=torch.uint8))


def test_convert_dtu_writes_the_reference_bytes(tmp_path):
    raw, conv = str(tmp_path / "raw"), tmp_path / "conv"
    conv.mkdir()
    scan_list = train_cases.write_raw_dtu_tree(raw)
    assert convert_dtu.main(["--input-folder", raw, "--output-folder", str(conv), "--scan-list", scan_list]) == 0
    files = sorted(os.path.relpath(os.path.join(d, f), conv) for d, _, fs in os.walk(conv) for f in fs)
    assert files == list(GOLDEN["convert_files"])
    for f, want in zip(files, GOLDEN["convert_sha256"]):
        assert hashlib.sha256(open(os.path.join(conv, f), "rb").read()).hexdigest() == want, f


def test_convert_dtu_messages(tmp_path):
    with pytest.raises(Exception, match="^Invalid input folder$"):
        convert_dtu.main(["--input-folder", str(tmp_path / "x")])
    with pytest.raises(Exception, match="^Invalid output folder$"):
        convert_dtu.main(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path / "x")])
    with pytest.raises(Exception, match="^Invalid input scan list$"):
        convert_dtu.main(["--input-folder", str(tmp_path), "--output-folder", str(tmp_path), "--scan-list", "nope.txt"])


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the machine without CUDA")
def test_train_raises_before_writing_without_cuda(tree, tmp_path):
    out = tmp_path / "out"
    args = train.parse_args(["--input-folder", tree, "--output-folder", str(out), "--train-list", os.path.join(tree, "scans.txt"),
                             "--test-list", os.path.join(tree, "scans.txt")])
    with pytest.raises(RuntimeError, match="CUDA"):
        train.run(args)
    assert not out.exists()
