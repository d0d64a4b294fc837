"""Generate tests/golden/train_io.npz: what the UNMODIFIED reference's training code returns on seeded inputs --
MVSDataset samples (datasets/mvs.py) of a converted training tree, create_stage_images + patchmatchnet_loss with the
depth-map gradients and both metrics (train.py, models/net.py, utils.py) on float64 tensors, the network's named_parameters,
find_latest_checkpoint on a listing, and the SHA-256 of every file convert_dtu_dataset.py writes from a seeded raw tree.
The seeded inputs come from tests/train_cases.py, so the tests regenerate them; only results are stored.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet):
    python tests/golden/make_train_golden.py <path to the reference checkout>"""
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "train_io.npz")
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REPO)
sys.path.insert(1, REF)
from tests import train_cases  # noqa: E402
from datasets.mvs import MVSDataset  # noqa: E402
from models.net import PatchmatchNet, patchmatchnet_loss  # noqa: E402
from train import create_stage_images, find_latest_checkpoint  # noqa: E402
from utils import absolute_depth_error_metrics, threshold_metrics  # noqa: E402

out = {}

# ---- MVSDataset samples ----------------------------------------------------------------------------------------------
with tempfile.TemporaryDirectory() as tmp:
    train_cases.write_training_tree(tmp)
    for tag, max_dim in (("full", -1), ("scaled", 40)):
        ds = MVSDataset(tmp, num_views=2, max_dim=max_dim, scan_list=os.path.join(tmp, "scans.txt"), num_light_idx=2)
        out[f"ds_{tag}_len"] = np.int64(len(ds))
        out[f"ds_{tag}_metas"] = np.array([f"{s}|{l}|{r}|{','.join(map(str, src))}" for s, l, r, src in ds.metas])
        for i in range(len(ds)):
            try:
                s = ds[i]
            except Exception as e:  # the reference's own failure (recorded, not worked around)
                out[f"ds_{tag}_{i}_error"] = np.array(f"{type(e).__name__}: {e}")
                continue
            out[f"ds_{tag}_{i}_images"] = np.stack(s["images"])
            for k in ("intrinsics", "extrinsics", "depth_gt", "mask"):
                out[f"ds_{tag}_{i}_{k}"] = np.asarray(s[k])
            out[f"ds_{tag}_{i}_range"] = np.array([s["depth_min"], s["depth_max"]])
            out[f"ds_{tag}_{i}_filename"] = np.array(s["filename"])

# ---- loss, gradients, metrics ----------------------------------------------------------------------------------------
for c, (B, H, W) in enumerate(train_cases.LOSS_CASES):
    case = train_cases.loss_case(B, H, W, seed=100 + c)
    gt = torch.from_numpy(case["gt"])
    mask = torch.from_numpy(case["mask"])
    maps = [torch.from_numpy(m).requires_grad_(True) for m in case["maps"]]
    per_level = {l: [m for m, lv in zip(maps, train_cases.LOSS_LEVELS) if lv == l] for l in range(4)}
    depth_gt = create_stage_images(gt)
    masks = [m.bool() for m in create_stage_images(mask.double())]
    loss = patchmatchnet_loss(per_level, depth_gt, masks)
    loss.backward()
    out[f"loss_{c}"] = np.float64(loss.item())
    for k, m in enumerate(maps):
        out[f"loss_{c}_grad_{k}"] = m.grad.numpy()
    with torch.no_grad():
        for b in range(B):  # per image: the batch mean of the metrics is then a plain mean of these
            sl = slice(b, b + 1)
            for l in range(4):
                out[f"metric_{c}_{b}_abs_{l}"] = np.float64(absolute_depth_error_metrics(per_level[l][-1][sl], depth_gt[l][sl], masks[l][sl]).item())
            for t in (1, 2, 4, 8):
                r = threshold_metrics(per_level[0][-1][sl], depth_gt[0][sl], masks[0][sl], float(t))
                out[f"metric_{c}_{b}_thr_{t}"] = np.float32(r.item())

# ---- parameters ------------------------------------------------------------------------------------------------------
net = PatchmatchNet([0.005, 0.0125, 0.025], [6, 4, 2], [1, 2, 2], [8, 8, 16], [0, 8, 16], [9, 9, 9])
named = list(net.named_parameters())
out["param_names"] = np.array([n for n, _ in named])
out["param_shapes"] = np.array([",".join(map(str, p.shape)) for _, p in named])
out["state_keys"] = np.array(list(torch.nn.DataParallel(net).state_dict()))

# ---- find_latest_checkpoint ------------------------------------------------------------------------------------------
LISTINGS = [
    ["params_000001.ckpt", "params_000010.ckpt", "params_000002.ckpt", "module_000099.pt", "notes.txt"],
    ["a_b_000005.ckpt", "params_000004.ckpt", "x_3.ckpt"],
    ["module_000001.pt"],
    [],
]
for k, names in enumerate(LISTINGS):
    with tempfile.TemporaryDirectory() as tmp:
        for n in names:
            open(os.path.join(tmp, n), "w").close()
        got = find_latest_checkpoint(tmp)
        out[f"latest_{k}_listing"] = np.array(names if names else [""])
        out[f"latest_{k}"] = np.array(os.path.basename(got))

# ---- convert_dtu_dataset.py ------------------------------------------------------------------------------------------
with tempfile.TemporaryDirectory() as tmp:
    raw, conv = os.path.join(tmp, "raw"), os.path.join(tmp, "conv")
    os.makedirs(conv)
    scan_list = train_cases.write_raw_dtu_tree(raw)
    subprocess.run([sys.executable, os.path.join(REF, "convert_dtu_dataset.py"), "--input_folder", raw, "--output_folder", conv,
                    "--scan_list", scan_list], check=True, cwd=REF)
    files = sorted(os.path.relpath(os.path.join(d, f), conv) for d, _, fs in os.walk(conv) for f in fs)
    out["convert_files"] = np.array(files)
    out["convert_sha256"] = np.array([hashlib.sha256(open(os.path.join(conv, f), "rb").read()).hexdigest() for f in files])

np.savez_compressed(OUT, **out)
print(f"wrote {OUT}: {len(out)} arrays")
