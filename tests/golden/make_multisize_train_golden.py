"""Generate tests/golden/multisize_train_case.pt from the UNMODIFIED reference: training on requests whose views differ in
size, and the ETH3D training-set converter.

Needs a checkout of the reference (FangjinhuaWang/PatchmatchNet) and cv2; tests/golden/weights_000007.pt must exist
(make_golden.py writes it):

    python tests/golden/make_multisize_train_golden.py <path to the reference checkout>

Two parts, inputs from tests/multisize_train_cases.py:
    train     PatchmatchNet (CPU, train() mode) on the 1 + 4 view request of tests/multisize_cases.py (B = 1) and on a B = 2
              request whose samples agree view by view; patchmatchnet_loss against per-level ground truth, backward.  Per
              case: the loss, the per-stage maps and every named parameter's gradient (None when it gets none), as
              multisize_train_cases.pack_grads stores them (12 bits of each tensor's largest magnitude).  The
              stage-3 random draw is the reference's own torch.rand after torch.manual_seed(case["seed"]), recorded in
              the case as rand48 (as make_multisize_golden.py does).
    eth3d     convert_eth3d_dataset.py on a small synthetic tree (index2prefix.txt, "_undistorted" image names): the
              relative path and SHA-256 of every file it writes.
"""
import hashlib
import os
import subprocess
import sys
import tempfile
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
if len(sys.argv) != 2:
    raise SystemExit(__doc__)
REFERENCE = os.path.abspath(sys.argv[1])
sys.path.insert(1, REFERENCE)
warnings.filterwarnings("ignore")

from models.net import PatchmatchNet as RefNet, patchmatchnet_loss  # noqa: E402

from tests import multisize_train_cases, pm_cases  # noqa: E402


def train_part(B):
    weights = torch.load(os.path.join(HERE, "weights_000007.pt"), map_location="cpu")
    net = RefNet(**pm_cases.NET_KWARGS)
    net.load_state_dict(weights, strict=True)
    net.train()
    case = multisize_train_cases.make_case(B)
    torch.manual_seed(case["seed"])
    _, _, per_stage = net([im.clone() for im in case["images"]], case["intrinsics"].clone(), case["extrinsics"].clone(),
                          case["depth_min"], case["depth_max"])
    loss = patchmatchnet_loss(per_stage, case["gts"], case["masks"])
    loss.backward()
    print("train B=%d loss %.6f" % (B, float(loss)))
    return {"checksum": pm_cases.checksum({k: case[k] for k in ("images", "intrinsics", "extrinsics", "depth_min", "depth_max", "rand48")}),
            "loss": loss.detach().clone(),
            "per_stage": {k: [d.detach().clone() for d in v] for k, v in per_stage.items()},
            "grads": multisize_train_cases.pack_grads({k: p.grad for k, p in net.named_parameters()})}


def eth3d_part():
    with tempfile.TemporaryDirectory() as tmp:
        raw, conv = os.path.join(tmp, "raw"), os.path.join(tmp, "conv")
        os.makedirs(conv)
        scan_list = multisize_train_cases.write_raw_eth3d_tree(raw)
        subprocess.run([sys.executable, os.path.join(REFERENCE, "convert_eth3d_dataset.py"), "--input_folder", raw,
                        "--output_folder", conv, "--scan_list", scan_list], check=True, cwd=REFERENCE)
        files = sorted(os.path.relpath(os.path.join(d, f), conv) for d, _, fs in os.walk(conv) for f in fs)
        print("eth3d", len(files), "files")
        return {"files": files, "sha256": [hashlib.sha256(open(os.path.join(conv, f), "rb").read()).hexdigest() for f in files]}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"train_b1": train_part(1), "train_b2": train_part(2), "eth3d": eth3d_part()}
    torch.save(out, os.path.join(HERE, "multisize_train_case.pt"))
    print("multisize_train_case.pt", os.path.getsize(os.path.join(HERE, "multisize_train_case.pt")))
