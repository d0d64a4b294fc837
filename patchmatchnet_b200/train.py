"""Training and validation from a dataset folder on this project's kernels -- the counterpart of the reference's train.py.

    python -m patchmatchnet_b200.train --input-folder dtu_train --output-folder runs/dtu --train-list lists/dtu/train.txt \\
        --test-list lists/dtu/val.txt --num-views 4 --batch-size 4 --epochs 8 --num-light-idx 7
    python -m torch.distributed.run --nproc-per-node 8 -m patchmatchnet_b200.train ...        # one process per GPU (NCCL)

Input per scan (datasets/mvs.py): pair.txt, images/[light/]%08d.jpg (--image-extension), cams/%08d_cam.txt, depth_gt/%08d.pfm.  Output in the
output folder: params_%06d.ckpt ({"epoch", "model", "optimizer"}; model keys carry the reference's DataParallel "module."
prefix, in its named_parameters order), module_%06d.pt (the eval-mode network scripted with TorchScript) and
train_log.jsonl (one line per scalar: {"tag", "step", "value"}, the reference's TensorBoard tags).

One step: the network forward, autograd.DepthLoss (the K-L loss kernels: no boolean indexing, no host round trip), the
backward, the optimiser step, and ops.depth_metrics for the logged scalars.  The printed loss is the step's one host
synchronisation; scalars are read back only when they are written.

Several GPUs follow nn.DataParallel's semantics (train.py:282): every rank draws the same permutation, global batch j is
perm[jB:(j+1)B] and each rank takes its distributed.shard_range slice; BatchNorm statistics are per shard; the loss terms
are summed over ranks before the loss is formed, the backward is scaled by the world size and FlatGradAllReduce averages, so
the gradient is that of the one global-batch loss.  Only rank 0 writes files and prints.
"""
from __future__ import annotations

import argparse
import datetime
import json
import os
import sys
import time
from typing import Callable, Dict, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset, Sampler, default_collate

from . import data_io, ops
from . import distributed as pmd
from .autograd import DepthLoss, loss_from_terms
from .net import PatchmatchNet, load_reference_state
from .reconstruct import precision

Tensor = torch.Tensor

THRESHOLDS = (1, 2, 4, 8)
SCALAR_TAGS = ["loss"] + [f"depth-error-stage-{l}" for l in range(4)] + [f"threshold-{t}mm-error" for t in THRESHOLDS]


def build_parser() -> argparse.ArgumentParser:
    """train.py:195-233 in this project's hyphen style, same defaults; plus --tf32 and --num-workers."""
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.train", description="PatchMatchNet for high-resolution multi-view stereo")
    ap.add_argument("--mode", type=str, default="train", help="Execution mode", choices=["train", "test"])
    ap.add_argument("--input-folder", type=str, help="input data path")
    ap.add_argument("--output-folder", type=str, default="", help="output path")
    ap.add_argument("--checkpoint-path", type=str, default="", help="load a specific checkpoint for parameters")
    ap.add_argument("--num-views", type=int, default=5, help="number of source views for each patch-match problem")
    ap.add_argument("--image-max-dim", type=int, default=640, help="max image dimension")
    ap.add_argument("--train-list", type=str, help="training scan list text file")
    ap.add_argument("--test-list", type=str, help="validation scan list text file")
    ap.add_argument("--num-light-idx", type=int, default=-1, help="Number of light indexes in source images")
    ap.add_argument("--batch-size", type=int, default=12, help="train batch size")
    ap.add_argument("--resume", action="store_true", default=False, help="continue to train the model")
    ap.add_argument("--epochs", type=int, default=16, help="number of epochs to train")
    ap.add_argument("--learning-rate", type=float, default=0.001, help="learning rate")
    ap.add_argument("--lr-epochs", type=str, default="10,12,14:2", help="epoch ids to downscale lr and the downscale rate")
    ap.add_argument("--weight-decay", type=float, default=0.0, help="weight decay")
    ap.add_argument("--summary-freq", type=int, default=20, help="print and summary frequency")
    ap.add_argument("--save-freq", type=int, default=1, help="save checkpoint frequency")
    ap.add_argument("--rand-seed", type=int, default=1, metavar="S", help="random seed")
    ap.add_argument("--patchmatch-interval-scale", nargs="+", type=float, default=[0.005, 0.0125, 0.025],
                    help="normalized interval in inverse depth range to generate samples in local perturbation")
    ap.add_argument("--propagation-range", nargs="+", type=int, default=[6, 4, 2],
                    help="fixed offset of sampling points for propagation of patch match on stages 1,2,3")
    ap.add_argument("--patchmatch-iteration", nargs="+", type=int, default=[1, 2, 2],
                    help="num of iteration of patch match on stages 1,2,3")
    ap.add_argument("--patchmatch-num-sample", nargs="+", type=int, default=[8, 8, 16],
                    help="num of generated samples in local perturbation on stages 1,2,3")
    ap.add_argument("--propagate-neighbors", nargs="+", type=int, default=[0, 8, 16],
                    help="num of neighbors for adaptive propagation on stages 1,2,3")
    ap.add_argument("--evaluate-neighbors", nargs="+", type=int, default=[9, 9, 9],
                    help="num of neighbors for adaptive matching cost aggregation of adaptive evaluation on stages 1,2,3")
    ap.add_argument("--tf32", action="store_true", help="TF32 operands in the convolutions (default: fp32-accurate)")
    ap.add_argument("--num-workers", type=int, default=8, help="training loader workers (validation uses half)")
    ap.add_argument("--image-extension", type=str, default=".jpg",
                    help="extension of the files under images/ (.png for convert_eth3d's output)")
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return build_parser().parse_args(argv)


def check_args(args: argparse.Namespace) -> None:
    """train.py:241-249's checks and messages; sets the default output folder."""
    if args.input_folder is None or not os.path.isdir(args.input_folder):
        raise Exception("Invalid input folder: {}".format(args.input_folder))
    if args.train_list is None or not os.path.isfile(args.train_list):
        raise Exception("Invalid training scan list file: {}".format(args.train_list))
    if args.test_list is None or not os.path.isfile(args.test_list):
        raise Exception("Invalid validation scan list file: {}".format(args.test_list))
    if not args.output_folder:
        args.output_folder = args.input_folder


def find_latest_checkpoint(path: str) -> str:
    """train.py:183-189: the .ckpt file of `path` with the largest number after its last '_', or "" when there is none."""
    saved = [fn for fn in os.listdir(path) if fn.endswith(".ckpt")]
    if not saved:
        return ""
    saved = sorted(saved, key=lambda x: int(x.split("_")[-1].split(".")[0]))
    return os.path.join(path, saved[-1])


# ---- dataset ------------------------------------------------------------------------------------------------------------

class MVSDataset(Dataset):
    """datasets/mvs.py's MVSDataset on data_io's readers: metas scan -> light -> pair entry; the reference view plus the first
    `num_views` source views; intrinsics scaled to the read image; depth_gt/%08d.pfm read with max_dim; mask = depth_gt >=
    depth_min.  A missing ground-truth file is an error naming the path."""

    def __init__(self, data_path: str, num_views: int = 10, max_dim: int = -1, scan_list: str = "", num_light_idx: int = -1,
                 image_extension: str = ".jpg") -> None:
        super().__init__()
        self.data_path, self.num_views, self.max_dim = data_path, num_views, max_dim
        self.image_extension = image_extension
        self.metas: List[Tuple[str, str, int, List[int]]] = []
        if os.path.isfile(scan_list):
            with open(scan_list) as f:
                scans = [line.rstrip() for line in f.readlines()]
        else:
            scans = [""]
        lights = [str(i) for i in range(num_light_idx)] if num_light_idx > 0 else [""]
        for scan in scans:
            pairs = data_io.read_pair_file(os.path.join(data_path, scan, "pair.txt"))
            for light in lights:
                self.metas += [(scan, light, ref, src) for ref, src in pairs]

    def __len__(self) -> int:
        return len(self.metas)

    def __getitem__(self, idx: int) -> Dict[str, object]:
        scan, light, ref, src = self.metas[idx]
        view_ids = [ref] + src[: min(len(src), self.num_views)]
        images, intrinsics, extrinsics = [], [], []
        depth_min = depth_max = -1.0
        depth_gt = mask = None
        for i, v in enumerate(view_ids):
            image, original_h, original_w = data_io.read_image(
                os.path.join(self.data_path, scan, "images", light, "{:0>8}{}".format(v, self.image_extension)), self.max_dim)
            images.append(image.transpose([2, 0, 1]))
            k, e, depth_params = data_io.read_cam_file(os.path.join(self.data_path, scan, "cams", "{:0>8}_cam.txt".format(v)))
            intrinsics.append(data_io.scale_intrinsics(k, image.shape[:2], original_h, original_w))
            extrinsics.append(e)
            if i == 0:
                depth_min, depth_max = depth_params[0], depth_params[1]
                path = os.path.join(self.data_path, scan, "depth_gt", "{:0>8}.pfm".format(v))
                if not os.path.isfile(path):
                    raise FileNotFoundError(f"missing ground-truth depth map: {path}")
                gt = data_io.read_map(path, self.max_dim)
                depth_gt = np.ascontiguousarray(gt.reshape(gt.shape[0], gt.shape[1], 1).transpose([2, 0, 1]))
                mask = depth_gt >= depth_min
        return {
            "images": images, "intrinsics": np.stack(intrinsics), "extrinsics": np.stack(extrinsics),
            "depth_min": depth_min, "depth_max": depth_max, "depth_gt": depth_gt, "mask": mask,
            "filename": os.path.join(scan, "{}", "{:0>8}".format(view_ids[0]) + "{}"),
        }


class GlobalBatchSampler(Sampler):
    """nn.DataParallel's batching over ranks: global batch j is perm[jB:(j+1)B] (or 0..n-1 in order without shuffling), and
    this rank yields its distributed.shard_range slice of it (possibly empty).  The permutation of an epoch comes from a
    generator seeded with (seed, epoch), so every rank draws the same one."""

    def __init__(self, n: int, batch_size: int, shuffle: bool, drop_last: bool, seed: int = 0, rank: int = 0, world: int = 1) -> None:
        self.n, self.batch_size, self.shuffle, self.drop_last = n, batch_size, shuffle, drop_last
        self.seed, self.rank, self.world, self.epoch = seed, rank, world, 0

    def set_epoch(self, epoch: int) -> None:
        self.epoch = epoch

    def global_batches(self) -> List[List[int]]:
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed * 1_000_003 + self.epoch)
            order = torch.randperm(self.n, generator=g).tolist()
        else:
            order = list(range(self.n))
        B = self.batch_size
        count = self.n // B if self.drop_last else (self.n + B - 1) // B
        return [order[j * B:(j + 1) * B] for j in range(count)]

    def __iter__(self) -> Iterator[List[int]]:
        for batch in self.global_batches():
            lo, hi = pmd.shard_range(len(batch), self.rank, self.world)
            yield batch[lo:hi]

    def __len__(self) -> int:
        return self.n // self.batch_size if self.drop_last else (self.n + self.batch_size - 1) // self.batch_size


def check_view_sizes(samples: Sequence[Dict[str, object]]) -> None:
    """Samples batched together must agree view by view in size (views may differ from each other within a sample).
    RuntimeError naming the two sizes otherwise, instead of default_collate's stack error."""
    first = samples[0]["images"]
    for s in samples[1:]:
        for v, (a, b) in enumerate(zip(first, s["images"])):
            if tuple(a.shape[-2:]) != tuple(b.shape[-2:]):
                raise RuntimeError(
                    "the samples of one batch disagree in the size of view {}: {}x{} and {}x{}; data whose samples differ "
                    "in size trains with one sample per rank (--batch-size equal to the number of processes)".format(
                        v, a.shape[-2], a.shape[-1], b.shape[-2], b.shape[-1]))


def collate(samples):
    """default_collate after check_view_sizes, and None for a rank's empty share of a small last batch."""
    if not samples:
        return None
    check_view_sizes(samples)
    return default_collate(samples)


def make_loader(dataset: Dataset, batch_size: int, shuffle: bool, num_workers: int, seed: int, rank: int, world: int) -> DataLoader:
    sampler = GlobalBatchSampler(len(dataset), batch_size, shuffle=shuffle, drop_last=shuffle, seed=seed, rank=rank, world=world)
    return DataLoader(dataset, batch_sampler=sampler, num_workers=num_workers, collate_fn=collate, pin_memory=True)


# ---- one step -----------------------------------------------------------------------------------------------------------

def to_device(sample: Dict[str, object], dev: torch.device) -> Dict[str, object]:
    return {
        "images": [im.to(dev, non_blocking=True) for im in sample["images"]],
        "intrinsics": sample["intrinsics"].to(dev, non_blocking=True),
        "extrinsics": sample["extrinsics"].to(dev, non_blocking=True),
        "depth_min": sample["depth_min"].to(dev, non_blocking=True),
        "depth_max": sample["depth_max"].to(dev, non_blocking=True),
        "depth_gt": sample["depth_gt"][:, 0].to(dev, non_blocking=True),
        "mask": sample["mask"][:, 0].to(dev, non_blocking=True),
    }


def loss_levels(patchmatch_iteration: Sequence[int]) -> List[int]:
    """The level of each map loss_maps returns: the refined map at level 0, then one per PatchMatch iteration of stages 1..3."""
    return [0] + [l for l in (1, 2, 3) for _ in range(patchmatch_iteration[l - 1])]


def loss_maps(per_stage: Dict[int, List[Tensor]]) -> Tuple[List[Tensor], List[int]]:
    """The maps patchmatchnet_loss sums over, in its order (level 0..3, every PatchMatch iteration), and their levels."""
    maps, levels = [], []
    for level in range(4):
        maps += list(per_stage[level])
        levels += [level] * len(per_stage[level])
    return maps, levels


def forward_loss(net: torch.nn.Module, s: Dict[str, object], all_reduce: Optional[Callable[[Tensor], None]] = None,
                 scale: float = 1.0) -> Tuple[Tensor, Dict[int, List[Tensor]]]:
    """Network forward and DepthLoss on a device batch -> (float32 loss on the device, per-level depth maps)."""
    _, _, per_stage = net(list(s["images"]), s["intrinsics"], s["extrinsics"], s["depth_min"], s["depth_max"])
    maps, levels = loss_maps(per_stage)
    return DepthLoss.apply(levels, s["depth_gt"], s["mask"], all_reduce, scale, *maps), per_stage


def threshold_rates(over: Tensor, count: Tensor) -> Tensor:
    """Rates from exact counts in float32, as torch's CUDA mean of err_mask.float() forms them: the float32 count times the
    float32 reciprocal of the number of pixels (nan for no pixels)."""
    return over.float() * (1.0 / count.float())


def batch_metric_sums(per_stage: Dict[int, List[Tensor]], s: Dict[str, object]) -> Tensor:
    """float64 [9] on the device: the sums over this rank's images of the 8 per-image metrics (depth-error-stage-0..3,
    threshold-{1,2,4,8}mm-error), then the number of images."""
    raw = ops.depth_metrics([per_stage[l][-1].detach() for l in range(4)], s["depth_gt"], s["mask"], THRESHOLDS)
    abs_err = raw[:, :4] / raw[:, 4:8]
    rates = threshold_rates(raw[:, 8:], raw[:, 4:5]).double()
    return torch.cat([abs_err.sum(0), rates.sum(0), raw.new_tensor([raw.shape[0]])])


class Session:
    """Per-process state of a run: device, rank, world, and the collectives (no-ops with one process)."""

    def __init__(self, device: torch.device, rank: int = 0, world: int = 1, loss_levels: Sequence[int] = (0, 1, 2, 2, 3, 3)) -> None:
        self.device, self.rank, self.world = device, rank, world
        self.loss_levels = list(loss_levels)  # the level of each map the loss sums over (loss_levels())

    def all_reduce(self, t: Tensor) -> None:
        if self.world > 1:
            torch.distributed.all_reduce(t)

    @property
    def reduce_fn(self) -> Optional[Callable[[Tensor], None]]:
        return self.all_reduce if self.world > 1 else None

    def log(self, *a, **k) -> None:
        if self.rank == 0:
            print(*a, **k, flush=True)


def empty_scalars(dev) -> Tensor:
    return torch.zeros(len(SCALAR_TAGS), dtype=torch.float64, device=dev)


def process_batch(net: torch.nn.Module, sample, sess: Session, optimizer=None, reducer=None) -> Tuple[Tensor, Tensor]:
    """train.py:127-171 for one global batch -> (float32 loss, float64 [9] batch scalars in SCALAR_TAGS order), on the device.
    With an optimizer: zero the gradients, backward, average them over ranks, step."""
    training = optimizer is not None
    if training:
        if reducer is not None:
            reducer.zero_()
        else:
            optimizer.zero_grad()
    dev = sess.device
    if sample is None:  # this rank's share of a small last validation batch is empty: contribute zeros to the sums
        n = len(sess.loss_levels)
        terms = torch.zeros(n + 4, dtype=torch.float64, device=dev)
        sess.all_reduce(terms)
        sums = torch.zeros(9, dtype=torch.float64, device=dev)
        sess.all_reduce(sums)
        loss = loss_from_terms(terms, sess.loss_levels)
    else:
        s = to_device(sample, dev)
        with torch.set_grad_enabled(training):
            loss, per_stage = forward_loss(net, s, sess.reduce_fn, float(sess.world))
        if training:
            loss.backward()
            if reducer is not None:
                reducer()
            optimizer.step()
        with torch.no_grad():
            sums = batch_metric_sums(per_stage, s)
            sess.all_reduce(sums)
    out = empty_scalars(dev)
    out[0] = loss.detach().double()
    out[1:] = sums[:8] / sums[8]
    return loss.detach(), out


# ---- the run ------------------------------------------------------------------------------------------------------------

def build_network(args: argparse.Namespace) -> PatchmatchNet:
    return PatchmatchNet(
        patchmatch_interval_scale=args.patchmatch_interval_scale,
        propagation_range=args.propagation_range,
        patchmatch_iteration=args.patchmatch_iteration,
        patchmatch_num_sample=args.patchmatch_num_sample,
        propagate_neighbors=args.propagate_neighbors,
        evaluate_neighbors=args.evaluate_neighbors,
    )


def make_scheduler(optimizer: torch.optim.Optimizer, lr_epochs: str, start_epoch: int):
    """train.py:27-29: MultiStepLR(milestones, gamma = 1 / rate, last_epoch = start_epoch - 1), stepped before each epoch.
    A fresh run uses lr * gamma^#{milestones <= e + 1} during epoch e; a run resumed at a milestone epoch decays once more
    (the constructor's own step), as the reference does."""
    milestones = [int(e) for e in lr_epochs.split(":")[0].split(",")]
    gamma = 1 / float(lr_epochs.split(":")[1])
    return torch.optim.lr_scheduler.MultiStepLR(optimizer, milestones, gamma=gamma, last_epoch=start_epoch - 1)


def checkpoint_state(net: torch.nn.Module, optimizer: torch.optim.Optimizer, epoch: int) -> Dict[str, object]:
    """train.py:46-48's checkpoint: model keys with nn.DataParallel's "module." prefix (the reference's eval.py and
    train.py --resume load them), in named_parameters order."""
    model = {"module." + k: v for k, v in net.state_dict().items()}
    return {"epoch": epoch, "model": model, "optimizer": optimizer.state_dict()}


def export_module(net: torch.nn.Module, path: str) -> None:
    """module_%06d.pt (train.py:50-55): `torch.jit.script(net.eval())`, a runnable TorchScript network over the
    `torch.ops.pmb200.*` operators whose state dict is the eval-mode network's under the reference's keys (no prefix: the
    reference scripts the child module).  `torch.jit.load` runs it after `import patchmatchnet_b200` (C++: after loading
    libpmb200_torch.so); `reconstruct --input-type module` loads its state dict."""
    was_training = net.training
    net.eval()  # freezes the eval-mode decisions and folded weights the scripted forward runs on
    torch.jit.script(net).save(path)
    net.train(was_training)


class ScalarLog:
    """train_log.jsonl: one line per scalar, {"tag": "<mode>/<name>", "step": global step, "value": float}."""

    def __init__(self, folder: str) -> None:
        self.path = os.path.join(folder, "train_log.jsonl")

    def write(self, mode: str, values: Sequence[float], step: int) -> None:
        with open(self.path, "a") as f:
            for tag, v in zip(SCALAR_TAGS, values):
                f.write(json.dumps({"tag": f"{mode}/{tag}", "step": int(step), "value": float(v)}) + "\n")


def process_samples(args, sess: Session, tag: str, log: Optional[ScalarLog], net, loader: DataLoader, epoch: int,
                    optimizer=None, reducer=None) -> List[float]:
    """train.py:79-111 for one pass over a loader -> the pass's mean scalars (DictAverageMeter: a mean over batches)."""
    n = len(loader)
    acc = empty_scalars(sess.device)
    global_step = n * epoch
    loader.batch_sampler.set_epoch(epoch)
    net.train(tag == "train")
    for batch_idx, sample in enumerate(loader):
        t0 = time.time()
        global_step = n * epoch + batch_idx
        loss, scalars = process_batch(net, sample, sess, optimizer if tag == "train" else None, reducer)
        acc += scalars
        loss_value = float(loss)  # the step's host synchronisation
        if global_step % args.summary_freq == 0 and log is not None:
            log.write(tag, scalars.tolist(), global_step)
        sess.log("Epoch {}/{}, Iter {}/{}, {} loss = {:.3f}, time = {:.3f}".format(
            epoch + 1, args.epochs, batch_idx + 1, n, tag, loss_value, time.time() - t0))
    sess.log("End of processing {} samples.".format(tag))
    mean = (acc / max(n, 1)).tolist()
    if tag == "test":
        if log is not None:
            log.write("full_test", mean, global_step)
        sess.log("avg_test_scalars:", dict(zip(SCALAR_TAGS, mean)))
    return mean


def validate(sess: Session, net, loader: DataLoader) -> Dict[str, float]:
    """train.py:65-76 (--mode test)."""
    n = len(loader)
    acc = empty_scalars(sess.device)
    net.eval()
    for batch_idx, sample in enumerate(loader):
        t0 = time.time()
        loss, scalars = process_batch(net, sample, sess)
        acc += scalars
        sess.log("Iter {}/{}, test loss = {:.3f}, time = {:3f}".format(batch_idx + 1, n, float(loss), time.time() - t0))
    final = dict(zip(SCALAR_TAGS, (acc / max(n, 1)).tolist()))
    sess.log("final", final)
    return final


def _session() -> Session:
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
    return Session(dev, rank, world)


def run(args: argparse.Namespace) -> Dict[str, object]:
    """The command's library call (args as parse_args returns them).  Raises before it writes anything when the arguments
    are invalid or there is no CUDA device.  -> {"start_epoch", "final"} (final: the --mode test scalars)."""
    check_args(args)
    if not torch.cuda.is_available():
        raise RuntimeError("train needs a CUDA device (H100); there is no CPU fallback")
    sess = _session()
    sess.loss_levels = loss_levels(args.patchmatch_iteration)
    try:
        return _run(args, sess)
    finally:
        if sess.world > 1:
            torch.distributed.destroy_process_group()


def _run(args: argparse.Namespace, sess: Session) -> Dict[str, object]:
    if args.batch_size < sess.world:
        raise ValueError(f"--batch-size {args.batch_size} is smaller than the number of processes ({sess.world})")
    sess.log("argv:", sys.argv[1:])
    torch.manual_seed(args.rand_seed)
    torch.cuda.manual_seed(args.rand_seed)
    torch.backends.cudnn.benchmark = True
    train_set = MVSDataset(args.input_folder, args.num_views, args.image_max_dim, args.train_list, args.num_light_idx,
                           args.image_extension)
    test_set = MVSDataset(args.input_folder, args.num_views, args.image_max_dim, args.test_list, args.num_light_idx,
                          args.image_extension)
    train_loader = make_loader(train_set, args.batch_size, True, args.num_workers, args.rand_seed, sess.rank, sess.world)
    test_loader = make_loader(test_set, args.batch_size, False, args.num_workers // 2, args.rand_seed, sess.rank, sess.world)
    result: Dict[str, object] = {"start_epoch": 0, "final": None}
    with precision(args.tf32):
        net = build_network(args).to(sess.device)
        optimizer = torch.optim.Adam(net.parameters(), lr=args.learning_rate, betas=(0.9, 0.999), weight_decay=args.weight_decay)
        if not args.checkpoint_path:
            args.checkpoint_path = find_latest_checkpoint(args.output_folder) if os.path.isdir(args.output_folder) else ""
        if args.mode == "test":
            if not os.path.isfile(args.checkpoint_path):
                raise Exception("Invalid checkpoint file: {}".format(args.checkpoint_path))
            sess.log("Validation using checkpoint: ", args.checkpoint_path)
            load_reference_state(net, torch.load(args.checkpoint_path, map_location=sess.device)["model"])
            result["final"] = validate(sess, net, test_loader)
            return result
        start = 0
        if args.resume:
            if not os.path.isfile(args.checkpoint_path):
                raise Exception("Invalid checkpoint file: {}".format(args.checkpoint_path))
            sess.log("Resume training from checkpoint: ", args.checkpoint_path)
            state = torch.load(args.checkpoint_path, map_location=sess.device)
            load_reference_state(net, state["model"])
            optimizer.load_state_dict(state["optimizer"])
            start = state["epoch"] + 1
        result["start_epoch"] = start
        sess.log("Start training at epoch {}".format(start + 1))
        sess.log("Number of model parameters: {}".format(sum(p.data.nelement() for p in net.parameters())))
        reducer = pmd.FlatGradAllReduce(net.parameters()) if sess.world > 1 else None
        scheduler = make_scheduler(optimizer, args.lr_epochs, start)
        log = None
        if sess.rank == 0:
            os.makedirs(args.output_folder, exist_ok=True)
            log = ScalarLog(args.output_folder)
        sess.log("current time: ", str(datetime.datetime.now().strftime("%Y%m%d_%H%M%S")))
        for epoch in range(start, args.epochs):
            sess.log("Epoch {}:".format(epoch + 1))
            scheduler.step()
            process_samples(args, sess, "train", log, net, train_loader, epoch, optimizer, reducer)
            if (epoch + 1) % args.save_freq == 0 and sess.rank == 0:
                torch.save(checkpoint_state(net, optimizer, epoch), os.path.join(args.output_folder, "params_{:0>6}.ckpt".format(epoch)))
                export_module(net, os.path.join(args.output_folder, "module_{:0>6}.pt".format(epoch)))
            with torch.no_grad():
                process_samples(args, sess, "test", log, net, test_loader, epoch)
    return result


def main(argv: Optional[Sequence[str]] = None) -> int:
    run(parse_args(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
