"""Whole-scene reconstruction: depth maps, geometric filtering and point fusion from a dataset folder to fused.ply, on this
project's kernels -- the counterpart of the reference's eval.py.

    python -m patchmatchnet_b200.reconstruct --input-folder dtu --output-folder outputs --checkpoint-path model.pt \\
        --scan-list lists/dtu/test.txt --num-views 5 --geo-mask-thres 3 --photo-thres 0.8
    python -m patchmatchnet_b200.dtu_eval --data-path "SampleSet/MVS Data" --outputs outputs

Input per scan (eval.py, datasets/mvs.py): pair.txt, images/%08d.jpg, cams/%08d_cam.txt.  Output per scan, in eval.py's
layout: depth_est/%08d{fmt} and confidence/%08d{fmt} (float32 [H,W]), mask/%08d_{photo,geo,final}.png, fused.ply.
Without --scan-list the input folder is one scene; with it, every line names a scan folder below it.

Depth stage, per scan: the requests are the pair.txt entries in file order, each the reference view plus its first
`--num-views` source views.  Every image the scan needs is decoded once (data_io.read_image) and uploaded once into a
device-resident image bank; a request is assembled on the device (DepthEngine.set_device_inputs).  Requests are grouped by
their size signature, the (H, W) of every view in request order (group_requests).  There is one DepthEngine per distinct
signature; request j of a group runs on slot j % n_slots, each slot on its own stream, so requests overlap.  Depth and
confidence are copied out of the graph-owned outputs on the slot's stream into a device map bank and then written with
data_io.save_map_from_device.  The network call is the one DepthEngine makes for any request, so the maps are bit-identical
to a direct engine run with the same seed, slot count and request order.  Engines of uniform signatures (every view the
reference's size) live for the whole call, so the stage-3 random initialisation continues its per-slot sequences from one
scan to the next.  A signature that mixes sizes (several cameras, portrait and landscape shots) gets an engine with
DepthEngine(view_sizes=...) and min(n_slots, group size) slots, released when its group is done, so a scene with many
signatures does not hold one engine per signature.

Fusion stage, per scan: the reference's filter_depth (eval.py:193-297) for every reference view in pair order, with every
source view pair.txt lists for it (not only --num-views): ops.compose_filter_cameras -> ops.geometric_filter
(pmb200_geometric_filter; pmb200_geometric_filter_views when the source maps differ in size) -> the three mask PNGs ->
ops.compose_fusion_camera -> ops.fuse_points (pmb200_fuse_points).  The vertex records stay on the device until
data_io.save_ply writes the scan's fused.ply once.  With --output-type both the maps come from the map bank; with
--output-type fusion each map file is read once per scan (data_io.read_map_to_device).

With --normals (off by default; it changes no other output) each reference view's normal map is estimated from its raw
depth map with that view's intrinsics (ops.estimate_normals, pmb200_depth_normals) and fused.ply is written oriented:
float x, y, z, nx, ny, nz, uchar red, green, blue per point (pmb200_fuse_points_oriented), which Poisson surface
reconstruction takes as is.  For COLMAP's own fusion and meshers, export the results instead:

    python -m patchmatchnet_b200.reconstruct --input-folder scene --output-folder outputs --checkpoint-path model.pt --normals
    PoissonRecon --in outputs/fused.ply --out mesh.ply            # or Open3D, or colmap poisson_mesher on this file
    python -m patchmatchnet_b200.colmap_output --input-folder scene --results-folder outputs --output-folder ws --normals
    colmap stereo_fusion --workspace_path ws --input_type geometric --output_path ws/fused.ply
    colmap poisson_mesher --input_path ws/fused.ply --output_path ws/meshed-poisson.ply

Device memory held besides the engines, for a scan of n_img images of H x W and n_ref reference views:
    image bank   n_img * 3 * H * W * 4 bytes
    map bank     n_ref * 2 * H * W * 4 bytes
e.g. 49 views at 1600 x 1200: 1.13 GB + 0.75 GB = 1.88 GB.

Differences from eval.py: checkpoints load strictly (a missing or unexpected key raises), TorchScript archives are loaded
into the native network, `--seed` seeds the random initialisation, `--tf32` opts into TF32 convolution operands (the default
is the fp32-accurate mode), and --batch_size, --display and --num_light_idx do not exist.  There is no CPU path.
"""
from __future__ import annotations

import argparse
import contextlib
import os
import sys
import time
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import data_io, ops
from .engine import DepthEngine
from .net import PatchmatchNet, load_reference_state

Tensor = torch.Tensor


def build_parser() -> argparse.ArgumentParser:
    """eval.py:303-347 in this project's hyphen style, same defaults; plus --seed and --tf32."""
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.reconstruct", description="Predict depth, filter, and fuse")
    ap.add_argument("--input-folder", type=str, help="input data path")
    ap.add_argument("--output-folder", type=str, default="", help="output path (default: the input folder)")
    ap.add_argument("--checkpoint-path", type=str, help="checkpoint: a state dict file (params) or a TorchScript archive (module)")
    ap.add_argument("--file-format", type=str, default=".pfm", choices=[".bin", ".pfm"], help="file format for depth maps")
    ap.add_argument("--input-type", type=str, default="params", choices=["params", "module"], help="input type of checkpoint")
    ap.add_argument("--output-type", type=str, default="both", choices=["depth", "fusion", "both"], help="outputs to produce")
    ap.add_argument("--num-views", type=int, default=20, help="number of source views for each patch-match problem")
    ap.add_argument("--image-max-dim", type=int, default=-1, help="max image dimension")
    ap.add_argument("--scan-list", type=str, default="", help="optional scan list text file to identify input folders")
    ap.add_argument("--patchmatch-interval-scale", nargs="+", type=float, default=[0.005, 0.0125, 0.025],
                    help="normalized interval in inverse depth range to generate samples in local perturbation")
    ap.add_argument("--patchmatch-range", nargs="+", type=int, default=[6, 4, 2],
                    help="fixed offset of sampling points for propagation of patch match on stages 1,2,3")
    ap.add_argument("--patchmatch-iteration", nargs="+", type=int, default=[1, 2, 2],
                    help="num of iteration of patch match on stages 1,2,3")
    ap.add_argument("--patchmatch-num-sample", nargs="+", type=int, default=[8, 8, 16],
                    help="num of generated samples in local perturbation on stages 1,2,3")
    ap.add_argument("--propagate-neighbors", nargs="+", type=int, default=[0, 8, 16],
                    help="num of neighbors for adaptive propagation on stages 1,2,3")
    ap.add_argument("--evaluate-neighbors", nargs="+", type=int, default=[9, 9, 9],
                    help="num of neighbors for adaptive matching cost aggregation of adaptive evaluation on stages 1,2,3")
    ap.add_argument("--geo-pixel-thres", type=float, default=1.0, help="pixel threshold for geometric consistency filtering")
    ap.add_argument("--geo-depth-thres", type=float, default=0.01, help="depth threshold for geometric consistency filtering")
    ap.add_argument("--geo-mask-thres", type=int, default=5, help="threshold for geometric consistency filtering")
    ap.add_argument("--photo-thres", type=float, default=0.5, help="threshold for photometric consistency filtering")
    ap.add_argument("--seed", type=int, default=0, help="seed of the stage-3 random initialisation (per request slot: seed + slot)")
    ap.add_argument("--tf32", action="store_true", help="TF32 operands in the convolutions (default: fp32-accurate)")
    ap.add_argument("--normals", action="store_true",
                    help="write an oriented fused.ply (float nx, ny, nz per point, for Poisson meshers) with normals estimated "
                         "from each reference view's depth map")
    return ap


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    return build_parser().parse_args(argv)


def list_scans(scan_list: str) -> List[str]:
    """eval.py:374-380: the lines of the scan list file, or one scene (the input folder itself) without a list."""
    if not scan_list:
        return [""]
    if not os.path.isfile(scan_list):
        raise Exception("Invalid scan list file: {}".format(scan_list))
    with open(scan_list) as f:
        return [line.rstrip() for line in f.readlines()]


def check_args(args: argparse.Namespace) -> List[str]:
    """eval.py:354-361's checks and messages, and the scan list; -> the scans.  Sets the default output folder."""
    if args.input_folder is None or not os.path.isdir(args.input_folder):
        raise Exception("Invalid input folder: {}".format(args.input_folder))
    if args.checkpoint_path is None or not os.path.isfile(args.checkpoint_path):
        raise Exception("Invalid checkpoint file: {}".format(args.checkpoint_path))
    scans = list_scans(args.scan_list)
    if not args.output_folder:
        args.output_folder = args.input_folder
    return scans


def scan_requests(pairs: Sequence[Tuple[int, List[int]]], num_views: int) -> List[List[int]]:
    """The depth requests of a scan (datasets/mvs.py:57-63): per pair entry, in order, [reference] + first num_views sources."""
    return [[ref] + list(src[:num_views]) for ref, src in pairs]


def scan_views(pairs: Sequence[Tuple[int, List[int]]], num_views: int, fusion: bool) -> List[int]:
    """The views whose images and cameras a scan needs, in order of first appearance: those of the depth requests, and with
    the fusion also every source view pair.txt lists (the filter uses them all, eval.py:226)."""
    seen: Dict[int, None] = {}
    for views in scan_requests(pairs, num_views):
        seen.update(dict.fromkeys(views))
    if fusion:
        for ref, src in pairs:
            seen.update(dict.fromkeys([ref] + list(src)))
    return list(seen)


class SceneBank:
    """One scan's images (device, [3,H,W] float32, decoded once) and cameras (host float32, intrinsics scaled to the
    decoded image size; eval.py:205-211, datasets/mvs.py:77-84), plus stacked device copies of the cameras and depth
    ranges from which requests are gathered on the device."""

    def __init__(self, scene_dir: str, views: Sequence[int], max_dim: int, device: torch.device) -> None:
        self.row = {v: i for i, v in enumerate(views)}
        self.images: Dict[int, Tensor] = {}
        self.intrinsics: Dict[int, np.ndarray] = {}
        self.extrinsics: Dict[int, np.ndarray] = {}
        self.has_range: Dict[int, bool] = {}
        ranges = np.zeros((len(views), 2), dtype=np.float32)
        for v in views:
            img, original_h, original_w = data_io.read_image(os.path.join(scene_dir, "images", "{:0>8}.jpg".format(v)), max_dim)
            if img.ndim != 3 or img.shape[2] != 3:
                raise ValueError(f"view {v}: expected an RGB image, got an array of shape {img.shape}")
            k, e, depth_params = data_io.read_cam_file(os.path.join(scene_dir, "cams", "{:0>8}_cam.txt".format(v)))
            self.intrinsics[v] = data_io.scale_intrinsics(k, img.shape[:2], original_h, original_w)
            self.extrinsics[v] = e
            self.has_range[v] = len(depth_params) >= 2
            if self.has_range[v]:
                ranges[self.row[v]] = depth_params[:2]
            self.images[v] = torch.from_numpy(np.ascontiguousarray(img.transpose(2, 0, 1))).to(device)
        self.K = torch.from_numpy(np.stack([self.intrinsics[v] for v in views])).to(device)
        self.E = torch.from_numpy(np.stack([self.extrinsics[v] for v in views])).to(device)
        self.ranges = torch.from_numpy(ranges).to(device)

    def shape(self, v: int) -> Tuple[int, int]:
        return tuple(self.images[v].shape[1:])


@contextlib.contextmanager
def precision(tf32: bool):
    """The convolution precision for the run: fp32-accurate (cuDNN / matmul TF32 off, the native convs' 3xTF32 split) by
    default, TF32 operands with tf32=True.  Set before the network is built (the kernels' precision is chosen at load time)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = bool(tf32)
    if not tf32:
        torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def load_network(args: argparse.Namespace) -> PatchmatchNet:
    """The native PatchmatchNet with eval.py's constructor arguments and the checkpoint's weights, loaded strictly.
    params: torch.load(path)["model"] (a file without a "model" entry is taken as the state dict itself);
    module: the state dict of a TorchScript archive (the reference's scripted PatchmatchNet has the same keys)."""
    net = PatchmatchNet(
        patchmatch_interval_scale=args.patchmatch_interval_scale,
        propagation_range=args.patchmatch_range,
        patchmatch_iteration=args.patchmatch_iteration,
        patchmatch_num_sample=args.patchmatch_num_sample,
        propagate_neighbors=args.propagate_neighbors,
        evaluate_neighbors=args.evaluate_neighbors,
    )
    if args.input_type == "params":
        state = torch.load(args.checkpoint_path, map_location="cpu")
        if isinstance(state, dict) and "model" in state:
            state = state["model"]
    else:
        state = torch.jit.load(args.checkpoint_path, map_location="cpu").state_dict()
    load_reference_state(net, state)
    return net.eval()


Signature = Tuple[Tuple[int, int], ...]


def group_requests(signatures: Sequence[Signature]) -> Dict[Signature, List[int]]:
    """Request indices grouped by size signature (the (H, W) of every view of a request, reference first), groups in order of
    first appearance and requests in their order within a group."""
    groups: Dict[Signature, List[int]] = {}
    for j, sig in enumerate(signatures):
        groups.setdefault(tuple(sig), []).append(j)
    return groups


def is_uniform(sig: Signature) -> bool:
    """Every view of the signature has the reference view's size."""
    return all(hw == sig[0] for hw in sig[1:])


class DepthStage:
    """The network side of the command: one DepthEngine (and one stream per slot) per size signature.  Engines of uniform
    signatures are kept across scans; an engine of a mixed signature is released when its group is done."""

    def __init__(self, net: PatchmatchNet, device: torch.device, n_slots: int = 3, seed: int = 0) -> None:
        self.net, self.device, self.n_slots, self.seed = net, device, n_slots, seed
        self.engines: Dict[Tuple[int, int, int], Tuple[DepthEngine, List[torch.cuda.Stream]]] = {}
        self.setup_seconds = 0.0
        self.engines_built = 0

    def _build(self, sig: Signature, n_slots: int, fill: Callable[[DepthEngine, int], None]):
        t0 = time.perf_counter()
        h, w = sig[0]
        eng = DepthEngine(self.net, 1, len(sig), h, w, device=str(self.device), n_slots=n_slots, seed=self.seed,
                          view_sizes=None if is_uniform(sig) else sig)
        for k in range(eng.n_slots):  # warm-up and capture need valid cameras in every slot
            fill(eng, k)
        torch.cuda.current_stream(self.device).synchronize()
        eng.prepare()
        self.setup_seconds += time.perf_counter() - t0
        self.engines_built += 1
        return eng, [torch.cuda.Stream(device=self.device) for _ in range(eng.n_slots)]

    def _engine(self, sig: Signature, group_size: int, fill: Callable[[DepthEngine, int], None]):
        if not is_uniform(sig):
            return self._build(sig, min(self.n_slots, group_size), fill)
        key = (len(sig),) + sig[0]
        if key not in self.engines:
            self.engines[key] = self._build(sig, self.n_slots, fill)
        return self.engines[key]

    def run(self, bank: SceneBank, requests: Sequence[List[int]]) -> Dict[int, Tuple[Tensor, Tensor]]:
        """All requests of a scan -> {reference view: (depth [H,W], confidence [H,W])} on the device, in the map bank."""
        for views in requests:
            if not bank.has_range[views[0]]:
                raise ValueError(f"view {views[0]}: its cam file has no depth range (line 12), which a depth request needs")
        groups = group_requests([tuple(bank.shape(v) for v in views) for views in requests])
        cur = torch.cuda.current_stream(self.device)
        maps: Dict[int, Tuple[Tensor, Tensor]] = {}
        for sig, js in groups.items():
            h, w = sig[0]
            rows = torch.tensor([[bank.row[v] for v in requests[j]] for j in js], dtype=torch.int64).to(self.device)
            out = torch.empty((len(js), 2, h, w), dtype=torch.float32, device=self.device)

            def fill(eng: DepthEngine, slot: int, i: int = 0) -> None:
                r = rows[i]
                depth_range = bank.ranges.index_select(0, r[:1])  # [1,2]: the reference view's depth_min, depth_max
                eng.set_device_inputs(slot, [bank.images[v] for v in requests[js[i]]], bank.K.index_select(0, r).unsqueeze(0),
                                      bank.E.index_select(0, r).unsqueeze(0), depth_range[:, 0], depth_range[:, 1])

            eng, streams = self._engine(sig, len(js), fill)
            for st in streams:
                st.wait_stream(cur)  # the banks were filled on the current stream
            for i, j in enumerate(js):
                k = i % eng.n_slots
                with torch.cuda.stream(streams[k]):
                    fill(eng, k, i)
                    depth, conf = eng.run_slot(k)
                    out[i, 0].copy_(depth[0, 0])
                    out[i, 1].copy_(conf[0])
                maps[requests[j][0]] = (out[i, 0], out[i, 1])
            for st in streams:
                cur.wait_stream(st)
            if not is_uniform(sig):
                # the graphs' private memory goes back to the allocator with the engine: let the replays finish first
                for st in streams:
                    st.synchronize()
                del eng, streams
        return maps


def _map_path(out_dir: str, kind: str, view: int, fmt: str) -> str:
    return os.path.join(out_dir, kind, "{:0>8}{}".format(view, fmt))


def save_maps(out_dir: str, maps: Dict[int, Tuple[Tensor, Tensor]], fmt: str) -> None:
    """depth_est/%08d{fmt}, confidence/%08d{fmt} (eval.py:75-82): float32 [H,W] each."""
    os.makedirs(os.path.join(out_dir, "depth_est"), exist_ok=True)
    os.makedirs(os.path.join(out_dir, "confidence"), exist_ok=True)
    for view, (depth, conf) in maps.items():
        data_io.save_map_from_device(_map_path(out_dir, "depth_est", view, fmt), depth)
        data_io.save_map_from_device(_map_path(out_dir, "confidence", view, fmt), conf)


class _DiskMaps:
    """Maps read from the files of a previous depth run, each file once per scan (eval.py:214-238 reads them per use)."""

    def __init__(self, out_dir: str, fmt: str, device: torch.device) -> None:
        self.out_dir, self.fmt, self.device = out_dir, fmt, device
        self.cache: Dict[Tuple[str, int], Tensor] = {}

    def _get(self, kind: str, view: int) -> Tensor:
        if (kind, view) not in self.cache:
            self.cache[(kind, view)] = data_io.read_map_to_device(_map_path(self.out_dir, kind, view, self.fmt), self.device)[..., 0]
        return self.cache[(kind, view)]

    def __getitem__(self, view: int) -> Tuple[Tensor, Tensor]:
        return self._get("depth_est", view), self._get("confidence", view)


def fuse_scan(args: argparse.Namespace, scan: str, bank: SceneBank, pairs: Sequence[Tuple[int, List[int]]], maps,
              log: Callable[..., None] = print) -> int:
    """filter_depth (eval.py:193-297) for one scan; `maps[view]` -> (depth [H,W], confidence [H,W]) on the device.
    Writes the mask PNGs and fused.ply (oriented with --normals); -> the number of points."""
    out_dir = os.path.join(args.output_folder, scan)
    os.makedirs(os.path.join(out_dir, "mask"), exist_ok=True)
    bodies = []
    for ref, srcs in pairs:
        ref_depth, conf = maps[ref]
        src_list = [maps[s][0] for s in srcs]
        same = all(d.shape == src_list[0].shape for d in src_list[1:])
        src_depths = torch.stack(src_list) if same else src_list  # sources of different sizes: the per-view filter
        cams = ops.compose_filter_cameras(bank.intrinsics[ref], bank.extrinsics[ref], [bank.intrinsics[s] for s in srcs],
                                          [bank.extrinsics[s] for s in srcs])
        photo, mask_sum, final, avg = ops.geometric_filter(ref_depth, conf, src_depths, cams, args.geo_pixel_thres,
                                                           args.geo_depth_thres, args.photo_thres, args.geo_mask_thres)
        photo_h, geo_h, final_h = (t.cpu().numpy() for t in (photo, mask_sum >= args.geo_mask_thres, final))
        data_io.save_image(os.path.join(out_dir, "mask", "{:0>8}_photo.png".format(ref)), photo_h)
        data_io.save_image(os.path.join(out_dir, "mask", "{:0>8}_geo.png".format(ref)), geo_h)
        data_io.save_image(os.path.join(out_dir, "mask", "{:0>8}_final.png".format(ref)), final_h)
        log("processing {}, ref-view{:0>3}, geo_mask:{:3f}, photo_mask:{:3f}, final_mask: {:3f}".format(
            os.path.join(args.input_folder, scan), ref, geo_h.mean(), photo_h.mean(), final_h.mean()))
        # --normals: from the raw depth map (depth_est), with the view's own intrinsics at that map's size
        normals = ops.estimate_normals(ref_depth, bank.intrinsics[ref]) if args.normals else None
        body = ops.fuse_points(final, avg, bank.images[ref].permute(1, 2, 0).contiguous(),
                               ops.compose_fusion_camera(bank.intrinsics[ref], bank.extrinsics[ref]), normals)
        bodies.append(body.clone())  # drop the [H*W,15] (or [H*W,27]) allocation behind the returned slice
    ply = os.path.join(out_dir, "fused.ply")
    data_io.save_ply(ply, bodies)
    log("saving the final model to", ply)
    return sum(int(b.shape[0]) for b in bodies)


def reconstruct(args: argparse.Namespace, *, device: str = "cuda:0", n_slots: int = 3,
                log: Callable[..., None] = print) -> Dict[str, float]:
    """The command's library call.  `args` as parse_args returns it.  -> seconds of the depth stage (image decoding and
    upload, engine set-up, network, map files), of the fusion stage (filter, masks, fusion, fused.ply) and end to end, plus
    counts (scans, depth maps, points, engines built and their set-up seconds).  Raises before it creates any output when the arguments are invalid or there is no CUDA device."""
    scans = check_args(args)
    if not torch.cuda.is_available():
        raise RuntimeError("reconstruct needs a CUDA device (H100); there is no CPU fallback")
    dev = torch.device(device)
    do_depth = args.output_type in ("depth", "both")
    do_fusion = args.output_type in ("fusion", "both")
    os.makedirs(args.output_folder, exist_ok=True)
    stats = {"depth_seconds": 0.0, "fusion_seconds": 0.0, "engine_setup_seconds": 0.0, "engines_built": 0, "scans": len(scans),
             "depth_maps": 0, "points": 0}
    t_start = time.perf_counter()
    with precision(args.tf32), torch.cuda.device(dev), torch.no_grad():
        stage = DepthStage(load_network(args).to(dev), dev, n_slots=n_slots, seed=args.seed) if do_depth else None
        for scan in scans:
            scene_dir = os.path.join(args.input_folder, scan)
            out_dir = os.path.join(args.output_folder, scan)
            pairs = data_io.read_pair_file(os.path.join(scene_dir, "pair.txt"))
            t0 = time.perf_counter()
            bank = SceneBank(scene_dir, scan_views(pairs, args.num_views, do_fusion), args.image_max_dim, dev)
            maps = None
            if do_depth:
                maps = stage.run(bank, scan_requests(pairs, args.num_views))
                save_maps(out_dir, maps, args.file_format)
                torch.cuda.synchronize(dev)
                t1 = time.perf_counter()
                stats["depth_seconds"] += t1 - t0
                stats["depth_maps"] += len(maps)
                log(f"depth {scene_dir}: {len(maps)} maps in {t1 - t0:.3f} s")
                t0 = t1
            if do_fusion:
                stats["points"] += fuse_scan(args, scan, bank, pairs,
                                             maps if maps is not None else _DiskMaps(out_dir, args.file_format, dev), log)
                torch.cuda.synchronize(dev)
                stats["fusion_seconds"] += time.perf_counter() - t0
            del bank, maps
        if stage is not None:
            stats["engine_setup_seconds"] = stage.setup_seconds
            stats["engines_built"] = stage.engines_built
    stats["total_seconds"] = time.perf_counter() - t_start
    return stats


def main(argv: Optional[Sequence[str]] = None) -> int:
    args = parse_args(argv)
    reconstruct(args)
    return 0


if __name__ == "__main__":
    sys.exit(main())
