"""ETH3D evaluation on the GPU: accuracy, completeness and F1 of a reconstruction against a high-resolution multi-view
training scene's laser-scan ground truth, at ETH3D's tolerances, computed in float64 throughout.  The protocol is restated in
full in INTEGRATION.md ("ETH3D evaluation (beyond the reference)") and include/patchmatch_b200.h; that restatement is the
definition.  It was not checked against ETH3D's own evaluation program.

Inputs of one scene: <gt>/<scene>/dslr_scan_eval/scan_alignment.mlp (a MeshLab project: per scan a PLY file, relative to the
.mlp's folder, and the 4 x 4 matrix that maps it into the scene frame) and the reconstruction (--ply-template), already in
the scene frame.

    1. ground truth     every scan's points through its matrix (ops.crop_points' transform); scan origin = the matrix's
                        translation column
    2. distances        d_acc (reconstruction -> ground truth) and d_comp (ground truth -> reconstruction), exact
                        (ops.nearest_distance, capped at 17/16 of the largest tolerance: no class depends on a
                        distance above the largest tolerance, and the search's cost grows with the cap's cube)
    3. visibility       observed(q): q lies in the free beam of some scan point (ops.beam_observed, one call per scan),
                        computed once, for the points with d_acc above the smallest tolerance
    4. scores per tau   accurate d_acc <= tau, inaccurate d_acc > tau and observed, else unobserved (excluded); covered
                        d_comp <= tau; accuracy and completeness are per-voxel means over voxels of edge tau anchored at the
                        world origin (ops.voxel_score); F1 = 2AC / (A + C)

Command line:
    python -m patchmatchnet_b200.eth3d_eval --gt-path eth3d_gt --outputs outputs --scenes courtyard pipes --json eth3d.json

With --surface the reconstruction is a triangle mesh scored as a surface: its samples (ops.sample_mesh, every point of the
surface within --surface-spacing of one, default half the smallest tolerance) instead of its vertices; the memory check
counts the samples.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time
import xml.etree.ElementTree as ET
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _native, data_io, ops, sample

MLP = os.path.join("dslr_scan_eval", "scan_alignment.mlp")
TOLERANCES = (0.01, 0.02, 0.05, 0.1, 0.2, 0.5)
# Faro Focus X 330: 2.25 mm beam exit diameter, 0.011 degrees divergence half-angle
BEAM_START_RADIUS = 0.001125
BEAM_DIVERGENCE_HALFANGLE_DEG = 0.011
CLOUD_TOLERANCE = 0.02
DISTANCE_CAP = 1.0625  # nearest distances are capped at this times the largest tolerance
GREEN, RED, BLUE = (0, 255, 0), (255, 0, 0), (0, 0, 255)


# ---- readers --------------------------------------------------------------------------------------------------------------

def read_mlp(path: str) -> List[Dict[str, object]]:
    """A MeshLab project -> per MLMesh element, in file order, {"filename": path joined to the .mlp's folder, "matrix" float64
    [4,4]} (MLMatrix44: 16 numbers, row-major, last row 0 0 0 1).  ValueError naming the file when it is malformed."""
    try:
        root = ET.parse(path).getroot()
    except ET.ParseError as e:
        raise ValueError(f"{path}: not a well-formed MeshLab project ({e})") from None
    meshes = root.iter("MLMesh")
    out = []
    for k, mesh in enumerate(meshes):
        name = mesh.get("filename")
        if not name:
            raise ValueError(f"{path}: MLMesh {k} has no filename attribute")
        m = mesh.find("MLMatrix44")
        if m is None or m.text is None:
            raise ValueError(f"{path}: MLMesh {k} ({name}) has no MLMatrix44")
        try:
            vals = [float(v) for v in m.text.split()]
        except ValueError:
            raise ValueError(f"{path}: MLMesh {k} ({name}): MLMatrix44 holds a value that is not a number") from None
        if len(vals) != 16:
            raise ValueError(f"{path}: MLMesh {k} ({name}): MLMatrix44 must hold 16 numbers, got {len(vals)}")
        mat = np.array(vals, dtype=np.float64).reshape(4, 4)
        if not np.isfinite(mat).all():
            raise ValueError(f"{path}: MLMesh {k} ({name}): MLMatrix44 must be finite")
        if mat[3].tolist() != [0.0, 0.0, 0.0, 1.0]:
            raise ValueError(f"{path}: MLMesh {k} ({name}): the last row of MLMatrix44 must be 0 0 0 1, got {mat[3].tolist()}")
        out.append({"filename": os.path.join(os.path.dirname(path), name), "matrix": mat})
    if not out:
        raise ValueError(f"{path}: the MeshLab project lists no MLMesh")
    return out


def load_scene_truth(gt_path: str, scene: str) -> Dict[str, object]:
    """<gt_path>/<scene>/dslr_scan_eval/scan_alignment.mlp and the scans it lists -> {"mlp": path, "scans": [{"filename",
    "matrix" [4,4], "origin" [3], "points" float64 [m,3] in the scan's own frame}]} (host memory)."""
    path = os.path.join(gt_path, scene, MLP)
    scans = read_mlp(path)
    for s in scans:
        s["origin"] = s["matrix"][:3, 3].copy()
        s["points"] = data_io.read_ply_points(s["filename"])
    return {"mlp": path, "scans": scans}


def find_scenes(gt_path: str) -> List[str]:
    """The folders under gt_path that hold dslr_scan_eval/scan_alignment.mlp, sorted."""
    return sorted(d for d in os.listdir(gt_path) if os.path.isfile(os.path.join(gt_path, d, MLP)))


# ---- evaluation -----------------------------------------------------------------------------------------------------------

def memory_bytes(n_rec: int, n_gt: int, max_scan: int) -> int:
    """Device memory a scene's evaluation holds at its peak: both clouds with their distances and flags, plus the largest of
    the stages' transient buffers (scan transform, nearest-distance search, beam index, voxel scores)."""
    lib = _native.lib()
    big = max(n_rec, n_gt)
    ws = [int(lib.pmb200_nearest_distance_workspace_bytes(n_gt)), int(lib.pmb200_nearest_distance_workspace_bytes(n_rec)),
          int(lib.pmb200_beam_index_workspace_bytes(max_scan)), int(lib.pmb200_voxel_score_workspace_bytes(big))]
    for w in ws:
        if w < 0:
            _native.check(w, "workspace size")
    stages = [2 * 24 * max_scan + max_scan, ws[0], ws[1], ws[2] + n_rec, ws[3] + 24 * big + 2 * big]
    return 32 * n_rec + 32 * n_gt + 2 * n_rec + max(stages)


def _free_bytes(dev: torch.device) -> int:
    return torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)


def _ratio(num: float, den: int) -> float:
    return num / den if den else 0.0


def _evaluate(rec_points, scans, tolerances, beam_start_radius, beam_divergence_halfangle_deg, device, extra_tau=None):
    """evaluate_scene's work; also returns the device state (reconstruction, ground truth, d_acc, d_comp, observed)."""
    taus = [float(t) for t in tolerances]
    if not taus or not all(t > 0 and math.isfinite(t) for t in taus):
        raise ValueError(f"tolerances must be positive and finite, got {tolerances}")
    if not (beam_start_radius >= 0 and math.isfinite(beam_start_radius)):
        raise ValueError(f"beam start radius must be finite and >= 0, got {beam_start_radius}")
    if not 0 <= beam_divergence_halfangle_deg < 90:
        raise ValueError(f"beam divergence half-angle must be in [0, 90) degrees, got {beam_divergence_halfangle_deg}")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError("eth3d_eval runs on a CUDA device; there is no CPU path")
    rec_h = np.ascontiguousarray(np.asarray(rec_points, dtype=np.float64).reshape(-1, 3))
    locals_h = [np.ascontiguousarray(np.asarray(s["points"], dtype=np.float64).reshape(-1, 3)) for s in scans]
    n, sizes = rec_h.shape[0], [p.shape[0] for p in locals_h]
    m = sum(sizes)
    with torch.cuda.device(dev):
        need, free = memory_bytes(n, m, max(sizes, default=0)), _free_bytes(dev)
        if need > free:
            raise ValueError(f"eth3d_eval: the scene needs about {need / 2 ** 30:.2f} GiB of device memory ({n} reconstruction and "
                             f"{m} ground-truth points), {free / 2 ** 30:.2f} GiB are free")
        rec = torch.from_numpy(rec_h).to(dev)
        gt = torch.empty((m, 3), dtype=torch.float64, device=dev)
        off = 0
        for s, p in zip(scans, locals_h):
            moved, _ = ops.crop_points(torch.from_numpy(p).to(dev), 2, -math.inf, math.inf, np.zeros((0, 3)), s["matrix"])
            gt[off:off + p.shape[0]] = moved
            off += p.shape[0]
        cap = DISTANCE_CAP * max(taus)
        both = [c for c in (rec, gt) if c.shape[0]]
        if both:
            lo = torch.stack([c.amin(0) for c in both]).amin(0) - cap
            hi = torch.stack([c.amax(0) for c in both]).amax(0) + cap
            box = [lo.cpu().tolist(), hi.cpu().tolist()]
        else:
            box = [[0.0] * 3, [1.0] * 3]
        d_acc = ops.nearest_distance(gt, rec, box, cap)
        d_comp = ops.nearest_distance(rec, gt, box, cap)
        observed = torch.zeros(n, dtype=torch.uint8, device=dev)
        mask = d_acc > min(taus + ([extra_tau] if extra_tau is not None else []))
        tan_half = math.tan(math.radians(beam_divergence_halfangle_deg))
        off = 0
        for s, k in zip(scans, sizes):
            ops.beam_observed(rec, gt[off:off + k], np.asarray(s["matrix"], np.float64)[:3, 3], beam_start_radius, tan_half,
                              observed, mask)
            off += k
        per_tau = []
        for tau in taus:
            a = ops.voxel_score(rec, d_acc, tau, observed)
            c = ops.voxel_score(gt, d_comp, tau)
            acc, comp = _ratio(a["fraction_sum"], a["voxels"]), _ratio(c["fraction_sum"], c["voxels"])
            per_tau.append({"tolerance": tau, "accuracy": acc, "completeness": comp,
                            "f1": 2 * acc * comp / (acc + comp) if acc + comp > 0 else 0.0,
                            "accurate": a["good"], "inaccurate": a["bad"], "unobserved": a["excluded"],
                            "covered": c["good"], "gt_points": m, "accuracy_voxels": a["voxels"],
                            "completeness_voxels": c["voxels"]})
    result = {"n_reconstruction": n, "n_gt": m, "n_scans": len(scans), "beam_start_radius": beam_start_radius,
              "beam_divergence_halfangle_deg": beam_divergence_halfangle_deg, "tolerances": per_tau}
    return result, (rec, gt, d_acc, d_comp, observed)


def evaluate_scene(rec_points, scans: Sequence[Dict[str, object]], tolerances: Sequence[float] = TOLERANCES, *,
                   beam_start_radius: float = BEAM_START_RADIUS,
                   beam_divergence_halfangle_deg: float = BEAM_DIVERGENCE_HALFANGLE_DEG, device="cuda") -> Dict[str, object]:
    """Accuracy, completeness, F1 and the class counts of one scene at each tolerance.  rec_points [n,3] in the scene frame;
    scans as load_scene_truth returns them ({"matrix" [4,4], "points" [m,3] in the scan's frame}).  ValueError before any
    device allocation when the scene would not fit in the device's free memory."""
    return _evaluate(rec_points, scans, tolerances, beam_start_radius, beam_divergence_halfangle_deg, device)[0]


def _coloured(points: torch.Tensor, colours: torch.Tensor) -> torch.Tensor:
    """uint8 [n,15] PLY vertex records (float32 xyz, uchar rgb) for data_io.save_ply."""
    xyz = points.float().contiguous().view(torch.uint8).view(-1, 12)
    return torch.cat([xyz, colours], 1)


def cloud_colours(d_acc, d_comp, observed, tau: float):
    """Reconstruction colours at tau (green accurate, red inaccurate, blue unobserved) and ground-truth colours (green
    covered, red missed): uint8 [n,3] and [m,3] on the distances' device."""
    dev = d_acc.device
    pal = torch.tensor([GREEN, RED, BLUE], dtype=torch.uint8, device=dev)
    rec_cls = torch.where(d_acc <= tau, 0, torch.where(observed.bool(), 1, 2))
    gt_cls = torch.where(d_comp <= tau, 0, 1)
    return pal[rec_cls], pal[gt_cls]


# ---- command --------------------------------------------------------------------------------------------------------------

def _tolerances(text: str) -> List[float]:
    try:
        vals = [float(v) for v in text.split(",") if v.strip()]
    except ValueError:
        raise argparse.ArgumentTypeError(f"expected comma-separated numbers, got {text!r}") from None
    if not vals or not all(v > 0 and math.isfinite(v) for v in vals):
        raise argparse.ArgumentTypeError(f"tolerances must be positive and finite, got {text!r}")
    return vals


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog="python -m patchmatchnet_b200.eth3d_eval", description=__doc__.split("\n\n")[0])
    ap.add_argument("--gt-path", required=True, help="ETH3D ground-truth folder holding <scene>/dslr_scan_eval/scan_alignment.mlp")
    ap.add_argument("--outputs", default="outputs", help="folder substituted for {outputs} in --ply-template")
    ap.add_argument("--ply-template", default="{outputs}/{scene}/fused.ply", help="path of a scene's reconstruction")
    ap.add_argument("--scenes", nargs="+", default=None, help="default: every folder under --gt-path that has the .mlp")
    ap.add_argument("--tolerances", type=_tolerances, default=list(TOLERANCES), help="comma-separated, in metres")
    ap.add_argument("--beam-start-radius", type=float, default=BEAM_START_RADIUS, help="laser beam radius at the scanner (m)")
    ap.add_argument("--beam-divergence-halfangle-deg", type=float, default=BEAM_DIVERGENCE_HALFANGLE_DEG,
                    help="laser beam divergence half-angle (degrees)")
    ap.add_argument("--accuracy-cloud", default=None,
                    help="path template ({outputs}, {scene}) of a PLY of the reconstruction coloured by class at --cloud-tolerance")
    ap.add_argument("--completeness-cloud", default=None,
                    help="path template ({outputs}, {scene}) of a PLY of the ground truth coloured by class at --cloud-tolerance")
    ap.add_argument("--cloud-tolerance", type=float, default=CLOUD_TOLERANCE)
    ap.add_argument("--json", default=None, help="write the results to this file")
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--surface", action="store_true",
                    help="score the mesh at --ply-template as a surface: its samples instead of its vertices")
    ap.add_argument("--surface-spacing", type=float, default=None,
                    help="sample spacing of --surface in metres (default half the smallest tolerance)")
    return ap


def check_args(args: argparse.Namespace) -> List[str]:
    """The argument checks, before any device work.  -> the scenes to evaluate."""
    if not os.path.isdir(args.gt_path):
        raise ValueError(f"--gt-path {args.gt_path!r} is not a folder")
    if not (args.beam_start_radius >= 0 and math.isfinite(args.beam_start_radius)):
        raise ValueError(f"--beam-start-radius must be finite and >= 0, got {args.beam_start_radius}")
    if not 0 <= args.beam_divergence_halfangle_deg < 90:
        raise ValueError(f"--beam-divergence-halfangle-deg must be in [0, 90), got {args.beam_divergence_halfangle_deg}")
    if not (args.cloud_tolerance > 0 and math.isfinite(args.cloud_tolerance)):
        raise ValueError(f"--cloud-tolerance must be positive and finite, got {args.cloud_tolerance}")
    if args.surface_spacing is not None and not args.surface:
        raise ValueError("--surface-spacing needs --surface")
    sample.check_spacing(args.surface_spacing, "--surface-spacing")
    scenes = args.scenes if args.scenes else find_scenes(args.gt_path)
    if not scenes:
        raise ValueError(f"no scene under {args.gt_path!r} has {MLP}")
    for scene in scenes:
        if not os.path.isfile(os.path.join(args.gt_path, scene, MLP)):
            raise ValueError(f"scene {scene!r}: {os.path.join(args.gt_path, scene, MLP)} does not exist")
    return scenes


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    scenes = check_args(args)
    if not torch.cuda.is_available() or torch.device(args.device).type != "cuda":
        raise RuntimeError("eth3d_eval needs a CUDA device; there is no CPU path")
    clouds = args.accuracy_cloud or args.completeness_cloud
    results = []
    for scene in scenes:
        t0 = time.perf_counter()
        truth = load_scene_truth(args.gt_path, scene)
        path = args.ply_template.format(outputs=args.outputs, scene=scene)
        surface = None
        if args.surface:
            spacing = min(args.tolerances) / 2 if args.surface_spacing is None else args.surface_spacing
            pts, surface = sample.mesh_samples(path, spacing, args.device)
            rec = pts.cpu().numpy()
            del pts
        else:
            rec = data_io.read_ply_points(path)
        r, state = _evaluate(rec, truth["scans"], args.tolerances, args.beam_start_radius, args.beam_divergence_halfangle_deg,
                             args.device, args.cloud_tolerance if clouds else None)
        if clouds:
            rec_t, gt_t, d_acc, d_comp, observed = state
            rec_c, gt_c = cloud_colours(d_acc, d_comp, observed, args.cloud_tolerance)
            for template, pts, col in ((args.accuracy_cloud, rec_t, rec_c), (args.completeness_cloud, gt_t, gt_c)):
                if template:
                    path = template.format(outputs=args.outputs, scene=scene)
                    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
                    data_io.save_ply(path, _coloured(pts, col))
        del state
        r["scene"] = scene
        r["seconds"] = time.perf_counter() - t0
        if surface is not None:
            r["surface"] = surface
        results.append(r)
    mean = [{"tolerance": tau, **{k: float(np.mean([r["tolerances"][i][k] for r in results]))
                                  for k in ("accuracy", "completeness", "f1")}}
            for i, tau in enumerate(args.tolerances)]
    print(f"{'scene':<20} {'tau (m)':>8} {'accuracy':>9} {'complete':>9} {'F1':>9}")
    for r in results:
        for t in r["tolerances"]:
            print(f"{r['scene']:<20} {t['tolerance']:>8g} {t['accuracy']:>9.4f} {t['completeness']:>9.4f} {t['f1']:>9.4f}")
    for t in mean:
        print(f"{'mean':<20} {t['tolerance']:>8g} {t['accuracy']:>9.4f} {t['completeness']:>9.4f} {t['f1']:>9.4f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"tolerances": args.tolerances, "beam_start_radius": args.beam_start_radius,
                       "beam_divergence_halfangle_deg": args.beam_divergence_halfangle_deg, "scenes": results, "mean": mean},
                      f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
