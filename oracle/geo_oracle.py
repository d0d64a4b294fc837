"""CPU restatement of the reference's geometric-consistency filtering (SURVEY.md 8f row f4).

TEST INFRASTRUCTURE ONLY: nothing under patchmatchnet_b200/ imports this file; only tests/ and bench-side baselines
may.  It follows, line by line, the reference's eval.py:

    reproject_with_depth          eval.py:86-146
    check_geometric_consistency   eval.py:149-190
    fuse_reference_view           the per-reference-view loop of filter_depth, eval.py:217-256 (masks and averaged depth)

The only arithmetic that is not numpy is `cv2.remap(depth_src, x_src, y_src, interpolation=cv2.INTER_LINEAR)`
(eval.py:128; OpenCV is a third-party dependency, requirements.txt unpinned, 4.13.0 installed).  `remap_linear` restates its
published algorithm for a float32 single-channel image, float32 maps, bilinear interpolation, BORDER_CONSTANT(0): map
coordinates are rounded to 1/32 pixel (INTER_BITS = 5, cvRound = nearest-even on the float32 product), the integer part is
floor(s / 32) saturated to int16, the four weights come from the float32 table (1-fy)(1-fx), (1-fy)fx, fy(1-fx), fy fx,
taps outside the image contribute the border value 0, and the sum runs left to right in float32.
Pin status: tests/test_geo.py checks `remap_linear` bit for bit against cv2.remap and the three functions bit for bit
against the reference's own source text executed in the build container; tests/golden/geo_case.npz carries
reference-generated outputs to the GPU box.
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

INTER_BITS = 5
INTER_TAB_SIZE = 1 << INTER_BITS


def remap_linear(src: np.ndarray, map_x: np.ndarray, map_y: np.ndarray) -> np.ndarray:
    """cv2.remap(src, map_x, map_y, cv2.INTER_LINEAR) for float32 HxW `src`, float32 maps, constant border 0."""
    src = np.ascontiguousarray(src, dtype=np.float32)
    H, W = src.shape
    sx = np.rint(map_x.astype(np.float32) * np.float32(INTER_TAB_SIZE))
    sy = np.rint(map_y.astype(np.float32) * np.float32(INTER_TAB_SIZE))
    # cvRound of non-finite / huge values is INT_MIN on x86 (cvtss2si); such taps are outside the image either way
    big = ~(np.isfinite(sx) & np.isfinite(sy) & (np.abs(sx) < 2.0 ** 31) & (np.abs(sy) < 2.0 ** 31))
    sx = np.where(big, -2.0 ** 31, sx).astype(np.int64)
    sy = np.where(big, -2.0 ** 31, sy).astype(np.int64)
    fx = (sx & (INTER_TAB_SIZE - 1)).astype(np.float32) / np.float32(INTER_TAB_SIZE)
    fy = (sy & (INTER_TAB_SIZE - 1)).astype(np.float32) / np.float32(INTER_TAB_SIZE)
    ix = np.clip(sx >> INTER_BITS, -32768, 32767)
    iy = np.clip(sy >> INTER_BITS, -32768, 32767)
    one = np.float32(1.0)
    w = [(one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx]  # float32 products, as the table holds them

    def tap(yy, xx):
        inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        return np.where(inside, src[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], np.float32(0.0)).astype(np.float32)

    out = tap(iy, ix) * w[0]
    out = out + tap(iy, ix + 1) * w[1]
    out = out + tap(iy + 1, ix) * w[2]
    out = out + tap(iy + 1, ix + 1) * w[3]
    return out.astype(np.float32)


def reproject_with_depth(depth_ref, intrinsics_ref, extrinsics_ref, depth_src, intrinsics_src, extrinsics_src,
                         remap=remap_linear) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """eval.py:86-146.  `remap(depth_src, x, y)` stands for cv2.remap(..., interpolation=cv2.INTER_LINEAR) (eval.py:128)."""
    width, height = depth_ref.shape[1], depth_ref.shape[0]
    x_ref, y_ref = np.meshgrid(np.arange(0, width), np.arange(0, height))
    x_ref, y_ref = x_ref.reshape([-1]), y_ref.reshape([-1])
    xyz_ref = np.matmul(np.linalg.inv(intrinsics_ref),
                        np.vstack((x_ref, y_ref, np.ones_like(x_ref))) * depth_ref.reshape([-1]))
    xyz_src = np.matmul(np.matmul(extrinsics_src, np.linalg.inv(extrinsics_ref)),
                        np.vstack((xyz_ref, np.ones_like(x_ref))))[:3]
    k_xyz_src = np.matmul(intrinsics_src, xyz_src)
    xy_src = k_xyz_src[:2] / k_xyz_src[2:3]
    x_src = xy_src[0].reshape([height, width]).astype(np.float32)
    y_src = xy_src[1].reshape([height, width]).astype(np.float32)
    sampled_depth_src = remap(depth_src, x_src, y_src)
    xyz_src = np.matmul(np.linalg.inv(intrinsics_src),
                        np.vstack((xy_src, np.ones_like(x_ref))) * sampled_depth_src.reshape([-1]))
    xyz_reprojected = np.matmul(np.matmul(extrinsics_ref, np.linalg.inv(extrinsics_src)),
                                np.vstack((xyz_src, np.ones_like(x_ref))))[:3]
    depth_reprojected = xyz_reprojected[2].reshape([height, width]).astype(np.float32)
    k_xyz_reprojected = np.matmul(intrinsics_ref, xyz_reprojected)
    xy_reprojected = k_xyz_reprojected[:2] / k_xyz_reprojected[2:3]
    x_reprojected = xy_reprojected[0].reshape([height, width]).astype(np.float32)
    y_reprojected = xy_reprojected[1].reshape([height, width]).astype(np.float32)
    return depth_reprojected, x_reprojected, y_reprojected


def check_geometric_consistency(depth_ref, intrinsics_ref, extrinsics_ref, depth_src, intrinsics_src, extrinsics_src,
                                geo_pixel_thres: float, geo_depth_thres: float, remap=remap_linear):
    """eval.py:149-190."""
    width, height = depth_ref.shape[1], depth_ref.shape[0]
    x_ref, y_ref = np.meshgrid(np.arange(0, width), np.arange(0, height))
    depth_reprojected, x2d_reprojected, y2d_reprojected = reproject_with_depth(
        depth_ref, intrinsics_ref, extrinsics_ref, depth_src, intrinsics_src, extrinsics_src, remap=remap)
    dist = np.sqrt((x2d_reprojected - x_ref) ** 2 + (y2d_reprojected - y_ref) ** 2)
    depth_diff = np.abs(depth_reprojected - depth_ref)
    relative_depth_diff = depth_diff / depth_ref
    mask = np.logical_and(dist < geo_pixel_thres, relative_depth_diff < geo_depth_thres)
    depth_reprojected[~mask] = 0
    return mask, depth_reprojected


def fuse_reference_view(ref_depth: np.ndarray, ref_intrinsics: np.ndarray, ref_extrinsics: np.ndarray,
                        src_depths: Sequence[np.ndarray], src_intrinsics: Sequence[np.ndarray],
                        src_extrinsics: Sequence[np.ndarray], confidence: np.ndarray, geo_pixel_thres: float = 1.0,
                        geo_depth_thres: float = 0.01, photo_thres: float = 0.8, geo_mask_thres: int = 3, remap=remap_linear):
    """The per-reference-view body of filter_depth (eval.py:217-256): photometric mask, geometric mask over the source
    views, final mask, and the averaged depth (eval.py:252).  -> (photo_mask, geo_mask_sum, final_mask, depth_averaged)."""
    photo_mask = confidence > photo_thres
    all_src: List[np.ndarray] = []
    geo_mask_sum = 0
    for d, k, e in zip(src_depths, src_intrinsics, src_extrinsics):
        geo_mask, depth_reprojected = check_geometric_consistency(
            ref_depth, ref_intrinsics, ref_extrinsics, d, k, e, geo_pixel_thres, geo_depth_thres, remap=remap)
        geo_mask_sum = geo_mask_sum + geo_mask.astype(np.int32)
        all_src.append(depth_reprojected)
    depth_est_averaged = (sum(all_src) + ref_depth) / (geo_mask_sum + 1)
    geo_mask = geo_mask_sum >= geo_mask_thres
    final_mask = np.logical_and(photo_mask, geo_mask)
    return photo_mask, geo_mask_sum, final_mask, depth_est_averaged


def fuse_points(final_mask: np.ndarray, depth_est_averaged: np.ndarray, ref_img: np.ndarray, ref_intrinsics: np.ndarray,
                ref_extrinsics: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """The point-cloud half of filter_depth for one reference view (eval.py:273-281): the pixels of `final_mask`, in row-major
    order, back-projected with the averaged depth into the world frame (float64 arithmetic on float32 camera inverses), and
    their colours.  -> (vertices float64 [n,3] -- the reference casts them to float32 when it assembles the PLY array,
    eval.py:285 -- , colours uint8 [n,3])."""
    height, width = depth_est_averaged.shape[:2]
    x, y = np.meshgrid(np.arange(0, width), np.arange(0, height))
    x, y, depth = x[final_mask], y[final_mask], depth_est_averaged[final_mask]
    color = ref_img[final_mask]
    xyz_ref = np.matmul(np.linalg.inv(ref_intrinsics), np.vstack((x, y, np.ones_like(x))) * depth)
    xyz_world = np.matmul(np.linalg.inv(ref_extrinsics), np.vstack((xyz_ref, np.ones_like(x))))[:3]
    return xyz_world.transpose((1, 0)), (color * 255).astype(np.uint8)


def ply_vertex_body(vertices: np.ndarray, colors: np.ndarray) -> bytes:
    """The binary little-endian body of the reference's fused.ply (eval.py:283-296): per vertex float32 x, y, z and uint8
    red, green, blue = 15 bytes, in order."""
    rec = np.empty(len(vertices), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v = np.asarray(vertices)
    rec["x"], rec["y"], rec["z"] = v[:, 0].astype(np.float32), v[:, 1].astype(np.float32), v[:, 2].astype(np.float32)
    rec["red"], rec["green"], rec["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
    return rec.tobytes()
