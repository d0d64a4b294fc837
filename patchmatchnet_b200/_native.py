"""ctypes binding of the C ABI in ``include/patchmatch_b200.h`` (libpmb200.so).

The library is built in-tree by ``build_library()`` (called from
``__graft_entry__.build()``): a single ``nvcc -gencode arch=compute_90a,code=sm_90a``
invocation, no torch headers.  There is NO fallback: if the shared object is
missing or a call is made on a non-CUDA tensor the binding raises.
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_void_p
from typing import Optional

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
_REPO_DIR = os.path.dirname(_PKG_DIR)
LIB_PATH = os.path.join(_PKG_DIR, "libpmb200.so")
SOURCES = [os.path.join(_PKG_DIR, "csrc", f) for f in ("pm_kernels.cu", "pm_backward.cu", "pm_conv.cu", "pm_conv5.cu", "pm_stem.cu", "pm_refine.cu", "pm_geo.cu", "pm_cloud.cu", "pm_scan.cu", "pm_colmap.cu", "pm_undistort.cu", "pm_mesh.cu", "pm_render.cu", "pm_train.cu", "pm_mapio.cpp")]
HEADERS = [
    os.path.join(_PKG_DIR, "csrc", "pm_math.cuh"),
    os.path.join(_PKG_DIR, "csrc", "pm_warpcorr4.cuh"),
    os.path.join(_PKG_DIR, "csrc", "pm_geo_math.cuh"),
    os.path.join(_PKG_DIR, "csrc", "pm_mesh_math.cuh"),
    os.path.join(_PKG_DIR, "csrc", "pm_camera_math.cuh"),
    os.path.join(_REPO_DIR, "include", "patchmatch_b200.h"),
]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC", "--threads", "0",
]

# TorchScript-facing shim: TORCH_LIBRARY(pmb200) over the same C ABI (csrc/torch_binding.cpp), host C++ only
TORCH_LIB_PATH = os.path.join(_PKG_DIR, "libpmb200_torch.so")
TORCH_SOURCE = os.path.join(_PKG_DIR, "csrc", "torch_binding.cpp")

_lib: Optional[ctypes.CDLL] = None
_torch_ops_loaded = False


class NativeLibraryMissing(RuntimeError):
    pass


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise NativeLibraryMissing("nvcc not found; cannot build libpmb200.so")
    return exe


def needs_rebuild() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    built = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(f) > built for f in SOURCES + HEADERS)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into patchmatchnet_b200/libpmb200.so (in-tree)."""
    global _lib
    if not force and not needs_rebuild():
        return LIB_PATH
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB_PATH] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    _lib = None
    return LIB_PATH


_PF = POINTER(c_float)
_PPF = POINTER(c_void_p)


class MlpStruct(ctypes.Structure):
    """pmb200_mlp (include/patchmatch_b200.h): folded G->16->8->1 head, host memory."""

    _fields_ = [
        ("w0", c_float * (16 * 8)),
        ("b0", c_float * 16),
        ("w1", c_float * (8 * 16)),
        ("b1", c_float * 8),
        ("w2", c_float * 8),
        ("b2", c_float),
    ]


_PMLP = POINTER(MlpStruct)


class MapInfo(ctypes.Structure):
    """pmb200_map_info (include/patchmatch_b200.h)."""

    _fields_ = [
        ("format", c_int), ("width", c_int), ("height", c_int), ("channels", c_int), ("big_endian", c_int),
        ("scale", c_double), ("data_offset", c_int64), ("payload_floats", c_int64),
    ]


_PMAP = POINTER(MapInfo)


class ViewExtent(ctypes.Structure):
    """pmb200_view_extent (include/patchmatch_b200.h): one source view of a ragged pack."""

    _fields_ = [("offset", c_int64), ("height", c_int), ("width", c_int)]


_PVIEW = POINTER(ViewExtent)


class TsdfView(ctypes.Structure):
    """pmb200_tsdf_view (include/patchmatch_b200.h): one view of the TSDF integration."""

    _fields_ = [("K", c_double * 9), ("Rt", c_double * 12), ("depth_offset", c_int64), ("image_offset", c_int64),
                ("height", c_int), ("width", c_int)]


class CameraStruct(ctypes.Structure):
    """pmb200_camera (include/patchmatch_b200.h): one COLMAP camera of the undistortion."""

    _fields_ = [("model", c_int), ("width", c_int), ("height", c_int), ("reserved", c_int), ("params", c_double * 12)]


_PCAM = POINTER(CameraStruct)
_SIGNATURES = {
    "pmb200_abi_version": (c_int, []),
    "pmb200_last_error": (c_char_p, []),
    "pmb200_set_tuning": (c_int, [c_char_p, c_int]),
    "pmb200_relative_projection": (c_int, [c_void_p, c_int64, _PPF, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "pmb200_pack_nhwc": (c_int, [_PPF, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "pmb200_photometric_confidence": (c_int, [c_void_p] * 2 + [c_int] * 6 + [c_void_p]),
    "pmb200_upsample2x_add_nhwc": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_void_p]),
    "pmb200_conv2d_filter_floats": (c_int, [c_int] * 4),
    "pmb200_conv2d_nhwc": (c_int, [c_void_p] * 5 + [c_int] * 15 + [c_void_p]),
    "pmb200_conv2d_tc5_supported": (c_int, [c_int] * 4),
    "pmb200_conv2d_tc5_filter_floats": (c_int, [c_int] * 3),
    "pmb200_conv2d_tc5": (c_int, [c_void_p] * 4 + [c_int] * 12 + [c_void_p]),
    "pmb200_conv2d_tc5h": (c_int, [c_void_p] * 4 + [c_int] * 11 + [c_void_p]),
    "pmb200_conv2d_tc5h_plan": (c_int, [c_int] * 7 + [POINTER(c_int)]),
    "pmb200_debug_conv5h_trace": (c_int, [c_void_p]),
    "pmb200_conv_stem": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_void_p]),
    "pmb200_refine_low": (c_int, [c_void_p] * 8 + [c_int] * 3 + [c_void_p]),
    "pmb200_refine_full": (c_int, [c_void_p] * 13 + [c_int] * 3 + [c_void_p]),
    "pmb200_geometric_filter": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_double, c_float, c_float, c_int] + [c_void_p] * 5),
    "pmb200_fuse_points": (c_int, [c_void_p] * 4 + [c_int] * 2 + [c_void_p] * 4),
    "pmb200_fuse_points_oriented": (c_int, [c_void_p] * 5 + [c_int] * 2 + [c_void_p] * 4),
    "pmb200_depth_normals": (c_int, [c_void_p, POINTER(c_double), c_int, c_int, c_int, c_double, c_int, c_void_p, c_void_p]),
    "pmb200_tsdf_alloc_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_tsdf_alloc": (c_int, [c_void_p, c_int64, c_double, c_int, POINTER(c_int64), c_void_p, c_int64, c_void_p]),
    "pmb200_tsdf_integrate_workspace_bytes": (c_int64, [c_int]),
    "pmb200_tsdf_integrate": (c_int, [c_void_p, c_int64, c_double, c_int, c_void_p, c_int] + [c_void_p] * 6 + [c_int64, c_void_p]),
    "pmb200_tsdf_mesh_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_tsdf_mesh_count": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_tsdf_mesh_write": (c_int, [c_void_p, c_int64, c_double] + [c_void_p] * 3 + [c_int] + [c_void_p] * 3 + [c_int64, c_void_p]),
    "pmb200_render_points_workspace_bytes": (c_int64, [c_int, c_int]),
    "pmb200_render_points": (c_int, [c_void_p] * 3 + [c_int64, _PF, _PF, c_int, c_int, c_int, c_float, c_int, POINTER(ctypes.c_ubyte)]
                             + [c_void_p] * 3 + [c_int64, c_void_p]),
    "pmb200_render_mesh_workspace_bytes": (c_int64, [c_int, c_int, c_int64, c_int64]),
    "pmb200_render_mesh": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, _PF, _PF, c_int, c_int, c_float, c_int,
                                   POINTER(ctypes.c_ubyte)] + [c_void_p] * 3 + [c_int64, c_void_p]),
    "pmb200_thin_points_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_thin_points": (c_int, [c_void_p, c_void_p, c_int64, c_double, c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_nearest_distance_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_nearest_distance": (c_int, [c_void_p, c_int64, c_void_p, c_int64, POINTER(c_double), c_double, c_double, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_crop_polygon": (c_int, [c_void_p, c_int64, POINTER(c_double), c_int, c_double, c_double, POINTER(c_double), c_int,
                                    c_void_p, c_void_p, c_void_p]),
    "pmb200_voxel_downsample_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_voxel_downsample": (c_int, [c_void_p, c_int64, POINTER(c_double), c_double, c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_icp_target_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_icp_target": (c_int, [c_void_p, c_int64, c_double, c_void_p, c_int64, c_void_p]),
    "pmb200_icp_query_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_icp_query": (c_int, [c_void_p, c_int64, POINTER(c_double), POINTER(c_double), c_double, c_void_p, c_int64, c_double,
                                 c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_beam_index_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_beam_index": (c_int, [c_void_p, c_int64, POINTER(c_double), c_void_p, c_int64, c_void_p]),
    "pmb200_beam_observed": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, POINTER(c_double), c_double, c_double, c_void_p,
                                     c_void_p]),
    "pmb200_voxel_score_workspace_bytes": (c_int64, [c_int64]),
    "pmb200_voxel_score": (c_int, [c_void_p, c_void_p, c_int64, c_double, c_void_p, POINTER(c_double), c_void_p, c_void_p, c_void_p,
                                   c_int64, c_void_p]),
    "pmb200_view_scores_workspace_bytes": (c_int64, [c_int, c_int64, c_int64]),
    "pmb200_view_scores_count": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_view_scores": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int64, c_double, c_double, c_double,
                                   c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_depth_ranges_workspace_bytes": (c_int64, [c_int, c_int64]),
    "pmb200_depth_ranges": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int64, c_void_p]),
    "pmb200_undistort_extents": (c_int, [_PCAM, c_int, c_void_p, c_void_p, c_void_p]),
    "pmb200_undistort_image": (c_int, [c_void_p, _PCAM, POINTER(c_double), c_int, c_int, c_void_p, c_void_p]),
    "pmb200_depth_loss_workspace_bytes": (c_int64, [POINTER(c_int), c_int, c_int, c_int, c_int]),
    "pmb200_depth_loss": (c_int, [_PPF, POINTER(c_int), c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int64,
                                  c_void_p]),
    "pmb200_depth_loss_backward": (c_int, [_PPF, POINTER(c_int), c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                           c_float, _PPF, c_void_p]),
    "pmb200_depth_metrics": (c_int, [_PPF, c_void_p, c_void_p, c_int, c_int, c_int, POINTER(c_float), c_int, c_void_p, c_void_p]),
    "pmb200_map_probe":(c_int, [c_char_p, c_int, _PMAP]),
    "pmb200_map_read": (c_int, [c_char_p, c_int, c_void_p, c_int64, _PMAP]),
    "pmb200_map_write": (c_int, [c_char_p, c_int, c_void_p, c_int, c_int, c_int, c_double]),
    "pmb200_warp_corr": (c_int, [c_void_p] * 6 + [c_int] * 9 + [c_void_p]),
    "pmb200_aggregate_views": (c_int, [c_void_p] * 3 + [c_int] * 6 + [c_void_p]),
    "pmb200_offset_corr": (c_int, [c_void_p] * 2 + [c_int, c_void_p] + [c_int] * 7 + [c_void_p]),
    "pmb200_warp_corr_score": (c_int, [c_void_p] * 5 + [_PMLP, c_void_p] + [c_int] * 10 + [c_void_p]),
    "pmb200_warp_corr_view_weights": (c_int, [c_void_p] * 4 + [_PMLP, c_void_p, c_void_p] + [c_int] * 9 + [c_void_p]),
    "pmb200_warp_corr_views": (c_int, [c_void_p, c_void_p, _PVIEW] + [c_void_p] * 4 + [c_int] * 7 + [c_void_p]),
    "pmb200_warp_corr_score_views": (c_int, [c_void_p, c_void_p, _PVIEW] + [c_void_p] * 3 + [_PMLP, c_void_p] + [c_int] * 8 + [c_void_p]),
    "pmb200_warp_corr_view_weights_views": (c_int, [c_void_p, c_void_p, _PVIEW] + [c_void_p] * 2 + [_PMLP, c_void_p, c_void_p]
                                            + [c_int] * 7 + [c_void_p]),
    "pmb200_geometric_filter_views": (c_int, [c_void_p] * 3 + [_PVIEW, c_void_p] + [c_int] * 3 + [c_double, c_float, c_float, c_int]
                                      + [c_void_p] * 5),
    "pmb200_aggregate_views_score": (c_int, [c_void_p] * 2 + [_PMLP, c_void_p] + [c_int] * 7 + [c_void_p]),
    "pmb200_offset_corr_weight": (c_int, [c_void_p] * 2 + [c_int, _PMLP, c_void_p] + [c_int] * 7 + [c_void_p]),
    "pmb200_init_propagate": (c_int, [c_void_p] * 2 + [c_int] + [c_void_p] * 4 + [c_int] * 8 + [c_float, c_void_p]),
    "pmb200_adaptive_eval": (c_int, [c_void_p] * 5 + [c_int] + [c_void_p] * 5 + [c_int] * 6 + [c_float, c_int, c_void_p]),
    "pmb200_adaptive_eval_plan": (c_int, [c_int] * 6 + [POINTER(c_int)]),
    "pmb200_warp_corr_backward": (c_int, [c_void_p] * 8 + [c_int] * 9 + [c_void_p]),
    "pmb200_warp_corr_views_backward": (c_int, [c_void_p, c_void_p, _PVIEW] + [c_void_p] * 6 + [c_int] * 7 + [c_void_p]),
    "pmb200_aggregate_views_backward": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_void_p]),
    "pmb200_offset_corr_backward": (c_int, [c_void_p] * 4 + [c_int] * 7 + [c_void_p]),
    "pmb200_init_propagate_backward": (c_int, [c_void_p] * 6 + [c_int] * 7 + [c_float, c_void_p]),
    "pmb200_adaptive_eval_backward": (c_int, [c_void_p] * 14 + [c_int] * 6 + [c_float, c_int, c_void_p]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def build_torch_library(force: bool = False) -> str:
    """Compile csrc/torch_binding.cpp (g++, torch headers) into patchmatchnet_b200/libpmb200_torch.so.  It links
    against libpmb200.so (rpath $ORIGIN), so build_library() must have run."""
    deps = [TORCH_SOURCE, HEADERS[-1]]
    if not force and os.path.exists(TORCH_LIB_PATH) and all(os.path.getmtime(TORCH_LIB_PATH) >= os.path.getmtime(f) for f in deps):
        return TORCH_LIB_PATH
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryMissing("build libpmb200.so first (build_library())")
    import torch

    tdir = os.path.dirname(os.path.abspath(torch.__file__))
    cuda_home = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    cmd = [
        shutil.which("g++") or "g++", "-O2", "-std=c++17", "-shared", "-fPIC",
        f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}",
        f"-I{tdir}/include", f"-I{tdir}/include/torch/csrc/api/include", f"-I{cuda_home}/include",
        TORCH_SOURCE, "-o", TORCH_LIB_PATH,
        f"-L{tdir}/lib", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
        f"-L{_PKG_DIR}", "-lpmb200", "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{tdir}/lib",
    ]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed on torch_binding.cpp:\n" + res.stdout + res.stderr)
    return TORCH_LIB_PATH


def load_torch_ops() -> None:
    """Register `torch.ops.pmb200.*` (needed before a PatchMatch is scripted, and before torch.jit.load of a scripted
    model that contains it).  Raises NativeLibraryMissing when the shim has not been built."""
    global _torch_ops_loaded
    if _torch_ops_loaded:
        return
    if not os.path.exists(TORCH_LIB_PATH):
        raise NativeLibraryMissing(
            f"{TORCH_LIB_PATH} is missing -- run `python -c 'import __graft_entry__ as g; g.build()'`"
        )
    import torch

    torch.ops.load_library(TORCH_LIB_PATH)
    _torch_ops_loaded = True


def lib() -> ctypes.CDLL:
    """The loaded library; raises NativeLibraryMissing when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                f"{LIB_PATH} is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the H100 path has no CPU or PyTorch fallback)"
            )
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        if handle.pmb200_abi_version() != 1:
            raise RuntimeError("libpmb200.so ABI version mismatch; rebuild")
        _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().pmb200_last_error().decode("utf-8", "replace")
        if rc == -2:
            raise NotImplementedError(f"{what}: {msg}")
        raise RuntimeError(f"{what} failed (code {rc}): {msg}")


def pointer_array(ptrs):
    arr = (c_void_p * len(ptrs))(*ptrs)
    return ctypes.cast(arr, _PPF), arr  # keep `arr` alive for the duration of the call
