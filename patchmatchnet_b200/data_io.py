"""Depth / confidence map files (PFM, COLMAP .bin) -- host-side mirror of the map functions of the reference's
``datasets/data_io.py`` (SURVEY.md 8f row f5) over the native readers / writers of libpmb200.so
(``csrc/pm_mapio.cpp``, C ABI ``pmb200_map_{probe,read,write}``).

Same names, arguments, return values, exception texts and -- byte for byte -- the same files:

    read_map  data_io.py:128-145      save_map  data_io.py:148-162
    read_bin  data_io.py:165-191      save_bin  data_io.py:194-223
    read_pfm  data_io.py:226-288      save_pfm  data_io.py:291-322

plus the two calls the H100 path itself uses so that a map never passes through a pageable temporary:

    read_map_to_device(path, device)   file -> pinned host buffer -> one async copy to the GPU
    save_map_from_device(path, tensor) GPU -> pinned host buffer -> file (row flip / planar order folded into the write)

There is no Python fallback: without libpmb200.so every call raises ``NativeLibraryMissing``.
"""
from __future__ import annotations

import os
from typing import Dict, List
from typing import Tuple

import numpy as np
import torch

from . import _native

PFM = 1  # PMB200_MAP_PFM
COLMAP_BIN = 2  # PMB200_MAP_COLMAP_BIN
_UNSUPPORTED = "Invalid input format; only pfm and bin are supported"  # data_io.py:145, :162
_BAD_SHAPE = "Image must have H x W x 3, H x W x 1 or H x W dimensions."


def _raise(rc: int) -> None:
    msg = _native.lib().pmb200_last_error().decode("utf-8", "replace")
    if rc == -3:  # PMB200_EIO: "<strerror>: '<path>'"
        if msg.startswith("No such file or directory"):
            raise FileNotFoundError(2, "No such file or directory", msg.split(": ", 1)[1].strip("'"))
        raise OSError(msg)
    if rc == -4 and (msg.startswith("cannot reshape") or msg.startswith("could not convert")):
        raise ValueError(msg)  # what np.reshape / float() raise in the reference
    raise Exception(msg)  # the reference raises bare Exception("Not a PFM file.") etc.


def _format_of(path: str) -> int:
    if path.endswith(".bin"):
        return COLMAP_BIN
    if path.endswith(".pfm"):
        return PFM
    raise Exception(_UNSUPPORTED)


def _probe(path: str, fmt: int) -> "_native.MapInfo":
    info = _native.MapInfo()
    rc = _native.lib().pmb200_map_probe(os.fsencode(path), fmt, info)
    if rc != 0:
        _raise(rc)
    return info


def _read_into(path: str, fmt: int, pinned: bool) -> Tuple[torch.Tensor, "_native.MapInfo"]:
    info = _probe(path, fmt)
    n = info.width * info.height * info.channels
    buf = torch.empty((info.height, info.width, info.channels), dtype=torch.float32, pin_memory=pinned)
    rc = _native.lib().pmb200_map_read(os.fsencode(path), fmt, buf.data_ptr(), n, info)
    if rc != 0:
        _raise(rc)
    return buf, info


def read_pfm(filename: str) -> Tuple[np.ndarray, float]:
    """data_io.py:226-288 -> (array [H,W,1] ('Pf') or [H,W,3] ('PF'), float32, top row first; scale)."""
    buf, info = _read_into(filename, PFM, pinned=False)
    return buf.numpy(), float(info.scale)


def read_bin(path: str) -> np.ndarray:
    """data_io.py:165-191 -> array [H,W,C] float32."""
    return _read_into(path, COLMAP_BIN, pinned=False)[0].numpy()


def scale_to_max_dim(image: np.ndarray, max_dim: int) -> Tuple[np.ndarray, int, int]:
    """data_io.py:13-31 (cv2.resize is the reference's own library call; only taken when max_dim shrinks the map)."""
    original_height, original_width = image.shape[0], image.shape[1]
    scale = max_dim / max(original_height, original_width)
    if 0 < scale < 1:
        import cv2

        image = cv2.resize(image, (int(scale * original_width), int(scale * original_height)), interpolation=cv2.INTER_LINEAR)
    return image, original_height, original_width


def read_image(filename: str, max_dim: int = -1) -> Tuple[np.ndarray, int, int]:
    """data_io.py:34-47 -> (image float32 [H,W,C] in [0,1], scaled to `max_dim` when that shrinks it; original_h; original_w)."""
    from PIL import Image

    np_image = np.array(Image.open(filename), dtype=np.float32) / 255.0
    return scale_to_max_dim(np_image, max_dim)


def save_image(filename: str, image: np.ndarray) -> None:
    """data_io.py:50-64: bool -> uint8 0 / 255, float32 / float64 -> uint8(value * 255), anything else -> uint8; PIL picks
    the file format from the extension (the mask PNGs of the fusion)."""
    from PIL import Image

    if image.dtype == bool:
        image = image.astype(np.uint8) * 255
    elif image.dtype == np.float32 or image.dtype == np.float64:
        image = (image * 255).astype(np.uint8)
    else:
        image = image.astype(np.uint8)
    Image.fromarray(image).save(filename)


def read_image_dictionary(filename: str) -> Dict[int, str]:
    """data_io.py:67-83 -> {image id: image file name} from an ETH3D index2prefix.txt: a count line, then "<id> <name>"
    lines, split on single spaces."""
    image_dict: Dict[int, str] = {}
    with open(filename) as f:
        num_entries = int(f.readline().strip())
        for _ in range(num_entries):
            parts = f.readline().strip().split(" ")
            image_dict[int(parts[0].strip())] = parts[1].strip()
    return image_dict


def read_cam_file(filename: str) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """data_io.py:85-106 -> (intrinsics float32 [3,3] from lines 8-10, extrinsics float32 [4,4] from lines 2-5, depth params
    float32 from line 12 -- (depth_min, depth_max) in the DTU files -- or an empty float64 array when the file has no line 12).
    The numbers go through np.fromstring(..., float32, sep=' ') as in the reference, so every value has the same bits."""
    with open(filename) as f:
        lines = [line.rstrip() for line in f.readlines()]
    extrinsics = np.fromstring(" ".join(lines[1:5]), dtype=np.float32, sep=" ").reshape((4, 4))
    intrinsics = np.fromstring(" ".join(lines[7:10]), dtype=np.float32, sep=" ").reshape((3, 3))
    if len(lines) >= 12:
        depth_params = np.fromstring(lines[11], dtype=np.float32, sep=" ")
    else:
        depth_params = np.empty(0)
    return intrinsics, extrinsics, depth_params


def read_pair_file(filename: str) -> List[Tuple[int, List[int]]]:
    """data_io.py:109-127 -> [(reference view, [source views in file order])]; entries without source views are dropped."""
    data = []
    with open(filename) as f:
        num_viewpoint = int(f.readline())
        for _ in range(num_viewpoint):
            ref_view = int(f.readline().rstrip())
            src_views = [int(x) for x in f.readline().rstrip().split()[1::2]]
            if len(src_views) != 0:
                data.append((ref_view, src_views))
    return data


def scale_intrinsics(intrinsics: np.ndarray, image_hw: Tuple[int, int], original_h: int, original_w: int) -> np.ndarray:
    """The intrinsics of a view whose image read_image scaled from original_h x original_w to image_hw: row 0 times
    width / original width, row 1 times height / original height, in float32 (datasets/mvs.py:83-84, eval.py:210-211).
    Returns a scaled copy."""
    k = np.array(intrinsics, dtype=np.float32, copy=True)
    k[0] *= image_hw[1] / original_w
    k[1] *= image_hw[0] / original_h
    return k


def read_map(path: str, max_dim: int = -1) -> np.ndarray:
    """data_io.py:128-145."""
    if path.endswith(".bin"):
        in_map = read_bin(path)
    elif path.endswith(".pfm"):
        in_map, _ = read_pfm(path)
    else:
        raise Exception(_UNSUPPORTED)
    return scale_to_max_dim(in_map, max_dim)[0]


def _hwc(data: np.ndarray) -> Tuple[int, int, int]:
    if data.ndim == 2:
        return data.shape[0], data.shape[1], 1
    if data.ndim == 3 and data.shape[2] in (1, 3):
        return data.shape[0], data.shape[1], data.shape[2]
    raise Exception(_BAD_SHAPE)


def _write(path: str, fmt: int, data: np.ndarray, scale: float) -> None:
    h, w, c = _hwc(data)
    arr = np.ascontiguousarray(data)
    rc = _native.lib().pmb200_map_write(os.fsencode(path), fmt, arr.ctypes.data, h, w, c, scale)
    if rc != 0:
        _raise(rc)


def save_pfm(filename: str, image: np.ndarray, scale: float = 1) -> None:
    """data_io.py:291-322.  (The reference opens the file before it validates, leaving an empty file behind a failed
    call; here nothing is created unless the arguments are valid.)"""
    if image.dtype.name != "float32":
        raise Exception("Image dtype must be float32.")
    if image.dtype.byteorder == ">":
        raise Exception("big-endian arrays are not supported on the H100 host path")
    # the library prints "%f" of -scale; keep Python's own sign arithmetic for the written value (int 0 stays "0.000000")
    _write(filename, PFM, image, -float(-scale))


def save_bin(filename: str, data: np.ndarray) -> None:
    """data_io.py:194-223."""
    if data.dtype != np.float32:
        raise Exception("Image data type must be float32.")
    _write(filename, COLMAP_BIN, data, 1.0)


def save_map(path: str, data: np.ndarray) -> None:
    """data_io.py:148-162."""
    if path.endswith(".bin"):
        save_bin(path, data)
    elif path.endswith(".pfm"):
        save_pfm(path, data)
    else:
        raise Exception(_UNSUPPORTED)


def read_map_to_device(path: str, device, non_blocking: bool = True) -> torch.Tensor:
    """File -> pinned host buffer -> device, [H,W,C] float32.  The copy is enqueued on the current stream of `device`."""
    buf, _ = _read_into(path, _format_of(path), pinned=True)
    return buf.to(device, non_blocking=non_blocking)


def save_map_from_device(path: str, tensor: torch.Tensor, scale: float = 1) -> None:
    """Device map ([H,W], [H,W,1] or [H,W,3], float32) -> pinned host buffer -> file."""
    fmt = _format_of(path)
    if tensor.dtype != torch.float32:
        raise Exception("Image dtype must be float32." if fmt == PFM else "Image data type must be float32.")
    if tensor.dim() not in (2, 3) or (tensor.dim() == 3 and tensor.shape[2] not in (1, 3)):
        raise Exception(_BAD_SHAPE)
    src = tensor.detach().contiguous()
    host = torch.empty(src.shape, dtype=torch.float32, pin_memory=src.is_cuda)
    host.copy_(src)  # synchronous with respect to the host: the data is there when copy_ returns
    h, w = host.shape[0], host.shape[1]
    c = host.shape[2] if host.dim() == 3 else 1
    rc = _native.lib().pmb200_map_write(os.fsencode(path), fmt, host.data_ptr(), h, w, c, -float(-scale) if fmt == PFM else 1.0)
    if rc != 0:
        _raise(rc)


def save_ply(path: str, body, faces=None) -> None:
    """Write the reference's fused.ply (eval.py:283-296: PlyData([PlyElement.describe(vertex_all, "vertex")]).write -- binary
    little endian, one `vertex` element with float x, y, z and uchar red, green, blue) from vertex records produced by
    ops.fuse_points: uint8 [n,15] tensor(s) (a list concatenates the per-reference-view clouds, eval.py:283-284).
    Oriented records, uint8 [n,27] (ops.fuse_points with normals), write float nx, ny, nz between z and red, the property
    order of COLMAP's fused.ply; every part of one file has the same record size.
    With `faces`, int32 [nf,3] vertex indices (ops.tsdf_mesh), a `face` element (property list uchar int vertex_indices)
    follows the vertices; without it the file is the vertex element alone."""
    import torch

    parts = list(body) if isinstance(body, (list, tuple)) else [body]
    parts = [b.detach().cpu().contiguous() for b in parts]
    width = int(parts[0].shape[1]) if parts and parts[0].dim() == 2 else 15
    for b in parts:
        if b.dtype != torch.uint8 or b.dim() != 2 or b.shape[1] not in (15, 27) or b.shape[1] != width:
            raise ValueError("save_ply: vertex records must be uint8 [n,15] or [n,27] tensors of one size (ops.fuse_points)")
    n = sum(int(b.shape[0]) for b in parts)
    normals = "property float nx\nproperty float ny\nproperty float nz\n" if width == 27 else ""
    face_rows = None
    if faces is not None:
        fc = faces.detach().cpu().contiguous()
        if fc.dtype != torch.int32 or fc.dim() != 2 or fc.shape[1] != 3:
            raise ValueError("save_ply: faces must be an int32 [nf,3] tensor (ops.tsdf_mesh)")
        if fc.numel() and (int(fc.min()) < 0 or int(fc.max()) >= n):
            raise ValueError(f"save_ply: a face refers to a vertex outside 0..{n - 1}")
        face_rows = np.empty(fc.shape[0], dtype=[("n", "u1"), ("v", "<i4", (3,))])
        face_rows["n"] = 3
        face_rows["v"] = fc.numpy()
    face_header = "element face %d\nproperty list uchar int vertex_indices\n" % face_rows.shape[0] if face_rows is not None else ""
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "%sproperty uchar red\nproperty uchar green\nproperty uchar blue\n%send_header\n" % (n, normals, face_header))
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        for b in parts:
            f.write(b.numpy().tobytes())
        if face_rows is not None:
            f.write(face_rows.tobytes())


_PLY_TYPES = {
    "char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
    "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8",
}


def read_ply_points(path: str) -> np.ndarray:
    """Vertex positions of a PLY file -> float64 [n,3] (float32 coordinates widen exactly).

    Reads `binary_little_endian` and `ascii` files whose `vertex` element has scalar properties x, y, z among any others
    (colours, normals, ...) in any order, e.g. this project's save_ply output and the DTU `stl%03d_total.ply` files.  The
    header becomes a numpy structured dtype, so the body is read in one call.  Other formats raise ValueError."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements, current = None, [], None
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: PLY header has no end_header")
            words = line.decode("ascii", "replace").split()
            if not words or words[0] in ("comment", "obj_info"):
                continue
            if words[0] == "end_header":
                break
            if words[0] == "format":
                fmt = words[1]
            elif words[0] == "element":
                current = (words[1], int(words[2]), [])
                elements.append(current)
            elif words[0] == "property":
                if current is None:
                    raise ValueError(f"{path}: PLY property outside an element")
                if words[1] == "list":
                    current[2].append((words[-1], None))
                else:
                    if words[1] not in _PLY_TYPES:
                        raise ValueError(f"{path}: unknown PLY property type {words[1]!r}")
                    current[2].append((words[2], _PLY_TYPES[words[1]]))
        if fmt not in ("binary_little_endian", "ascii"):
            raise ValueError(f"{path}: PLY format {fmt!r} is not supported (binary_little_endian or ascii)")
        for name, count, props in elements:
            if name == "vertex":
                break
            if count:  # an element before the vertices would have to be skipped row by row
                raise ValueError(f"{path}: PLY element {name!r} precedes the vertex element")
        else:
            raise ValueError(f"{path}: PLY file has no vertex element")
        if any(t is None for _, t in props):
            raise ValueError(f"{path}: list properties in the vertex element are not supported")
        names = [p for p, _ in props]
        if not all(a in names for a in ("x", "y", "z")):
            raise ValueError(f"{path}: PLY vertex element lacks x, y or z")
        if fmt == "ascii":
            data = np.loadtxt(f, dtype=np.float64, max_rows=count, ndmin=2) if count else np.zeros((0, len(names)))
            if data.shape != (count, len(names)):
                raise ValueError(f"{path}: PLY body has {data.shape[0]} rows of {data.shape[1]} values, header says {count} of {len(names)}")
            return np.ascontiguousarray(data[:, [names.index(a) for a in ("x", "y", "z")]])
        dtype = np.dtype([(p, "<" + t) for p, t in props])
        data = np.fromfile(f, dtype=dtype, count=count)
        if data.shape[0] != count:
            raise ValueError(f"{path}: PLY body holds {data.shape[0]} vertices, header says {count}")
        out = np.empty((count, 3), dtype=np.float64)
        for a, axis in enumerate(("x", "y", "z")):
            out[:, a] = data[axis]
        return out


_PLY_FACE_LISTS = ("vertex_indices", "vertex_index")


def _ply_header(f, path: str):
    """(format, [(element name, count, [(property name, numpy type or ("list", count type, item type))])]) of an open PLY."""
    if f.readline().strip() != b"ply":
        raise ValueError(f"{path}: not a PLY file")
    fmt, elements, current = None, [], None
    while True:
        line = f.readline()
        if not line:
            raise ValueError(f"{path}: PLY header has no end_header")
        words = line.decode("ascii", "replace").split()
        if not words or words[0] in ("comment", "obj_info"):
            continue
        if words[0] == "end_header":
            break
        if words[0] == "format":
            fmt = words[1]
        elif words[0] == "element":
            current = (words[1], int(words[2]), [])
            elements.append(current)
        elif words[0] == "property":
            if current is None:
                raise ValueError(f"{path}: PLY property outside an element")
            types = words[2:4] if words[1] == "list" else words[1:2]
            for t in types:
                if t not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY property type {t!r}")
            if words[1] == "list":
                current[2].append((words[4], ("list", _PLY_TYPES[words[2]], _PLY_TYPES[words[3]])))
            else:
                current[2].append((words[2], _PLY_TYPES[words[1]]))
    if fmt not in ("binary_little_endian", "ascii"):
        raise ValueError(f"{path}: PLY format {fmt!r} is not supported (binary_little_endian or ascii)")
    return fmt, elements


def _ply_colour(v: np.ndarray) -> np.ndarray:
    """One colour channel -> uint8: integer types clamped to 0..255, floating types as 255 * v rounded and clamped."""
    if v.dtype.kind == "f":
        v = np.rint(v.astype(np.float64) * 255.0)
    return np.clip(v, 0, 255).astype(np.uint8)


def read_ply(path: str):
    """A point cloud or triangle mesh from a PLY file -> (xyz float32 [n,3], colours uint8 [n,3] or None, normals float32
    [n,3] or None, faces int32 [nf,3] or None).

    Reads `binary_little_endian` and `ascii` files: this project's fused.ply (plain and oriented), mesh.ply and the coloured
    class clouds of the evaluations, and ground-truth scans such as DTU's stl*.ply.  The `vertex` element comes first with
    scalar properties x, y, z and optionally red, green, blue (uchar as they are; other integer types clamped to 0..255,
    floating types in [0,1] scaled by 255 and rounded) and nx, ny, nz.  Double coordinates are narrowed to float32, which
    rounds ground-truth scans to float32.  A `face` element holds one list property `vertex_indices` (or `vertex_index`)
    with an integer count type (uchar, int, uint, ...).  Other elements after the vertices are skipped.  ValueError on a
    polygon that is not a triangle, a vertex index out of range, and on every malformed file read_ply_points rejects."""
    with open(path, "rb") as f:
        fmt, elements = _ply_header(f, path)
        if not elements or elements[0][0] != "vertex":
            for name, count, _ in elements:
                if name == "vertex":
                    break
                if count:
                    raise ValueError(f"{path}: PLY element {name!r} precedes the vertex element")
            else:
                raise ValueError(f"{path}: PLY file has no vertex element")
            elements = [e for e in elements if e[1] or e[0] == "vertex"]
            elements = elements[[e[0] for e in elements].index("vertex"):]
        ascii_rows = None
        if fmt == "ascii":
            ascii_rows = iter(f.read().decode("ascii", "replace").splitlines())
        xyz = colours = normals = faces = None
        for name, count, props in elements:
            lists = [p for p, t in props if isinstance(t, tuple)]
            if name == "vertex":
                if lists:
                    raise ValueError(f"{path}: list properties in the vertex element are not supported")
                names = [p for p, _ in props]
                if not all(a in names for a in ("x", "y", "z")):
                    raise ValueError(f"{path}: PLY vertex element lacks x, y or z")
                data = _ply_scalar_rows(f, ascii_rows, props, count, path)
                xyz = np.stack([data[a] for a in ("x", "y", "z")], axis=1).astype(np.float32)
                if all(a in names for a in ("red", "green", "blue")):
                    colours = np.stack([_ply_colour(data[a]) for a in ("red", "green", "blue")], axis=1)
                if all(a in names for a in ("nx", "ny", "nz")):
                    normals = np.stack([data[a] for a in ("nx", "ny", "nz")], axis=1).astype(np.float32)
            elif name == "face":
                if len(props) != 1 or props[0][0] not in _PLY_FACE_LISTS:
                    raise ValueError(f"{path}: the face element must hold one list property vertex_indices (or vertex_index)")
                _, count_t, item_t = props[0][1]
                if count_t[0] not in "iu" or item_t[0] not in "iu":
                    raise ValueError(f"{path}: face lists need integer count and index types")
                faces = _ply_triangles(f, ascii_rows, count_t, item_t, count, path)
                if faces.size and (faces.min() < 0 or faces.max() >= xyz.shape[0]):
                    raise ValueError(f"{path}: a face refers to a vertex outside 0..{xyz.shape[0] - 1}")
                faces = faces.astype(np.int32)
            else:
                if lists:
                    raise ValueError(f"{path}: list properties in the PLY element {name!r} are not supported")
                _ply_scalar_rows(f, ascii_rows, props, count, path)
        return xyz, colours, normals, faces


def _ply_scalar_rows(f, ascii_rows, props, count: int, path: str) -> np.ndarray:
    dtype = np.dtype([(p, "<" + t) for p, t in props])
    if ascii_rows is None:
        data = np.fromfile(f, dtype=dtype, count=count)
        if data.shape[0] != count:
            raise ValueError(f"{path}: PLY body holds {data.shape[0]} rows, header says {count}")
        return data
    lines = [next(ascii_rows, "") for _ in range(count)]
    vals = np.array(" ".join(lines).split(), dtype=np.float64)
    if vals.size != count * len(props) or any(len(line.split()) != len(props) for line in lines):
        raise ValueError(f"{path}: PLY body does not hold {count} rows of {len(props)} values")
    out = np.zeros(count, dtype=dtype)
    for k, (p, _) in enumerate(props):
        out[p] = vals[k::len(props)]
    return out


def _ply_triangles(f, ascii_rows, count_t: str, item_t: str, count: int, path: str) -> np.ndarray:
    if ascii_rows is None:
        rows = np.fromfile(f, dtype=np.dtype([("n", "<" + count_t), ("v", "<" + item_t, (3,))]), count=count)
        bad = np.flatnonzero(rows["n"] != 3)
        if bad.size:  # rows up to the first non-triangle are aligned, so its count is read where it is
            raise ValueError(f"{path}: face {int(bad[0])} has {int(rows['n'][bad[0]])} vertices; only triangles are supported")
        if rows.shape[0] != count:
            raise ValueError(f"{path}: PLY body holds {rows.shape[0]} faces, header says {count}")
        v = rows["v"].astype(np.int64)
    else:
        v = np.zeros((count, 3), dtype=np.int64)
        for i in range(count):
            words = next(ascii_rows, "").split()
            if not words or int(words[0]) != 3 or len(words) != 4:
                raise ValueError(f"{path}: face {i} is not a triangle ({' '.join(words) or 'missing'})")
            v[i] = [int(w) for w in words[1:]]
    return v
