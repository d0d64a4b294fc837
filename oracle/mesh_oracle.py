"""Oracle of the TSDF mesher (include/patchmatch_b200.h "Meshes"; beyond the reference, which has no mesher): allocation,
integration and marching cubes restated in numpy float64.  The triangle table is read from the text of
patchmatchnet_b200/csrc/pm_mesh_math.cuh; the tests check it with invariants of their own.  Never imported by the product.
"""
from __future__ import annotations

import os
import re
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "patchmatchnet_b200", "csrc",
                       "pm_mesh_math.cuh")
KEY_BIAS = 1 << 20
VOXEL_LIMIT = 1 << 23
# corner c at offset (x, y, z); edges as (lower corner offset, axis)
CORNERS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)], dtype=np.int64)
EDGE_OFFSET = np.array([(0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (0, 0, 1), (0, 0, 0),
                        (1, 0, 0), (1, 1, 0), (0, 1, 0)], dtype=np.int64)
EDGE_AXIS = np.array([0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2], dtype=np.int64)
UNIT = np.eye(3, dtype=np.int64)


def read_table(path: str = _HEADER) -> np.ndarray:
    """kTriTable of the header -> int8 [256,16] (edge triples, -1 after the last)."""
    text = open(path).read()
    body = text[text.index("kTriTable[256][kTableWidth] = {") :]
    body = body[body.index("{") + 1 : body.index("};")]
    rows = re.findall(r"\{([^{}]*)\}", body)
    tab = np.array([[int(v) for v in r.split(",") if v.strip()] for r in rows], dtype=np.int8)
    assert tab.shape == (256, 16), tab.shape
    return tab


def block_key(b: np.ndarray) -> np.ndarray:
    """[..., 3] int block coordinates -> uint64 keys."""
    b = b.astype(np.int64) + KEY_BIAS
    return (b[..., 2].astype(np.uint64) << np.uint64(42)) | (b[..., 1].astype(np.uint64) << np.uint64(21)) | b[..., 0].astype(np.uint64)


def key_blocks(keys: np.ndarray) -> np.ndarray:
    k = keys.astype(np.uint64)
    m = np.uint64((1 << 21) - 1)
    return np.stack([(k & m), (k >> np.uint64(21)) & m, (k >> np.uint64(42)) & m], -1).astype(np.int64) - KEY_BIAS


def allocate(points: np.ndarray, s: float, trunc: int) -> np.ndarray:
    """Sorted unique uint64 keys of the blocks the cubes [p - tau, p + tau] meet; ValueError when a voxel index does not fit."""
    p = np.asarray(points, dtype=np.float32).astype(np.float64)
    tau = trunc * s
    lo, hi = np.floor((p - tau) / s), np.floor((p + tau) / s)
    if not (np.all(lo >= -VOXEL_LIMIT) and np.all(hi < VOXEL_LIMIT)):
        raise ValueError("a seed point's voxel index does not fit")
    lo, hi = lo.astype(np.int64) >> 3, hi.astype(np.int64) >> 3
    keys = [block_key(np.stack([np.where(c & 1, hi[:, 0], lo[:, 0]), np.where(c & 2, hi[:, 1], lo[:, 1]),
                                np.where(c & 4, hi[:, 2], lo[:, 2])], -1)) for c in range(8)]
    return np.unique(np.concatenate(keys)) if len(p) else np.zeros(0, np.uint64)


def voxel_coords(keys: np.ndarray) -> np.ndarray:
    """[n_blocks * 512, 3] int64 voxel indices in the volume's order (block, then x fastest)."""
    b = key_blocks(keys)
    v = np.arange(512)
    local = np.stack([v & 7, (v >> 3) & 7, v >> 6], -1)
    return (8 * b[:, None, :] + local[None]).reshape(-1, 3)


def integrate(keys, s: float, trunc: int, depths, images, Ks, Es):
    """-> (tsdf float32, weight float32, colour uint8 [.,3]) per voxel of the volume's order."""
    tau = trunc * s
    X = (voxel_coords(keys).astype(np.float64) + 0.5) * s
    n = np.zeros(len(X), np.int64)
    F = np.zeros(len(X))
    C = np.zeros((len(X), 3))
    for d, img, K, E in zip(depths, images, Ks, Es):
        d = np.asarray(d, np.float32)
        img = np.asarray(img, np.float32)
        K = np.asarray(K, np.float32).astype(np.float64)
        Rt = np.asarray(E, np.float32).astype(np.float64)[:3]
        H, W = d.shape
        xc = ((Rt[0, 0] * X[:, 0] + Rt[0, 1] * X[:, 1]) + Rt[0, 2] * X[:, 2]) + Rt[0, 3]
        yc = ((Rt[1, 0] * X[:, 0] + Rt[1, 1] * X[:, 1]) + Rt[1, 2] * X[:, 2]) + Rt[1, 3]
        zc = ((Rt[2, 0] * X[:, 0] + Rt[2, 1] * X[:, 1]) + Rt[2, 2] * X[:, 2]) + Rt[2, 3]
        front = zc > 0
        zs = np.where(front, zc, 1.0)
        with np.errstate(invalid="ignore", over="ignore"):
            u = ((K[0, 0] * xc + K[0, 1] * yc) + K[0, 2] * zc) / zs
            v = ((K[1, 0] * xc + K[1, 1] * yc) + K[1, 2] * zc) / zs
            fx, fy = np.floor(u + 0.5), np.floor(v + 0.5)
        ok = front & (fx >= 0) & (fx < W) & (fy >= 0) & (fy < H)
        px, py = np.where(ok, fx, 0).astype(np.int64), np.where(ok, fy, 0).astype(np.int64)
        dv = d[py, px].astype(np.float64)
        ok &= np.isfinite(dv) & (dv > 0)
        sdf = dv - zc
        ok &= ~(sdf < -tau)
        n += ok
        F += np.where(ok, np.minimum(1.0, sdf / tau), 0.0)
        C += np.where(ok[:, None], img[:, py, px].T.astype(np.float64), 0.0)
    nn = np.maximum(n, 1)
    tsdf = np.where(n > 0, F / nn, 1.0).astype(np.float32)
    colour = np.where(n[:, None] > 0, np.clip(np.rint(255.0 * (C / nn[:, None])), 0, 255), 0).astype(np.uint8)
    return tsdf, n.astype(np.float32), colour


def marching_cubes(keys, s: float, tsdf, weight, colour, min_weight: int = 1, table=None):
    """Marching cubes over a volume in the layout integrate returns (colour [.,3] or [.,4]) -> (positions float32 [nv,3],
    colours uint8 [nv,3], faces int32 [nf,3]) in the documented order."""
    tab = read_table() if table is None else table
    keys = np.asarray(keys, np.uint64)
    coords = voxel_coords(keys)
    tsdf = np.asarray(tsdf, np.float32)
    valid = np.asarray(weight) >= min_weight
    colour = np.asarray(colour)[:, :3]

    def lookup(c):
        """voxel indices of coordinates [m,3] -> global index or -1 (a block outside the key range would alias another
        key: its coordinate field overflows into the next one)"""
        b = c >> 3
        inside = ((b >= -KEY_BIAS) & (b < KEY_BIAS)).all(-1)
        k = block_key(np.where(inside[:, None], b, 0))
        pos = np.searchsorted(keys, k)
        posc = np.minimum(pos, len(keys) - 1)
        hit = inside & (pos < len(keys)) & (keys[posc] == k)
        local = (c[:, 0] & 7) + 8 * (c[:, 1] & 7) + 64 * (c[:, 2] & 7)
        return np.where(hit, posc * 512 + local, -1)

    G = len(coords)
    corner_idx = np.stack([lookup(coords + CORNERS[c]) for c in range(8)], -1)  # [G,8]
    corner_valid = (corner_idx >= 0) & valid[np.maximum(corner_idx, 0)]
    cube_ok = corner_valid.all(1)
    neg = tsdf[np.maximum(corner_idx, 0)] < 0
    case = (neg * (1 << np.arange(8))).sum(1)
    meshed = cube_ok & (case != 0) & (case != 255)
    meshed_ext = np.append(meshed, False)  # index -1 -> False

    # owned edges: (voxel, axis), sign change between two valid voxels, one of the four cubes meshed
    owned = np.zeros((G, 3), bool)
    other = np.zeros((G, 3), np.int64)
    for k in range(3):
        b = lookup(coords + UNIT[k])
        other[:, k] = b
        ok = valid & (b >= 0)
        ok &= valid[np.maximum(b, 0)]
        ok &= (tsdf < 0) != (tsdf[np.maximum(b, 0)] < 0)
        j, l = [a for a in range(3) if a != k]
        any_meshed = np.zeros(G, bool)
        for dj in (0, 1):
            for dl in (0, 1):
                any_meshed |= meshed_ext[lookup(coords - dj * UNIT[j] - dl * UNIT[l])]
        owned[:, k] = ok & any_meshed
    vid = np.full((G, 3), -1, np.int64)
    flat = owned.ravel()
    vid.ravel()[flat] = np.arange(int(flat.sum()))
    a_idx, axis = np.nonzero(owned)
    b_idx = other[a_idx, axis]
    Xa = (coords[a_idx].astype(np.float64) + 0.5) * s
    Xb = (coords[b_idx].astype(np.float64) + 0.5) * s
    ta, tb = tsdf[a_idx].astype(np.float64), tsdf[b_idx].astype(np.float64)
    t = ta / (ta - tb)
    pos = (Xa + t[:, None] * (Xb - Xa)).astype(np.float32)
    ca, cb = colour[a_idx].astype(np.float64), colour[b_idx].astype(np.float64)
    col = np.clip(np.rint(ca + t[:, None] * (cb - ca)), 0, 255).astype(np.uint8)

    cubes = np.nonzero(meshed)[0]
    rows = tab[case[cubes]].astype(np.int64)  # [m,16]
    faces = []
    per_cube = []
    for q in range(5):
        e = rows[:, 3 * q : 3 * q + 3]
        has = e[:, 0] >= 0
        ee = np.maximum(e, 0)
        vox = lookup((coords[cubes][:, None, :] + EDGE_OFFSET[ee]).reshape(-1, 3)).reshape(-1, 3)
        f = vid[vox, EDGE_AXIS[ee]]
        per_cube.append(np.where(has[:, None], f, -2))
    tri = np.stack(per_cube, 1).reshape(-1, 3)  # cube-major, then table order
    faces = tri[tri[:, 0] != -2]
    assert (faces >= 0).all(), "a meshed cube refers to an edge without a vertex"
    return pos, col, faces.astype(np.int32)


# ---- chunked forms: any subset of a large volume, memory linear in the chunk ------------------------------------------------

def integrate_blocks(keys, s: float, trunc: int, depths, images, Ks, Es, chunk: int = 256):
    """integrate() of the blocks `keys` (any subset of a volume's keys, in any order), `chunk` blocks at a time: every voxel's
    sums depend on that voxel alone, so the result is integrate(keys, ...) bit for bit."""
    keys = np.asarray(keys, np.uint64)
    parts = [integrate(keys[i : i + chunk], s, trunc, depths, images, Ks, Es) for i in range(0, len(keys), chunk)]
    if not parts:
        return np.zeros(0, np.float32), np.zeros(0, np.float32), np.zeros((0, 3), np.uint8)
    return tuple(np.concatenate(p) for p in zip(*parts))


# neighbour n of a block at offset NEIGHBOURS[n] = (dx, dy, dz), n = (dx + 1) + 3 (dy + 1) + 9 (dz + 1)
NEIGHBOURS = np.array([(dx, dy, dz) for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1)], dtype=np.int64)
_TILE = np.arange(-1, 9)  # voxel coordinates -1..8 of a block's tile along one axis


def neighbour_blocks(keys: np.ndarray, blocks: np.ndarray) -> np.ndarray:
    """[len(blocks), 27] indices into the sorted `keys` of the neighbours of blocks keys[blocks], -1 where a neighbour is not
    allocated or lies outside the key range."""
    c = key_blocks(keys[blocks])[:, None, :] + NEIGHBOURS
    inside = ((c >= -KEY_BIAS) & (c < KEY_BIAS)).all(-1)
    k = block_key(np.where(inside[..., None], c, 0))
    pos = np.minimum(np.searchsorted(keys, k), len(keys) - 1)
    return np.where(inside & (keys[pos] == k), pos, -1)


def _tiles(keys, blocks, tsdf, valid):
    """Per block the voxels -1..8 along each axis, [B,10,10,10] indexed [z,y,x]: (global voxel index or -1, tsdf with NaN
    where the voxel is not valid), and the neighbour table."""
    nb = neighbour_blocks(keys, blocks)
    n = (_TILE >> 3) + 1
    local = _TILE & 7
    tb = nb[:, (9 * n)[:, None, None] + (3 * n)[None, :, None] + n[None, None, :]]
    g = np.where(tb >= 0, tb * 512 + (64 * local[:, None, None] + 8 * local[None, :, None] + local[None, None, :]), -1)
    ok = g >= 0
    ok[ok] = valid[g[ok]]
    return g, np.where(ok, tsdf[np.maximum(g, 0)], np.float32(np.nan)), nb


def _owned_and_cases(t):
    """tsdf tiles [B,10,10,10] -> (owned [B,8,8,8,3]: the voxel's edge along x / y / z has a vertex, case int16 [B,9,9,9] of
    the cubes with minimum corner -1..7, -1 unless the cube is meshed)."""
    valid, neg = ~np.isnan(t), t < 0
    allv = np.ones(t.shape[:1] + (9, 9, 9), bool)
    case = np.zeros(t.shape[:1] + (9, 9, 9), np.int16)
    for c, (ox, oy, oz) in enumerate(CORNERS):
        allv &= valid[:, oz : oz + 9, oy : oy + 9, ox : ox + 9]
        case |= neg[:, oz : oz + 9, oy : oy + 9, ox : ox + 9].astype(np.int16) << c
    meshed = allv & (case != 0) & (case != 255)
    owned = np.zeros(t.shape[:1] + (8, 8, 8, 3), bool)
    a_valid, a_neg = valid[:, 1:9, 1:9, 1:9], neg[:, 1:9, 1:9, 1:9]
    for k in range(3):
        ux, uy, uz = UNIT[k]
        b = (slice(None), slice(1 + uz, 9 + uz), slice(1 + uy, 9 + uy), slice(1 + ux, 9 + ux))
        any_meshed = np.zeros_like(a_valid)
        j, l = [a for a in range(3) if a != k]
        for dj in (0, 1):
            for dl in (0, 1):
                dx, dy, dz = dj * UNIT[j] + dl * UNIT[l]
                any_meshed |= meshed[:, 1 - dz : 9 - dz, 1 - dy : 9 - dy, 1 - dx : 9 - dx]
        owned[..., k] = a_valid & valid[b] & (a_neg != neg[b]) & any_meshed
    return owned, np.where(meshed, case, np.int16(-1))


def _map_chunks(fn, blocks, chunk):
    """[fn(part) for each chunk of blocks], the chunks on a thread pool (numpy releases the GIL in its array loops)."""
    parts = [blocks[i : i + chunk] for i in range(0, len(blocks), chunk)]
    with ThreadPoolExecutor(max_workers=min(len(parts), os.cpu_count() or 1) or 1) as ex:
        return list(ex.map(fn, parts))


def marching_cubes_blocks(keys, s: float, tsdf, weight, colour, emit, min_weight: int = 1, table=None, chunk: int = 1024):
    """marching_cubes() restricted to the blocks keys[emit] (emit: increasing block indices): the vertices those blocks' voxels
    own and the faces of their cubes, with the global vertex numbering of the whole volume.  A count pass over every block
    and a prefix sum give each block's first vertex and face; each block reads its 26 neighbours from the full key array
    and its voxels -1..8 along each axis; the faces of an emitted block read the vertex numbering of its neighbours.  Work
    goes `chunk` blocks at a time.  -> (positions float32 [m,3], colours uint8 [m,3], faces int32 [f,3], the vertices' global
    indices int64 [m], the faces' global indices int64 [f]).  Over emit = every block this is marching_cubes()."""
    tab = read_table() if table is None else table
    ntri = (tab[:, ::3] >= 0).sum(1)
    ntri[[0, 255]] = 0
    keys = np.asarray(keys, np.uint64)
    tsdf = np.asarray(tsdf, np.float32)
    valid = np.asarray(weight) >= min_weight
    colour = np.asarray(colour)[:, :3]
    emit = np.asarray(emit, np.int64)
    assert (np.diff(emit) > 0).all()

    def owned_of(blocks):
        return _owned_and_cases(_tiles(keys, blocks, tsdf, valid)[1])[0].reshape(len(blocks), 1536)

    def counts(blocks):
        owned, case = _owned_and_cases(_tiles(keys, blocks, tsdf, valid)[1])
        c = case[:, 1:, 1:, 1:].reshape(len(blocks), -1)
        return owned.reshape(len(blocks), -1).sum(1), np.where(c >= 0, ntri[np.maximum(c, 0)], 0).sum(1)

    cnt = _map_chunks(counts, np.arange(len(keys)), chunk)
    nv = np.concatenate([c[0] for c in cnt]) if cnt else np.zeros(0, np.int64)
    nf = np.concatenate([c[1] for c in cnt]) if cnt else np.zeros(0, np.int64)
    vbase = np.concatenate([[0], np.cumsum(nv)])
    fbase = np.concatenate([[0], np.cumsum(nf)])

    def emit_chunk(blocks):
        B = len(blocks)
        g, t, nb = _tiles(keys, blocks, tsdf, valid)
        owned, case = _owned_and_cases(t)
        # vertices: block, voxel (x fastest), axis
        bi, z, y, x, k = np.nonzero(owned)
        ga = g[bi, z + 1, y + 1, x + 1]
        gb = g[bi, z + 1 + UNIT[k, 2], y + 1 + UNIT[k, 1], x + 1 + UNIT[k, 0]]
        ia = key_blocks(keys[blocks[bi]]) * 8 + np.stack([x, y, z], -1)
        Xa = (ia.astype(np.float64) + 0.5) * s
        Xb = ((ia + UNIT[k]).astype(np.float64) + 0.5) * s
        ta, tb = tsdf[ga].astype(np.float64), tsdf[gb].astype(np.float64)
        tt = ta / (ta - tb)
        pos = (Xa + tt[:, None] * (Xb - Xa)).astype(np.float32)
        cA, cB = colour[ga].astype(np.float64), colour[gb].astype(np.float64)
        col = np.clip(np.rint(cA + tt[:, None] * (cB - cA)), 0, 255).astype(np.uint8)
        vid = vbase[blocks[bi]] + np.cumsum(owned.reshape(B, -1), 1)[bi, 3 * (x + 8 * y + 64 * z) + k] - 1
        # the owned edges of these blocks and their neighbours, and their exclusive prefix per block
        near = np.unique(nb[nb >= 0])
        own = np.zeros((len(near), 1536), bool)
        own[np.searchsorted(near, blocks)] = owned.reshape(B, -1)
        rest = np.setdiff1d(near, blocks)
        if len(rest):
            own[np.searchsorted(near, rest)] = owned_of(rest)
        pre = np.cumsum(own, 1) - 1
        # faces: cube (the voxel's order), then table order
        cb, cz, cy, cx = np.nonzero(case[:, 1:, 1:, 1:] >= 0)
        rows = tab[case[cb, cz + 1, cy + 1, cx + 1]].astype(np.int64)
        tri = np.full((len(cb), 5, 3), -2, np.int64)
        for q in range(5):
            e = rows[:, 3 * q : 3 * q + 3]
            has = e[:, 0] >= 0
            ee = np.maximum(e, 0)
            w = np.stack([cx, cy, cz], -1)[:, None, :] + EDGE_OFFSET[ee]  # [m, 3 vertices, xyz], each in 0..8
            n = (w >> 3) + 1
            blk = nb[cb[:, None], n[..., 0] + 3 * n[..., 1] + 9 * n[..., 2]]
            lw = w & 7
            slot = 3 * (lw[..., 0] + 8 * lw[..., 1] + 64 * lw[..., 2]) + EDGE_AXIS[ee]
            r = np.searchsorted(near, blk)
            assert own[r[has], slot[has]].all(), "a meshed cube refers to an edge without a vertex"
            tri[:, q] = np.where(has[:, None], vbase[blk] + pre[r, slot], -2)
        tri = tri.reshape(-1, 3)
        faces = tri[tri[:, 0] != -2]
        fid = np.repeat(fbase[blocks], nf[blocks]) + (np.arange(int(nf[blocks].sum())) - np.repeat(np.cumsum(nf[blocks]) - nf[blocks], nf[blocks]))
        assert len(fid) == len(faces)
        return pos, col, faces.astype(np.int32), vid, fid

    out = _map_chunks(emit_chunk, emit, chunk)
    if not out:
        return (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint8), np.zeros((0, 3), np.int32), np.zeros(0, np.int64),
                np.zeros(0, np.int64))
    return tuple(np.concatenate(p) for p in zip(*out))


def mesh(points, depths, images, Ks, Es, s: float, trunc: int = 3, min_weight: int = 1):
    """Allocation, integration and marching cubes -> (positions, colours, faces, keys, (tsdf, weight, colour))."""
    keys = allocate(points, s, trunc)
    vol = integrate(keys, s, trunc, depths, images, Ks, Es)
    pos, col, faces = marching_cubes(keys, s, *vol, min_weight=min_weight)
    return pos, col, faces, keys, vol
