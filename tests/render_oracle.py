"""numpy restatement of the rendering definition in include/patchmatch_b200.h (pmb200_render_points / pmb200_render_mesh), in
float32 with the kernels' operation order, so its images equal the GPU's bit for bit (test infrastructure).

Every product, sum and difference below is one float32 numpy operation, rounded on its own; `/` and sqrt are IEEE, np.rint
rounds half to even.  The z-buffer is a uint64 per pixel holding min((float_bits(z) << 32) | index)."""
from __future__ import annotations

import numpy as np

F = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
GREY = F(160.0)
MAX_COORD = F(4194304.0)  # 2^22
SMALL_BOX = 16


def camera(P) -> tuple:
    """A 3 x 4 float64 camera -> (P float32 [3,4], centre float32 [3]), as ops.render_camera_arrays rounds them."""
    P64 = np.asarray(P, dtype=np.float64)
    return P64.astype(F), (-np.linalg.solve(P64[:, :3], P64[:, 3])).astype(F)


def project(P32, xyz):
    """(u, v, z) float32 arrays: u' = ((P00 x + P01 y) + P02 z) + P03, u = u' / z."""
    x, y, z = (np.asarray(xyz, F)[:, a] for a in range(3))
    row = lambda r: ((P32[r, 0] * x + P32[r, 1] * y) + P32[r, 2] * z) + P32[r, 3]
    with np.errstate(all="ignore"):
        zz = row(2)
        return row(0) / zz, row(1) / zz, zz


def keys(z, index):
    return (z.astype(F).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(index, np.uint64)


def zmin(zbuf, pix, key):
    """zbuf[pix] = min(zbuf[pix], key) with repeated pixels (the atomicMin of every fragment)."""
    if pix.size == 0:
        return
    order = np.lexsort((key, pix))
    p, k = pix[order], key[order]
    first = np.r_[True, p[1:] != p[:-1]]
    zbuf[p[first]] = np.minimum(zbuf[p[first]], k[first])


def shade_factor(n, d):
    """0.25 + 0.75 |n . d| / (|n| |d|), 1 where |n| |d| is not finite and > 0.  n, d float32 [m,3]."""
    dot3 = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    with np.errstate(all="ignore"):
        den = np.sqrt(dot3(n, n)) * np.sqrt(dot3(d, d))
        f = F(0.25) + F(0.75) * np.abs(dot3(n, d) / den)
    ok = (den > 0) & (den < np.inf) & (f < np.inf)
    return np.where(ok, f, F(1.0)).astype(F)


def channels(c, f):
    return np.clip(np.rint(c * f[:, None]), 0, 255).astype(np.uint8)


def _resolve_empty(zbuf, background):
    H, W = zbuf.shape
    rgb = np.empty((H, W, 3), np.uint8)
    rgb[...] = np.asarray(background, np.uint8)
    depth = np.zeros((H, W), F)
    hit = zbuf != EMPTY
    depth[hit] = (zbuf[hit] >> np.uint64(32)).astype(np.uint32).view(F)
    return rgb, depth, hit


def point_zbuffer(xyz, P32, W, H, point_size, near):
    u, v, z = project(P32, xyz)
    near = F(near)
    ok = (z > near) & (z < np.inf) & (np.abs(u) < np.inf) & (np.abs(v) < np.inf)
    idx = np.flatnonzero(ok)
    cx, cy, z = np.rint(u[idx]), np.rint(v[idx]), z[idx]
    key = keys(z, idx)
    r = point_size // 2
    zbuf = np.full(H * W, EMPTY)
    for dy in range(-r, r + 1):
        for dx in range(-r, r + 1):
            with np.errstate(all="ignore"):
                px, py = cx + F(dx), cy + F(dy)
            inside = (px >= 0) & (px <= W - 1) & (py >= 0) & (py <= H - 1)
            zmin(zbuf, py[inside].astype(np.int64) * W + px[inside].astype(np.int64), key[inside])
    return zbuf.reshape(H, W)


def render_points(xyz, rgb, normals, P, W, H, near, point_size=1, shade=False, background=(255, 255, 255)):
    """-> (rgb uint8 [H,W,3], depth float32 [H,W]).  P is the 3 x 4 float64 camera."""
    P32, C = camera(P)
    xyz = np.asarray(xyz, F)
    zbuf = point_zbuffer(xyz, P32, W, H, point_size, near)
    out, depth, hit = _resolve_empty(zbuf, background)
    i = (zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    c = np.asarray(rgb, F)[i] if rgb is not None else np.full((i.size, 3), GREY, F)
    f = np.ones(i.size, F)
    if shade and normals is not None:
        f = shade_factor(np.asarray(normals, F)[i], C[None, :] - xyz[i])
    out[hit] = channels(c, f)
    return out, depth


# ---- triangles ------------------------------------------------------------------------------------------------------------


def top_left(ax, ay, bx, by):
    dx, dy = bx - ax, by - ay
    return (dy < 0) | ((dy == 0) & (dx > 0))


def edge_at(ax, ay, bx, by, px, py):
    """The edge function of a -> b at p, evaluated from the lower endpoint (smaller v, then u), negated when that is b."""
    flip = (by < ay) | ((by == ay) & (bx < ax))
    sx, sy, ex, ey = np.where(flip, bx, ax), np.where(flip, by, ay), np.where(flip, ax, bx), np.where(flip, ay, by)
    e = (ex - sx) * (py - sy) - (ey - sy) * (px - sx)
    return np.where(flip, -e, e)


def project_vertices(P32, xyz, W, H, near):
    """(u, v, z, ok) per vertex: ok when z > near, |u|, |v| <= 2^22, all finite."""
    u, v, z = project(P32, xyz)
    ok = (z > F(near)) & (z < np.inf) & (np.abs(u) <= MAX_COORD) & (np.abs(v) <= MAX_COORD)
    return np.where(ok, u, 0).astype(F), np.where(ok, v, 0).astype(F), np.where(ok, z, 1).astype(F), ok


def setup(proj, faces, W, H):
    """Vectorised over faces [m,3]: dict of slot arrays x, y, z, v [m,3] (slots 1, 2 swapped when A < 0), area, tl [m,3],
    box x0, x1, y0, y1, and ok (the face is rasterised)."""
    u, v, z, vok = proj
    nv = u.shape[0]
    fv = np.asarray(faces, np.int64).reshape(-1, 3)
    ok = ((fv >= 0) & (fv < nv)).all(1)
    idx = np.where(ok[:, None], fv, 0)
    ok &= vok[idx].all(1) if nv else np.zeros_like(ok)
    idx = np.where(ok[:, None], idx, 0)
    if nv == 0:
        x = y = np.zeros(idx.shape, F)
        zz = np.ones(idx.shape, F)
    else:
        x, y, zz = u[idx], v[idx], z[idx]
    A = (x[:, 1] - x[:, 0]) * (y[:, 2] - y[:, 0]) - (y[:, 1] - y[:, 0]) * (x[:, 2] - x[:, 0])
    ok &= A != 0
    sw = A < 0
    perm = np.where(sw[:, None], [0, 2, 1], [0, 1, 2])
    take = lambda a: np.take_along_axis(a, perm, 1)
    t = {"x": take(x), "y": take(y), "z": take(zz), "v": take(idx), "area": np.where(sw, -A, A).astype(F), "face": fv}
    X, Y = t["x"], t["y"]
    t["tl"] = np.stack([top_left(X[:, 1], Y[:, 1], X[:, 2], Y[:, 2]), top_left(X[:, 2], Y[:, 2], X[:, 0], Y[:, 0]),
                        top_left(X[:, 0], Y[:, 0], X[:, 1], Y[:, 1])], 1)
    t["x0"] = np.maximum(np.ceil(X.min(1)), 0).astype(np.int64)
    t["x1"] = np.minimum(np.floor(X.max(1)), W - 1).astype(np.int64)
    t["y0"] = np.maximum(np.ceil(Y.min(1)), 0).astype(np.int64)
    t["y1"] = np.minimum(np.floor(Y.max(1)), H - 1).astype(np.int64)
    t["ok"] = ok & (t["x0"] <= t["x1"]) & (t["y0"] <= t["y1"])
    return t


def cover(t, sel, px, py):
    """Faces t[sel] at pixels (px, py) (int arrays of sel's length): (covered, b [m,3], z)."""
    X, Y, Z, tl, A = t["x"][sel], t["y"][sel], t["z"][sel], t["tl"][sel], t["area"][sel]
    fx, fy = px.astype(F), py.astype(F)
    e = [edge_at(X[:, 1], Y[:, 1], X[:, 2], Y[:, 2], fx, fy), edge_at(X[:, 2], Y[:, 2], X[:, 0], Y[:, 0], fx, fy),
         edge_at(X[:, 0], Y[:, 0], X[:, 1], Y[:, 1], fx, fy)]
    inside = np.ones(px.shape, bool)
    for i in range(3):
        inside &= (e[i] > 0) | ((e[i] == 0) & tl[:, i])
    with np.errstate(all="ignore"):
        b = np.stack([e[i] / A for i in range(3)], 1)
        s = (b[:, 0] / Z[:, 0] + b[:, 1] / Z[:, 1]) + b[:, 2] / Z[:, 2]
        zz = F(1.0) / s
    inside &= (s > 0) & (zz < np.inf)
    return inside, b, zz


def mesh_zbuffer(proj, faces, W, H, count=False):
    """-> (zbuf uint64 [H,W], fragments per pixel int64 [H,W] when count else None).  Small faces (box at most 16 x 16) are
    visited by box offset, vectorised over faces; larger faces one at a time over their box."""
    t = setup(proj, faces, W, H)
    zbuf = np.full(H * W, EMPTY)
    frags = np.zeros(H * W, np.int64) if count else None
    bw, bh = t["x1"] - t["x0"] + 1, t["y1"] - t["y0"] + 1
    small = np.flatnonzero(t["ok"] & (bw <= SMALL_BOX) & (bh <= SMALL_BOX))
    large = np.flatnonzero(t["ok"] & ((bw > SMALL_BOX) | (bh > SMALL_BOX)))

    def emit(sel, px, py):
        inside, _, z = cover(t, sel, px, py)
        pix = py[inside] * W + px[inside]
        zmin(zbuf, pix, keys(z[inside], sel[inside]))
        if count:
            np.add.at(frags, pix, 1)

    for oy in range(SMALL_BOX):
        for ox in range(SMALL_BOX):
            sel = small[(ox < bw[small]) & (oy < bh[small])]
            emit(sel, t["x0"][sel] + ox, t["y0"][sel] + oy)
    for f in large:
        py, px = np.mgrid[t["y0"][f]:t["y1"][f] + 1, t["x0"][f]:t["x1"][f] + 1]
        emit(np.full(px.size, f), px.ravel(), py.ravel())
    return zbuf.reshape(H, W), (frags.reshape(H, W) if count else None)


def render_mesh(xyz, rgb, faces, P, W, H, near, shade=False, background=(255, 255, 255)):
    """-> (rgb uint8 [H,W,3], depth float32 [H,W])."""
    P32, C = camera(P)
    xyz = np.asarray(xyz, F)
    proj = project_vertices(P32, xyz, W, H, near)
    zbuf, _ = mesh_zbuffer(proj, faces, W, H)
    out, depth, hit = _resolve_empty(zbuf, background)
    f_idx = (zbuf[hit] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    py, px = np.nonzero(hit)
    t = setup(proj, np.asarray(faces, np.int64).reshape(-1, 3)[f_idx], W, H)
    sel = np.arange(f_idx.size)
    _, b, z = cover(t, sel, px, py)
    w = np.stack([(b[:, k] / t["z"][:, k]) * z for k in range(3)], 1)
    slots = t["v"]
    if rgb is not None:
        col = np.asarray(rgb, F)[slots]  # [m,3 slots,3 channels]
        c = (w[:, 0:1] * col[:, 0] + w[:, 1:2] * col[:, 1]) + w[:, 2:3] * col[:, 2]
    else:
        c = np.full((sel.size, 3), GREY, F)
    f = np.ones(sel.size, F)
    if shade:
        P3 = xyz[slots]
        X = (w[:, 0:1] * P3[:, 0] + w[:, 1:2] * P3[:, 1]) + w[:, 2:3] * P3[:, 2]
        own = xyz[t["face"]]  # the face's own vertex order
        e1, e2 = own[:, 1] - own[:, 0], own[:, 2] - own[:, 0]
        n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
        f = shade_factor(n, C[None, :] - X)
    out[hit] = channels(c, f)
    return out, depth
