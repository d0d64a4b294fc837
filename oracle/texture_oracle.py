"""numpy restatement of the mesh texturing definition in include/patchmatch_b200.h (pmb200_texture_mesh / _pack / _write),
so labels, charts, placements, texture coordinates and page bytes equal the GPU's bit for bit (test infrastructure).

float64 arithmetic below is one numpy operation per rounding, in the order of patchmatchnet_b200/csrc/pm_texture_math.cuh;
the z-buffer is tests/render_oracle.py's."""
from __future__ import annotations

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from tests import render_oracle as ro

ROUNDS = 3
LAMBDA = 0.5
MARGIN = 2
CELL = 4
MIN_PAGE = 4096
MAX_PAGE = 16384
GREY = 160


def box_centre(xyz):
    """Centre of the per-axis 1st-99th percentile box (float64 [3])."""
    x = np.asarray(xyz, np.float32)
    n = len(x)
    if n == 0:
        return np.zeros(3)
    k = int(0.01 * (n - 1))
    s = np.sort(x, axis=0)
    return (s[k].astype(np.float64) + s[n - 1 - k].astype(np.float64)) / 2.0


def views(Ks, Es, sizes, centre):
    """[(P float64 [3,4], C float64 [3], near, W, H)] as ops.texture_view_table builds them."""
    out = []
    for K, E, (H, W) in zip(Ks, Es, sizes):
        P = np.asarray(K, np.float64) @ np.asarray(E, np.float64)[:3, :4]
        C = -np.linalg.solve(P[:, :3], P[:, 3])
        out.append((P, C, 1e-3 * max(float(np.linalg.norm(C - centre)), 1e-30), W, H))
    return out


def project64(P, X):
    """(u, v, z) float64 of points X float64 [...,3]."""
    x, y, z = X[..., 0], X[..., 1], X[..., 2]
    row = lambda r: ((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3]
    with np.errstate(all="ignore"):
        zz = row(2)
        return row(0) / zz, row(1) / zz, zz


def front_facing(X0, X1, X2, C):
    a, b = X1 - X0, X2 - X0
    d = C[None, :] - ((X0 + X1) + X2) / 3.0
    n0 = a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1]
    n1 = a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2]
    n2 = a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]
    return ((n0 * d[:, 0] + n1 * d[:, 1]) + n2 * d[:, 2]) > 0


def visibility(xyz, faces, view):
    """(visible int64 [nf], covered int64 [nf]) of one view."""
    P, C, near, W, H = view
    P32 = P.astype(np.float32)
    xyz = np.asarray(xyz, np.float32)
    nf = len(faces)
    proj = ro.project_vertices(P32, xyz, W, H, np.float32(near))
    t = ro.setup(proj, faces, W, H)
    zbuf = np.full(H * W, ro.EMPTY)
    covered = np.zeros(nf, np.int64)
    bw, bh = t["x1"] - t["x0"] + 1, t["y1"] - t["y0"] + 1
    small = np.flatnonzero(t["ok"] & (bw <= ro.SMALL_BOX) & (bh <= ro.SMALL_BOX))
    large = np.flatnonzero(t["ok"] & ((bw > ro.SMALL_BOX) | (bh > ro.SMALL_BOX)))

    def emit(sel, px, py):
        inside, _, z = ro.cover(t, sel, px, py)
        ro.zmin(zbuf, py[inside] * W + px[inside], ro.keys(z[inside], sel[inside]))
        np.add.at(covered, sel[inside], 1)

    for oy in range(ro.SMALL_BOX):
        for ox in range(ro.SMALL_BOX):
            sel = small[(ox < bw[small]) & (oy < bh[small])]
            emit(sel, t["x0"][sel] + ox, t["y0"][sel] + oy)
    for f in large:
        py, px = np.mgrid[t["y0"][f]:t["y1"][f] + 1, t["x0"][f]:t["x1"][f] + 1]
        emit(np.full(px.size, f), px.ravel(), py.ravel())
    hit = zbuf[zbuf != ro.EMPTY]
    visible = np.bincount((hit & np.uint64(0xFFFFFFFF)).astype(np.int64), minlength=nf)[:nf]
    return visible, covered


def candidates(xyz, faces, view, visible, covered):
    """bool [nf]: the candidate test of every face in one view."""
    P, C, near, W, H = view
    ok = (visible >= 1) & (10 * visible >= 9 * covered)
    X = np.asarray(xyz, np.float32).astype(np.float64)[faces]  # [nf,3,3]
    u, v, z = project64(P, X)
    inside = (z > near) & (z < np.inf) & (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1)
    return ok & inside.all(1) & front_facing(X[:, 0], X[:, 1], X[:, 2], C)


def neighbour_pairs(faces):
    """(f, g) int64 arrays: one pair per shared undirected edge (a != b) and ordered pair of distinct faces on it."""
    f = np.asarray(faces, np.int64)
    nf = len(f)
    a = f.ravel()
    b = f[:, [1, 2, 0]].ravel()
    face = np.repeat(np.arange(nf), 3)
    keep = a != b
    key = np.minimum(a, b)[keep] * (1 << 32) + np.maximum(a, b)[keep]
    face = face[keep]
    order = np.argsort(key, kind="stable")
    key, face = key[order], face[order]
    fs, gs = [], []
    d = 1
    while d < len(key):
        same = key[d:] == key[:-d]
        if not same.any():
            break
        i = np.flatnonzero(same)
        fs += [face[i], face[i + d]]
        gs += [face[i + d], face[i]]
        d += 1
    if not fs:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    F, G = np.concatenate(fs), np.concatenate(gs)
    k = F != G
    return F[k], G[k]


def select(xyz, faces, vws):
    """-> (label int64 [nf], entries (face, view, D) sorted by face then view)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nf = len(faces)
    ef, ev, ed = [], [], []
    for vi, view in enumerate(vws):
        vis, cov = visibility(xyz, faces, view)
        c = np.flatnonzero(candidates(xyz, faces, view, vis, cov))
        ef.append(c); ev.append(np.full(c.size, vi)); ed.append(vis[c])
    ef, ev, ed = np.concatenate(ef), np.concatenate(ev), np.concatenate(ed)
    order = np.lexsort((ev, ef))
    ef, ev, ed = ef[order], ev[order], ed[order]
    label = np.full(nf, -1, np.int64)
    if ef.size == 0:
        return label, (ef, ev, ed)
    starts = np.r_[0, np.flatnonzero(ef[1:] != ef[:-1]) + 1]
    rows = ef[starts]
    maxd = np.maximum.reduceat(ed, starts)
    per_entry_max = np.repeat(maxd, np.diff(np.r_[starts, ef.size]))

    def first_best(score):
        best = np.repeat(np.maximum.reduceat(score, starts), np.diff(np.r_[starts, ef.size]))
        hit = score == best
        idx = np.flatnonzero(hit)
        first = np.r_[True, ef[idx][1:] != ef[idx][:-1]]
        out = label.copy()
        out[ef[idx[first]]] = ev[idx[first]]
        return out

    label = first_best(ed.astype(np.float64))
    F, G = neighbour_pairs(faces)
    V = len(vws)
    for _ in range(ROUNDS):
        lg = label[G]
        k = lg >= 0
        code, cnt = np.unique(F[k] * V + lg[k], return_counts=True)
        q = ef * V + ev
        pos = np.searchsorted(code, q)
        pos = np.minimum(pos, max(code.size - 1, 0))
        same = np.where((code.size > 0) & (code[pos] == q), cnt[pos] if code.size else 0, 0)
        score = ed.astype(np.float64) / per_entry_max.astype(np.float64) + LAMBDA * same.astype(np.float64)
        label = first_best(score)
    del rows
    return label, (ef, ev, ed)


def charts(faces, label, xyz, vws):
    """-> (chart int64 [nf], -1 untextured; table int64 [n,6]: id, view, x0, y0, width, height by ascending id)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nf = len(faces)
    F, G = neighbour_pairs(faces)
    k = (label[F] >= 0) & (label[F] == label[G])
    graph = coo_matrix((np.ones(int(k.sum())), (F[k], G[k])), shape=(nf, nf))
    _, comp = connected_components(graph, directed=False)
    root = np.full(comp.max() + 1 if nf else 0, nf, np.int64)
    np.minimum.at(root, comp, np.arange(nf))
    chart = np.where(label >= 0, root[comp] if nf else 0, -1)
    ids = np.flatnonzero((chart == np.arange(nf)) & (label >= 0))
    X = np.asarray(xyz, np.float32).astype(np.float64)[faces]
    lo = np.full((nf, 2), np.iinfo(np.int64).max)
    hi = np.full((nf, 2), np.iinfo(np.int64).min)
    for vi, (P, _, _, _, _) in enumerate(vws):
        sel = np.flatnonzero(label == vi)
        if sel.size == 0:
            continue
        u, v, _ = project64(P, X[sel])
        for a, q in enumerate((u, v)):
            np.minimum.at(lo[:, a], chart[sel], np.floor(q).min(1).astype(np.int64))
            np.maximum.at(hi[:, a], chart[sel], np.ceil(q).max(1).astype(np.int64))
    x0, y0 = lo[ids, 0] - MARGIN, lo[ids, 1] - MARGIN
    table = np.stack([ids, label[ids], x0, y0, hi[ids, 0] + MARGIN - x0 + 1, hi[ids, 1] + MARGIN - y0 + 1], 1) if ids.size else np.zeros((0, 6), np.int64)
    return chart, table


def pack(sizes, n_cells):
    """Shelf packing -> (places int64 [n + n_cells,3] (page, x, y), S, pages)."""
    sizes = np.asarray(sizes, np.int64).reshape(-1, 2)
    n = len(sizes)
    largest = max([CELL] + sizes.ravel().tolist())
    if largest > MAX_PAGE:
        raise ValueError("a rectangle side > 16384")
    S = MIN_PAGE
    while S < largest:
        S *= 2
    order = sorted(range(n), key=lambda i: (-sizes[i, 1], -sizes[i, 0], i))
    places = np.zeros((n + n_cells, 3), np.int64)
    page = x = y = shelf = 0
    todo = [(i, int(sizes[i, 0]), int(sizes[i, 1])) for i in order] + [(n + j, CELL, CELL) for j in range(n_cells)]
    for i, w, h in todo:
        if x + w > S:
            y += shelf; x = 0; shelf = 0
        if y + h > S:
            page += 1; x = y = shelf = 0
        places[i] = (page, x, y)
        x += w
        shelf = max(shelf, h)
    return places, S, (page + 1 if todo else 0)


def texture(xyz, rgb, faces, images, Ks, Es):
    """The whole texturer -> dict(label, chart, table, places, S, uv float32 [nf,3,2], page int32 [nf], pages uint8
    [P,S,S,3]).  images float32 [3,H,W] numpy arrays."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    nf = len(faces)
    xyz = np.asarray(xyz, np.float32)
    vws = views(Ks, Es, [im.shape[1:] for im in images], box_centre(xyz))
    label, entries = select(xyz, faces, vws)
    chart, table = charts(faces, label, xyz, vws)
    untex = np.flatnonzero(label < 0)
    places, S, P = pack(table[:, 4:6], untex.size)
    pages = np.zeros((P, S, S, 3), np.uint8)
    for r, (cid, v, x0, y0, w, h) in enumerate(table):
        img = images[v]
        H, W = img.shape[1:]
        ys = np.clip(np.arange(y0, y0 + h), 0, H - 1)
        xs = np.clip(np.arange(x0, x0 + w), 0, W - 1)
        block = img[:, ys][:, :, xs].transpose(1, 2, 0)
        pg, ox, oy = places[r]
        pages[pg, oy:oy + h, ox:ox + w] = np.clip(np.rint(np.float32(255.0) * block), 0, 255).astype(np.uint8)
    row_of = np.full(nf, -1, np.int64)
    row_of[table[:, 0]] = np.arange(len(table))
    slot = np.where(label >= 0, row_of[np.maximum(chart, 0)], 0)
    slot[untex] = len(table) + np.arange(untex.size)
    uv = np.zeros((nf, 3, 2), np.float32)
    page = places[slot, 0].astype(np.int32) if nf else np.zeros(0, np.int32)
    X = xyz.astype(np.float64)[faces]
    for vi, (Pm, _, _, _, _) in enumerate(vws):
        sel = np.flatnonzero(label == vi)
        if sel.size == 0:
            continue
        u, v, _ = project64(Pm, X[sel])
        rows = table[slot[sel]]
        pl = places[slot[sel]]
        a = (u - rows[:, 2:3].astype(np.float64)) + pl[:, 1:2].astype(np.float64)
        b = (v - rows[:, 3:4].astype(np.float64)) + pl[:, 2:3].astype(np.float64)
        uv[sel, :, 0] = ((a + 0.5) / S).astype(np.float32)
        uv[sel, :, 1] = (1.0 - (b + 0.5) / S).astype(np.float32)
    if untex.size:
        pl = places[slot[untex]]
        uv[untex, :, 0] = ((pl[:, 1:2] + CELL // 2).astype(np.float64) / S).astype(np.float32)
        uv[untex, :, 1] = (1.0 - (pl[:, 2:3] + CELL // 2).astype(np.float64) / S).astype(np.float32)
        if rgb is None:
            col = np.full((untex.size, 3), GREY, np.uint8)
        else:
            c = np.asarray(rgb, np.uint8).astype(np.float64)[faces[untex]]
            col = np.rint(((c[:, 0] + c[:, 1]) + c[:, 2]) / 3.0).astype(np.uint8)
        for j in range(untex.size):
            pg, ox, oy = pl[j]
            pages[pg, oy:oy + CELL, ox:ox + CELL] = col[j]
    return {"label": label, "chart": chart, "table": table, "places": places, "S": S, "uv": uv, "page": page, "pages": pages,
            "entries": entries, "views": vws}
