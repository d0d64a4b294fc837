"""Float64 numpy oracle of the mesh simplifier (include/patchmatch_b200.h "Mesh simplification"; pm_simplify.cu).

Test infrastructure: never imported by the product.  Each round is one vectorised function (`round_step`), restating the
kernels' rounds of independent collapses; `simplify` drives them.  Arithmetic is elementwise numpy float64 in the order
pm_simplify_math.cuh writes it (no `@`, dot, sum or einsum on a compared value), so the GPU agrees bit for bit.  The
constants are read from pm_simplify_math.cuh."""
from __future__ import annotations

import os
import re

import numpy as np

_HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "patchmatchnet_b200", "csrc",
                       "pm_simplify_math.cuh")


def _constants(path: str = _HEADER):
    text = open(path).read()
    out = {}
    for name in ("kBoundaryWeight", "kDetRel", "kFarEdges", "kFlatRel", "kMaxValence"):
        m = re.search(r"constexpr\s+(?:double|int)\s+%s\s*=\s*([0-9.eE+-]+)\s*;" % name, text)
        out[name] = float(m.group(1)) if "." in m.group(1) or "e" in m.group(1).lower() else int(m.group(1))
    return out


_C = _constants()
BOUNDARY_WEIGHT = float(_C["kBoundaryWeight"])
DET_REL = float(_C["kDetRel"])
FAR_EDGES = float(_C["kFarEdges"])
FLAT_REL = float(_C["kFlatRel"])
MAX_VALENCE = int(_C["kMaxValence"])
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)

# (i, j) of the 10 unique quadric entries: xx xy xz xd yy yz yd zz zd dd
_IJ = [(i, j) for i in range(4) for j in range(i, 4)]


# ---- per-edge arithmetic (pm_simplify_math.cuh) ---------------------------------------------------------------------------

def dot3(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross3(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def face_normal(x0, x1, x2):
    return cross3(x1 - x0, x2 - x0)


def plane_terms(m, x, w):
    """w (p p^T) for p = (m / |m|, -(m / |m|) . x) -> ([n,10] terms, mask where |m| > 0; elsewhere nothing is added)."""
    with np.errstate(all="ignore"):
        ln = np.sqrt(dot3(m, m))
        ok = ln > 0
        u = m / ln[..., None]
        p = np.concatenate([u, -dot3(u, x)[..., None]], -1)
        terms = np.stack([w * (p[..., i] * p[..., j]) for i, j in _IJ], -1)
    return terms, ok


def face_terms(x0, x1, x2):
    n = face_normal(x0, x1, x2)
    return plane_terms(n, x0, np.sqrt(dot3(n, n)) * 0.5)


def border_terms(xa, xb, x0, x1, x2):
    n = face_normal(x0, x1, x2)
    e = xb - xa
    return plane_terms(cross3(e, n), xa, BOUNDARY_WEIGHT * dot3(e, e))


def _qrow(a, b, c, d, v):
    return ((a * v[..., 0] + b * v[..., 1]) + c * v[..., 2]) + d


def quadric_cost(q, v):
    r0, r1 = _qrow(q[..., 0], q[..., 1], q[..., 2], q[..., 3], v), _qrow(q[..., 1], q[..., 4], q[..., 5], q[..., 6], v)
    r2, r3 = _qrow(q[..., 2], q[..., 5], q[..., 7], q[..., 8], v), _qrow(q[..., 3], q[..., 6], q[..., 8], q[..., 9], v)
    c = ((v[..., 0] * r0 + v[..., 1] * r1) + v[..., 2] * r2) + r3
    return np.where(c > 0, c, 0.0)


def _clamp01(t):
    return np.where(t > 0, np.where(t < 1, t, 1.0), 0.0)


def segment_param(xa, e, v):
    ee = dot3(e, e)
    with np.errstate(all="ignore"):
        t = dot3(v - xa, e) / ee
    return np.where(ee > 0, _clamp01(t), 0.0)


def placement(q, xa, xb):
    """-> (v [n,3], solved [n] bool): the minimiser of q when the 3x3 system passes the determinant test and lies within
    FAR_EDGES |e| of the segment, else the minimiser on the segment a + t e (t = 1/2 when flat)."""
    q = [q[..., k] for k in range(10)]
    e = xb - xa
    ee = dot3(e, e)
    c00, c01, c02 = q[4] * q[7] - q[5] * q[5], q[5] * q[2] - q[1] * q[7], q[1] * q[5] - q[4] * q[2]
    c11, c12, c22 = q[0] * q[7] - q[2] * q[2], q[2] * q[1] - q[0] * q[5], q[0] * q[4] - q[1] * q[1]
    det = (q[0] * c00 + q[1] * c01) + q[2] * c02
    s = np.maximum(np.maximum(np.abs(q[0]), np.abs(q[4])), np.abs(q[7]))
    g = np.stack([_qrow(q[0], q[1], q[2], q[3], xa), _qrow(q[1], q[4], q[5], q[6], xa), _qrow(q[2], q[5], q[7], q[8], xa)], -1)
    g0, g1, g2 = g[..., 0], g[..., 1], g[..., 2]
    with np.errstate(all="ignore"):
        w = xa - np.stack([((c00 * g0 + c01 * g1) + c02 * g2) / det, ((c01 * g0 + c11 * g1) + c12 * g2) / det,
                           ((c02 * g0 + c12 * g1) + c22 * g2) / det], -1)
        t = segment_param(xa, e, w)
        d = w - (xa + t[..., None] * e)
        solved = (np.abs(det) > DET_REL * ((s * s) * s)) & (ee > 0) & (dot3(d, d) <= (FAR_EDGES * FAR_EDGES) * ee)
        ae = np.stack([(q[0] * e[..., 0] + q[1] * e[..., 1]) + q[2] * e[..., 2], (q[1] * e[..., 0] + q[4] * e[..., 1]) + q[5] * e[..., 2],
                       (q[2] * e[..., 0] + q[5] * e[..., 1]) + q[7] * e[..., 2]], -1)
        eae, eg = dot3(e, ae), dot3(e, g)
        tr = (q[0] + q[4]) + q[7]
        ts = np.where(eae > (FLAT_REL * tr) * ee, _clamp01(-(eg / eae)), 0.5)
    vs = xa + ts[..., None] * e
    return np.where(solved[..., None], w, vs), solved


def placement_colour(xa, xb, v, ca, cb):
    t = segment_param(xa, xb - xa, v)[..., None]
    ca, cb = ca.astype(np.float64), cb.astype(np.float64)
    return np.rint(ca + t * (cb - ca)).astype(np.uint8)


def keeps_orientation(x0, x1, x2, slot, v):
    """A face with vertex `slot` moved to v: False when its old normal is non-zero and new . old <= 0."""
    n0 = face_normal(x0, x1, x2)
    y = [np.where((slot == k)[..., None], v, x) for k, x in enumerate((x0, x1, x2))]
    n1 = face_normal(*y)
    zero = (n0[..., 0] == 0) & (n0[..., 1] == 0) & (n0[..., 2] == 0)
    return zero | (dot3(n1, n0) > 0)


def edge_key(cost, edge):
    bits = cost.astype(np.float32).view(np.uint32).astype(np.uint64)
    return (bits << np.uint64(32)) | edge.astype(np.uint64)


# ---- topology and quadrics -------------------------------------------------------------------------------------------------

def clean_faces(faces, nv):
    """Faces with an index outside 0..nv-1 or a repeated index are dropped."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ok = ((f >= 0) & (f < nv)).all(1) & (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    return f[ok]


def component_labels(faces, nv):
    """Per face, the smallest vertex index of its component (faces joined through shared vertices)."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components

    if len(faces) == 0:
        return np.zeros(0, np.int64)
    r = np.concatenate([faces[:, 0], faces[:, 1]])
    c = np.concatenate([faces[:, 1], faces[:, 2]])
    _, comp = connected_components(coo_matrix((np.ones(len(r)), (r, c)), shape=(nv, nv)), directed=False)
    smallest = np.full(comp.max() + 1, nv, np.int64)
    np.minimum.at(smallest, comp, np.arange(nv))
    return smallest[comp[faces[:, 0]]]


def remove_small_components(faces, nv, min_faces):
    if min_faces <= 0 or len(faces) == 0:
        return faces
    lab = component_labels(faces, nv)
    count = np.bincount(lab, minlength=nv)
    return faces[count[lab] >= min_faces]


class Topology:
    """Edges (a < b) sorted by (a, b) with face counts, per-vertex face counts, border / lock flags, the vertex -> face
    incidences sorted by (vertex, face)."""

    def __init__(self, faces, nv):
        self.faces, self.nv = faces, nv
        nf = len(faces)
        fa, fb = faces, np.roll(faces, -1, axis=1)  # edge k of a face runs v_k -> v_{k+1}
        lo, hi = np.minimum(fa, fb), np.maximum(fa, fb)
        keys = (lo * nv + hi).ravel()
        self.keys, self.count = np.unique(keys, return_counts=True)
        self.a, self.b = self.keys // nv, self.keys % nv
        self.face_edge = np.searchsorted(self.keys, keys).reshape(nf, 3)  # edge id of face edge k
        self.deg = np.bincount(faces.ravel(), minlength=nv)
        self.border = np.zeros(nv, bool)
        self.locked = np.zeros(nv, bool)
        for m, flag in ((self.count == 1, self.border), (self.count > 2, self.locked)):
            flag[self.a[m]] = True
            flag[self.b[m]] = True
        inc_v = faces.ravel()
        inc_f = np.repeat(np.arange(nf), 3)
        order = np.lexsort((inc_f, inc_v))
        self.inc_v, self.inc_f = inc_v[order], inc_f[order]
        self.off = np.concatenate([[0], np.cumsum(self.deg)])

    def edge_id(self, x, y):
        """Ids of edges {x, y}, -1 where there is none."""
        k = np.minimum(x, y) * self.nv + np.maximum(x, y)
        if len(self.keys) == 0:
            return np.full(len(k), -1, np.int64)
        i = np.clip(np.searchsorted(self.keys, k), 0, len(self.keys) - 1)
        return np.where(self.keys[i] == k, i, -1)

    def star_pairs(self, centre):
        """(edge index, face) for every edge e and face of the star of centre[e], in incidence order."""
        n = self.deg[centre]
        e = np.repeat(np.arange(len(centre)), n)
        start = np.repeat(self.off[centre], n)
        rank = np.arange(len(e)) - np.repeat(np.cumsum(n) - n, n)
        return e, self.inc_f[start + rank]


def _ranked_add(q, vert, terms, ok):
    """q[vert[i]] += terms[i] (where ok[i]) in the order of the rows: rows of one vertex added one rank at a time."""
    if len(vert) == 0:
        return q
    order = np.argsort(vert, kind="stable")
    vert, terms, ok = vert[order], terms[order], ok[order]
    first = np.searchsorted(vert, vert)
    rank = np.arange(len(vert)) - first
    for r in range(rank.max() + 1):
        m = (rank == r) & ok
        q[vert[m]] = q[vert[m]] + terms[m]
    return q


def quadrics(pos, topo: Topology):
    """Per vertex: incident faces by ascending index, then border edges by ascending key."""
    f = topo.faces
    q = np.zeros((topo.nv, 10))
    ft = f[topo.inc_f]
    terms, ok = face_terms(pos[ft[:, 0]], pos[ft[:, 1]], pos[ft[:, 2]])
    q = _ranked_add(q, topo.inc_v, terms, ok)
    bf, bk = np.nonzero(topo.count[topo.face_edge] == 1)  # (face, slot) of each border edge; its only face
    eid = topo.face_edge[bf, bk]
    order = np.argsort(eid)
    bf, eid = bf[order], eid[order]
    a, b = topo.a[eid], topo.b[eid]
    t = f[bf]
    terms, ok = border_terms(pos[a], pos[b], pos[t[:, 0]], pos[t[:, 1]], pos[t[:, 2]])
    vert = np.concatenate([a, b])
    order = np.argsort(np.concatenate([eid, eid]), kind="stable")  # ascending key within each vertex
    return _ranked_add(q, vert[order], np.concatenate([terms, terms])[order], np.concatenate([ok, ok])[order])


# ---- one round -------------------------------------------------------------------------------------------------------------

def _member(sorted_keys, k):
    if len(sorted_keys) == 0:
        return np.zeros(len(k), bool)
    i = np.clip(np.searchsorted(sorted_keys, k), 0, len(sorted_keys) - 1)
    return sorted_keys[i] == k


def evaluate(pos, q, topo: Topology):
    """Per edge: the selection key, NONE where the collapse is not valid."""
    f, nv = topo.faces, topo.nv
    a, b, cnt = topo.a, topo.b, topo.count
    E = len(a)
    ok = ((cnt <= 2) & ~topo.locked[a] & ~topo.locked[b] & (topo.deg[a] <= MAX_VALENCE) & (topo.deg[b] <= MAX_VALENCE)
          & ~((cnt == 2) & topo.border[a] & topo.border[b]))
    # opposite vertices: (edge, third vertex) of every face edge; triangles: (edge, third vertex) keys
    third = np.stack([f[:, 2], f[:, 0], f[:, 1]], 1)
    opp_keys = np.unique((topo.face_edge * nv + third).ravel())
    # link condition over the faces of a's star without b
    e, t = topo.star_pairs(a)
    tv = f[t]
    keep = ~(tv == b[e][:, None]).any(1)
    e, tv = e[keep], tv[keep]
    slot = np.argmax(tv == a[e][:, None], 1)
    x, y = tv[np.arange(len(e)), (slot + 1) % 3], tv[np.arange(len(e)), (slot + 2) % 3]
    hx, hy = topo.edge_id(b[e], x) >= 0, topo.edge_id(b[e], y) >= 0
    ox, oy = _member(opp_keys, e * nv + x), _member(opp_keys, e * nv + y)
    hxy = _member(opp_keys, topo.edge_id(x, y) * nv + b[e])
    bad = hxy | (hx & ~ox) | (hy & ~oy)
    ok &= np.bincount(e[bad], minlength=E) == 0
    # placement and the flip test
    qs = q[a] + q[b]
    v, _ = placement(qs, pos[a], pos[b])
    for c, o in ((a, b), (b, a)):
        e, t = topo.star_pairs(c)
        tv = f[t]
        keep = ~(tv == o[e][:, None]).any(1)
        e, tv = e[keep], tv[keep]
        slot = np.argmax(tv == c[e][:, None], 1)
        good = keeps_orientation(pos[tv[:, 0]], pos[tv[:, 1]], pos[tv[:, 2]], slot, v[e])
        ok &= np.bincount(e[~good], minlength=E) == 0
    key = edge_key(quadric_cost(qs, v), np.arange(E))
    return np.where(ok, key, NONE)


def select(key, topo: Topology):
    """Edges whose key is the minimum over both endpoints' neighbourhoods."""
    a, b = topo.a, topo.b
    m = np.full(topo.nv, NONE, np.uint64)
    valid = key != NONE
    np.minimum.at(m, a[valid], key[valid])
    np.minimum.at(m, b[valid], key[valid])
    M = m.copy()
    np.minimum.at(M, a, m[b])
    np.minimum.at(M, b, m[a])
    return np.nonzero(valid & (key == M[a]) & (key == M[b]))[0]


def apply(pos, col, q, faces, edges_a, edges_b):
    """Collapse the independent edges (a, b) together: a takes v, its colour and Q_a + Q_b; b's references become a; faces
    with both disappear; the others keep their order."""
    pos, col, q = pos.copy(), col.copy(), q.copy()
    a, b = edges_a, edges_b
    qs = q[a] + q[b]
    v, _ = placement(qs, pos[a], pos[b])
    c = placement_colour(pos[a], pos[b], v, col[a], col[b])
    pos[a], col[a], q[a] = v, c, qs
    rep = np.arange(len(pos))
    rep[b] = a
    f = rep[faces]
    keep = (f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])
    return pos, col, q, f[keep]


def round_step(pos, col, q, faces, target, topo=None):
    """One round -> (pos, col, q, faces, kept edge ids in key order or selection order, topology), or None when no edge is
    valid."""
    topo = topo or Topology(faces, len(pos))
    key = evaluate(pos, q, topo)
    sel = select(key, topo)
    if len(sel) == 0:
        return None
    nf = len(faces)
    removed = int(topo.count[sel].astype(np.int64).sum())
    if nf - removed < target:
        sel = sel[np.argsort(key[sel])]
        incl = np.cumsum(topo.count[sel])
        sel = sel[(incl - topo.count[sel]) < nf - target]
    pos, col, q, faces = apply(pos, col, q, faces, topo.a[sel], topo.b[sel])
    return pos, col, q, faces, sel, topo


def prepare(xyz, rgb, faces, min_component_faces=0):
    nv = len(xyz)
    f = remove_small_components(clean_faces(faces, nv), nv, min_component_faces)
    pos = np.asarray(xyz, np.float32).astype(np.float64).reshape(-1, 3)
    col = np.zeros((nv, 3), np.uint8) if rgb is None else np.asarray(rgb, np.uint8).reshape(-1, 3).copy()
    topo = Topology(f, nv)
    return pos, col, quadrics(pos, topo), f, topo


def finish(pos, col, faces, nv):
    used = np.zeros(nv, bool)
    used[faces.ravel()] = True
    idx = np.cumsum(used) - 1
    return pos[used].astype(np.float32), col[used], idx[faces].astype(np.int32)


def simplify(xyz, rgb, faces, target_faces, min_component_faces=0, max_rounds=None):
    """-> (xyz float32 [n,3], rgb uint8 [n,3] or None, faces int32 [nf,3], rounds)."""
    nv = len(xyz)
    pos, col, q, f, topo = prepare(xyz, rgb, faces, min_component_faces)
    rounds = 0
    while len(f) > target_faces and (max_rounds is None or rounds < max_rounds):
        r = round_step(pos, col, q, f, target_faces, topo)
        if r is None:
            break
        pos, col, q, f, _, _ = r
        topo = None
        rounds += 1
    p, c, fo = finish(pos, col, f, nv)
    return p, (None if rgb is None else c), fo, rounds
