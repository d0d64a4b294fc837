"""numpy restatement of the mesh refinement definition in include/patchmatch_b200.h (pmb200_refine_mesh), so the per-vertex
sums and the refined positions equal the GPU's bit for bit (test infrastructure).

float64 arithmetic below is one numpy operation per rounding, in the order of patchmatchnet_b200/csrc/pm_refine_mesh_math.cuh;
grey levels are float32; the z-buffer is tests/render_oracle.py's and the near plane oracle/texture_oracle.py's.
`frozen` runs (finite differences) keep one iteration's coverage, validity and counted windows and skip the fixed-point
rounding."""
from __future__ import annotations

import numpy as np

from oracle import texture_oracle as to
from tests import render_oracle as ro

F = np.float32
RADIUS = 2
MIN_COUNT = 13
MIN_VARIANCE = 1e-4
DEPTH_TOLERANCE = 0.01
GRAD_UNIT = 2.0 ** 20
WEIGHT_UNIT = 2.0 ** 32
ENERGY_UNIT = 2.0 ** 24
MIN_COSINE = 0.3


# ---- views and levels -----------------------------------------------------------------------------------------------------

def level_K(K, levels):
    """[K_0 .. K_{levels-1}] float64: fx/2, skew/2, fy/2, c' = (c + 0.5)/2 - 0.5 per level."""
    out = [np.asarray(K, np.float64).copy()]
    for _ in range(levels - 1):
        k = out[-1].copy()
        k[0, 0] = k[0, 0] / 2.0
        k[0, 1] = k[0, 1] / 2.0
        k[1, 1] = k[1, 1] / 2.0
        k[0, 2] = (k[0, 2] + 0.5) / 2.0 - 0.5
        k[1, 2] = (k[1, 2] + 0.5) / 2.0 - 0.5
        out.append(k)
    return out


def grey_levels(image, levels):
    """image float32 [3,H,W] -> [float32 [H_l, W_l]]."""
    im = np.asarray(image, F)
    g = (F(0.299) * im[0] + F(0.587) * im[1]) + F(0.114) * im[2]
    out = [g]
    for _ in range(levels - 1):
        p = out[-1]
        h, w = p.shape[0] // 2, p.shape[1] // 2
        q = p[:2 * h, :2 * w]
        out.append(((q[0::2, 0::2] + q[0::2, 1::2]) + (q[1::2, 0::2] + q[1::2, 1::2])) * F(0.25))
    return out


def box_diagonal(xyz):
    """L: the diagonal of the per-axis 1st-99th percentile box, sqrt((dx dx + dy dy) + dz dz) in float64 (1 when 0)."""
    x = np.asarray(xyz, F)
    n = len(x)
    if n == 0:
        return 1.0
    k = int(0.01 * (n - 1))
    s = np.sort(x, axis=0)
    d = s[n - 1 - k].astype(np.float64) - s[k].astype(np.float64)
    L = float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
    return L if L > 0 else 1.0


def views(Ks, Es, images, levels, box_centre):
    """[level][view] dicts: P, K, Rt, C (float64), near, W, H, grey (float32 [H,W])."""
    out = [[] for _ in range(levels)]
    for K, E, img in zip(Ks, Es, images):
        Rt = np.asarray(E, np.float64)[:3, :4]
        (P0, _, near, _, _), = to.views([K], [E], [np.asarray(img).shape[1:]], box_centre)
        g = grey_levels(img, levels)
        C = -((Rt[0, :3] * Rt[0, 3] + Rt[1, :3] * Rt[1, 3]) + Rt[2, :3] * Rt[2, 3])
        for l, Kl in enumerate(level_K(K, levels)):
            out[l].append({"P": Kl @ Rt, "K": Kl, "Rt": Rt, "C": C, "near": near, "W": g[l].shape[1], "H": g[l].shape[0], "grey": g[l]})
    return out


def zbuffer(xyz, faces, v):
    P32 = v["P"].astype(F)
    return ro.mesh_zbuffer(ro.project_vertices(P32, np.asarray(xyz, F), v["W"], v["H"], F(v["near"])), faces, v["W"], v["H"])[0].ravel()


# ---- per pixel ------------------------------------------------------------------------------------------------------------

def dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def rays(v, x, y):
    K, R = v["K"], v["Rt"]
    yy = (y - K[1, 2]) / K[1, 1]
    xx = ((x - K[0, 2]) - K[0, 1] * yy) / K[0, 0]
    return np.stack([(R[0, c] * xx + R[1, c] * yy) + R[2, c] for c in range(3)], -1)


def hits(xyz, faces, f, C, r):
    """(ok, n, nr, t, X, beta [m,3]) of rays r [m,3] from C on faces f."""
    X0, X1, X2 = (xyz[faces[f, k]].astype(np.float64) for k in range(3))
    n = cross(X1 - X0, X2 - X0)
    nr = dot(n, r)
    with np.errstate(all="ignore"):
        t = dot(n, X0 - C) / nr
        ok = (nr < 0) & (t > 0) & (t < np.inf)
        X = C + t[:, None] * r
        nn = dot(n, n)
        xs = (X0, X1, X2)
        beta = np.stack([dot(n, cross(xs[(k + 1) % 3] - X, xs[(k + 2) % 3] - X)) / nn for k in range(3)], -1)
    return ok, n, nr, t, X, beta


def oblique_ok(n, nr, r, X, Cj):
    """-(n . r) > c sqrt((n . n) (r . r)) and n . d > c sqrt((n . n) (d . d)), d = Cj - X, c = MIN_COSINE."""
    dj = Cj - X
    nn = dot(n, n)
    with np.errstate(all="ignore"):
        return (-nr > MIN_COSINE * np.sqrt(nn * dot(r, r))) & (dot(n, dj) > MIN_COSINE * np.sqrt(nn * dot(dj, dj)))


def bilinear(img, u, v):
    H, W = img.shape
    x0, y0 = np.floor(u).astype(np.int64), np.floor(v).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    fx, fy = u - x0, v - y0
    g = img.astype(np.float64)
    p, q, s, t = g[y0, x0], g[y0, x1], g[y1, x0], g[y1, x1]
    dq, dt = q - p, t - s
    top, bot = p + fx * dq, s + fx * dt
    return top + fy * (bot - top), dq + fy * (dt - dq), bot - top


def db_dt(P, u, v, z, r, du, dv):
    pr = [(P[k, 0] * r[:, 0] + P[k, 1] * r[:, 1]) + P[k, 2] * r[:, 2] for k in range(3)]
    return du * ((pr[0] - u * pr[2]) / z) + dv * ((pr[1] - v * pr[2]) / z)


def pair_pixels(xyz, faces, vi, vj, zi, zj, frozen=None):
    """The pixels of view i in pair (i, j): dict(valid bool [H,W], a, b, dbdt [H,W] float64, face, t, nr, n, beta at the
    valid pixels, idx their flat indices).  `frozen` (a previous result) keeps its valid pixels and faces."""
    W, H = vi["W"], vi["H"]
    if frozen is None:
        idx = np.flatnonzero(zi != ro.EMPTY)
        f = (zi[idx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    else:
        idx, f = frozen["idx"], frozen["face"]
    x, y = (idx % W).astype(np.float64), (idx // W).astype(np.float64)
    r = rays(vi, x, y)
    ok, n, nr, t, X, beta = hits(xyz, faces, f, vi["C"], r)
    if frozen is None:
        ok &= dot(n, vj["C"] - xyz[faces[f, 0]].astype(np.float64)) > 0
        ok &= oblique_ok(n, nr, r, X, vj["C"])
    P = vj["P"]
    with np.errstate(all="ignore"):
        zz = (P[2, 0] * X[:, 0] + P[2, 1] * X[:, 1]) + P[2, 2] * X[:, 2] + P[2, 3]
        u = ((P[0, 0] * X[:, 0] + P[0, 1] * X[:, 1]) + P[0, 2] * X[:, 2] + P[0, 3]) / zz
        v = ((P[1, 0] * X[:, 0] + P[1, 1] * X[:, 1]) + P[1, 2] * X[:, 2] + P[1, 3]) / zz
    if frozen is None:
        ok &= (zz > vj["near"]) & (zz < np.inf) & (u >= 0) & (u <= vj["W"] - 1) & (v >= 0) & (v <= vj["H"] - 1)
        pix = np.where(ok, np.rint(np.where(ok, v, 0)).astype(np.int64) * vj["W"] + np.rint(np.where(ok, u, 0)).astype(np.int64), 0)
        key = zj[pix]
        zb = (key >> np.uint64(32)).astype(np.uint32).view(F).astype(np.float64)
        ok &= (key != ro.EMPTY) & (zz <= (1.0 + DEPTH_TOLERANCE) * zb)
    else:
        u, v = np.clip(u, 0, vj["W"] - 1), np.clip(v, 0, vj["H"] - 1)
    sel = np.flatnonzero(ok)
    b, du, dv = bilinear(vj["grey"], u[sel], v[sel])
    out = {"valid": np.zeros(H * W, bool), "a": np.zeros(H * W), "b": np.zeros(H * W), "dbdt": np.zeros(H * W)}
    q = idx[sel]
    out["valid"][q] = True
    out["a"][q] = vi["grey"].ravel()[q].astype(np.float64)
    out["b"][q] = b
    out["dbdt"][q] = db_dt(P, u[sel], v[sel], zz[sel], r[sel], du, dv)
    out.update(idx=q, face=f[sel], t=t[sel], nr=nr[sel], n=n[sel], beta=beta[sel])
    for k in ("valid", "a", "b", "dbdt"):
        out[k] = out[k].reshape(H, W)
    return out


def _shifted(a, dy, dx, fill):
    """a[y + dy, x + dx] with `fill` outside."""
    H, W = a.shape
    out = np.full_like(a, fill)
    ys, xs = slice(max(0, -dy), min(H, H - dy)), slice(max(0, -dx), min(W, W - dx))
    out[ys, xs] = a[max(0, dy):min(H, H + dy), max(0, dx):min(W, W + dx)]
    return out


OFFSETS = [(dy, dx) for dy in range(-RADIUS, RADIUS + 1) for dx in range(-RADIUS, RADIUS + 1)]


def windows(px, counted=None):
    """-> (counted bool [H,W], energy [H,W], coefficients [3,H,W]).  `counted` (frozen) keeps the counted windows."""
    valid, a, b = px["valid"], px["a"], px["b"]
    n = np.zeros(valid.shape, np.int64)
    S = [np.zeros(valid.shape) for _ in range(5)]
    for dy, dx in OFFSETS:
        m = _shifted(valid, dy, dx, False)
        av, bv = np.where(m, _shifted(a, dy, dx, 0.0), 0.0), np.where(m, _shifted(b, dy, dx, 0.0), 0.0)
        n += m
        for k, term in enumerate((av, bv, av * av, bv * bv, av * bv)):
            S[k] = np.where(m, S[k] + term, S[k])
    dn = np.maximum(n, 1).astype(np.float64)
    with np.errstate(all="ignore"):
        ma, mb = S[0] / dn, S[1] / dn
        va, vb = S[2] / dn - ma * ma, S[3] / dn - mb * mb
        cov = S[4] / dn - ma * mb
        sigma = np.sqrt(va * vb)
        Z = cov / sigma
        ns, nv = dn * sigma, dn * vb
        c = np.stack([ma / ns - (Z * mb) / nv, -(1.0 / ns), Z / nv])
    use = valid & (n >= MIN_COUNT) & (va > MIN_VARIANCE) & (vb > MIN_VARIANCE) if counted is None else counted
    E = np.where(use, 1.0 - Z, 0.0)
    return use, E, np.where(use[None], c, 0.0)


def pixel_gradient(px, use, c):
    """dE/dt at the valid pixels (px['idx'] order) and whether a counted window contains each."""
    H, W = use.shape
    s = np.zeros((3, H, W))
    anyw = np.zeros((H, W), bool)
    for dy, dx in OFFSETS:
        m = _shifted(use, dy, dx, False)
        anyw |= m
        for k in range(3):
            s[k] = np.where(m, s[k] + _shifted(c[k], dy, dx, 0.0), s[k])
    q = px["idx"]
    sk = [s[k].ravel()[q] for k in range(3)]
    a, b = px["a"].ravel()[q], px["b"].ravel()[q]
    g = ((sk[1] * a + sk[2] * b) + sk[0]) * px["dbdt"].ravel()[q]
    return g, anyw.ravel()[q]


def scatter(px, g, has, faces, fx, L, nv, fixed=True):
    """Per-vertex sums [nv,5] (G xyz, W, S): int64 fixed point, or float64 unrounded with fixed=False."""
    acc = np.zeros((nv, 5), np.int64 if fixed else np.float64)
    sel = np.flatnonzero(has)
    g, f, beta, nr, n, t = g[sel], px["face"][sel], px["beta"][sel], px["nr"][sel], px["n"][sel], px["t"][sel]
    rnd = (lambda v: np.rint(v).astype(np.int64)) if fixed else (lambda v: v)
    for k in range(3):
        vert = faces[f, k]
        s = (g * beta[:, k]) / nr
        for c in range(3):
            np.add.at(acc[:, c], vert, rnd(((s * n[:, c]) * L) * GRAD_UNIT) if fixed else s * n[:, c])
        np.add.at(acc[:, 3], vert, rnd(beta[:, k] * WEIGHT_UNIT) if fixed else beta[:, k])
        np.add.at(acc[:, 4], vert, rnd((((beta[:, k] * t) / fx) / L) * WEIGHT_UNIT) if fixed else (beta[:, k] * t) / fx)
    return acc


# ---- update ---------------------------------------------------------------------------------------------------------------

def adjacency(faces, nv):
    """(rows: vertex, face of the sorted (vertex, face) slots; neighbour entries (vertex, w) in the kernels' order)."""
    nf = len(faces)
    key = faces.ravel().astype(np.int64) * (1 << 32) + np.repeat(np.arange(nf), 3)
    key = np.sort(key)
    rv, rf = key >> 32, key & 0xFFFFFFFF
    ev = np.repeat(rv, 3)
    ew = faces[rf].ravel().astype(np.int64)
    keep = ew != ev
    code = ev * (1 << 32) + ew
    _, first = np.unique(code, return_index=True)
    isfirst = np.zeros(code.size, bool)
    isfirst[first] = True
    keep &= isfirst
    return (rv, rf), (ev[keep], ew[keep])


def update(xyz, faces, acc, alpha, lam, L):
    """The new float32 positions from the sums acc [nv,5] (int64)."""
    nv = len(xyz)
    x = np.asarray(xyz, F)
    (rv, rf), (ev, ew) = adjacency(faces, nv)
    X = x.astype(np.float64)
    fn = cross(X[faces[:, 1]] - X[faces[:, 0]], X[faces[:, 2]] - X[faces[:, 0]])
    nsum = np.zeros((nv, 3))
    for c in range(3):
        np.add.at(nsum[:, c], rv, fn[rf, c])
    ln = np.sqrt(dot(nsum, nsum))
    with np.errstate(all="ignore"):
        normal = np.where(ln[:, None] > 0, nsum / ln[:, None], 0.0)
    cnt = np.bincount(ev, minlength=nv)
    U = np.zeros((nv, 3))
    for c in range(3):
        np.add.at(U[:, c], ev, X[ew, c] - X[ev, c])
    U = np.where(cnt[:, None] > 0, U / np.maximum(cnt, 1)[:, None], 0.0)
    U2 = np.zeros((nv, 3))
    for c in range(3):
        np.add.at(U2[:, c], ev, U[ew, c] - U[ev, c])
    U2 = np.where(cnt[:, None] > 0, U2 / np.maximum(cnt, 1)[:, None], 0.0)
    return step_positions(x, acc, normal, U2, alpha, lam, L)


def step_positions(x, acc, normal, U2, alpha, lam, L):
    """float32((x + d n) - lambda U2) with the photometric step d of the sums acc [nv,5]."""
    X = np.asarray(x, F).astype(np.float64)
    Wf, Sf = acc[:, 3], acc[:, 4]
    with np.errstate(all="ignore"):
        w = Wf.astype(np.float64) / WEIGHT_UNIT
        s = ((Sf.astype(np.float64) / WEIGHT_UNIT) * L) / w
        G = (acc[:, :3].astype(np.float64) / GRAD_UNIT) / L
        g = dot(normal, G) / w
        d = ((alpha * s) * s) * g
        lim = 0.5 * s
        d = -np.where(d > lim, lim, np.where(d < -lim, -lim, d))
    d = np.where(Wf > 0, d, 0.0)
    return ((X + d[:, None] * normal) - lam * U2).astype(F)


# ---- the whole refinement -------------------------------------------------------------------------------------------------

def iteration(xyz, faces, vl, pairs, L, alpha, lam):
    """One iteration at one level -> (new xyz float32, acc int64 [nv,5], energy, counted windows)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    xyz = np.asarray(xyz, F)
    zb = [zbuffer(xyz, faces, v) for v in vl]
    acc = np.zeros((len(xyz), 5), np.int64)
    energy, count = 0, 0
    for i, j in pairs:
        px = pair_pixels(xyz, faces, vl[i], vl[j], zb[i], zb[j])
        use, E, c = windows(px)
        energy += int(np.rint(E[use] * ENERGY_UNIT).astype(np.int64).sum())
        count += int(use.sum())
        g, has = pixel_gradient(px, use, c)
        acc += scatter(px, g, has, faces, vl[i]["K"][0, 0], L, len(xyz))
    return update(xyz, faces, acc, alpha, lam, L), acc, energy / ENERGY_UNIT, count


def refine(xyz, faces, images, Ks, Es, pairs, iterations, levels, alpha, smoothness):
    """The whole refinement -> (xyz float32, [(energy, windows)] per iteration coarse to fine, acc of the last iteration)."""
    xyz = np.asarray(xyz, F)
    L = box_diagonal(xyz)
    vw = views(Ks, Es, images, levels, to.box_centre(xyz))
    stats, acc = [], None
    for l in range(levels - 1, -1, -1):
        for _ in range(iterations):
            xyz, acc, e, n = iteration(xyz, faces, vw[l], pairs, L, alpha, smoothness)
            stats.append((e, n))
    return xyz, stats, acc


# ---- frozen energy and gradient (finite differences) ----------------------------------------------------------------------

def freeze(xyz, faces, vl, pairs):
    """One iteration's coverage, validity and counted windows per pair."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    zb = [zbuffer(xyz, faces, v) for v in vl]
    out = []
    for i, j in pairs:
        px = pair_pixels(xyz, faces, vl[i], vl[j], zb[i], zb[j])
        use, _, _ = windows(px)
        out.append((px, use))
    return out


def frozen_energy_and_gradient(xyz, faces, vl, pairs, frozen):
    """(E, dE/dx float64 [nv,3]) with the frozen pixels and windows, in float64 without fixed-point rounding."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    xyz = np.asarray(xyz, np.float64)
    E, G = 0.0, np.zeros((len(xyz), 3))
    for (i, j), (fp, use) in zip(pairs, frozen):
        px = pair_pixels(xyz, faces, vl[i], vl[j], None, None, frozen=fp)
        _, e, c = windows(px, counted=use)
        E += float(e[use].sum())
        g, has = pixel_gradient(px, use, c)
        G += scatter(px, g, has, faces, vl[i]["K"][0, 0], 1.0, len(xyz), fixed=False)[:, :3]
    return E, G
