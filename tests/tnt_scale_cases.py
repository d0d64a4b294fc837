"""Tanks and Temples evaluation inputs at the sizes of real scenes, generated from seeds (no T&T data is needed or stored).

The real T&T ground-truth and fused-cloud point counts are not restated here; the rows are of their order: a fused cloud of
tens of millions of points, ground truth of millions.  Coordinates are float32-representable (PLY files store float32), except
where a row places a point on a float64 value on purpose (block_gap).

    object        Ignatius-like, tau = 0.003: a 3.2 m surface patch tens of metres from the origin.  The reconstruction has
                  more than 2^24 points (the patch, a floor outside the crop, 3% outliers above it), in a frame related to the
                  GT frame by the similarity S; more than 1.5 * 4 * 2^20 of them survive the crop, so refinement round 3
                  strides by 2.  GT: 5M samples of the patch.  Noise 0.3 tau and a missed strip, as in tnt_cases.make_scene.
    large         Courthouse-like, tau = 0.025: 120 m of terrain, a concave 20-vertex crop polygon.
    stride_half   exactly 2.5 * 2^22 = 10 485 760 reconstruction points inside the crop (round(2.5) = 2, half to even); the GT is
                  the same points in another order, so ICP converges at once and the row costs little beyond its size.
    block_gap     MaxDistCP's blocks over the score box (min / max -+ 5 tau) leave gaps of one rounding step
                  (Low_k + 5 tau < Low_{k+1}); the cloud's minimum is chosen so that gaps fall inside it, and points sit exactly
                  on the gap values, each with a point of the other cloud within tau.
    hist_edges    single-point voxels whose nearest distances are exactly the histogram edges np.arange(0, 5 tau, tau / 100)
                  and exactly tau (precision and recall count d < tau strictly).
    voxel_keys    voxel-index bit widths 22/21/21 (a 64-bit key, not split), 22/21/22 (split), and an x extent at the int32
                  limit of Open3D's bound check (accepted) and one voxel beyond it (refused).
    polygon_limits  crop polygons of 128 vertices (the kernel's limit) and 129 (refused).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from tests import tnt_cases

OFFSET = tnt_cases.OFFSET
UNIFORM_MAX_POINTS = 4 * 2 ** 20   # tnt_eval.UNIFORM_MAX_POINTS
STRIDE_HALF = 10 * 2 ** 20         # 2.5 * 4 * 2^20


def f32(p) -> np.ndarray:
    return tnt_cases.f32(p)


def _height(x, y):
    return 0.3 * np.sin(1.3 * x) * np.cos(1.1 * y) + 0.1 * x * y


def _patch(rng, n, half):
    x, y = rng.uniform(-half, half, n), rng.uniform(-half, half, n)
    return np.stack([x, y, _height(x, y)], axis=1) + OFFSET


def object_crop():
    ang = np.arange(6) * (np.pi / 3) + 0.2
    poly = np.stack([OFFSET[0] + 1.45 * np.cos(ang), OFFSET[1] + 1.45 * np.sin(ang), np.full(6, OFFSET[2])], axis=1)
    return {"orthogonal_axis": 2, "axis_min": OFFSET[2] - 0.8, "axis_max": OFFSET[2] + 0.8, "polygon": f32(poly)}


def object_row(seed: int = 0, n_patch: int = 13_500_000, n_floor: int = 3_900_000, n_gt: int = 5_000_000):
    """-> {"rec" (reconstruction frame), "gt", "crop", "S" (rec -> GT), "tau"}."""
    tau = 0.003
    rng = np.random.RandomState(seed)
    gt = f32(_patch(rng, n_gt, 1.6))
    rec = _patch(rng, n_patch, 1.6)
    rec = rec[~((rec[:, 0] - OFFSET[0] > 0.3) & (rec[:, 0] - OFFSET[0] < 0.5))]  # a strip the reconstruction missed
    rec += rng.normal(0.0, 0.3 * tau, rec.shape)
    floor = np.stack([rng.uniform(-3.0, 3.0, n_floor), rng.uniform(-3.0, 3.0, n_floor), np.full(n_floor, -1.0)], 1) + OFFSET
    floor[:, 2] += rng.normal(0.0, 0.3 * tau, n_floor)  # below axis_min: outside the crop
    k = int(0.03 * len(rec))
    far = rng.uniform(-1, 1, (k, 3)) * 1.5 + OFFSET + np.array([0.0, 0.0, 2.5])  # above axis_max
    rec = np.concatenate([rec, floor, far])[rng.permutation(len(rec) + n_floor + k)]
    s = tnt_cases.similarity(1.3, [0.2, -0.4, 0.9], 0.5, [-2.0, 1.5, 0.75])
    return {"rec": f32(tnt_cases.apply(np.linalg.inv(s), rec)), "gt": gt, "crop": object_crop(), "S": s, "tau": tau}


def large_row(seed: int = 1, n_rec: int = 3_000_000, n_gt: int = 2_000_000):
    """-> {"rec", "gt", "crop", "tau"}: 120 m of terrain around (200, -150, 30); the concave polygon alternates radii."""
    tau = 0.025
    rng = np.random.RandomState(seed)
    o = np.array([200.0, -150.0, 30.0])

    def terrain(n, noise):
        x, y = rng.uniform(-60, 60, n), rng.uniform(-60, 60, n)
        z = 2.0 * np.sin(x / 15.0) * np.cos(y / 20.0) + 0.02 * x
        return f32(np.stack([x, y, z], 1) + o + rng.normal(0.0, noise, (n, 3)))

    ang = np.arange(20) * (2 * np.pi / 20)
    rad = np.where(np.arange(20) % 2 == 0, 55.0, 32.0)
    poly = f32(np.stack([o[0] + rad * np.cos(ang), o[1] + rad * np.sin(ang), np.full(20, o[2])], 1))
    crop = {"orthogonal_axis": 2, "axis_min": o[2] - 4.0, "axis_max": o[2] + 4.0, "polygon": poly}
    return {"rec": terrain(n_rec, 0.3 * tau), "gt": terrain(n_gt, 0.0), "crop": crop, "tau": tau}


def stride_half_row(seed: int = 2):
    """STRIDE_HALF reconstruction points well inside the crop of object_row (x, y within 0.88 of its centre: inside the
    hexagon's inradius 1.256 whatever ICP's small corrections), 1% above it; identity frame.  GT: the inside points
    permuted."""
    tau = 0.003
    rng = np.random.RandomState(seed)
    inside = f32(_patch(rng, STRIDE_HALF, 0.88))
    out = f32(_patch(rng, STRIDE_HALF // 100, 0.88) + np.array([0.0, 0.0, 2.0]))
    rec = np.concatenate([inside, out])[rng.permutation(STRIDE_HALF + len(out))]
    return {"rec": rec, "gt": inside[rng.permutation(STRIDE_HALF)], "crop": object_crop(), "S": np.eye(4), "tau": tau}


# ---- MaxDistCP block gaps ---------------------------------------------------------------------------------------------------

def block_gaps(lo: float, m: float, k_max: int) -> np.ndarray:
    """The values High_k = (lo + k m) + m, k < k_max, that lie below Low_{k+1} = lo + (k + 1) m: in no block (each operation
    rounded on its own, as MaxDistCP and the kernel's block test compute them)."""
    k = np.arange(k_max, dtype=np.float64)
    high = (lo + k * m) + m
    return high[high < lo + (k + 1) * m]


def block_gaps_fused(lo: float, m: float, k_max: int) -> np.ndarray:
    """The same with Low_k = fma(k, m, lo) (one rounding), the arithmetic of a contracted multiply-add."""
    low = [float(Fraction(k) * Fraction(m) + Fraction(lo)) for k in range(k_max + 1)]
    return np.array([low[k] + m for k in range(k_max) if low[k] + m < low[k + 1]])


def _gap_minimum(base: float, m: float, k_lo: int, k_hi: int) -> float:
    """The first float32 minimum near `base` whose box (minimum - m) has a gap between blocks k_lo and k_hi."""
    for j in range(20000):
        a = float(np.float32(base + j * 1.1e-4))
        if (block_gaps(a - m, m, k_hi) > a + k_lo * m).any():
            return a
    raise AssertionError("no minimum with block gaps found")


def block_gap_row():
    """-> {"rec", "gt", "crop", "tau", "lo", "gaps" [(axis, value)], "gap_rec" (rec rows on a gap), "gap_gt" (gt rows)}.
    One anchor rec point holds the minimum of both clouds on every axis, so the score box is lo = anchor - 5 tau.  Every point
    is alone in its tau / 2 voxel (the down-sampled clouds keep its coordinates exactly)."""
    tau = 0.003
    m = 5 * tau
    k_hi = 400
    anchor = np.array([_gap_minimum(b, m, 4, k_hi) for b in (30.0, -17.0, 6.0)])
    lo = anchor - m
    rng = np.random.RandomState(3)
    rec, gt, gap_rec, gap_gt, gaps = [anchor], [], [], [], []
    slot = 0
    for a in range(3):
        vals = np.union1d(block_gaps(lo[a], m, k_hi), block_gaps_fused(lo[a], m, k_hi))
        vals = vals[vals > anchor[a] + 3 * m]
        for v in vals:
            for side in (0, 1):  # side 0: the rec point on the gap, 1: the GT point
                slot += 1
                p = anchor + 0.5 + 0.05 * np.array([slot % 40, (slot // 40) % 40, slot // 1600], np.float64)
                p = f32(p)
                p[a] = v
                q = p.copy()
                b = (a + 1) % 3
                q[b] = float(np.float32(p[b] + (0.4 if side == 0 else 0.7) * tau))  # the partner: within tau, off the gap axis
                if side == 0:
                    gap_rec.append(len(rec)); rec.append(p); gt.append(q)
                else:
                    gap_gt.append(len(gt)); gt.append(p); rec.append(q)
                gaps.append((a, float(v)))
    filler = f32(anchor + 0.5 + rng.uniform(0, 2.0, (3000, 3)))  # scattered pairs, 0.2 tau to 8 tau apart
    rec += list(filler)
    gt += list(f32(filler + rng.uniform(0.2, 8.0, (3000, 1)) * tau * np.array([0.6, 0.0, 0.8])))
    crop = {"orthogonal_axis": 2, "axis_min": -1e3, "axis_max": 1e3,
            "polygon": np.array([[-1e3, -1e3, 0.0], [1e3, -1e3, 0.0], [1e3, 1e3, 0.0], [-1e3, 1e3, 0.0]])}
    return {"rec": np.array(rec), "gt": np.array(gt), "crop": crop, "tau": tau, "lo": lo, "gaps": gaps,
            "gap_rec": np.array(gap_rec), "gap_gt": np.array(gap_gt)}


def hist_edges_row():
    """Pairs (0, Y, Z) and (e, Y, Z), Y and Z on a 0.1 grid: both nearest distances are exactly e (dx = e - 0, dy = dz = 0,
    and sqrt(e * e) = e in binary floating point).  e: every histogram edge, exactly tau, and its neighbours."""
    tau = 0.003
    edges = np.arange(0, 5 * tau, tau / 100)
    e = np.concatenate([edges, [tau, np.nextafter(tau, 0), np.nextafter(tau, 1), 5 * tau, np.nextafter(5 * tau, 0)]])
    j = np.arange(len(e))
    yz = np.stack([0.1 * (j % 30), 0.1 * (j // 30)], 1)
    rec = np.concatenate([np.zeros((len(e), 1)), yz], 1)
    gt = np.concatenate([e[:, None], yz], 1)
    crop = {"orthogonal_axis": 2, "axis_min": -10.0, "axis_max": 10.0,
            "polygon": np.array([[-10.0, -10.0, 0.0], [10.0, -10.0, 0.0], [10.0, 10.0, 0.0], [-10.0, 10.0, 0.0]])}
    return {"rec": rec, "gt": gt, "crop": crop, "tau": tau, "distances": e}


# ---- voxel keys and polygon limits ------------------------------------------------------------------------------------------

def voxel_keys_rows():
    """-> {name: (points, voxel size, refusal message or None)}.  Voxel 1.0 and minimum 0: a coordinate c is in voxel
    floor(c + 0.5); the largest index per axis sets its key bits."""
    rng = np.random.RandomState(4)

    def row(top):
        top = np.asarray(top, np.float64)
        p = np.floor(rng.uniform(0, 1, (20000, 3)) * (top + 1)) + rng.uniform(-0.4, 0.4, (20000, 3))
        p[:3000] = p[rng.randint(3000, 20000, 3000)] + rng.uniform(-0.05, 0.05, (3000, 3))  # shared voxels
        p = np.clip(p, 0.0, top)
        p[0], p[1] = 0.0, top  # the extremes: bits exactly
        return f32(p) if top.max() < 2 ** 24 else p

    return {"64_bits": (row([2 ** 21 + 5, 2 ** 20 + 3, 2 ** 20 + 7]), 1.0, None),      # 22 + 21 + 21
            "65_bits": (row([2 ** 21 + 5, 2 ** 20 + 3, 2 ** 21 + 7]), 1.0, None),      # 22 + 21 + 22: split
            "x_int32": (row([2.0 ** 31 - 2, 100.0, 100.0]), 1.0, None),                # largest accepted extent
            "x_int32_over": (row([2.0 ** 31 - 1, 100.0, 100.0]), 1.0, "int32")}        # one voxel more


def star_polygon(n: int, centre=(0.0, 0.0), r_out: float = 1.0, r_in: float = 0.6) -> np.ndarray:
    a = np.arange(n) * (2 * np.pi / n)
    r = np.where(np.arange(n) % 2 == 0, r_out, r_in)
    return f32(np.stack([centre[0] + r * np.cos(a), centre[1] + r * np.sin(a), np.zeros(n)], 1))


# ---- cell faces of the nearest-neighbour search -----------------------------------------------------------------------------

def _cell(x: float, inv: float) -> int:
    return int(np.floor(x * inv))  # the kernel's fine_coord: floor(x * (1 / cell)), rounded products


def _ulps_around(v: float, n: int):
    out, u, d = [v], v, v
    for _ in range(n):
        u, d = float(np.nextafter(u, np.inf)), float(np.nextafter(d, -np.inf))
        out += [u, d]
    return out


def cell_face_trios(cell: float, y0: float = 0.0, z0: float = 0.0):
    """Queries whose computed fine cell f = floor(x (1 / c)) is one above their true one, each with two targets on the same
    x line (y, z equal, so |t - x| is an exact difference of x):
        x   a query a few ulps from a cell face, its product x (1 / c) rounded up across the integer;
        t   the true nearest target, whose computed cell is f -+ (k + 1): unvisited after fine ring k, yet at exact distance
            |t - x| < k c;
        v   a visited target on the other side (computed cell within f -+ k): the mirror of t moved 1.5e-9 off the line,
            at a distance in (|t - x|, k c] (the x grid has no value strictly between at these magnitudes).
    Such trios need the two faces' products to round differently, which happens where the product crosses a power of two
    (face indices 2^15 and 2^16 here).  After ring k the best distance is |x - v| <= k c: a search that stops at best <= k c
    (no slack for the rounding of floor(x / c)) returns v; the library's stops only at best <= (k - 1e-6) c and goes on to
    find t.  Trios sit 0.1 apart in y.  -> (queries [m,3], visited [m,3], true [m,3], k [m])."""
    c, inv = Fraction(cell), 1.0 / cell
    q, vis, tru, ks = [], [], [], []
    for centre in (2 ** 15, 2 ** 16):
        for a in range(centre - 4, centre + 5):
            for x in _ulps_around(float(a * c), 8):
                f = _cell(x, inv)
                if f == int(np.floor(Fraction(x) / c)):
                    continue
                for k in (1, 2):
                    best = None
                    for b in range(a - k - 3, a + k + 4):
                        for t in _ulps_around(float(b * c), 8):
                            d = abs(Fraction(t) - Fraction(x))
                            if abs(_cell(t, inv) - f) >= k + 1 and d < k * c and Fraction(abs(t - x)) == d:
                                best = t if best is None or d < abs(Fraction(best) - Fraction(x)) else best
                    if best is None:
                        continue
                    v = x + (x - best)  # the mirror of t, then moved off the line by dy: just farther than t
                    dy = 1.5e-9
                    d_true = abs(x - best)
                    d_vis = float(np.sqrt((v - x) * (v - x) + dy * dy))
                    if abs(v - x) != d_true or abs(_cell(v, inv) - f) > k or not d_true < d_vis <= k * cell:
                        continue
                    if any(r[0] == x for r in q):
                        continue
                    y = y0 + 0.1 * len(q)
                    q.append([x, y, z0]); vis.append([v, y + dy, z0]); tru.append([best, y, z0]); ks.append(k)
    assert len(q) >= 2, "no cell-face trios"
    return np.array(q), np.array(vis), np.array(tru), np.array(ks)


def lattice_ties(base, n_side: int = 16, n_src: int = 4000, seed: int = 5):
    """An exact lattice of spacing 2^-8 at `base` (every coordinate exact in float64) and sources on its half-integer
    positions: up to 8 targets at exactly the same distance (at most sqrt(3) 2^-9 < 0.0034).  -> (targets, sources)."""
    s = 2.0 ** -8
    g = np.arange(n_side) * s
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + np.asarray(base, np.float64)
    rng = np.random.RandomState(seed)
    idx = rng.randint(1, n_side - 1, (n_src, 3)) * s
    half = rng.randint(0, 2, (n_src, 3)) * (s / 2)
    half[:, 0] = s / 2  # at least one half coordinate: two or more candidates tie
    return lat, idx + half + np.asarray(base, np.float64)
