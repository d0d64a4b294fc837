"""Undistortion of COLMAP cameras restated in numpy float64 (INTEGRATION.md "Undistortion (beyond the reference)"): the 11
camera models, ImageToWorld by Newton's method, the border extents and scale of COLMAP's UndistortCamera, and the bilinear
warp.  TEST INFRASTRUCTURE: the tests compare csrc/pm_camera_math.cuh (host build and GPU) and the ops against it.

Every operation is written in the order pm_camera_math.cuh performs it, so the host build agrees bit for bit.  atan and tan
are libm's (math.atan / math.tan element by element), as the host build calls them; numpy's vectorised versions differ from
libm in the last bit on some machines."""
from __future__ import annotations

import math
from typing import Sequence, Tuple

import numpy as np

DBL_EPSILON = np.finfo(np.float64).eps
NEWTON_ITERATIONS = 100
NEWTON_STEP_NORM2 = 1e-20
NEWTON_REL_STEP = 1e-6
FOV_EPSILON = 1e-4
MIN_SCALE, MAX_SCALE = 0.2, 2.0

SINGLE_FOCAL = {"SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE"}
USES_ATAN = {"OPENCV_FISHEYE", "FOV", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE", "THIN_PRISM_FISHEYE"}

_atan_obj = np.frompyfunc(math.atan, 1, 1)
_tan_obj = np.frompyfunc(math.tan, 1, 1)


def atan(x):
    return np.asarray(_atan_obj(np.asarray(x, dtype=np.float64)), dtype=np.float64)


def tan(x):
    return np.asarray(_tan_obj(np.asarray(x, dtype=np.float64)), dtype=np.float64)


def pinhole_part(model: str, p: Sequence[float]) -> Tuple[float, float, float, float]:
    if model in SINGLE_FOCAL:
        return p[0], p[0], p[1], p[2]
    return p[0], p[1], p[2], p[3]


def _fisheye(model, k, u, v, r2):
    r = np.sqrt(r2)
    th = atan(r)
    th2 = th * th
    if model == "SIMPLE_RADIAL_FISHEYE":
        poly = 1.0 + k[0] * th2
    elif model == "RADIAL_FISHEYE":
        poly = (1.0 + k[0] * th2) + k[1] * (th2 * th2)
    else:
        th4 = th2 * th2
        th6, th8 = th4 * th2, th4 * th4
        poly = (((1.0 + k[0] * th2) + k[1] * th4) + k[2] * th6) + k[3] * th8
    thd = th * poly
    big = r > DBL_EPSILON
    return np.where(big, (u * thd) / r, u), np.where(big, (v * thd) / r, v)


def distort(model: str, p: Sequence[float], u, v):
    """Distorted normalised coordinates (xd, yd) of the normalised points (u, v): x = fx xd + cx."""
    u, v = np.asarray(u, dtype=np.float64), np.asarray(v, dtype=np.float64)
    with np.errstate(all="ignore"):
        u2, v2 = u * u, v * v
        r2 = u2 + v2
        if model in ("SIMPLE_PINHOLE", "PINHOLE"):
            return u.copy(), v.copy()
        if model == "SIMPLE_RADIAL":
            radial = p[3] * r2
            return u + u * radial, v + v * radial
        if model == "RADIAL":
            radial = p[3] * r2 + p[4] * (r2 * r2)
            return u + u * radial, v + v * radial
        if model == "OPENCV":
            k1, k2, p1, p2 = p[4:8]
            uv = u * v
            radial = k1 * r2 + k2 * (r2 * r2)
            du = (u * radial + (2.0 * p1) * uv) + p2 * (r2 + 2.0 * u2)
            dv = (v * radial + (2.0 * p2) * uv) + p1 * (r2 + 2.0 * v2)
            return u + du, v + dv
        if model == "FULL_OPENCV":
            k1, k2, p1, p2, k3, k4, k5, k6 = p[4:12]
            r4 = r2 * r2
            r6, uv = r4 * r2, u * v
            radial = (((1.0 + k1 * r2) + k2 * r4) + k3 * r6) / (((1.0 + k4 * r2) + k5 * r4) + k6 * r6)
            du = ((u * radial + (2.0 * p1) * uv) + p2 * (r2 + 2.0 * u2)) - u
            dv = ((v * radial + (2.0 * p2) * uv) + p1 * (r2 + 2.0 * v2)) - v
            return u + du, v + dv
        if model in ("OPENCV_FISHEYE", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE"):
            return _fisheye(model, p[4:] if model == "OPENCV_FISHEYE" else p[3:], u, v, r2)
        if model == "FOV":
            w = p[4]
            w2 = w * w
            if w2 < FOV_EPSILON:
                f = ((w2 * r2) / 3.0 - w2 / 12.0) + 1.0
            else:
                t = float(tan(w / 2.0))
                small = (-2.0 * t) * ((((4.0 * r2) * t) * t) - 3.0) / (3.0 * w)
                r = np.sqrt(r2)
                general = atan((r * 2.0) * float(tan(w / 2.0))) / (r * w)
                f = np.where(r2 < FOV_EPSILON, small, general)
            return u * f, v * f
        if model == "THIN_PRISM_FISHEYE":
            k1, k2, p1, p2, k3, k4, sx1, sy1 = p[4:12]
            r = np.sqrt(r2)
            th = atan(r)
            big = r > DBL_EPSILON
            uu, vv = np.where(big, (u * th) / r, u), np.where(big, (v * th) / r, v)
            uu2, vv2 = uu * uu, vv * vv
            rho2 = uu2 + vv2
            rho4 = rho2 * rho2
            rho6, rho8, uv = rho4 * rho2, rho4 * rho4, uu * vv
            radial = ((k1 * rho2 + k2 * rho4) + k3 * rho6) + k4 * rho8
            xd = (((uu + uu * radial) + (2.0 * p1) * uv) + p2 * (rho2 + 2.0 * uu2)) + sx1 * rho2
            yd = (((vv + vv * radial) + (2.0 * p2) * uv) + p1 * (rho2 + 2.0 * vv2)) + sy1 * rho2
            return xd, yd
    raise ValueError(f"unknown camera model {model}")


def world_to_image(model: str, p: Sequence[float], u, v):
    fx, fy, cx, cy = pinhole_part(model, p)
    xd, yd = distort(model, p, u, v)
    return fx * xd + cx, fy * yd + cy


def image_to_world(model: str, p: Sequence[float], x, y):
    """Newton's method on distort(u, v) = ((x - cx) / fx, (y - cy) / fy) from that point (FOV: from its closed-form inverse),
    central-difference Jacobian, per point until the squared step is below 1e-20 or 100 iterations; NaN on breakdown."""
    fx, fy, cx, cy = pinhole_part(model, p)
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    xn, yn = (x - cx) / fx, (y - cy) / fy
    u, v = xn.copy(), yn.copy()
    if model in ("SIMPLE_PINHOLE", "PINHOLE"):
        return u, v
    if model == "FOV" and not (p[4] * p[4] < FOV_EPSILON):
        w = p[4]
        rd = np.sqrt(xn * xn + yn * yn)
        big = rd > DBL_EPSILON
        with np.errstate(all="ignore"):
            f = tan(rd * w) / ((rd * 2.0) * float(tan(w / 2.0)))
        u, v = np.where(big, xn * f, u), np.where(big, yn * f, v)
    active = np.ones(u.shape, dtype=bool)
    with np.errstate(all="ignore"):
        for _ in range(NEWTON_ITERATIONS):
            if not active.any():
                break
            a_u, a_v, a_xn, a_yn = u[active], v[active], xn[active], yn[active]
            s0 = np.maximum(DBL_EPSILON, np.abs(NEWTON_REL_STEP * a_u))
            s1 = np.maximum(DBL_EPSILON, np.abs(NEWTON_REL_STEP * a_v))
            ex, ey = distort(model, p, a_u, a_v)
            ax, ay = distort(model, p, a_u - s0, a_v)
            bx, by = distort(model, p, a_u + s0, a_v)
            cx_, cy_ = distort(model, p, a_u, a_v - s1)
            dx_, dy_ = distort(model, p, a_u, a_v + s1)
            j00, j01 = (bx - ax) / (2.0 * s0), (dx_ - cx_) / (2.0 * s1)
            j10, j11 = (by - ay) / (2.0 * s0), (dy_ - cy_) / (2.0 * s1)
            rx, ry = ex - a_xn, ey - a_yn
            det = j00 * j11 - j01 * j10
            sx, sy = (j11 * rx - j01 * ry) / det, (j00 * ry - j10 * rx) / det
            nu, nv = a_u - sx, a_v - sy
            n2 = sx * sx + sy * sy
            bad = ~(n2 < np.inf)
            nu[bad], nv[bad] = np.nan, np.nan
            u[active], v[active] = nu, nv
            idx = np.nonzero(active)[0]
            active[idx[(n2 < NEWTON_STEP_NORM2) | bad]] = False
    return u, v


def border_points(W: int, H: int):
    """(px, py, side) of the 2H + 2W border pixel centres: left and right of each row, then top and bottom of each column."""
    ys, xs = np.arange(H) + 0.5, np.arange(W) + 0.5
    px = np.concatenate([np.full(H, 0.5), np.full(H, W - 0.5), xs, xs])
    py = np.concatenate([ys, ys, np.full(W, 0.5), np.full(W, H - 0.5)])
    side = np.repeat([0, 1, 2, 3], [H, H, W, W])
    return px, py, side


def extents(model: str, p: Sequence[float], W: int, H: int) -> np.ndarray:
    """float64 [8]: (min, max) of the mapped x on the left and right border, then of the mapped y on the top and bottom
    border; points whose Newton iteration broke down are skipped."""
    fx, fy, cx, cy = pinhole_part(model, p)
    px, py, side = border_points(W, H)
    u, v = image_to_world(model, p, px, py)
    mapped = np.where(side < 2, fx * u + cx, fy * v + cy)
    out = np.empty(8)
    for s in range(4):
        m = mapped[side == s]
        m = m[~np.isnan(m)]
        out[2 * s] = m.min() if m.size else np.inf
        out[2 * s + 1] = m.max() if m.size else -np.inf
    return out


def undistorted_camera(model: str, p: Sequence[float], W: int, H: int, ext, blank_pixels: float = 0.0):
    """COLMAP's UndistortCamera scale with min_scale 0.2, max_scale 2.0: (W', H', [fx, fy, cx', cy']); ValueError when a scale is
    not finite."""
    fx, fy, cx, cy = pinhole_part(model, p)
    b = np.float64(blank_pixels)
    dims = []
    with np.errstate(all="ignore"):
        for c, n, e in ((np.float64(cx), W, ext[0:4]), (np.float64(cy), H, ext[4:8])):
            lo_min, lo_max, hi_min, hi_max = (np.float64(t) for t in e)
            min_s = min(c / (c - lo_min), (n - 0.5 - c) / (hi_max - c))
            max_s = max(c / (c - lo_max), (n - 0.5 - c) / (hi_min - c))
            s = 1.0 / (min_s * b + max_s * (1.0 - b))
            if not np.isfinite(s):
                raise ValueError("scale is not finite")
            dims.append(int(max(1.0, float(np.clip(s, MIN_SCALE, MAX_SCALE)) * n)))
    w, h = dims
    return w, h, [fx, fy, cx * w / W, cy * h / H]


def _round_half_away(x):
    a = np.abs(x)
    f = np.floor(a)
    return np.copysign(f + (a - f >= 0.5), x)


def undistort_image(model: str, p: Sequence[float], src: np.ndarray, kp: Sequence[float], out_w: int, out_h: int,
                    rows_per_chunk: int = 256) -> np.ndarray:
    """uint8 [out_h,out_w,3] warp of src uint8 [H,W,3] (the camera's size) into the pinhole camera kp = (fx', fy', cx', cy')."""
    H, W = src.shape[:2]
    out = np.zeros((out_h, out_w, 3), dtype=np.uint8)
    xs_pix = np.arange(out_w, dtype=np.float64)
    srcf = src.astype(np.float64)
    for y0 in range(0, out_h, rows_per_chunk):
        ys_pix = np.arange(y0, min(out_h, y0 + rows_per_chunk), dtype=np.float64)
        X, Y = np.meshgrid(xs_pix, ys_pix)
        u = ((X + 0.5) - kp[2]) / kp[0]
        v = ((Y + 0.5) - kp[3]) / kp[1]
        xs, ys = world_to_image(model, p, u, v)
        with np.errstate(all="ignore"):
            xs, ys = xs - 0.5, ys - 0.5
            valid = (xs >= 0.0) & (xs <= W - 1) & (ys >= 0.0) & (ys <= H - 1)
        xv, yv = xs[valid], ys[valid]
        fx0, fy0 = np.floor(xv), np.floor(yv)
        x0, y0i = fx0.astype(np.int64), fy0.astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0i + 1, H - 1)
        dx, dy = xv - fx0, yv - fy0
        ex, ey = 1.0 - dx, 1.0 - dy
        a = ex[:, None] * srcf[y0i, x0] + dx[:, None] * srcf[y0i, x1]
        b = ex[:, None] * srcf[y1, x0] + dx[:, None] * srcf[y1, x1]
        val = np.clip(_round_half_away(ey[:, None] * a + dy[:, None] * b), 0, 255)
        block = out[int(ys_pix[0]):int(ys_pix[-1]) + 1]
        block[valid] = val.astype(np.uint8)
    return out
