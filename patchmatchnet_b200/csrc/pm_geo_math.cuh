// pm_geo_math.cuh -- per-pixel arithmetic of the geometric-consistency filter (reference eval.py:86-190, :220-256).
//
// __host__ __device__ like pm_math.cuh: inlined into geometric_filter_kernel (pm_geo.cu) and compiled with g++ into
// tests/_hostmath.so, where the formulas are checked on the CPU build box against the oracle and the reference-generated
// fixture.  The host build is test infrastructure only; the product path never uses it.
//
// Arithmetic follows the reference's dtypes step by step so that the thresholded masks agree with it: camera matrices
// arrive already composed the way numpy composes them (float32 inverses / products, see ops.compose_filter_cameras), the
// projections run in float64, the map coordinates are rounded to float32 before sampling, and the bilinear sample is
// cv2.remap's published algorithm -- coordinates rounded to 1/32 pixel (nearest-even), float32 weight table, taps outside
// the image contribute the constant border 0, float32 multiply and add WITHOUT contraction.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PMG_HD __host__ __device__ __forceinline__
#else
#define PMG_HD inline
#endif

namespace pmgeo {

constexpr int kCamDoubles = 60;  // Kref^-1 (9) | T_ref->src (3x4) | Ksrc (9) | Ksrc^-1 (9) | T_src->ref (3x4) | Kref (9)

// float32 operations that must not be contracted into FMAs (the host build is compiled with -ffp-contract=off)
#if defined(__CUDA_ARCH__)
PMG_HD float mul32(float a, float b) { return __fmul_rn(a, b); }
PMG_HD float add32(float a, float b) { return __fadd_rn(a, b); }
PMG_HD float sub32(float a, float b) { return __fsub_rn(a, b); }
PMG_HD float div32(float a, float b) { return __fdiv_rn(a, b); }
PMG_HD float load32(const float *p) { return __ldg(p); }
#else
PMG_HD float mul32(float a, float b) { return a * b; }
PMG_HD float add32(float a, float b) { return a + b; }
PMG_HD float sub32(float a, float b) { return a - b; }
PMG_HD float div32(float a, float b) { return a / b; }
PMG_HD float load32(const float *p) { return *p; }
#endif

PMG_HD void mat3(const double *m, double x, double y, double z, double &ox, double &oy, double &oz) {
    ox = m[0] * x + m[1] * y + m[2] * z;
    oy = m[3] * x + m[4] * y + m[5] * z;
    oz = m[6] * x + m[7] * y + m[8] * z;
}

PMG_HD void mat34(const double *m, double x, double y, double z, double &ox, double &oy, double &oz) {
    ox = m[0] * x + m[1] * y + m[2] * z + m[3];
    oy = m[4] * x + m[5] * y + m[6] * z + m[7];
    oz = m[8] * x + m[9] * y + m[10] * z + m[11];
}

// cvRound(v * 32) as OpenCV computes it on the float32 product: nearest-even; non-finite / out-of-int-range -> INT_MIN
PMG_HD int fixed_coord(float v) {
    const float s = rintf(mul32(v, 32.0f));
    if (!(fabsf(s) < 2147483648.0f)) return INT32_MIN;  // also catches NaN
    return (int)s;
}

// cv2.remap(src, x, y, INTER_LINEAR), float32 single channel, BORDER_CONSTANT(0)
PMG_HD float remap_linear(const float *src, int rows, int cols, float x, float y) {
    const int sx = fixed_coord(x), sy = fixed_coord(y);
    const float fx = (float)(sx & 31) * 0.03125f, fy = (float)(sy & 31) * 0.03125f;
    int ix = sx >> 5, iy = sy >> 5;
    ix = ix < -32768 ? -32768 : (ix > 32767 ? 32767 : ix);
    iy = iy < -32768 ? -32768 : (iy > 32767 ? 32767 : iy);
    const float gx = sub32(1.0f, fx), gy = sub32(1.0f, fy);
    const float w0 = mul32(gy, gx), w1 = mul32(gy, fx), w2 = mul32(fy, gx), w3 = mul32(fy, fx);
    const bool x0 = ix >= 0 && ix < cols, x1 = ix + 1 >= 0 && ix + 1 < cols;
    const bool y0 = iy >= 0 && iy < rows, y1 = iy + 1 >= 0 && iy + 1 < rows;
    const float t00 = (x0 && y0) ? load32(src + (size_t)iy * cols + ix) : 0.0f;
    const float t01 = (x1 && y0) ? load32(src + (size_t)iy * cols + ix + 1) : 0.0f;
    const float t10 = (x0 && y1) ? load32(src + (size_t)(iy + 1) * cols + ix) : 0.0f;
    const float t11 = (x1 && y1) ? load32(src + (size_t)(iy + 1) * cols + ix + 1) : 0.0f;
    float out = mul32(t00, w0);
    out = add32(out, mul32(t01, w1));
    out = add32(out, mul32(t10, w2));
    out = add32(out, mul32(t11, w3));
    return out;
}

// One reference pixel against one source view (eval.py:86-146 + :180-188): -> consistent?, reprojected depth.
PMG_HD bool check_view(const double *c, const float *src_depth, int Hs, int Ws, int x, int y, float dref, double pixel_thres,
                       float depth_thres, float *drep_out) {
    const double dx = (double)x, dy = (double)y, dd = (double)dref;
    double rx, ry, rz, sxw, syw, szw, kx, ky, kz;
    mat3(c, dx * dd, dy * dd, dd, rx, ry, rz);                  // eval.py:116-117
    mat34(c + 9, rx, ry, rz, sxw, syw, szw);                    // :119-120
    mat3(c + 21, sxw, syw, szw, kx, ky, kz);                    // :122
    const double xs = kx / kz, ys = ky / kz;                    // :123
    const float sampled = remap_linear(src_depth, Hs, Ws, (float)xs, (float)ys);  // :126-128
    const double sd = (double)sampled;
    double bx, by, bz, qx, qy, qz;
    mat3(c + 30, xs * sd, ys * sd, sd, bx, by, bz);             // :132-133
    mat34(c + 39, bx, by, bz, qx, qy, qz);                      // :135-136
    const float drep = (float)qz;                               // :138
    mat3(c + 51, qx, qy, qz, kx, ky, kz);                       // :139
    const float x2 = (float)(kx / kz), y2 = (float)(ky / kz);   // :140-142
    const double ex = (double)x2 - dx, ey = (double)y2 - dy;
    const double dist = sqrt(ex * ex + ey * ey);                // :180
    const float rel = div32(fabsf(sub32(drep, dref)), dref);    // :183-184 (float32)
    *drep_out = drep;
    return dist < pixel_thres && rel < depth_thres;             // :187 (NaN compares false)
}

struct PixelResult {
    int count;          // geo_mask_sum (eval.py:248)
    bool photo, final;  // :220, :254-255
    double depth_avg;   // :252
};

// One reference pixel against all V source views (the per-reference-view body of filter_depth, eval.py:220-256).
PMG_HD PixelResult filter_pixel(const double *cams, const float *src_depths, int V, int Hs, int Ws, int x, int y, float dref,
                                float confidence, double pixel_thres, float depth_thres, float photo_thres, int mask_thres) {
    float sum = 0.0f;  // Python's sum(): 0 + a_0 + a_1 + ... in float32
    int cnt = 0;
    for (int v = 0; v < V; ++v) {
        float drep;
        const bool ok = check_view(cams + v * kCamDoubles, src_depths + (size_t)v * Hs * Ws, Hs, Ws, x, y, dref, pixel_thres,
                                   depth_thres, &drep);
        sum = add32(sum, ok ? drep : 0.0f);  // :188, :249
        cnt += ok ? 1 : 0;                   // :248
    }
    PixelResult r;
    r.count = cnt;
    r.photo = confidence > photo_thres;
    r.final = r.photo && cnt >= mask_thres;
    r.depth_avg = (double)add32(sum, dref) / (double)(cnt + 1);  // float32 / int32 -> float64 in numpy
    return r;
}

// One source depth map of a ragged pack: [rows, cols] at src_flat + offset
struct SourceMap {
    long long offset;
    int rows, cols;
};

// filter_pixel with a size per source view: view v samples its own [rows_v, cols_v] map (eval.py:129 remaps each source at
// its own size).  Same arithmetic, same order as filter_pixel.
PMG_HD PixelResult filter_pixel(const double *cams, const float *src_flat, const SourceMap *views, int V, int x, int y, float dref,
                                float confidence, double pixel_thres, float depth_thres, float photo_thres, int mask_thres) {
    float sum = 0.0f;
    int cnt = 0;
    for (int v = 0; v < V; ++v) {
        float drep;
        const bool ok = check_view(cams + v * kCamDoubles, src_flat + views[v].offset, views[v].rows, views[v].cols, x, y, dref,
                                   pixel_thres, depth_thres, &drep);
        sum = add32(sum, ok ? drep : 0.0f);
        cnt += ok ? 1 : 0;
    }
    PixelResult r;
    r.count = cnt;
    r.photo = confidence > photo_thres;
    r.final = r.photo && cnt >= mask_thres;
    r.depth_avg = (double)add32(sum, dref) / (double)(cnt + 1);
    return r;
}

// One fused point (reference eval.py:273-281).  cam: Kref^-1 (9, row-major) | Eref^-1 (16): float32 inverses widened to double,
// composed on the host the way numpy composes them (ops.compose_fusion_camera).  The reference multiplies (x, y, 1) by the
// float64 averaged depth first, then applies the two matrices in float64 (BLAS: one fused multiply-add chain per output, k
// ascending); the result is cast to float32 when the PLY array is assembled.  Colour: float32 image value * 255 in float32,
// truncated to uint8.
constexpr int kFuseCamDoubles = 25;
constexpr int kPlyVertexBytes = 15;
constexpr int kPlyOrientedVertexBytes = 27;  // float32 x, y, z, nx, ny, nz, uint8 r, g, b: the order of COLMAP's fused.ply

PMG_HD void fuse_position(const double *cam, int x, int y, double depth, unsigned char *rec) {
    const double px = (double)x * depth, py = (double)y * depth, pz = depth;
    const double *K = cam, *E = cam + 9;
    const double rx = fma(K[2], pz, fma(K[1], py, K[0] * px));
    const double ry = fma(K[5], pz, fma(K[4], py, K[3] * px));
    const double rz = fma(K[8], pz, fma(K[7], py, K[6] * px));
    float out[3];
    out[0] = (float)fma(E[3], 1.0, fma(E[2], rz, fma(E[1], ry, E[0] * rx)));
    out[1] = (float)fma(E[7], 1.0, fma(E[6], rz, fma(E[5], ry, E[4] * rx)));
    out[2] = (float)fma(E[11], 1.0, fma(E[10], rz, fma(E[9], ry, E[8] * rx)));
    const unsigned char *b = reinterpret_cast<const unsigned char *>(out);
    for (int i = 0; i < 12; ++i) rec[i] = b[i];
}

PMG_HD void fuse_colour(const float *rgb, unsigned char *rec) {
    for (int c = 0; c < 3; ++c) rec[c] = (unsigned char)mul32(load32(rgb + c), 255.0f);
}

PMG_HD void fuse_point(const double *cam, int x, int y, double depth, const float *rgb, unsigned char *rec) {
    fuse_position(cam, x, y, depth, rec);
    fuse_colour(rgb, rec + 12);
}

// fuse_point with the pixel's camera-frame normal (a pmb200_depth_normals output) rotated into the world frame by the rotation
// block of inverse(extrinsics) (cam + 9, rows of 4); a zero normal (no estimate) stays exactly zero.
PMG_HD void fuse_point_oriented(const double *cam, int x, int y, double depth, const float *rgb, const float *normal,
                                unsigned char *rec) {
    fuse_position(cam, x, y, depth, rec);
    const double nx = (double)load32(normal), ny = (double)load32(normal + 1), nz = (double)load32(normal + 2);
    const double *E = cam + 9;
    float out[3] = {0.0f, 0.0f, 0.0f};
    if (nx != 0.0 || ny != 0.0 || nz != 0.0) {
        out[0] = (float)fma(E[2], nz, fma(E[1], ny, E[0] * nx));
        out[1] = (float)fma(E[6], nz, fma(E[5], ny, E[4] * nx));
        out[2] = (float)fma(E[10], nz, fma(E[9], ny, E[8] * nx));
    }
    const unsigned char *b = reinterpret_cast<const unsigned char *>(out);
    for (int i = 0; i < 12; ++i) rec[12 + i] = b[i];
    fuse_colour(rgb, rec + 24);
}

// ---- surface normals from one depth map (pmb200_depth_normals; this project's own definition, the reference has none) ----
// The normal of pixel p = (x, y) is the direction of least spread of the back-projected points P(q) = D(q) K^-1 (x_q, y_q, 1)
// of its inliers: the valid pixels q (finite depth > 0) of the (2r+1)^2 window around p, clipped at the image border, whose
// depth is within depth_thres * D(p) of D(p) (p included).  Everything runs in float64.  The points are shifted by P(p) before
// the covariance about their centroid is formed (two passes: centroid, then covariance), so ~10^3 mm coordinates do not
// cancel.  Zero normal: p invalid, fewer than min_inliers inliers, or lambda_mid <= 1e-6 lambda_max (collinear or coincident
// points).  Otherwise the unit eigenvector of lambda_min, turned to face the camera (n . P(p) < 0), in the camera frame.
constexpr int kNormalMaxRadius = 7;
constexpr double kNormalDegenerate = 1e-6;

#if defined(__CUDA_ARCH__)
PMG_HD double cos_pi(double v) { return cospi(v); }  // no Payne-Hanek slow path: cos(pi * v) without a stack frame
PMG_HD double rsqrt64(double v) { return rsqrt(v); }
#else
PMG_HD double cos_pi(double v) { return cos(3.14159265358979323846 * v); }
PMG_HD double rsqrt64(double v) { return 1.0 / sqrt(v); }
#endif

PMG_HD bool valid_depth(float d) { return isfinite(d) && d > 0.0f; }

// Eigenvalues l0 <= l1 <= l2 of the symmetric matrix [a0 a1 a2; a1 a3 a4; a2 a4 a5] (trigonometric closed form).
PMG_HD void sym3_eigenvalues(const double *a, double &l0, double &l1, double &l2) {
    const double off = a[1] * a[1] + a[2] * a[2] + a[4] * a[4];
    const double q = (a[0] + a[3] + a[5]) * (1.0 / 3.0);
    const double b0 = a[0] - q, b3 = a[3] - q, b5 = a[5] - q;
    const double p2 = (b0 * b0 + b3 * b3 + b5 * b5 + 2.0 * off) * (1.0 / 6.0);
    if (p2 == 0.0) {  // a multiple of the identity
        l0 = l1 = l2 = q;
        return;
    }
    const double ip = rsqrt64(p2), p = p2 * ip;
    const double c0 = b0 * ip, c1 = a[1] * ip, c2 = a[2] * ip, c3 = b3 * ip, c4 = a[4] * ip, c5 = b5 * ip;
    double hdet = 0.5 * (c0 * (c3 * c5 - c4 * c4) - c1 * (c1 * c5 - c4 * c2) + c2 * (c1 * c4 - c3 * c2));
    hdet = hdet < -1.0 ? -1.0 : (hdet > 1.0 ? 1.0 : hdet);
    const double t = acos(hdet) * (1.0 / (3.0 * 3.14159265358979323846));  // phi / pi, phi in [0, pi/3]
    l2 = q + 2.0 * p * cos_pi(t);
    l0 = q + 2.0 * p * cos_pi(t + 2.0 / 3.0);
    l1 = 3.0 * q - l0 - l2;
}

// Unit eigenvector of the symmetric matrix `a` (as above) for its eigenvalue `lam`: the largest cross product of two rows of
// a - lam I.  False when every cross product vanishes.
PMG_HD void cross_keep_largest(double u0, double u1, double u2, double w0, double w1, double w2, double &best, double *v) {
    const double c0 = u1 * w2 - u2 * w1, c1 = u2 * w0 - u0 * w2, c2 = u0 * w1 - u1 * w0;
    const double n2 = c0 * c0 + c1 * c1 + c2 * c2;
    if (n2 > best) {
        best = n2;
        v[0] = c0; v[1] = c1; v[2] = c2;
    }
}

PMG_HD bool sym3_eigenvector(const double *a, double lam, double *v) {
    const double m0 = a[0] - lam, m3 = a[3] - lam, m5 = a[5] - lam;
    double best = 0.0;
    cross_keep_largest(m0, a[1], a[2], a[1], m3, a[4], best, v);  // row 0 x row 1
    cross_keep_largest(m0, a[1], a[2], a[2], a[4], m5, best, v);  // row 0 x row 2
    cross_keep_largest(a[1], m3, a[4], a[2], a[4], m5, best, v);  // row 1 x row 2
    if (!(best > 0.0)) return false;
    const double s = rsqrt64(best);
    v[0] *= s; v[1] *= s; v[2] *= s;
    return true;
}

// The normal of pixel (x, y).  dp points at the pixel's depth in a row-major map (or a tile of it) of row pitch `pitch`; the
// window is dx in [dx0, dx1], dy in [dy0, dy1], already clipped at the image border.  kinv: K^-1 row-major.  -> out[3].
PMG_HD void normal_pixel(const float *dp, int pitch, int x, int y, int dx0, int dx1, int dy0, int dy1, const double *kinv,
                         double depth_thres, int min_inliers, float *out) {
    out[0] = out[1] = out[2] = 0.0f;
    const float dpf = dp[0];
    if (!valid_depth(dpf)) return;
    const double d0 = (double)dpf, tol = depth_thres * d0;
    const double px = d0 * (kinv[0] * x + kinv[1] * y + kinv[2]);
    const double py = d0 * (kinv[3] * x + kinv[4] * y + kinv[5]);
    const double pz = d0 * (kinv[6] * x + kinv[7] * y + kinv[8]);
    int n = 0;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int dy = dy0; dy <= dy1; ++dy)
        for (int dx = dx0; dx <= dx1; ++dx) {
            const float df = dp[dy * pitch + dx];
            if (!valid_depth(df) || !(fabs((double)df - d0) <= tol)) continue;
            const double d = (double)df, u = (double)(x + dx), w = (double)(y + dy);
            sx += d * (kinv[0] * u + kinv[1] * w + kinv[2]) - px;
            sy += d * (kinv[3] * u + kinv[4] * w + kinv[5]) - py;
            sz += d * (kinv[6] * u + kinv[7] * w + kinv[8]) - pz;
            ++n;
        }
    if (n < min_inliers) return;
    const double inv_n = 1.0 / (double)n, cx = sx * inv_n, cy = sy * inv_n, cz = sz * inv_n;
    double a[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int dy = dy0; dy <= dy1; ++dy)
        for (int dx = dx0; dx <= dx1; ++dx) {
            const float df = dp[dy * pitch + dx];
            if (!valid_depth(df) || !(fabs((double)df - d0) <= tol)) continue;
            const double d = (double)df, u = (double)(x + dx), w = (double)(y + dy);
            const double ex = d * (kinv[0] * u + kinv[1] * w + kinv[2]) - px - cx;
            const double ey = d * (kinv[3] * u + kinv[4] * w + kinv[5]) - py - cy;
            const double ez = d * (kinv[6] * u + kinv[7] * w + kinv[8]) - pz - cz;
            a[0] += ex * ex; a[1] += ex * ey; a[2] += ex * ez;
            a[3] += ey * ey; a[4] += ey * ez; a[5] += ez * ez;
        }
    double scale = 0.0;  // the solve runs on the matrix scaled to a largest entry in [1, 2)
    for (int i = 0; i < 6; ++i) scale = fabs(a[i]) > scale ? fabs(a[i]) : scale;
    if (!(scale > 0.0)) return;
    const int e = ilogb(scale);  // a power-of-two scale: exact
    for (int i = 0; i < 6; ++i) a[i] = ldexp(a[i], -e);
    double l0, l1, l2, v[3];
    sym3_eigenvalues(a, l0, l1, l2);
    if (!(l1 > kNormalDegenerate * l2)) return;
    if (!sym3_eigenvector(a, l0, v)) return;
    if (v[0] * px + v[1] * py + v[2] * pz > 0.0) {
        v[0] = -v[0]; v[1] = -v[1]; v[2] = -v[2];
    }
    out[0] = (float)v[0];
    out[1] = (float)v[1];
    out[2] = (float)v[2];
}

}  // namespace pmgeo
