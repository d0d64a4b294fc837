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

PMG_HD void fuse_point(const double *cam, int x, int y, double depth, const float *rgb, unsigned char *rec) {
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
    for (int c = 0; c < 3; ++c) rec[12 + c] = (unsigned char)mul32(load32(rgb + c), 255.0f);
}

}  // namespace pmgeo
