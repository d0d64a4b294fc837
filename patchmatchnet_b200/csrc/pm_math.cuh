// pm_math.cuh -- per-element arithmetic of the learned-PatchMatch path.
//
// Everything here is __host__ __device__ so the same source is (a) inlined into the
// sm_90a kernels and (b) compiled with g++ into tests/_hostmath.so, where the
// formulas (not the kernels) are checked against the oracle on the CPU build box.
// The host build is test infrastructure only; it is never used by the product path.
#pragma once

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PM_HD __host__ __device__ __forceinline__
#else
#define PM_HD inline
#endif

namespace pm {

// A bilinear footprint: the four taps are texels r0, r0+dx, r0+dy*row, r0+dy*row+dx of a
// [rows, cols] map and `w` their weights (already zeroed for taps that fall outside).
// key packs (r0, dx, dy) so two footprints over the same four texels compare equal.
struct Cell {
    float w00, w01, w10, w11;
    int key;
};

constexpr int kKeyDxShift = 29;
constexpr int kKeyDyShift = 30;
constexpr int kKeyIndexMask = (1 << kKeyDxShift) - 1;
constexpr int kKeyNone = -2;  // all four taps outside: contributes exactly 0, nothing is read

PM_HD int cell_r0(int key) { return key & kKeyIndexMask; }
PM_HD int cell_dx(int key) { return (key >> kKeyDxShift) & 1; }
PM_HD int cell_dy(int key) { return (key >> kKeyDyShift) & 1; }

// Zero-padded bilinear footprint at pixel coordinates (u, v) of a [rows, cols] map.
// Equivalent to F.grid_sample(mode=bilinear, padding_mode=zeros, align_corners=True) fed
// with the normalised coordinates 2u/(cols-1)-1 (reference models/module.py:170-181).
PM_HD Cell zero_pad_cell(float u, float v, int rows, int cols) {
    Cell c;
    // taps exist only if floor(u) in [-1, cols-1] and floor(v) in [-1, rows-1]; NaN fails both tests
    if (!(u >= -1.0f && u < (float)cols && v >= -1.0f && v < (float)rows)) {
        c.w00 = c.w01 = c.w10 = c.w11 = 0.0f;
        c.key = kKeyNone;
        return c;
    }
    const float xf = floorf(u), yf = floorf(v);
    const float fx = u - xf, fy = v - yf;
    const int x0 = (int)xf, y0 = (int)yf;
    const float gx = 1.0f - fx, gy = 1.0f - fy;
    const bool x0in = x0 >= 0, x1in = x0 + 1 <= cols - 1;
    const bool y0in = y0 >= 0, y1in = y0 + 1 <= rows - 1;
    c.w00 = (x0in && y0in) ? gx * gy : 0.0f;
    c.w01 = (x1in && y0in) ? fx * gy : 0.0f;
    c.w10 = (x0in && y1in) ? gx * fy : 0.0f;
    c.w11 = (x1in && y1in) ? fx * fy : 0.0f;
    const int x0c = x0in ? x0 : 0, y0c = y0in ? y0 : 0;
    // when one column (row) is outside, both taps alias the inside one: the outside tap already
    // has weight 0, the inside tap keeps its own weight, so no memory outside the map is touched
    const int dx = (x0in && x1in) ? 1 : 0;
    const int dy = (y0in && y1in) ? 1 : 0;
    c.key = (y0c * cols + x0c) | (dx << kKeyDxShift) | (dy << kKeyDyShift);
    return c;
}

// Border-clamped bilinear footprint for a *normalised* coordinate pair produced by the
// reference's get_grid (models/patchmatch.py:420-421: g = p/((size-1)/2) - 1) and consumed
// by F.grid_sample(padding_mode=border, align_corners=False): un-normalise with
// ((g+1)*size-1)/2, clamp to [0,size-1], then bilinear.
PM_HD Cell border_cell(float px, float py, int rows, int cols) {
    const float gx = px / ((float)(cols - 1) * 0.5f) - 1.0f;
    const float gy = py / ((float)(rows - 1) * 0.5f) - 1.0f;
    float ix = ((gx + 1.0f) * (float)cols - 1.0f) * 0.5f;
    float iy = ((gy + 1.0f) * (float)rows - 1.0f) * 0.5f;
    ix = fminf((float)(cols - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(rows - 1), fmaxf(iy, 0.0f));
    const float xf = floorf(ix), yf = floorf(iy);
    const float fx = ix - xf, fy = iy - yf;
    const int x0 = (int)xf, y0 = (int)yf;
    const int dx = (x0 + 1 <= cols - 1) ? 1 : 0;
    const int dy = (y0 + 1 <= rows - 1) ? 1 : 0;
    Cell c;
    const float hx = 1.0f - fx, hy = 1.0f - fy;
    c.w00 = hx * hy;
    c.w01 = dx ? fx * hy : 0.0f;
    c.w10 = dy ? hx * fy : 0.0f;
    c.w11 = (dx && dy) ? fx * fy : 0.0f;
    c.key = (y0 * cols + x0) | (dx << kKeyDxShift) | (dy << kKeyDyShift);
    return c;
}

// Projection of reference pixel (x, y) at depth d into a source view
// (reference models/module.py:161-173).  rt = rot row-major (9) then trans (3).
// (sx, sy) = ((cols_src-1)/(W-1), (rows_src-1)/(H-1)) -- 1 when both maps have the same size.
struct Ray {
    float ax, ay, az;  // rot . (x, y, 1)
};

PM_HD Ray pixel_ray(const float *rt, float x, float y) {
    Ray r;
    r.ax = rt[0] * x + rt[1] * y + rt[2];
    r.ay = rt[3] * x + rt[4] * y + rt[5];
    r.az = rt[6] * x + rt[7] * y + rt[8];
    return r;
}

PM_HD void project(const Ray &r, const float *rt, float d, int W, int H, float sx, float sy, float *u, float *v) {
    float X = r.ax * d + rt[9];
    float Y = r.ay * d + rt[10];
    float Z = r.az * d + rt[11];
    if (Z <= 1e-3f) {  // behind the camera: send to (W, H) so that every tap is outside (module.py:166-169)
        X = (float)W;
        Y = (float)H;
        Z = 1.0f;
    }
    *u = (X / Z) * sx;
    *v = (Y / Z) * sy;
}

#if defined(__CUDACC__) || defined(PM_EMU)
// Device-only variants used by the third-generation K-A kernel: division by MUFU.RCP (<= 2 ulp, i.e.
// < 2e-4 px at 640 px -- far below the fp32 noise of the reference's own normalise/un-normalise round
// trip) and a footprint routine with a branch-free interior fast path.
__device__ __forceinline__ void project_fast(const Ray &r, const float *rt, float d, int W, int H, float sx, float sy,
                                             float *u, float *v) {
    float X = fmaf(r.ax, d, rt[9]);
    float Y = fmaf(r.ay, d, rt[10]);
    float Z = fmaf(r.az, d, rt[11]);
    if (Z <= 1e-3f) {
        X = (float)W;
        Y = (float)H;
        Z = 1.0f;
    }
    const float iz = __fdividef(1.0f, Z);
    *u = X * iz * sx;
    *v = Y * iz * sy;
}

__device__ __forceinline__ Cell zero_pad_cell_fast(float u, float v, int rows, int cols) {
    const float xf = floorf(u), yf = floorf(v);
    const float fx = u - xf, fy = v - yf;
    const float gx = 1.0f - fx, gy = 1.0f - fy;
    // interior: all four taps inside.  (NaN / huge coordinates fail the comparisons and take the general path.)
    if (xf >= 0.0f && xf < (float)(cols - 1) && yf >= 0.0f && yf < (float)(rows - 1)) {
        Cell c;
        c.w00 = gx * gy;
        c.w01 = fx * gy;
        c.w10 = gx * fy;
        c.w11 = fx * fy;
        c.key = ((int)yf * cols + (int)xf) | (1 << kKeyDxShift) | (1 << kKeyDyShift);
        return c;
    }
    return zero_pad_cell(u, v, rows, cols);
}
#endif

// Fixed neighbour offset (dy, dx) tables, reference models/patchmatch.py:331-392.
// Returns false for the counts the reference raises NotImplementedError on.
PM_HD bool neighbour_offset(bool evaluation, int count, int dilation, int k, int *dy, int *dx) {
    const int d = evaluation ? dilation - 1 : dilation;
    int a = 0, b = 0;
    if (evaluation) {
        if (count != 9 && count != 17) return false;
        int kk = k, m = 1;
        if (k >= 9) {  // doubled ring without the centre
            kk = k - 9;
            if (kk >= 4) kk += 1;
            m = 2;
        }
        a = (kk / 3 - 1) * d * m;
        b = (kk % 3 - 1) * d * m;
    } else {
        if (count == 4) {
            const int t4y[4] = {-1, 0, 0, 1}, t4x[4] = {0, -1, 1, 0};
            a = t4y[k] * d;
            b = t4x[k] * d;
        } else if (count == 8 || count == 16) {
            int kk = k % 8, m = (k >= 8) ? 2 : 1;
            if (kk >= 4) kk += 1;  // 3x3 ring without the centre
            a = (kk / 3 - 1) * d * m;
            b = (kk % 3 - 1) * d * m;
        } else {
            return false;
        }
    }
    *dy = a;
    *dx = b;
    return true;
}

// One stratified random hypothesis, reference models/patchmatch.py:61-71 (48 bins).
PM_HD float random_hypothesis(float u01, int bin, float inv_min, float inv_max) {
    float s = u01 + (float)bin;
    s = inv_max + s / 48.0f * (inv_min - inv_max);
    return 1.0f / s;
}

// One local perturbation, reference models/patchmatch.py:78-94.  k_off = floor(-Ns/2) + k.
PM_HD float perturbed_hypothesis(float depth, int k_off, float inv_min, float inv_max, float interval_scale) {
    const float step = (inv_min - inv_max) * interval_scale;
    float s = 1.0f / depth + step * (float)k_off;
    s = fminf(fmaxf(s, inv_max), inv_min);
    return 1.0f / s;
}

PM_HD int floor_div2_neg(int ns) {  // Python's -ns // 2
    return -((ns + 1) / 2);
}

// Depth-similarity weight of one neighbour, reference models/patchmatch.py:657-669.
PM_HD float depth_similarity(float x_centre, float x_neighbour, float interval_scale) {
    float t = fabsf(x_neighbour - x_centre) / interval_scale;
    t = fminf(fmaxf(t, 0.0f), 4.0f);
    const float z = 4.0f - 2.0f * t;
    return 1.0f / (1.0f + expf(-z));
}

PM_HD float normalised_inverse_depth(float depth, float inv_min, float inv_max) {
    return (1.0f / depth - inv_max) / (inv_min - inv_max);
}

}  // namespace pm
