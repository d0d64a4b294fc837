// pm_raster.cuh -- the mesh rasteriser's camera, triangle set-up and coverage rule, shared by pm_render.cu (images) and
// pm_texture.cu (per-face visibility for texturing).  float32, every product, sum and difference rounded on its own (no
// fused multiply-add); definition in include/patchmatch_b200.h ("Rendering"), restated by tests/render_oracle.py.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace pmraster {

constexpr int kSmallBox = 16;            // a triangle whose clipped box is at most 16 x 16 pixels is rasterised by one thread
constexpr float kMaxCoord = 4194304.0f;  // 2^22: a triangle vertex farther out in u or v is not rasterised
constexpr unsigned long long kEmpty = ~0ull;

struct Camera {
    float P[12];   // K [R | t], row-major 3 x 4
    float C[3];    // camera centre
    int W, H;
    float near_z;
    int shade;
    float bg[3];
};

// ((r0 x + r1 y) + r2 z) + r3
__device__ inline float row(const float *r, float x, float y, float z) {
    return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r[0], x), __fmul_rn(r[1], y)), __fmul_rn(r[2], z)), r[3]);
}

// (u, v, z) of a world point; u = u' / z and v = v' / z, IEEE division
__device__ inline float3 project(const Camera &c, float x, float y, float z) {
    const float zz = row(c.P + 8, x, y, z);
    return make_float3(row(c.P, x, y, z) / zz, row(c.P + 4, x, y, z) / zz, zz);
}

struct Tri {
    float x[3], y[3], z[3];
    int v[3];      // mesh vertex of each slot (slots 1 and 2 swapped when the signed area is negative)
    float area;    // > 0
    bool tl[3];    // the edge opposite slot i is a top or left edge
    int x0, x1, y0, y1;  // clipped box, inclusive
};

__device__ inline bool top_left(float ax, float ay, float bx, float by) {
    const float dx = __fsub_rn(bx, ax), dy = __fsub_rn(by, ay);
    return dy < 0.0f || (dy == 0.0f && dx > 0.0f);
}

// the edge function of a -> b at p, evaluated from the edge's lower endpoint (smaller v, then smaller u) and negated when
// that is b, so the two faces of a shared edge get the same magnitude with opposite signs
__device__ inline float edge_at(float ax, float ay, float bx, float by, float px, float py) {
    const bool flip = by < ay || (by == ay && bx < ax);
    const float sx = flip ? bx : ax, sy = flip ? by : ay, ex = flip ? ax : bx, ey = flip ? ay : by;
    const float e = __fsub_rn(__fmul_rn(__fsub_rn(ex, sx), __fsub_rn(py, sy)), __fmul_rn(__fsub_rn(ey, sy), __fsub_rn(px, sx)));
    return flip ? -e : e;
}

// false for a triangle that is not rasterised (a vertex index out of range, a vertex skipped by the projection, zero area,
// or an empty clipped box)
__device__ inline bool setup(const Camera &c, const float4 *proj, const int *faces, long long f, long long nv, Tri &t) {
    for (int k = 0; k < 3; ++k) {
        const int v = faces[3 * f + k];
        if (v < 0 || v >= nv) return false;
        const float4 q = proj[v];
        if (q.w == 0.0f) return false;
        t.x[k] = q.x; t.y[k] = q.y; t.z[k] = q.z; t.v[k] = v;
    }
    float a = __fsub_rn(__fmul_rn(__fsub_rn(t.x[1], t.x[0]), __fsub_rn(t.y[2], t.y[0])),
                        __fmul_rn(__fsub_rn(t.y[1], t.y[0]), __fsub_rn(t.x[2], t.x[0])));
    if (a == 0.0f) return false;
    if (a < 0.0f) {
        float s;
        s = t.x[1]; t.x[1] = t.x[2]; t.x[2] = s;
        s = t.y[1]; t.y[1] = t.y[2]; t.y[2] = s;
        s = t.z[1]; t.z[1] = t.z[2]; t.z[2] = s;
        const int w = t.v[1]; t.v[1] = t.v[2]; t.v[2] = w;
        a = -a;
    }
    t.area = a;
    t.tl[0] = top_left(t.x[1], t.y[1], t.x[2], t.y[2]);
    t.tl[1] = top_left(t.x[2], t.y[2], t.x[0], t.y[0]);
    t.tl[2] = top_left(t.x[0], t.y[0], t.x[1], t.y[1]);
    const float umin = fminf(fminf(t.x[0], t.x[1]), t.x[2]), umax = fmaxf(fmaxf(t.x[0], t.x[1]), t.x[2]);
    const float vmin = fminf(fminf(t.y[0], t.y[1]), t.y[2]), vmax = fmaxf(fmaxf(t.y[0], t.y[1]), t.y[2]);
    t.x0 = (int)fmaxf(ceilf(umin), 0.0f); t.x1 = (int)fminf(floorf(umax), (float)(c.W - 1));
    t.y0 = (int)fmaxf(ceilf(vmin), 0.0f); t.y1 = (int)fminf(floorf(vmax), (float)(c.H - 1));
    return t.x0 <= t.x1 && t.y0 <= t.y1;
}

// pixel (px, py) inside the triangle: its barycentrics b and depth z (0 < z < inf), else false
__device__ inline bool cover(const Tri &t, int px, int py, float b[3], float &z) {
    const float fx = (float)px, fy = (float)py;
    const float e0 = edge_at(t.x[1], t.y[1], t.x[2], t.y[2], fx, fy);
    const float e1 = edge_at(t.x[2], t.y[2], t.x[0], t.y[0], fx, fy);
    const float e2 = edge_at(t.x[0], t.y[0], t.x[1], t.y[1], fx, fy);
    if (!(e0 > 0.0f || (e0 == 0.0f && t.tl[0])) || !(e1 > 0.0f || (e1 == 0.0f && t.tl[1])) ||
        !(e2 > 0.0f || (e2 == 0.0f && t.tl[2])))
        return false;
    b[0] = e0 / t.area; b[1] = e1 / t.area; b[2] = e2 / t.area;
    const float s = __fadd_rn(__fadd_rn(b[0] / t.z[0], b[1] / t.z[1]), b[2] / t.z[2]);
    if (!(s > 0.0f)) return false;
    z = 1.0f / s;
    return z < INFINITY;
}

// the fragment pixel (px, py) of face f offers the z-buffer; true when it covers the pixel
__device__ inline bool raster_pixel(const Camera &c, const Tri &t, int px, int py, uint32_t f, unsigned long long *zbuf) {
    float b[3], z;
    if (!cover(t, px, py, b, z)) return false;
    atomicMin(zbuf + (size_t)py * c.W + px, ((unsigned long long)__float_as_uint(z) << 32) | (unsigned long long)f);
    return true;
}

}  // namespace pmraster
