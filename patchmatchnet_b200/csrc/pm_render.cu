// pm_render.cu -- headless rendering of point clouds and triangle meshes (beyond the reference; INTEGRATION.md "Rendering
// (beyond the reference)", definition and contract in include/patchmatch_b200.h).  float32 throughout, every product, sum and
// difference rounded on its own (no fused multiply-add), so tests/render_oracle.py reproduces every pixel bit for bit.
//
// Z-buffer: one uint64 per pixel, cleared to all ones; a fragment writes atomicMin((float_bits(z) << 32) | primitive index).
// z > 0, so the nearest fragment wins and an exact depth tie goes to the lower index, whatever the launch order.  The resolve
// then recomputes the winner's attributes at the pixel.
//
// Points: one thread per point splats its s x s square.  Meshes: vertices are projected once; one thread per triangle
// rasterises the triangles whose clipped box is at most kSmallBox pixels on a side, larger ones are appended to a list (atomic
// counter) that a grid of CTAs rasterises, one triangle per CTA at a time, striding over its box.  Both call cover()
// (pm_raster.cuh, shared with the texturer's visibility pass).
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "../../include/patchmatch_b200.h"
#include "pm_raster.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmraster;

constexpr int kBlock = 256;
constexpr int kLargeCtas = 1056;    // CTAs of the large-triangle pass (8 per SM of an H100 SXM)
constexpr int kMaxSide = 16384;     // width and height
constexpr float kGrey = 160.0f;     // colour of a PLY without colours

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 * 8 ? 65535 * 8 : b));
}

// 0.25 + 0.75 |n . l| with l = d / |d| (d = camera centre - surface point); 1 where that is undefined
__device__ inline float shade_factor(float nx, float ny, float nz, float dx, float dy, float dz) {
    const float dot = __fadd_rn(__fadd_rn(__fmul_rn(nx, dx), __fmul_rn(ny, dy)), __fmul_rn(nz, dz));
    const float nn = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
    const float ll = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    const float den = __fmul_rn(nn, ll);
    if (!(den > 0.0f) || !(den < INFINITY)) return 1.0f;
    const float f = __fadd_rn(0.25f, __fmul_rn(0.75f, fabsf(dot / den)));
    return f < INFINITY ? f : 1.0f;
}

__device__ inline unsigned char channel(float c, float f) {
    const int v = __float2int_rn(__fmul_rn(c, f));
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__device__ inline void write_background(const Camera &c, size_t p, unsigned char *out_rgb, float *out_depth) {
    for (int k = 0; k < 3; ++k) out_rgb[3 * p + k] = (unsigned char)c.bg[k];
    out_depth[p] = 0.0f;
}

// ---- points ---------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) splat_kernel(const Camera c, const float *xyz, long long n, int half,
                                                       unsigned long long *zbuf) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock) {
        const float3 q = project(c, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        if (!(q.z > c.near_z) || !(q.z < INFINITY) || !(fabsf(q.x) < INFINITY) || !(fabsf(q.y) < INFINITY)) continue;
        const float cx = rintf(q.x), cy = rintf(q.y), r = (float)half;
        const float x0 = fmaxf(cx - r, 0.0f), x1 = fminf(cx + r, (float)(c.W - 1));
        const float y0 = fmaxf(cy - r, 0.0f), y1 = fminf(cy + r, (float)(c.H - 1));
        if (!(x0 <= x1) || !(y0 <= y1)) continue;
        const unsigned long long key = ((unsigned long long)__float_as_uint(q.z) << 32) | (unsigned long long)(uint32_t)i;
        for (int y = (int)y0; y <= (int)y1; ++y)
            for (int x = (int)x0; x <= (int)x1; ++x) atomicMin(zbuf + (size_t)y * c.W + x, key);
    }
}

__global__ void __launch_bounds__(kBlock) resolve_points_kernel(const Camera c, const float *xyz, const unsigned char *rgb,
                                                                const float *normals, const unsigned long long *zbuf,
                                                                unsigned char *out_rgb, float *out_depth) {
    const size_t npix = (size_t)c.W * c.H;
    for (size_t p = blockIdx.x * (size_t)kBlock + threadIdx.x; p < npix; p += (size_t)gridDim.x * kBlock) {
        const unsigned long long key = zbuf[p];
        if (key == kEmpty) {
            write_background(c, p, out_rgb, out_depth);
            continue;
        }
        const size_t i = (uint32_t)key;
        float f = 1.0f;
        if (c.shade && normals) {
            f = shade_factor(normals[3 * i], normals[3 * i + 1], normals[3 * i + 2], __fsub_rn(c.C[0], xyz[3 * i]),
                             __fsub_rn(c.C[1], xyz[3 * i + 1]), __fsub_rn(c.C[2], xyz[3 * i + 2]));
        }
        for (int k = 0; k < 3; ++k) out_rgb[3 * p + k] = channel(rgb ? (float)rgb[3 * i + k] : kGrey, f);
        out_depth[p] = __uint_as_float((uint32_t)(key >> 32));
    }
}

// ---- meshes ---------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) project_kernel(const Camera c, const float *xyz, long long nv, float4 *proj) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < nv; i += (long long)gridDim.x * kBlock) {
        const float3 q = project(c, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        const bool ok = q.z > c.near_z && q.z < INFINITY && fabsf(q.x) <= kMaxCoord && fabsf(q.y) <= kMaxCoord;
        proj[i] = make_float4(q.x, q.y, q.z, ok ? 1.0f : 0.0f);
    }
}

__global__ void __launch_bounds__(kBlock) raster_small_kernel(const Camera c, const float4 *proj, const int *faces, long long nf,
                                                              long long nv, unsigned long long *zbuf, int *large, int *n_large) {
    for (long long f = blockIdx.x * (long long)kBlock + threadIdx.x; f < nf; f += (long long)gridDim.x * kBlock) {
        Tri t;
        if (!setup(c, proj, faces, f, nv, t)) continue;
        if (t.x1 - t.x0 >= kSmallBox || t.y1 - t.y0 >= kSmallBox) {
            large[atomicAdd(n_large, 1)] = (int)f;  // nf < 2^31 for a list entry: checked on the host
            continue;
        }
        for (int y = t.y0; y <= t.y1; ++y)
            for (int x = t.x0; x <= t.x1; ++x) raster_pixel(c, t, x, y, (uint32_t)f, zbuf);
    }
}

__global__ void __launch_bounds__(kBlock) raster_large_kernel(const Camera c, const float4 *proj, const int *faces, long long nv,
                                                              const int *large, const int *n_large, unsigned long long *zbuf) {
    const int m = *n_large;
    for (int j = blockIdx.x; j < m; j += gridDim.x) {
        const int f = large[j];
        Tri t;
        setup(c, proj, faces, f, nv, t);  // true: the small pass listed it
        const int bw = t.x1 - t.x0 + 1;
        const long long npix = (long long)bw * (t.y1 - t.y0 + 1);
        for (long long k = threadIdx.x; k < npix; k += kBlock)
            raster_pixel(c, t, t.x0 + (int)(k % bw), t.y0 + (int)(k / bw), (uint32_t)f, zbuf);
    }
}

__global__ void __launch_bounds__(kBlock) resolve_mesh_kernel(const Camera c, const float *xyz, const unsigned char *rgb,
                                                              const float4 *proj, const int *faces, long long nv,
                                                              const unsigned long long *zbuf, unsigned char *out_rgb,
                                                              float *out_depth) {
    const size_t npix = (size_t)c.W * c.H;
    for (size_t p = blockIdx.x * (size_t)kBlock + threadIdx.x; p < npix; p += (size_t)gridDim.x * kBlock) {
        const unsigned long long key = zbuf[p];
        if (key == kEmpty) {
            write_background(c, p, out_rgb, out_depth);
            continue;
        }
        const long long f = (uint32_t)key;
        Tri t;
        float b[3], z;
        setup(c, proj, faces, f, nv, t);
        cover(t, (int)(p % c.W), (int)(p / c.W), b, z);  // the winner covers its pixel, with the same b and z
        float w[3];  // perspective-correct weights
        for (int k = 0; k < 3; ++k) w[k] = __fmul_rn(b[k] / t.z[k], z);
        float f_shade = 1.0f;
        if (c.shade) {
            float X[3], e1[3], e2[3];
            const int v0 = faces[3 * f], v1 = faces[3 * f + 1], v2 = faces[3 * f + 2];  // the face's own order
            for (int a = 0; a < 3; ++a) {
                X[a] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], xyz[3 * (size_t)t.v[0] + a]), __fmul_rn(w[1], xyz[3 * (size_t)t.v[1] + a])),
                                 __fmul_rn(w[2], xyz[3 * (size_t)t.v[2] + a]));
                e1[a] = __fsub_rn(xyz[3 * (size_t)v1 + a], xyz[3 * (size_t)v0 + a]);
                e2[a] = __fsub_rn(xyz[3 * (size_t)v2 + a], xyz[3 * (size_t)v0 + a]);
            }
            f_shade = shade_factor(__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1])),
                                   __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2])),
                                   __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0])), __fsub_rn(c.C[0], X[0]),
                                   __fsub_rn(c.C[1], X[1]), __fsub_rn(c.C[2], X[2]));
        }
        for (int k = 0; k < 3; ++k) {
            float col = kGrey;
            if (rgb)
                col = __fadd_rn(__fadd_rn(__fmul_rn(w[0], (float)rgb[3 * (size_t)t.v[0] + k]), __fmul_rn(w[1], (float)rgb[3 * (size_t)t.v[1] + k])),
                                __fmul_rn(w[2], (float)rgb[3 * (size_t)t.v[2] + k]));
            out_rgb[3 * p + k] = channel(col, f_shade);
        }
        out_depth[p] = __uint_as_float((uint32_t)(key >> 32));
    }
}

// a textured face's colour: the nearest texel of the perspective-correct texture coordinate (the PLY path above is untouched)
__global__ void __launch_bounds__(kBlock) resolve_textured_kernel(const Camera c, const float *xyz, const float4 *proj, const int *faces,
                                                                  long long nv, const float *uv, const int *page,
                                                                  const unsigned char *pages, int n_pages, int S,
                                                                  const unsigned long long *zbuf, unsigned char *out_rgb,
                                                                  float *out_depth) {
    const size_t npix = (size_t)c.W * c.H;
    for (size_t p = blockIdx.x * (size_t)kBlock + threadIdx.x; p < npix; p += (size_t)gridDim.x * kBlock) {
        const unsigned long long key = zbuf[p];
        if (key == kEmpty) {
            write_background(c, p, out_rgb, out_depth);
            continue;
        }
        const long long f = (uint32_t)key;
        Tri t;
        float b[3], z;
        setup(c, proj, faces, f, nv, t);
        cover(t, (int)(p % c.W), (int)(p / c.W), b, z);
        float w[3];
        for (int k = 0; k < 3; ++k) w[k] = __fmul_rn(b[k] / t.z[k], z);
        const bool swapped = t.v[1] != faces[3 * f + 1];  // setup swapped corners 1 and 2 (a rasterised face has distinct corners)
        const int corner[3] = {0, swapped ? 2 : 1, swapped ? 1 : 2};
        float st[2];
        for (int a = 0; a < 2; ++a)
            st[a] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], uv[6 * f + 2 * corner[0] + a]), __fmul_rn(w[1], uv[6 * f + 2 * corner[1] + a])),
                              __fmul_rn(w[2], uv[6 * f + 2 * corner[2] + a]));
        float f_shade = 1.0f;
        if (c.shade) {
            float X[3], e1[3], e2[3];
            const int v0 = faces[3 * f], v1 = faces[3 * f + 1], v2 = faces[3 * f + 2];
            for (int a = 0; a < 3; ++a) {
                X[a] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], xyz[3 * (size_t)t.v[0] + a]), __fmul_rn(w[1], xyz[3 * (size_t)t.v[1] + a])),
                                 __fmul_rn(w[2], xyz[3 * (size_t)t.v[2] + a]));
                e1[a] = __fsub_rn(xyz[3 * (size_t)v1 + a], xyz[3 * (size_t)v0 + a]);
                e2[a] = __fsub_rn(xyz[3 * (size_t)v2 + a], xyz[3 * (size_t)v0 + a]);
            }
            f_shade = shade_factor(__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1])),
                                   __fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2])),
                                   __fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0])), __fsub_rn(c.C[0], X[0]),
                                   __fsub_rn(c.C[1], X[1]), __fsub_rn(c.C[2], X[2]));
        }
        const int pg = page[f];
        const float fs = (float)S;
        const int tx = (int)fminf(fmaxf(floorf(__fmul_rn(st[0], fs)), 0.0f), fs - 1.0f);
        const int ty = (int)fminf(fmaxf(floorf(__fmul_rn(__fsub_rn(1.0f, st[1]), fs)), 0.0f), fs - 1.0f);
        const unsigned char *texel = pages + 3 * (((size_t)pg * S + ty) * S + tx);
        for (int k = 0; k < 3; ++k)
            out_rgb[3 * p + k] = channel(pg >= 0 && pg < n_pages ? (float)texel[k] : kGrey, f_shade);
        out_depth[p] = __uint_as_float((uint32_t)(key >> 32));
    }
}

// ---- host -----------------------------------------------------------------------------------------------------------------

int check_camera(const char *what, const float *P_host, const float *centre_host, int W, int H, float near_z,
                 const unsigned char *background_host, int shade, Camera &c) {
    if (!P_host || !centre_host || !background_host) return pmb200_internal_fail(PMB200_EINVAL, what);
    if (W < 1 || H < 1 || W > kMaxSide || H > kMaxSide) return pmb200_internal_fail(PMB200_EINVAL, what);
    for (int k = 0; k < 12; ++k)
        if (!std::isfinite(P_host[k])) return pmb200_internal_fail(PMB200_EINVAL, what);
    for (int k = 0; k < 3; ++k)
        if (!std::isfinite(centre_host[k])) return pmb200_internal_fail(PMB200_EINVAL, what);
    if (!(near_z > 0.0f) || !(near_z < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, what);
    for (int k = 0; k < 12; ++k) c.P[k] = P_host[k];
    for (int k = 0; k < 3; ++k) c.C[k] = centre_host[k];
    for (int k = 0; k < 3; ++k) c.bg[k] = (float)background_host[k];
    c.W = W; c.H = H; c.near_z = near_z; c.shade = shade ? 1 : 0;
    return 0;
}

struct MeshLayout {
    unsigned long long *zbuf;
    float4 *proj;
    int *large, *n_large;
};

long long mesh_layout(char *base, int W, int H, long long nv, long long nf, MeshLayout &w) {
    size_t used = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + used : nullptr; used += align256(bytes); return p; };
    w.zbuf = reinterpret_cast<unsigned long long *>(take((size_t)W * H * 8));
    w.proj = reinterpret_cast<float4 *>(take((size_t)nv * sizeof(float4)));
    w.large = reinterpret_cast<int *>(take((size_t)nf * sizeof(int)));
    w.n_large = reinterpret_cast<int *>(take(sizeof(int)));
    return (long long)used;
}

}  // namespace

extern "C" int64_t pmb200_render_points_workspace_bytes(int width, int height) {
    if (width < 1 || height < 1 || width > kMaxSide || height > kMaxSide)
        return pmb200_internal_fail(PMB200_EINVAL, "render_points_workspace_bytes: 1 <= width, height <= 16384");
    return (int64_t)align256((size_t)width * height * 8);
}

extern "C" int pmb200_render_points(const float *xyz, const unsigned char *rgb, const float *normals, int64_t n, const float *P_host,
                                   const float *centre_host, int width, int height, int point_size, float near_z, int shade,
                                   const unsigned char *background_host, unsigned char *out_rgb, float *out_depth, void *workspace,
                                   int64_t workspace_bytes, void *stream) {
    if ((!xyz && n > 0) || !out_rgb || !out_depth || !workspace) return pmb200_internal_fail(PMB200_EINVAL, "render_points: null pointer");
    if (n < 0 || n > 0xffffffffll) return pmb200_internal_fail(PMB200_EINVAL, "render_points: 0 <= n < 2^32");
    if (point_size < 1 || point_size > 15 || point_size % 2 == 0)
        return pmb200_internal_fail(PMB200_EINVAL, "render_points: point_size must be odd, 1..15");
    Camera c;
    if (check_camera("render_points: null camera, a size outside 1..16384, a non-finite camera or near not finite and > 0", P_host,
                     centre_host, width, height, near_z, background_host, shade, c))
        return PMB200_EINVAL;
    if (workspace_bytes < pmb200_render_points_workspace_bytes(width, height))
        return pmb200_internal_fail(PMB200_EINVAL, "render_points: workspace smaller than render_points_workspace_bytes(width, height)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned long long *zbuf = static_cast<unsigned long long *>(workspace);
    const size_t npix = (size_t)width * height;
    cudaMemsetAsync(zbuf, 0xff, npix * 8, st);
    if (n > 0) splat_kernel<<<grid_blocks(n), kBlock, 0, st>>>(c, xyz, n, point_size / 2, zbuf);
    resolve_points_kernel<<<grid_blocks((long long)npix), kBlock, 0, st>>>(c, xyz, rgb, normals, zbuf, out_rgb, out_depth);
    return pmb200_internal_launch_status("render_points");
}

extern "C" int64_t pmb200_render_mesh_workspace_bytes(int width, int height, int64_t n_vertices, int64_t n_faces) {
    if (width < 1 || height < 1 || width > kMaxSide || height > kMaxSide || n_vertices < 0 || n_vertices >= (1ll << 31) ||
        n_faces < 0 || n_faces >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL,
                                    "render_mesh_workspace_bytes: 1 <= width, height <= 16384, 0 <= n_vertices, n_faces < 2^31");
    MeshLayout w;
    return mesh_layout(nullptr, width, height, n_vertices, n_faces, w);
}

extern "C" int pmb200_render_mesh(const float *xyz, const unsigned char *rgb, int64_t n_vertices, const int *faces, int64_t n_faces,
                                 const float *P_host, const float *centre_host, int width, int height, float near_z, int shade,
                                 const unsigned char *background_host, unsigned char *out_rgb, float *out_depth, void *workspace,
                                 int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !out_rgb || !out_depth || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh: null pointer");
    if (n_vertices < 0 || n_vertices >= (1ll << 31) || n_faces < 0 || n_faces >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh: 0 <= n_vertices, n_faces < 2^31");
    Camera c;
    if (check_camera("render_mesh: null camera, a size outside 1..16384, a non-finite camera or near not finite and > 0", P_host,
                     centre_host, width, height, near_z, background_host, shade, c))
        return PMB200_EINVAL;
    MeshLayout w;
    const long long need = mesh_layout(static_cast<char *>(workspace), width, height, n_vertices, n_faces, w);
    if (workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh: workspace smaller than render_mesh_workspace_bytes(...)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t npix = (size_t)width * height;
    cudaMemsetAsync(w.zbuf, 0xff, npix * 8, st);
    cudaMemsetAsync(w.n_large, 0, sizeof(int), st);
    if (n_vertices > 0) project_kernel<<<grid_blocks(n_vertices), kBlock, 0, st>>>(c, xyz, n_vertices, w.proj);
    if (n_faces > 0) {
        raster_small_kernel<<<grid_blocks(n_faces), kBlock, 0, st>>>(c, w.proj, faces, n_faces, n_vertices, w.zbuf, w.large, w.n_large);
        raster_large_kernel<<<kLargeCtas, kBlock, 0, st>>>(c, w.proj, faces, n_vertices, w.large, w.n_large, w.zbuf);
    }
    resolve_mesh_kernel<<<grid_blocks((long long)npix), kBlock, 0, st>>>(c, xyz, rgb, w.proj, faces, n_vertices, w.zbuf, out_rgb,
                                                                         out_depth);
    return pmb200_internal_launch_status("render_mesh");
}

extern "C" int pmb200_render_mesh_textured(const float *xyz, int64_t n_vertices, const int *faces, int64_t n_faces, const float *uv,
                                          const int *page, const unsigned char *pages, int n_pages, int side, const float *P_host,
                                          const float *centre_host, int width, int height, float near_z, int shade,
                                          const unsigned char *background_host, unsigned char *out_rgb, float *out_depth,
                                          void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || ((!uv || !page) && n_faces > 0) || (!pages && n_pages > 0) || !out_rgb ||
        !out_depth || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh_textured: null pointer");
    if (n_vertices < 0 || n_vertices >= (1ll << 31) || n_faces < 0 || n_faces >= (1ll << 31) || n_pages < 0 || side < 1 || side > kMaxSide)
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh_textured: 0 <= n_vertices, n_faces < 2^31, n_pages >= 0, 1 <= side <= 16384");
    Camera c;
    if (check_camera("render_mesh_textured: null camera, a size outside 1..16384, a non-finite camera or near not finite and > 0", P_host,
                     centre_host, width, height, near_z, background_host, shade, c))
        return PMB200_EINVAL;
    MeshLayout w;
    const long long need = mesh_layout(static_cast<char *>(workspace), width, height, n_vertices, n_faces, w);
    if (workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "render_mesh_textured: workspace smaller than render_mesh_workspace_bytes(...)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t npix = (size_t)width * height;
    cudaMemsetAsync(w.zbuf, 0xff, npix * 8, st);
    cudaMemsetAsync(w.n_large, 0, sizeof(int), st);
    if (n_vertices > 0) project_kernel<<<grid_blocks(n_vertices), kBlock, 0, st>>>(c, xyz, n_vertices, w.proj);
    if (n_faces > 0) {
        raster_small_kernel<<<grid_blocks(n_faces), kBlock, 0, st>>>(c, w.proj, faces, n_faces, n_vertices, w.zbuf, w.large, w.n_large);
        raster_large_kernel<<<kLargeCtas, kBlock, 0, st>>>(c, w.proj, faces, n_vertices, w.large, w.n_large, w.zbuf);
    }
    resolve_textured_kernel<<<grid_blocks((long long)npix), kBlock, 0, st>>>(c, xyz, w.proj, faces, n_vertices, uv, page, pages, n_pages,
                                                                             side, w.zbuf, out_rgb, out_depth);
    return pmb200_internal_launch_status("render_mesh_textured");
}
