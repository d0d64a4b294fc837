// pm_refine_mesh.cu -- photometric refinement of triangle meshes (beyond the reference; INTEGRATION.md "Mesh refinement
// (beyond the reference)", definition and contract in include/patchmatch_b200.h, per-pixel arithmetic in
// pm_refine_mesh_math.cuh).
//
// Per level, per iteration:
//   z-buffers  one per view at the level's size, with the renderer's set-up, coverage rule and key (pm_raster.cuh);
//   pixels     per ordered pair (i, j) three launches over view i's pixels: the hit on the winning face, validity, a, b and
//              db/dt; the window sums and ZNCC coefficients at every valid centre; dE/db of every valid pixel from the
//              counted windows around it and its scatter onto the face's corners;
//   update     per-vertex unit normals and umbrella vectors over a vertex -> face CSR (built once per call), then the step.
// Every sum that crosses threads is an integer: fixed-point int64 atomics (units in pm_refine_mesh_math.cuh), so reruns
// give the same bits whatever the order of the atomics.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_raster.cuh"
#include "pm_refine_mesh_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmraster;

constexpr int kBlock = 256;
constexpr int kLargeCtas = 1056;  // CTAs of the large-triangle pass (8 per SM of an H100 SXM)
constexpr int kMaxSide = 16384;
constexpr int kTile = 16;         // pixel tiles of the window and gradient passes

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 * 8 ? 65535 * 8 : b));
}

#define GRID_LOOP(i, n) for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < (n); i += (long long)gridDim.x * kBlock)

// ---- grey levels ----------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) grey_kernel(const float *rgb, long long npix, float *out) {
    GRID_LOOP(p, npix) out[p] = pmrm::grey(rgb[p], rgb[npix + p], rgb[2 * npix + p]);
}

__global__ void __launch_bounds__(kBlock) box_kernel(const float *in, int W, int w, int h, float *out) {
    GRID_LOOP(p, (long long)w * h) {
        const int x = (int)(p % w), y = (int)(p / w);
        const float *a = in + (size_t)(2 * y) * W + 2 * x;
        out[p] = pmrm::box(a[0], a[1], a[W], a[W + 1]);
    }
}

// ---- z-buffers (pm_raster.cuh) --------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) project_kernel(const Camera c, const float *xyz, long long nv, float4 *proj) {
    GRID_LOOP(i, nv) {
        const float3 q = project(c, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        const bool ok = q.z > c.near_z && q.z < INFINITY && fabsf(q.x) <= kMaxCoord && fabsf(q.y) <= kMaxCoord;
        proj[i] = make_float4(q.x, q.y, q.z, ok ? 1.0f : 0.0f);
    }
}

__global__ void __launch_bounds__(kBlock) raster_small_kernel(const Camera c, const float4 *proj, const int *faces, long long nf,
                                                              long long nv, unsigned long long *zbuf, int *large, int *n_large) {
    GRID_LOOP(f, nf) {
        Tri t;
        if (!setup(c, proj, faces, f, nv, t)) continue;
        if (t.x1 - t.x0 >= kSmallBox || t.y1 - t.y0 >= kSmallBox) {
            large[atomicAdd(n_large, 1)] = (int)f;
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

// ---- pixels ---------------------------------------------------------------------------------------------------------------

struct View {
    double P[12], K[9], Rt[12], C[3];
    double near_z;
    int W, H;
};

// the hit of pixel (x, y) of view v on its z-buffer winner; false when the pixel is not covered or the ray misses the
// winner's front
__device__ inline bool pixel_hit(const View &v, const unsigned long long *zbuf, const float *xyz, const int *faces, int x, int y,
                                 int &f, pmrm::Hit &h, double *r) {
    const unsigned long long key = zbuf[(size_t)y * v.W + x];
    if (key == kEmpty) return false;
    f = (int)(uint32_t)key;
    pmrm::ray(v.K, v.Rt, (double)x, (double)y, r);
    const int *fv = faces + 3 * (size_t)f;
    return pmrm::hit(v.C, r, xyz + 3 * (size_t)fv[0], xyz + 3 * (size_t)fv[1], xyz + 3 * (size_t)fv[2], h);
}

// per pixel of view i in pair (i, j): valid, a = G_i, b = G_j(pi_j(X)), db/dt
__global__ void __launch_bounds__(kBlock) pixel_kernel(const View vi, const View vj, const unsigned long long *zb_i,
                                                       const unsigned long long *zb_j, const float *gi, const float *gj,
                                                       const float *xyz, const int *faces, unsigned char *valid, float *a,
                                                       double *b, double *dbdt) {
    GRID_LOOP(p, (long long)vi.W * vi.H) {
        const int x = (int)(p % vi.W), y = (int)(p / vi.W);
        int f;
        pmrm::Hit h;
        unsigned char ok = 0;
        double r[3];
        if (pixel_hit(vi, zb_i, xyz, faces, x, y, f, h, r) && pmrm::faces_point(h.n, xyz + 3 * (size_t)faces[3 * (size_t)f], vj.C) &&
            pmrm::oblique_ok(h, r, vj.C)) {
            double q[3];
            pmtex::project(vj.P, h.X[0], h.X[1], h.X[2], q);
            if (pmrm::lands(q, vj.near_z, vj.W, vj.H)) {
                const unsigned long long key = zb_j[(size_t)(int)rint(q[1]) * vj.W + (int)rint(q[0])];
                if (key != kEmpty && pmrm::depth_ok(q[2], __uint_as_float((uint32_t)(key >> 32)))) {
                    double bb, du, dv;
                    pmrm::bilinear(gj, vj.W, vj.H, q[0], q[1], bb, du, dv);
                    b[p] = bb;
                    dbdt[p] = pmrm::db_dt(vj.P, q, r, du, dv);
                    a[p] = gi[p];
                    ok = 1;
                }
            }
        }
        valid[p] = ok;
    }
}

// tile of (kTile + 2 kRadius)^2 pixels around a kTile x kTile block of centres, loaded into shared memory
constexpr int kHalo = kTile + 2 * pmrm::kRadius;

__device__ inline void warp_add(long long v, unsigned long long *dst) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v != 0) atomicAdd(dst, (unsigned long long)v);
}

// per valid centre p: the window sums in row-major order over the clipped window, whether it counts, its coefficients and
// (fixed point) energy
__global__ void __launch_bounds__(kTile *kTile) window_kernel(int W, int H, const unsigned char *valid, const float *a, const double *b,
                                                              unsigned char *counted, double *coef, unsigned long long *energy,
                                                              unsigned long long *windows) {
    __shared__ float sa[kHalo][kHalo];
    __shared__ double sb[kHalo][kHalo];
    __shared__ unsigned char sv[kHalo][kHalo];
    const int bx = blockIdx.x * kTile - pmrm::kRadius, by = blockIdx.y * kTile - pmrm::kRadius;
    for (int k = threadIdx.x; k < kHalo * kHalo; k += kTile * kTile) {
        const int ty = k / kHalo, tx = k % kHalo, x = bx + tx, y = by + ty;
        const bool in = x >= 0 && x < W && y >= 0 && y < H;
        const size_t q = (size_t)y * W + x;
        const unsigned char v = in ? valid[q] : 0;
        sv[ty][tx] = v;
        sa[ty][tx] = v ? a[q] : 0.0f;
        sb[ty][tx] = v ? b[q] : 0.0;
    }
    __syncthreads();
    const int lx = threadIdx.x % kTile, ly = threadIdx.x / kTile;
    const int x = blockIdx.x * kTile + lx, y = blockIdx.y * kTile + ly;
    long long e = 0, cnt = 0;
    if (x < W && y < H) {
        const size_t p = (size_t)y * W + x;
        unsigned char use = 0;
        if (sv[ly + pmrm::kRadius][lx + pmrm::kRadius]) {
            int n = 0;
            double Sa = 0.0, Sb = 0.0, Saa = 0.0, Sbb = 0.0, Sab = 0.0;
            for (int dy = 0; dy <= 2 * pmrm::kRadius; ++dy)
                for (int dx = 0; dx <= 2 * pmrm::kRadius; ++dx) {
                    if (!sv[ly + dy][lx + dx]) continue;
                    const double av = sa[ly + dy][lx + dx], bv = sb[ly + dy][lx + dx];
                    ++n;
                    Sa = pmrm::add(Sa, av);
                    Sb = pmrm::add(Sb, bv);
                    Saa = pmrm::add(Saa, pmrm::mul(av, av));
                    Sbb = pmrm::add(Sbb, pmrm::mul(bv, bv));
                    Sab = pmrm::add(Sab, pmrm::mul(av, bv));
                }
            double E, c[3];
            if (pmrm::window(n, Sa, Sb, Saa, Sbb, Sab, E, c)) {
                use = 1;
                coef[3 * p] = c[0];
                coef[3 * p + 1] = c[1];
                coef[3 * p + 2] = c[2];
                e = pmrm::to_fixed(pmrm::mul(E, pmrm::kEnergyUnit));
                cnt = 1;
            }
        }
        counted[p] = use;
    }
    warp_add(e, energy);
    warp_add(cnt, windows);
}

// the exact int64 sum of v over the lanes of `peers` (every lane of it calls this): v split into 22-, 22- and 20-bit parts,
// each summed by one redux over at most 32 lanes without overflow, and the parts recombined modulo 2^64 (the sum's own
// value when it fits in an int64)
__device__ inline long long peer_sum(unsigned peers, long long v) {
    const unsigned long long u = (unsigned long long)v;
    const unsigned lo = __reduce_add_sync(peers, (unsigned)(u & 0x3FFFFFu));
    const unsigned mid = __reduce_add_sync(peers, (unsigned)((u >> 22) & 0x3FFFFFu));
    const int hi = (int)__reduce_add_sync(peers, (unsigned)(int)(v >> 44));
    return (long long)((unsigned long long)lo + ((unsigned long long)mid << 22) + ((unsigned long long)(long long)hi << 44));
}

// per valid pixel q: the coefficients of the counted windows around it summed in row-major order, dE/dt and the scatter of
// the gradient, weight and footprint onto its face's corners
__global__ void __launch_bounds__(kTile *kTile) grad_kernel(const View vi, const unsigned long long *zb_i, const float *xyz,
                                                            const int *faces, const unsigned char *valid, const float *a,
                                                            const double *b, const double *dbdt, const unsigned char *counted,
                                                            const double *coef, double L, unsigned long long *acc) {
    __shared__ double sc[3][kHalo][kHalo];
    __shared__ unsigned char su[kHalo][kHalo];
    const int W = vi.W, H = vi.H;
    const int bx = blockIdx.x * kTile - pmrm::kRadius, by = blockIdx.y * kTile - pmrm::kRadius;
    for (int k = threadIdx.x; k < kHalo * kHalo; k += kTile * kTile) {
        const int ty = k / kHalo, tx = k % kHalo, x = bx + tx, y = by + ty;
        const bool in = x >= 0 && x < W && y >= 0 && y < H;
        const size_t q = (size_t)y * W + x;
        const unsigned char u = in ? counted[q] : 0;
        su[ty][tx] = u;
        for (int c = 0; c < 3; ++c) sc[c][ty][tx] = u ? coef[3 * q + c] : 0.0;
    }
    __syncthreads();
    const int lx = threadIdx.x % kTile, ly = threadIdx.x / kTile;
    const int x = blockIdx.x * kTile + lx, y = blockIdx.y * kTile + ly;
    if (x >= W || y >= H) return;
    const size_t p = (size_t)y * W + x;
    if (!valid[p]) return;
    double c[3] = {0.0, 0.0, 0.0};
    bool any = false;
    for (int dy = 0; dy <= 2 * pmrm::kRadius; ++dy)
        for (int dx = 0; dx <= 2 * pmrm::kRadius; ++dx) {
            if (!su[ly + dy][lx + dx]) continue;
            any = true;
            for (int k = 0; k < 3; ++k) c[k] = pmrm::add(c[k], sc[k][ly + dy][lx + dx]);
        }
    if (!any) return;
    const double g = pmrm::mul(pmrm::de_db(c, (double)a[p], b[p]), dbdt[p]);
    int f;
    pmrm::Hit h;
    double r[3];
    pixel_hit(vi, zb_i, xyz, faces, x, y, f, h, r);  // true: the pixel is valid
    // the lanes on the same face sum their integer contributions first and one of them adds the sums: neighbouring pixels
    // mostly share a face, and on coarse meshes many warps would otherwise contend on the same corners
    const unsigned peers = __match_any_sync(__activemask(), f);
    const bool leader = (threadIdx.x & 31) == __ffs(peers) - 1;
    for (int k = 0; k < 3; ++k) {
        long long o[5];
        pmrm::contributions(g, h, k, vi.K[0], L, o);
        unsigned long long *dst = acc + 5 * (size_t)faces[3 * (size_t)f + k];
        for (int m = 0; m < 5; ++m) {
            const long long s = peer_sum(peers, o[m]);
            if (leader && s != 0) atomicAdd(dst + m, (unsigned long long)s);
        }
    }
}

// ---- update ---------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) slot_keys_kernel(const int *faces, long long nf, unsigned long long *key) {
    GRID_LOOP(s, 3 * nf) key[s] = ((unsigned long long)(uint32_t)faces[s] << 32) | (unsigned long long)(s / 3);
}

// row_off[v] = the first sorted key of vertex v or later (lower bound), v in 0..nv
__global__ void __launch_bounds__(kBlock) row_kernel(const unsigned long long *key, long long ns, long long nv, long long *row_off) {
    GRID_LOOP(v, nv + 1) {
        long long lo = 0, hi = ns;
        const unsigned long long k = (unsigned long long)v << 32;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (key[mid] < k) lo = mid + 1; else hi = mid;
        }
        row_off[v] = lo;
    }
}

// calls fn(w) for each distinct edge neighbour w != v of v: incident faces in face order, in each the corners in slot order
template <typename Fn>
__device__ inline void for_each_neighbour(long long v, const unsigned long long *key, const long long *row_off, const int *faces, Fn fn) {
    const long long r0 = row_off[v], r1 = row_off[v + 1];
    for (long long e = r0; e < r1; ++e) {
        const int *fv = faces + 3 * (size_t)(uint32_t)key[e];
        for (int s = 0; s < 3; ++s) {
            const int w = fv[s];
            if (w == v) continue;
            bool seen = false;
            for (long long e2 = r0; e2 <= e && !seen; ++e2) {
                const int *gv = faces + 3 * (size_t)(uint32_t)key[e2];
                for (int s2 = 0; s2 < (e2 == e ? s : 3); ++s2) seen = seen || gv[s2] == w;
            }
            if (!seen) fn(w);
        }
    }
}

// unit vertex normal (sum of incident face normals in face order, divided by its length; 0 when the length is 0) and the
// umbrella vector U(v) = (sum over neighbours of (x_w - x_v)) / their count
__global__ void __launch_bounds__(kBlock) vertex_kernel(const float *xyz, const int *faces, long long nv, const unsigned long long *key,
                                                        const long long *row_off, double *normal, double *umb) {
    GRID_LOOP(v, nv) {
        double n[3] = {0.0, 0.0, 0.0};
        for (long long e = row_off[v]; e < row_off[v + 1]; ++e) {
            const int *fv = faces + 3 * (size_t)(uint32_t)key[e];
            double m[3];
            pmrm::face_normal(xyz + 3 * (size_t)fv[0], xyz + 3 * (size_t)fv[1], xyz + 3 * (size_t)fv[2], m);
            for (int c = 0; c < 3; ++c) n[c] = pmrm::add(n[c], m[c]);
        }
        const double len = pmrm::dsqrt(pmrm::dot3(n, n));
        for (int c = 0; c < 3; ++c) normal[3 * v + c] = len > 0.0 ? pmrm::dvd(n[c], len) : 0.0;
        double u[3] = {0.0, 0.0, 0.0};
        int cnt = 0;
        const float *xv = xyz + 3 * v;
        for_each_neighbour(v, key, row_off, faces, [&](int w) {
            ++cnt;
            for (int c = 0; c < 3; ++c) u[c] = pmrm::add(u[c], pmrm::sub((double)xyz[3 * (size_t)w + c], (double)xv[c]));
        });
        for (int c = 0; c < 3; ++c) umb[3 * v + c] = cnt ? pmrm::dvd(u[c], (double)cnt) : 0.0;
    }
}

// U2(v) = (sum over neighbours of (U(w) - U(v))) / their count; x <- float32((x + d n) - lambda U2)
__global__ void __launch_bounds__(kBlock) update_kernel(float *xyz, const int *faces, long long nv, const unsigned long long *key,
                                                        const long long *row_off, const double *normal, const double *umb,
                                                        const unsigned long long *acc, double alpha, double lambda, double L) {
    GRID_LOOP(v, nv) {
        double u2[3] = {0.0, 0.0, 0.0};
        int cnt = 0;
        for_each_neighbour(v, key, row_off, faces, [&](int w) {
            ++cnt;
            for (int c = 0; c < 3; ++c) u2[c] = pmrm::add(u2[c], pmrm::sub(umb[3 * (size_t)w + c], umb[3 * v + c]));
        });
        const long long *s = (const long long *)acc + 5 * v;
        const double d = pmrm::step(s, s[3], s[4], normal + 3 * v, alpha, L);
        for (int c = 0; c < 3; ++c)
            xyz[3 * v + c] = pmrm::moved(xyz[3 * v + c], d, normal[3 * v + c], lambda, cnt ? pmrm::dvd(u2[c], (double)cnt) : 0.0);
    }
}

// ---- host -----------------------------------------------------------------------------------------------------------------

struct Layout {
    unsigned long long *zbuf;  // every view at level 0 sizes, in view order
    float4 *proj;
    int *large, *n_large;
    unsigned char *valid, *counted;
    float *a;
    double *b, *dbdt, *coef;
    unsigned long long *acc, *sums;
    unsigned long long *key_in, *key;
    long long *row_off;
    double *normal, *umb;
    void *cub;
    size_t cub_bytes;
};

bool cub_bytes(long long nf, size_t &out) {
    out = 0;
    return cub::DeviceRadixSort::SortKeys(nullptr, out, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int)(3 * nf)) ==
           cudaSuccess;
}

long long layout(char *base, long long nv, long long nf, const pmb200_refine_view *views, int n_views, size_t cubb, Layout &w) {
    size_t used = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + used : nullptr; used += align256(bytes); return (void *)p; };
    long long max_pix = 0, all_pix = 0;
    for (int v = 0; v < n_views; ++v) {
        const long long n = (long long)views[v].width * views[v].height;
        max_pix = std::max(max_pix, n);
        all_pix += n;
    }
    w.zbuf = (unsigned long long *)take(all_pix * 8);
    w.proj = (float4 *)take(nv * sizeof(float4));
    w.large = (int *)take(nf * 4);
    w.n_large = (int *)take(4);
    w.valid = (unsigned char *)take(max_pix);
    w.counted = (unsigned char *)take(max_pix);
    w.a = (float *)take(max_pix * 4);
    w.b = (double *)take(max_pix * 8);
    w.dbdt = (double *)take(max_pix * 8);
    w.coef = (double *)take(max_pix * 24);
    w.acc = (unsigned long long *)take(nv * 40);
    w.sums = (unsigned long long *)take(16);
    w.key_in = (unsigned long long *)take(3 * nf * 8);
    w.key = (unsigned long long *)take(3 * nf * 8);
    w.row_off = (long long *)take((nv + 1) * 8);
    w.normal = (double *)take(nv * 24);
    w.umb = (double *)take(nv * 24);
    w.cub = take(cubb);
    w.cub_bytes = cubb;
    return (long long)used;
}

bool finite_view(const pmb200_refine_view &x) {
    for (int k = 0; k < 12; ++k)
        if (!std::isfinite(x.P[k]) || !std::isfinite((float)x.P[k]) || !std::isfinite(x.Rt[k])) return false;
    for (int k = 0; k < 9; ++k)
        if (!std::isfinite(x.K[k])) return false;
    return x.K[0] != 0.0 && x.K[4] != 0.0 && x.near_z > 0.0 && (float)x.near_z > 0.0f && (float)x.near_z < INFINITY;
}

// levels x n_views records, level-major; each level halves the previous (floor), down to at least 1 x 1
bool check_views(const pmb200_refine_view *views, int n_views, int levels, int64_t grey_floats) {
    if (!views || n_views < 1 || n_views > 65535 || levels < 1 || levels > 16) return false;
    for (int l = 0; l < levels; ++l)
        for (int v = 0; v < n_views; ++v) {
            const pmb200_refine_view &x = views[(size_t)l * n_views + v];
            if (x.width < 1 || x.height < 1 || x.width > kMaxSide || x.height > kMaxSide || !finite_view(x)) return false;
            if (l > 0 && (x.width != views[(size_t)(l - 1) * n_views + v].width / 2 || x.height != views[(size_t)(l - 1) * n_views + v].height / 2))
                return false;
            if (grey_floats >= 0 && (x.offset < 0 || x.offset + (int64_t)x.width * x.height > grey_floats)) return false;
        }
    return true;
}

bool sizes_ok(long long nv, long long nf) { return nv >= 0 && nv < (1ll << 31) && nf >= 0 && nf < (1ll << 29); }

View device_view(const pmb200_refine_view &x) {
    View v;
    for (int k = 0; k < 12; ++k) { v.P[k] = x.P[k]; v.Rt[k] = x.Rt[k]; }
    for (int k = 0; k < 9; ++k) v.K[k] = x.K[k];
    pmrm::centre(x.Rt, v.C);
    v.near_z = x.near_z;
    v.W = x.width;
    v.H = x.height;
    return v;
}

Camera raster_camera(const pmb200_refine_view &x, const double *C) {
    Camera c;
    for (int k = 0; k < 12; ++k) c.P[k] = (float)x.P[k];
    for (int k = 0; k < 3; ++k) { c.C[k] = (float)C[k]; c.bg[k] = 0.0f; }
    c.W = x.width; c.H = x.height; c.near_z = (float)x.near_z; c.shade = 0;
    return c;
}

}  // namespace

extern "C" int pmb200_refine_mesh_pyramid(const float *rgb, int width, int height, int levels, float *grey_out, void *stream) {
    if (!rgb || !grey_out) return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh_pyramid: null pointer");
    if (width < 1 || height < 1 || width > kMaxSide || height > kMaxSide || levels < 1 || levels > 16 || (width >> (levels - 1)) < 1 ||
        (height >> (levels - 1)) < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh_pyramid: 1..16384 pixels a side, 1..16 levels of at least 1 x 1");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long npix = (long long)width * height;
    grey_kernel<<<grid_blocks(npix), kBlock, 0, st>>>(rgb, npix, grey_out);
    float *in = grey_out;
    int W = width, H = height;
    for (int l = 1; l < levels; ++l) {
        float *out = in + (size_t)W * H;
        box_kernel<<<grid_blocks((long long)(W / 2) * (H / 2)), kBlock, 0, st>>>(in, W, W / 2, H / 2, out);
        in = out;
        W /= 2;
        H /= 2;
    }
    return pmb200_internal_launch_status("refine_mesh_pyramid");
}

extern "C" int64_t pmb200_refine_mesh_workspace_bytes(int64_t n_vertices, int64_t n_faces, const pmb200_refine_view *views_host,
                                                      int n_views) {
    if (!sizes_ok(n_vertices, n_faces) || !check_views(views_host, n_views, 1, -1))
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh_workspace_bytes: 0 <= nv < 2^31, 0 <= nf < 2^29, 1..65535 valid views");
    size_t cubb;
    if (!cub_bytes(n_faces, cubb))
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh_workspace_bytes: no CUDA device to size the CUB sort for");
    Layout w;
    return layout(nullptr, n_vertices, n_faces, views_host, n_views, cubb, w);
}

extern "C" int pmb200_refine_mesh(float *xyz, int64_t n_vertices, const int *faces, int64_t n_faces, const float *grey,
                                  int64_t grey_floats, const pmb200_refine_view *views_host, int n_views, int levels,
                                  const int *pairs_host, int64_t n_pairs, int iterations, double alpha, double smoothness,
                                  double unit_length, int64_t *acc_out, double *stats_host, void *workspace, int64_t workspace_bytes,
                                  void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !grey || !pairs_host || !stats_host || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh: null pointer");
    if (!sizes_ok(n_vertices, n_faces) || !check_views(views_host, n_views, levels, grey_floats))
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh: 0 <= nv < 2^31, 0 <= nf < 2^29, 1..16 levels of 1..65535 views of "
                                                   "1..16384 pixels a side, each level half the previous, with finite cameras, "
                                                   "near > 0 and images inside the grey buffer");
    if (n_pairs < 0 || n_pairs > (1ll << 31) || iterations < 0 || !(alpha >= 0.0 && alpha < INFINITY) ||
        !(smoothness >= 0.0 && smoothness < INFINITY) || !(unit_length > 0.0 && unit_length < INFINITY))
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh: n_pairs >= 0, iterations >= 0, finite alpha, smoothness >= 0 and "
                                                   "unit length > 0");
    for (long long k = 0; k < 2 * n_pairs; ++k)
        if (pairs_host[k] < 0 || pairs_host[k] >= n_views || (k % 2 == 1 && pairs_host[k] == pairs_host[k - 1]))
            return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh: a pair names a view that does not exist, or a view and itself");
    size_t cubb;
    if (!cub_bytes(n_faces, cubb)) return pmb200_internal_launch_status("refine_mesh (CUB sizes)");
    Layout w;
    if (workspace_bytes < layout(static_cast<char *>(workspace), n_vertices, n_faces, views_host, n_views, cubb, w))
        return pmb200_internal_fail(PMB200_EINVAL, "refine_mesh: workspace smaller than refine_mesh_workspace_bytes(...)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long nv = n_vertices, nf = n_faces;
    // vertex -> face CSR: (vertex, face) keys sorted, rows by lower bound
    if (nf > 0) {
        slot_keys_kernel<<<grid_blocks(3 * nf), kBlock, 0, st>>>(faces, nf, w.key_in);
        size_t bytes = w.cub_bytes;
        if (cub::DeviceRadixSort::SortKeys(w.cub, bytes, w.key_in, w.key, (int)(3 * nf), 0, 64, st) != cudaSuccess)
            return pmb200_internal_launch_status("refine_mesh (vertex rows)");
    }
    row_kernel<<<grid_blocks(nv + 1), kBlock, 0, st>>>(w.key, 3 * nf, nv, w.row_off);
    if (nv > 0) cudaMemsetAsync(w.acc, 0, nv * 40, st);
    std::vector<long long> zoff(n_views + 1, 0);
    for (int v = 0; v < n_views; ++v) zoff[v + 1] = zoff[v] + (long long)views_host[v].width * views_host[v].height;
    cudaEvent_t ev[4];
    for (auto &e : ev) cudaEventCreate(&e);
    int rc = 0;
    int row = 0;
    for (int l = levels - 1; l >= 0 && rc == 0; --l) {
        const pmb200_refine_view *lv = views_host + (size_t)l * n_views;
        std::vector<View> dv(n_views);
        for (int v = 0; v < n_views; ++v) dv[v] = device_view(lv[v]);
        for (int it = 0; it < iterations && rc == 0; ++it, ++row) {
            cudaEventRecord(ev[0], st);
            for (int v = 0; v < n_views; ++v) {
                const Camera c = raster_camera(lv[v], dv[v].C);
                unsigned long long *zb = w.zbuf + zoff[v];
                cudaMemsetAsync(zb, 0xff, (size_t)lv[v].width * lv[v].height * 8, st);
                if (nf == 0) continue;
                cudaMemsetAsync(w.n_large, 0, 4, st);
                project_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(c, xyz, nv, w.proj);
                raster_small_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(c, w.proj, faces, nf, nv, zb, w.large, w.n_large);
                raster_large_kernel<<<kLargeCtas, kBlock, 0, st>>>(c, w.proj, faces, nv, w.large, w.n_large, zb);
            }
            cudaEventRecord(ev[1], st);
            cudaMemsetAsync(w.acc, 0, nv * 40, st);
            cudaMemsetAsync(w.sums, 0, 16, st);
            for (long long k = 0; k < n_pairs && nf > 0; ++k) {
                const int i = pairs_host[2 * k], j = pairs_host[2 * k + 1];
                const View &vi = dv[i], &vj = dv[j];
                const long long npix = (long long)vi.W * vi.H;
                pixel_kernel<<<grid_blocks(npix), kBlock, 0, st>>>(vi, vj, w.zbuf + zoff[i], w.zbuf + zoff[j], grey + lv[i].offset,
                                                                   grey + lv[j].offset, xyz, faces, w.valid, w.a, w.b, w.dbdt);
                const dim3 tiles((vi.W + kTile - 1) / kTile, (vi.H + kTile - 1) / kTile);
                window_kernel<<<tiles, kTile * kTile, 0, st>>>(vi.W, vi.H, w.valid, w.a, w.b, w.counted, w.coef, w.sums, w.sums + 1);
                grad_kernel<<<tiles, kTile * kTile, 0, st>>>(vi, w.zbuf + zoff[i], xyz, faces, w.valid, w.a, w.b, w.dbdt, w.counted,
                                                            w.coef, unit_length, w.acc);
            }
            cudaEventRecord(ev[2], st);
            if (nv > 0) {
                vertex_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(xyz, faces, nv, w.key, w.row_off, w.normal, w.umb);
                update_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(xyz, faces, nv, w.key, w.row_off, w.normal, w.umb, w.acc, alpha,
                                                                  smoothness, unit_length);
            }
            cudaEventRecord(ev[3], st);
            long long sums[2];
            if (cudaMemcpyAsync(sums, w.sums, 16, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
                rc = pmb200_internal_launch_status("refine_mesh (iteration)");
                break;
            }
            double *s = stats_host + 6 * (size_t)row;
            s[0] = (double)sums[0] / pmrm::kEnergyUnit;
            s[1] = (double)sums[1];
            s[2] = 0.0;
            for (long long k = 0; k < n_pairs; ++k) s[2] += (double)lv[pairs_host[2 * k]].width * lv[pairs_host[2 * k]].height;
            for (int m = 0; m < 3; ++m) {
                float ms = 0.0f;
                cudaEventElapsedTime(&ms, ev[m], ev[m + 1]);
                s[3 + m] = 1e-3 * ms;
            }
        }
    }
    for (auto &e : ev) cudaEventDestroy(e);
    if (rc) return rc;
    if (acc_out && nv > 0) cudaMemcpyAsync(acc_out, w.acc, nv * 40, cudaMemcpyDeviceToDevice, st);
    return pmb200_internal_launch_status("refine_mesh");
}
