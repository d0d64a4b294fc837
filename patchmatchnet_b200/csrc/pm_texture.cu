// pm_texture.cu -- texturing of triangle meshes from the scene's views (beyond the reference; INTEGRATION.md "Textured meshes
// (beyond the reference)", definition and contract in include/patchmatch_b200.h, per-face arithmetic in pm_texture_math.cuh).
//
// Visibility, one view at a time: the vertices are projected with the renderer's camera and the faces rasterised into a
// z-buffer with its set-up and coverage rule (pm_raster.cuh).  The raster pass also counts each face's covered pixels: a
// thread counts its own face in the small-triangle pass, a CTA reduces its face's count in the large one.  A pass over the
// pixels counts each face's winning pixels (integer atomics).  The faces that pass the candidate test append (face, count)
// entries to a list (one host read per view for its length); after the last view the entries are scattered into a CSR by
// face, in view order, without a sort.
// Labels: argmax of the data term, then kRounds Jacobi rounds over the edge neighbours (the edges sorted by vertex pair).
// Charts: min-label propagation over edges whose faces share a label (hooking with integer atomicMin and pointer jumping,
// one host read per pass); rectangles by integer atomicMin / atomicMax.  No atomic touches a float.
// Pages: the host packs the rectangles into shelves (pmb200_texture_pack); one thread per chart texel copies the nearest
// image pixel of its view, so every texel is written once; one thread per face writes its texture coordinates and, for an
// untextured face, its cell.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <vector>

#include <cub/block/block_reduce.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_raster.cuh"
#include "pm_texture_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmraster;

constexpr int kBlock = 256;
constexpr int kLargeCtas = 1056;  // CTAs of the large-triangle pass (8 per SM of an H100 SXM)
constexpr int kMaxSide = 16384;
constexpr unsigned long long kNoEdge = ~0ull;

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 * 8 ? 65535 * 8 : b));
}

#define GRID_LOOP(i, n) for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < (n); i += (long long)gridDim.x * kBlock)

// ---- visibility -----------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) project_kernel(const Camera c, const float *xyz, long long nv, float4 *proj) {
    GRID_LOOP(i, nv) {
        const float3 q = project(c, xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
        const bool ok = q.z > c.near_z && q.z < INFINITY && fabsf(q.x) <= kMaxCoord && fabsf(q.y) <= kMaxCoord;
        proj[i] = make_float4(q.x, q.y, q.z, ok ? 1.0f : 0.0f);
    }
}

__global__ void __launch_bounds__(kBlock) raster_small_kernel(const Camera c, const float4 *proj, const int *faces, long long nf,
                                                              long long nv, unsigned long long *zbuf, int *large, int *n_large,
                                                              int *covered) {
    GRID_LOOP(f, nf) {
        Tri t;
        if (!setup(c, proj, faces, f, nv, t)) {
            covered[f] = 0;
            continue;
        }
        if (t.x1 - t.x0 >= kSmallBox || t.y1 - t.y0 >= kSmallBox) {
            large[atomicAdd(n_large, 1)] = (int)f;  // covered[f] is written by the large pass
            continue;
        }
        int n = 0;
        for (int y = t.y0; y <= t.y1; ++y)
            for (int x = t.x0; x <= t.x1; ++x) n += raster_pixel(c, t, x, y, (uint32_t)f, zbuf) ? 1 : 0;
        covered[f] = n;
    }
}

__global__ void __launch_bounds__(kBlock) raster_large_kernel(const Camera c, const float4 *proj, const int *faces, long long nv,
                                                              const int *large, const int *n_large, unsigned long long *zbuf,
                                                              int *covered) {
    typedef cub::BlockReduce<int, kBlock> Reduce;
    __shared__ typename Reduce::TempStorage tmp;
    const int m = *n_large;
    for (int j = blockIdx.x; j < m; j += gridDim.x) {
        const int f = large[j];
        Tri t;
        setup(c, proj, faces, f, nv, t);  // true: the small pass listed it
        const int bw = t.x1 - t.x0 + 1;
        const long long npix = (long long)bw * (t.y1 - t.y0 + 1);
        int n = 0;
        for (long long k = threadIdx.x; k < npix; k += kBlock)
            n += raster_pixel(c, t, t.x0 + (int)(k % bw), t.y0 + (int)(k / bw), (uint32_t)f, zbuf) ? 1 : 0;
        const int total = Reduce(tmp).Sum(n);
        if (threadIdx.x == 0) covered[f] = total;
        __syncthreads();  // tmp is reused by the next face
    }
}

__global__ void __launch_bounds__(kBlock) winners_kernel(const unsigned long long *zbuf, long long npix, int *visible) {
    GRID_LOOP(p, npix) {
        const unsigned long long key = zbuf[p];
        if (key != kEmpty) atomicAdd(visible + (uint32_t)key, 1);
    }
}

__global__ void __launch_bounds__(kBlock) candidates_kernel(const pmb200_texture_view view, const float *xyz, const int *faces,
                                                            long long nf, const int *covered, const int *visible, int *ent_face,
                                                            int *ent_count, unsigned long long *n_ent, long long *row_count) {
    GRID_LOOP(f, nf) {
        const int vis = visible[f];
        if (!pmtex::visible_enough(vis, covered[f])) continue;
        double q[9];
        const int *fv = faces + 3 * f;
        if (!pmtex::candidate(view.P, view.centre, view.near_z, view.width, view.height, xyz + 3 * (size_t)fv[0],
                              xyz + 3 * (size_t)fv[1], xyz + 3 * (size_t)fv[2], q))
            continue;
        const unsigned long long e = atomicAdd(n_ent, 1ull);  // the capacity covers every face of the view
        ent_face[e] = (int)f;
        ent_count[e] = vis;
        row_count[f] += 1;  // one entry per face and view: no other thread touches row_count[f] in this launch
    }
}

// the view's entries into their CSR rows: a face's entries land in view order
__global__ void __launch_bounds__(kBlock) scatter_kernel(const int *ent_face, const int *ent_count, long long n, int view,
                                                         const long long *row_off, int *cursor, int *csr_view, int *csr_count) {
    GRID_LOOP(i, n) {
        const int f = ent_face[i];
        const long long p = row_off[f] + cursor[f]++;
        csr_view[p] = view;
        csr_count[p] = ent_count[i];
    }
}

// ---- labels ---------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) edge_keys_kernel(const int *faces, long long nf, unsigned long long *key, int *slot) {
    GRID_LOOP(s, 3 * nf) {
        const long long f = s / 3;
        const int k = (int)(s % 3);
        const unsigned a = (unsigned)faces[3 * f + k], b = (unsigned)faces[3 * f + (k + 1) % 3];
        key[s] = a == b ? kNoEdge : ((unsigned long long)(a < b ? a : b) << 32) | (a < b ? b : a);
        slot[s] = (int)s;
    }
}

__global__ void __launch_bounds__(kBlock) slot_pos_kernel(const int *slot, long long n, int *pos) {
    GRID_LOOP(p, n) pos[slot[p]] = (int)p;
}

// calls fn(g) for every face g != f that shares an edge with f, once per shared edge (sorted edge keys; runs are short)
template <typename Fn>
__device__ inline void for_each_neighbour(long long f, const unsigned long long *key, const int *slot, const int *pos, long long ns,
                                          Fn fn) {
    for (int k = 0; k < 3; ++k) {
        const long long p = pos[3 * f + k];
        const unsigned long long e = key[p];
        if (e == kNoEdge) continue;
        for (long long q = p - 1; q >= 0 && key[q] == e; --q)
            if (slot[q] / 3 != f) fn(slot[q] / 3);
        for (long long q = p + 1; q < ns && key[q] == e; ++q)
            if (slot[q] / 3 != f) fn(slot[q] / 3);
    }
}

__global__ void __launch_bounds__(kBlock) init_labels_kernel(const long long *row_off, const int *csr_view, const int *csr_count,
                                                             long long nf, int *label) {
    GRID_LOOP(f, nf) {
        int best = -1, bd = 0;
        for (long long p = row_off[f]; p < row_off[f + 1]; ++p)
            if (csr_count[p] > bd) { bd = csr_count[p]; best = csr_view[p]; }
        label[f] = best;
    }
}

__global__ void __launch_bounds__(kBlock) smooth_labels_kernel(const long long *row_off, const int *csr_view, const int *csr_count,
                                                               long long nf, const unsigned long long *key, const int *slot,
                                                               const int *pos, const int *label_in, int *label_out) {
    GRID_LOOP(f, nf) {
        const long long p0 = row_off[f], p1 = row_off[f + 1];
        int max_d = 0;
        for (long long p = p0; p < p1; ++p) max_d = max(max_d, csr_count[p]);
        int best = -1;
        double bs = -INFINITY;
        for (long long p = p0; p < p1; ++p) {
            const int v = csr_view[p];
            int same = 0;
            for_each_neighbour(f, key, slot, pos, 3 * nf, [&](long long g) { same += label_in[g] == v ? 1 : 0; });
            const double s = pmtex::score(csr_count[p], max_d, same);
            if (s > bs) { bs = s; best = v; }
        }
        label_out[f] = best;
    }
}

// ---- charts ---------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) chart_init_kernel(const int *label, long long nf, int *chart, int *rect) {
    GRID_LOOP(f, nf) {
        chart[f] = label[f] >= 0 ? (int)f : -1;
        rect[4 * f] = rect[4 * f + 1] = INT_MAX;
        rect[4 * f + 2] = rect[4 * f + 3] = INT_MIN;
    }
}

__global__ void __launch_bounds__(kBlock) chart_hook_kernel(const int *label, long long nf, const unsigned long long *key,
                                                            const int *slot, const int *pos, int *chart, int *changed) {
    GRID_LOOP(f, nf) {
        const int l = label[f];
        if (l < 0) continue;
        for_each_neighbour(f, key, slot, pos, 3 * nf, [&](long long g) {
            if (label[g] != l) return;
            const int a = chart[f], b = chart[g];
            if (a == b) return;
            atomicMin(chart + (a > b ? a : b), a < b ? a : b);
            *changed = 1;
        });
    }
}

__global__ void __launch_bounds__(kBlock) chart_jump_kernel(long long nf, int *chart) {
    GRID_LOOP(f, nf) {
        int c = chart[f];
        if (c < 0) continue;
        while (chart[c] != c) c = chart[c];
        chart[f] = c;
    }
}

__global__ void __launch_bounds__(kBlock) chart_rect_kernel(const pmb200_texture_view *views, const float *xyz, const int *faces,
                                                            long long nf, const int *label, const int *chart, int *rect) {
    GRID_LOOP(f, nf) {
        const int l = label[f];
        if (l < 0) continue;
        const pmb200_texture_view &v = views[l];
        int *r = rect + 4 * (size_t)chart[f];
        for (int k = 0; k < 3; ++k) {
            const float *x = xyz + 3 * (size_t)faces[3 * f + k];
            double q[3];
            pmtex::project(v.P, x[0], x[1], x[2], q);
            atomicMin(r, pmtex::lo_pixel(q[0]));
            atomicMin(r + 1, pmtex::lo_pixel(q[1]));
            atomicMax(r + 2, pmtex::hi_pixel(q[0]));
            atomicMax(r + 3, pmtex::hi_pixel(q[1]));
        }
    }
}

__global__ void __launch_bounds__(kBlock) slot_flags_kernel(const int *label, const int *chart, long long nf, int *is_root, int *is_cell) {
    GRID_LOOP(f, nf) {
        is_root[f] = chart[f] == f ? 1 : 0;
        is_cell[f] = label[f] < 0 ? 1 : 0;
    }
}

// slot of each face (its chart's row, or n_charts + its rank among the untextured faces) and the chart table
__global__ void __launch_bounds__(kBlock) slots_kernel(const int *label, const int *chart, const int *rect, const int *root_rank,
                                                       const int *cell_rank, long long nf, int n_charts, int *slot_out,
                                                       int *charts_out) {
    GRID_LOOP(f, nf) {
        if (label[f] < 0) {
            slot_out[f] = n_charts + cell_rank[f];
            continue;
        }
        slot_out[f] = root_rank[chart[f]];
        if (chart[f] != f) continue;
        const int *r = rect + 4 * f;
        int *o = charts_out + 6 * (size_t)root_rank[f];
        const int x0 = r[0] - pmtex::kMargin, y0 = r[1] - pmtex::kMargin;
        o[0] = (int)f;
        o[1] = label[f];
        o[2] = x0;
        o[3] = y0;
        o[4] = r[2] + pmtex::kMargin - x0 + 1;
        o[5] = r[3] + pmtex::kMargin - y0 + 1;
    }
}

// ---- pages ----------------------------------------------------------------------------------------------------------------

// one thread per texel of the view's charts: rows[j] is a chart-table row, prefix its exclusive texel offsets
__global__ void __launch_bounds__(kBlock) fill_kernel(const float *image, int W, int H, const int *charts, const int *places,
                                                      const int *rows, const long long *prefix, int m, int S, unsigned char *pages) {
    const long long total = prefix[m];
    GRID_LOOP(t, total) {
        int lo = 0, hi = m - 1;  // the last j with prefix[j] <= t
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (prefix[mid] <= t) lo = mid; else hi = mid - 1;
        }
        const int *c = charts + 6 * (size_t)rows[lo];
        const int *pl = places + 3 * (size_t)rows[lo];
        const long long i = t - prefix[lo];
        const int dx = (int)(i % c[4]), dy = (int)(i / c[4]);
        const int px = min(max(c[2] + dx, 0), W - 1), py = min(max(c[3] + dy, 0), H - 1);
        unsigned char *dst = pages + 3 * (((size_t)pl[0] * S + pl[2] + dy) * S + pl[1] + dx);
        const size_t plane = (size_t)W * H, src = (size_t)py * W + px;
        for (int k = 0; k < 3; ++k) {
            const int b = __float2int_rn(__fmul_rn(255.0f, image[k * plane + src]));
            dst[k] = (unsigned char)(b < 0 ? 0 : (b > 255 ? 255 : b));
        }
    }
}

__global__ void __launch_bounds__(kBlock) uv_kernel(const pmb200_texture_view *views, const float *xyz, const unsigned char *rgb,
                                                    const int *faces, long long nf, const int *label, const int *slot,
                                                    const int *charts, const int *places, int S, float *uv_out, int *page_out,
                                                    unsigned char *pages) {
    GRID_LOOP(f, nf) {
        const int s = slot[f];
        const int *pl = places + 3 * (size_t)s;
        page_out[f] = pl[0];
        float *uv = uv_out + 6 * f;
        const int l = label[f];
        if (l >= 0) {
            const int *c = charts + 6 * (size_t)s;
            for (int k = 0; k < 3; ++k) {
                const float *x = xyz + 3 * (size_t)faces[3 * f + k];
                double q[3];
                pmtex::project(views[l].P, x[0], x[1], x[2], q);
                pmtex::corner_uv(q[0], q[1], c[2], c[3], pl[1], pl[2], S, uv + 2 * k);
            }
            continue;
        }
        float cu[2];
        pmtex::cell_uv(pl[1], pl[2], S, cu);
        for (int k = 0; k < 3; ++k) { uv[2 * k] = cu[0]; uv[2 * k + 1] = cu[1]; }
        const unsigned char *c0 = rgb ? rgb + 3 * (size_t)faces[3 * f] : nullptr;
        const unsigned char *c1 = rgb ? rgb + 3 * (size_t)faces[3 * f + 1] : nullptr;
        const unsigned char *c2 = rgb ? rgb + 3 * (size_t)faces[3 * f + 2] : nullptr;
        unsigned char col[3];
        for (int k = 0; k < 3; ++k) col[k] = pmtex::cell_colour(c0, c1, c2, k);
        for (int dy = 0; dy < pmtex::kCell; ++dy)
            for (int dx = 0; dx < pmtex::kCell; ++dx) {
                unsigned char *dst = pages + 3 * (((size_t)pl[0] * S + pl[2] + dy) * S + pl[1] + dx);
                dst[0] = col[0]; dst[1] = col[1]; dst[2] = col[2];
            }
    }
}

// ---- host -----------------------------------------------------------------------------------------------------------------

struct Layout {
    pmb200_texture_view *views;
    float4 *proj;
    unsigned long long *zbuf;
    int *large, *n_large, *covered, *visible;
    int *ent_face, *ent_count;
    unsigned long long *n_ent;
    long long *row_count, *row_off;
    int *cursor, *csr_view, *csr_count;
    int *lab_a, *lab_b;
    unsigned long long *key_in, *key;
    int *slot_in, *slot, *pos;
    int *chart, *rect, *root_rank, *cell_rank, *flag_a, *flag_b, *changed;
    void *cub;
    size_t cub_bytes;
};

bool cub_bytes(long long nf, size_t &out) {
    size_t b = 0;
    out = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int *)nullptr,
                                        (int *)nullptr, (int)(3 * nf)) != cudaSuccess)
        return false;
    out = std::max(out, b);
    if (cub::DeviceScan::ExclusiveSum(nullptr, b, (long long *)nullptr, (long long *)nullptr, (int)(nf + 1)) != cudaSuccess) return false;
    out = std::max(out, b);
    if (cub::DeviceScan::ExclusiveSum(nullptr, b, (int *)nullptr, (int *)nullptr, (int)nf) != cudaSuccess) return false;
    out = std::max(out, b);
    return true;
}

long long entry_capacity(const pmb200_texture_view *views, int n_views, long long nf) {
    long long cap = 0;
    for (int v = 0; v < n_views; ++v) cap += std::min(nf, (long long)views[v].width * views[v].height);
    return cap;
}

long long layout(char *base, long long nv, long long nf, const pmb200_texture_view *views, int n_views, size_t cubb, Layout &w) {
    size_t used = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + used : nullptr; used += align256(bytes); return (void *)p; };
    long long max_pix = 0;
    for (int v = 0; v < n_views; ++v) max_pix = std::max(max_pix, (long long)views[v].width * views[v].height);
    const long long cap = entry_capacity(views, n_views, nf);
    w.views = (pmb200_texture_view *)take(n_views * sizeof(pmb200_texture_view));
    w.proj = (float4 *)take(nv * sizeof(float4));
    w.zbuf = (unsigned long long *)take(max_pix * 8);
    w.large = (int *)take(nf * 4);
    w.n_large = (int *)take(4);
    w.covered = (int *)take(nf * 4);
    w.visible = (int *)take(nf * 4);
    w.ent_face = (int *)take(cap * 4);
    w.ent_count = (int *)take(cap * 4);
    w.n_ent = (unsigned long long *)take(8);
    w.row_count = (long long *)take((nf + 1) * 8);
    w.row_off = (long long *)take((nf + 1) * 8);
    w.cursor = (int *)take(nf * 4);
    w.csr_view = (int *)take(cap * 4);
    w.csr_count = (int *)take(cap * 4);
    w.lab_a = (int *)take(nf * 4);
    w.lab_b = (int *)take(nf * 4);
    w.key_in = (unsigned long long *)take(3 * nf * 8);
    w.key = (unsigned long long *)take(3 * nf * 8);
    w.slot_in = (int *)take(3 * nf * 4);
    w.slot = (int *)take(3 * nf * 4);
    w.pos = (int *)take(3 * nf * 4);
    w.chart = (int *)take(nf * 4);
    w.rect = (int *)take(4 * nf * 4);
    w.root_rank = (int *)take(nf * 4);
    w.cell_rank = (int *)take(nf * 4);
    w.flag_a = (int *)take(nf * 4);
    w.flag_b = (int *)take(nf * 4);
    w.changed = (int *)take(4);
    w.cub = take(cubb);
    w.cub_bytes = cubb;
    return (long long)used;
}

bool check_views(const pmb200_texture_view *views, int n_views) {
    if (!views || n_views < 1 || n_views > 65535) return false;
    for (int v = 0; v < n_views; ++v) {
        const pmb200_texture_view &x = views[v];
        if (x.width < 1 || x.height < 1 || x.width > kMaxSide || x.height > kMaxSide) return false;
        for (int k = 0; k < 12; ++k)
            if (!std::isfinite(x.P[k]) || !std::isfinite((float)x.P[k])) return false;
        for (int k = 0; k < 3; ++k)
            if (!std::isfinite(x.centre[k]) || !std::isfinite((float)x.centre[k])) return false;
        if (!(x.near_z > 0.0) || !((float)x.near_z > 0.0f) || !((float)x.near_z < INFINITY)) return false;
    }
    return true;
}

bool sizes_ok(long long nv, long long nf) { return nv >= 0 && nv < (1ll << 31) && nf >= 0 && nf < (1ll << 29); }

int read_back(void *host, const void *dev, size_t bytes, cudaStream_t st, const char *what) {
    if (cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status(what);
    return 0;
}

}  // namespace

extern "C" int64_t pmb200_texture_mesh_workspace_bytes(int64_t n_vertices, int64_t n_faces, const pmb200_texture_view *views_host,
                                                       int n_views) {
    if (!sizes_ok(n_vertices, n_faces) || !check_views(views_host, n_views))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_mesh_workspace_bytes: 0 <= nv < 2^31, 0 <= nf < 2^29, 1..65535 valid views");
    size_t cubb;
    if (!cub_bytes(n_faces, cubb))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_mesh_workspace_bytes: no CUDA device to size the CUB passes for");
    Layout w;
    return layout(nullptr, n_vertices, n_faces, views_host, n_views, cubb, w);
}

extern "C" int pmb200_texture_mesh(const float *xyz, int64_t n_vertices, const int *faces, int64_t n_faces,
                                   const pmb200_texture_view *views_host, int n_views, int *label_out, int *slot_out,
                                   int *charts_out, int64_t *counts_host, void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !label_out || !slot_out || !charts_out || !counts_host || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "texture_mesh: null pointer");
    if (!sizes_ok(n_vertices, n_faces) || !check_views(views_host, n_views))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_mesh: 0 <= nv < 2^31, 0 <= nf < 2^29, 1..65535 views of 1..16384 pixels a "
                                                   "side with finite cameras and near > 0");
    size_t cubb;
    if (!cub_bytes(n_faces, cubb)) return pmb200_internal_launch_status("texture_mesh (CUB sizes)");
    Layout w;
    if (workspace_bytes < layout(static_cast<char *>(workspace), n_vertices, n_faces, views_host, n_views, cubb, w))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_mesh: workspace smaller than texture_mesh_workspace_bytes(...)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long nv = n_vertices, nf = n_faces;
    counts_host[0] = counts_host[1] = counts_host[2] = 0;
    if (nf == 0) return 0;
    cudaMemcpyAsync(w.views, views_host, n_views * sizeof(pmb200_texture_view), cudaMemcpyHostToDevice, st);
    cudaMemsetAsync(w.row_count, 0, (nf + 1) * 8, st);
    cudaMemsetAsync(w.n_ent, 0, 8, st);
    std::vector<unsigned long long> seg(n_views + 1, 0);
    for (int v = 0; v < n_views; ++v) {
        const pmb200_texture_view &x = views_host[v];
        Camera c;
        for (int k = 0; k < 12; ++k) c.P[k] = (float)x.P[k];
        for (int k = 0; k < 3; ++k) { c.C[k] = (float)x.centre[k]; c.bg[k] = 0.0f; }
        c.W = x.width; c.H = x.height; c.near_z = (float)x.near_z; c.shade = 0;
        const long long npix = (long long)x.width * x.height;
        cudaMemsetAsync(w.zbuf, 0xff, npix * 8, st);
        cudaMemsetAsync(w.n_large, 0, 4, st);
        cudaMemsetAsync(w.visible, 0, nf * 4, st);
        if (nv > 0) project_kernel<<<grid_blocks(nv), kBlock, 0, st>>>(c, xyz, nv, w.proj);
        raster_small_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(c, w.proj, faces, nf, nv, w.zbuf, w.large, w.n_large, w.covered);
        raster_large_kernel<<<kLargeCtas, kBlock, 0, st>>>(c, w.proj, faces, nv, w.large, w.n_large, w.zbuf, w.covered);
        winners_kernel<<<grid_blocks(npix), kBlock, 0, st>>>(w.zbuf, npix, w.visible);
        candidates_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(x, xyz, faces, nf, w.covered, w.visible, w.ent_face, w.ent_count,
                                                               w.n_ent, w.row_count);
        if (int rc = read_back(&seg[v + 1], w.n_ent, 8, st, "texture_mesh (visibility)")) return rc;
    }
    const long long n_ent = (long long)seg[n_views];
    size_t bytes = w.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(w.cub, bytes, w.row_count, w.row_off, (int)(nf + 1), st) != cudaSuccess)
        return pmb200_internal_launch_status("texture_mesh (rows)");
    cudaMemsetAsync(w.cursor, 0, nf * 4, st);
    for (int v = 0; v < n_views; ++v) {
        const long long n = (long long)(seg[v + 1] - seg[v]);
        if (n > 0)
            scatter_kernel<<<grid_blocks(n), kBlock, 0, st>>>(w.ent_face + seg[v], w.ent_count + seg[v], n, v, w.row_off, w.cursor,
                                                              w.csr_view, w.csr_count);
    }
    // labels
    edge_keys_kernel<<<grid_blocks(3 * nf), kBlock, 0, st>>>(faces, nf, w.key_in, w.slot_in);
    bytes = w.cub_bytes;
    if (cub::DeviceRadixSort::SortPairs(w.cub, bytes, w.key_in, w.key, w.slot_in, w.slot, (int)(3 * nf), 0, 64, st) != cudaSuccess)
        return pmb200_internal_launch_status("texture_mesh (edge sort)");
    slot_pos_kernel<<<grid_blocks(3 * nf), kBlock, 0, st>>>(w.slot, 3 * nf, w.pos);
    init_labels_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(w.row_off, w.csr_view, w.csr_count, nf, w.lab_a);
    int *lab = w.lab_a, *other = w.lab_b;
    for (int r = 0; r < pmtex::kRounds; ++r) {
        smooth_labels_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(w.row_off, w.csr_view, w.csr_count, nf, w.key, w.slot, w.pos, lab, other);
        std::swap(lab, other);
    }
    // charts
    chart_init_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(lab, nf, w.chart, w.rect);
    for (;;) {
        int changed = 0;
        cudaMemsetAsync(w.changed, 0, 4, st);
        chart_hook_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(lab, nf, w.key, w.slot, w.pos, w.chart, w.changed);
        chart_jump_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(nf, w.chart);
        if (int rc = read_back(&changed, w.changed, 4, st, "texture_mesh (charts)")) return rc;
        if (!changed) break;
    }
    chart_rect_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(w.views, xyz, faces, nf, lab, w.chart, w.rect);
    slot_flags_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(lab, w.chart, nf, w.flag_a, w.flag_b);
    bytes = w.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(w.cub, bytes, w.flag_a, w.root_rank, (int)nf, st) != cudaSuccess)
        return pmb200_internal_launch_status("texture_mesh (chart ranks)");
    bytes = w.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(w.cub, bytes, w.flag_b, w.cell_rank, (int)nf, st) != cudaSuccess)
        return pmb200_internal_launch_status("texture_mesh (cell ranks)");
    int tail[4];
    if (int rc = read_back(tail, w.root_rank + nf - 1, 4, st, "texture_mesh (counts)")) return rc;
    if (int rc = read_back(tail + 1, w.flag_a + nf - 1, 4, st, "texture_mesh (counts)")) return rc;
    if (int rc = read_back(tail + 2, w.cell_rank + nf - 1, 4, st, "texture_mesh (counts)")) return rc;
    if (int rc = read_back(tail + 3, w.flag_b + nf - 1, 4, st, "texture_mesh (counts)")) return rc;
    const int n_charts = tail[0] + tail[1];
    slots_kernel<<<grid_blocks(nf), kBlock, 0, st>>>(lab, w.chart, w.rect, w.root_rank, w.cell_rank, nf, n_charts, slot_out, charts_out);
    cudaMemcpyAsync(label_out, lab, nf * 4, cudaMemcpyDeviceToDevice, st);
    counts_host[0] = n_ent;
    counts_host[1] = n_charts;
    counts_host[2] = tail[2] + tail[3];
    return pmb200_internal_launch_status("texture_mesh");
}

extern "C" int pmb200_texture_pack(const int *sizes_host, int64_t n_charts, int64_t n_cells, int *places_host, int *side_out,
                                   int *pages_out) {
    if ((!sizes_host && n_charts > 0) || (!places_host && n_charts + n_cells > 0) || !side_out || !pages_out)
        return pmb200_internal_fail(PMB200_EINVAL, "texture_pack: null pointer");
    if (n_charts < 0 || n_cells < 0 || n_charts + n_cells >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_pack: 0 <= n_charts, n_cells and n_charts + n_cells < 2^31");
    int largest = pmtex::kCell;
    for (long long i = 0; i < 2 * n_charts; ++i) {
        if (sizes_host[i] < 1) return pmb200_internal_fail(PMB200_EINVAL, "texture_pack: a rectangle side < 1");
        largest = std::max(largest, sizes_host[i]);
    }
    if (largest > pmtex::kMaxPage) return pmb200_internal_fail(PMB200_EINVAL, "texture_pack: a rectangle side > 16384");
    int S = pmtex::kMinPage;
    while (S < largest) S *= 2;
    std::vector<int> order(n_charts);
    for (long long i = 0; i < n_charts; ++i) order[i] = (int)i;
    std::sort(order.begin(), order.end(), [&](int a, int b) {
        const int ha = sizes_host[2 * a + 1], hb = sizes_host[2 * b + 1], wa = sizes_host[2 * a], wb = sizes_host[2 * b];
        if (ha != hb) return ha > hb;
        if (wa != wb) return wa > wb;
        return a < b;
    });
    int page = 0, x = 0, y = 0, shelf = 0;
    auto place = [&](long long i, int rw, int rh) {
        if (x + rw > S) { y += shelf; x = 0; shelf = 0; }
        if (y + rh > S) { ++page; x = 0; y = 0; shelf = 0; }
        places_host[3 * i] = page;
        places_host[3 * i + 1] = x;
        places_host[3 * i + 2] = y;
        x += rw;
        shelf = std::max(shelf, rh);
    };
    for (long long j = 0; j < n_charts; ++j) place(order[j], sizes_host[2 * order[j]], sizes_host[2 * order[j] + 1]);
    for (long long j = 0; j < n_cells; ++j) place(n_charts + j, pmtex::kCell, pmtex::kCell);
    *side_out = S;
    *pages_out = n_charts + n_cells > 0 ? page + 1 : 0;
    return 0;
}

extern "C" int64_t pmb200_texture_write_workspace_bytes(int n_views) {
    if (n_views < 1 || n_views > 65535) return pmb200_internal_fail(PMB200_EINVAL, "texture_write_workspace_bytes: 1..65535 views");
    return (int64_t)align256(n_views * sizeof(pmb200_texture_view));
}

extern "C" int pmb200_texture_write(int view, const float *image, int width, int height, const int *rows, const int64_t *prefix,
                                    int n_rows, const float *xyz, const unsigned char *rgb, int64_t n_vertices, const int *faces,
                                    int64_t n_faces, const pmb200_texture_view *views_host, int n_views, const int *label,
                                    const int *slot, const int *charts, const int *places, int side, int n_pages, float *uv_out,
                                    int *page_out, unsigned char *pages, void *workspace, int64_t workspace_bytes, void *stream) {
    if (!charts || !places || !pages || !workspace) return pmb200_internal_fail(PMB200_EINVAL, "texture_write: null pointer");
    if (side < pmtex::kMinPage || side > pmtex::kMaxPage || (side & (side - 1)) || n_pages < 1 || !sizes_ok(n_vertices, n_faces))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_write: a page side outside 4096..16384 or not a power of two, or bad sizes");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (view >= 0) {
        if (!image || !rows || !prefix || n_rows < 0 || width < 1 || height < 1 || width > kMaxSide || height > kMaxSide)
            return pmb200_internal_fail(PMB200_EINVAL, "texture_write: a view needs its image, size, rows and prefix");
        if (n_rows == 0) return 0;
        int64_t total;
        if (int rc = read_back(&total, prefix + n_rows, 8, st, "texture_write (texels)")) return rc;
        if (total > 0)
            fill_kernel<<<grid_blocks(total), kBlock, 0, st>>>(image, width, height, charts, places, rows, (const long long *)prefix,
                                                               n_rows, side, pages);
        return pmb200_internal_launch_status("texture_write (view)");
    }
    if (view != -1 || (!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !label || !slot || !uv_out || !page_out ||
        !check_views(views_host, n_views))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_write: view -1 needs the mesh, the labels and slots and valid views");
    if (workspace_bytes < pmb200_texture_write_workspace_bytes(n_views))
        return pmb200_internal_fail(PMB200_EINVAL, "texture_write: workspace smaller than texture_write_workspace_bytes(n_views)");
    if (n_faces == 0) return 0;
    pmb200_texture_view *views = static_cast<pmb200_texture_view *>(workspace);
    cudaMemcpyAsync(views, views_host, n_views * sizeof(pmb200_texture_view), cudaMemcpyHostToDevice, st);
    uv_kernel<<<grid_blocks(n_faces), kBlock, 0, st>>>(views, xyz, rgb, faces, n_faces, label, slot, charts, places, side, uv_out,
                                                       page_out, pages);
    return pmb200_internal_launch_status("texture_write (coordinates)");
}
