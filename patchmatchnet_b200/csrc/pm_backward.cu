// pm_backward.cu -- backward kernels of the learned-PatchMatch path (training configuration).
//
// Which gradients exist is dictated by the reference's graph (SURVEY.md 3.4):
//   * the warp grid is built under no_grad (models/module.py:147): K-A has gradients w.r.t. the source
//     features (bilinear scatter-add) and the reference feature only;
//   * depth_weight is detached (models/patchmatch.py:503,506,669), DepthInitialization detaches the
//     incoming depth (:74,:85): K-C only differentiates the propagated gathers w.r.t. the learned
//     propagation offsets, K-B differentiates w.r.t. the raw score, the hypotheses (regression), the
//     learned evaluation offsets (through the score gather only) and the feature weight;
//   * FeatureWeightNet sees a detached reference feature (:475): K-A' differentiates w.r.t. the offsets only.
// Layouts and argument meaning follow the forward entry points (include/patchmatch_b200.h).
#if !defined(PM_EMU)  // host emulation build (tests/warp_emu.h) brings its own CUDA vocabulary
#include <cuda_runtime.h>
#endif
#include <math.h>

#include "../../include/patchmatch_b200.h"
#include "pm_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

#if !defined(PM_EMU)
cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }
#endif

// ------------------------------------------------------------------------------------------
// bilinear footprints with the quantities a backward pass needs
// ------------------------------------------------------------------------------------------

struct BorderTap {
    int r0, dx, dy;       // texels r0, r0+dx, r0+dy*cols, r0+dy*cols+dx
    float fx, fy;         // fractional position inside the cell
    float gmx, gmy;       // d(ix)/d(px), d(iy)/d(py): size/(size-1) inside the map, 0 once clamped (ATen grid_sampler)
};

__device__ __forceinline__ BorderTap border_tap(float px, float py, int rows, int cols) {
    const float gx = px / ((float)(cols - 1) * 0.5f) - 1.0f;
    const float gy = py / ((float)(rows - 1) * 0.5f) - 1.0f;
    float ix = ((gx + 1.0f) * (float)cols - 1.0f) * 0.5f;
    float iy = ((gy + 1.0f) * (float)rows - 1.0f) * 0.5f;
    BorderTap t;
    // clip_coordinates_set_grad: zero gradient at or beyond either border
    t.gmx = (ix <= 0.0f || ix >= (float)(cols - 1)) ? 0.0f : (float)cols / (float)(cols - 1);
    t.gmy = (iy <= 0.0f || iy >= (float)(rows - 1)) ? 0.0f : (float)rows / (float)(rows - 1);
    ix = fminf((float)(cols - 1), fmaxf(ix, 0.0f));
    iy = fminf((float)(rows - 1), fmaxf(iy, 0.0f));
    const float xf = floorf(ix), yf = floorf(iy);
    t.fx = ix - xf;
    t.fy = iy - yf;
    const int x0 = (int)xf, y0 = (int)yf;
    t.dx = (x0 + 1 <= cols - 1) ? 1 : 0;
    t.dy = (y0 + 1 <= rows - 1) ? 1 : 0;
    t.r0 = y0 * cols + x0;
    return t;
}

// d(bilinear)/d(ix), d(bilinear)/d(iy) from the four tap values (taps outside the map never carry weight
// when the gradient multiplier is non-zero, see border_tap)
__device__ __forceinline__ void bilinear_grad(const BorderTap &t, float v00, float v01, float v10, float v11,
                                              float *gix, float *giy) {
    *gix = (v01 - v00) * (1.0f - t.fy) + (v11 - v10) * t.fy;
    *giy = (v10 - v00) * (1.0f - t.fx) + (v11 - v01) * t.fx;
}

// ------------------------------------------------------------------------------------------
// K-A backward
// ------------------------------------------------------------------------------------------

struct WarpCorrBwdParams {
    const float *ref, *src, *rt, *depth, *vw, *gout;
    float *dref, *dsrc;
    int V, B, H, W, Hs, Ws, D;
    float sx, sy;
};

template <int C, int G>
struct BwdMap {
    static constexpr int CPL = 8;
    static constexpr int LPP = C / CPL;
    static constexpr int PPW = 32 / LPP;
    static constexpr int CPG = C / G;
    static constexpr int GPL = CPL / CPG;
};

// Per-view source extents of a ragged source pack (pmb200_warp_corr_views_backward): view v, batch b starts at float
// base[v] + b * hs[v] * ws[v] * C of p.src (and of p.dsrc); sx / sy are that view's align_corners=True scales.  A kernel
// parameter of its own, so that the uniform instantiations keep the parameter block (and the code) they always had.
struct BwdViewTable {
    long long base[PMB200_MAX_VIEWS];
    int hs[PMB200_MAX_VIEWS], ws[PMB200_MAX_VIEWS];
    float sx[PMB200_MAX_VIEWS], sy[PMB200_MAX_VIEWS];
};

// One lane group (C/8 lanes) per reference pixel, all hypotheses and all views in the group.
// d_ref is owned by the group (plain stores); d_src is scattered with 128-bit vector atomics, accumulated
// in registers while consecutive hypotheses stay in the same source cell.
// VIEWS = false: one (Hs, Ws) for every source view, read from p (vt is null).  VIEWS = true: view v's extent, base and
// scales come from vt.
template <int C, int G, bool VIEWS>
__device__ __forceinline__ void warp_corr_backward_body(const WarpCorrBwdParams &p, const BwdViewTable *vt) {
    using M = BwdMap<C, G>;
    constexpr int V4 = C / 4;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int HW = p.H * p.W;
    const int b = blockIdx.y;
    const int grp = lane / M::LPP, li = lane % M::LPP;
    const int n = warp * M::PPW + grp;
    if (n >= HW) return;
    const float x = (float)(n % p.W), y = (float)(n / p.W);
    const int g0 = li * M::GPL;
    constexpr float inv_cpg = 1.0f / (float)M::CPG;

    float r[8], dref[8];
    {
        const float4 *rp = reinterpret_cast<const float4 *>(p.ref + ((size_t)b * HW + n) * C) + li * 2;
        const float4 q0 = __ldg(rp), q1 = __ldg(rp + 1);
        r[0] = q0.x; r[1] = q0.y; r[2] = q0.z; r[3] = q0.w;
        r[4] = q1.x; r[5] = q1.y; r[6] = q1.z; r[7] = q1.w;
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) dref[c] = 0.0f;

    float wsum = 1e-5f;
    if (p.vw)
        for (int v = 0; v < p.V; ++v) wsum += __ldg(p.vw + ((size_t)b * p.V + v) * HW + n);

    for (int v = 0; v < p.V; ++v) {
        float rt[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) rt[i] = __ldg(p.rt + ((size_t)v * p.B + b) * 12 + i);
        const pm::Ray ray = pm::pixel_ray(rt, x, y);
        const float vscale = p.vw ? __ldg(p.vw + ((size_t)b * p.V + v) * HW + n) / wsum : 1.0f;
        const int Hs = VIEWS ? vt->hs[v] : p.Hs, Ws = VIEWS ? vt->ws[v] : p.Ws;
        const float sx = VIEWS ? vt->sx[v] : p.sx, sy = VIEWS ? vt->sy[v] : p.sy;
        const size_t vbase = VIEWS ? (size_t)vt->base[v] + (size_t)b * Hs * Ws * C : ((size_t)v * p.B + b) * Hs * Ws * C;
        const float4 *sv = reinterpret_cast<const float4 *>(p.src + vbase) + li * 2;
        float4 *dv = reinterpret_cast<float4 *>(p.dsrc + vbase) + li * 2;

        int pkey = pm::kKeyNone;
        float ta[4][8], tg[4][8];
#pragma unroll
        for (int t = 0; t < 4; ++t)
#pragma unroll
            for (int c = 0; c < 8; ++c) { ta[t][c] = 0.0f; tg[t][c] = 0.0f; }

        auto flush = [&](int key) {
            const int r0 = pm::cell_r0(key), dx = pm::cell_dx(key), dy = pm::cell_dy(key);
            float4 *t0 = dv + (size_t)r0 * V4;
            float4 *tp[4] = {t0, t0 + dx * V4, t0 + (size_t)dy * Ws * V4, t0 + (size_t)dy * Ws * V4 + dx * V4};
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                atomicAdd(tp[t], make_float4(tg[t][0], tg[t][1], tg[t][2], tg[t][3]));
                atomicAdd(tp[t] + 1, make_float4(tg[t][4], tg[t][5], tg[t][6], tg[t][7]));
            }
        };

        for (int d = 0; d < p.D; ++d) {
            const float dep = __ldg(p.depth + ((size_t)b * p.D + d) * HW + n);
            float uu, vv;
            pm::project(ray, rt, dep, p.W, p.H, sx, sy, &uu, &vv);
            const pm::Cell c = pm::zero_pad_cell(uu, vv, Hs, Ws);
            if (c.key == pm::kKeyNone) continue;
            float gs[M::GPL];
#pragma unroll
            for (int g = 0; g < M::GPL; ++g) {
                const size_t o = p.vw ? (((size_t)b * G + g0 + g) * p.D + d) * HW + n
                                      : ((((size_t)v * p.B + b) * G + g0 + g) * p.D + d) * HW + n;
                gs[g] = __ldg(p.gout + o) * vscale * inv_cpg;
            }
            if (c.key != pkey) {
                if (pkey != pm::kKeyNone) flush(pkey);
                const int r0 = pm::cell_r0(c.key), dx = pm::cell_dx(c.key), dy = pm::cell_dy(c.key);
                const float4 *t0 = sv + (size_t)r0 * V4;
                const float4 *tq[4] = {t0, t0 + dx * V4, t0 + (size_t)dy * Ws * V4, t0 + (size_t)dy * Ws * V4 + dx * V4};
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const float4 a = __ldg(tq[t]), bq = __ldg(tq[t] + 1);
                    ta[t][0] = a.x; ta[t][1] = a.y; ta[t][2] = a.z; ta[t][3] = a.w;
                    ta[t][4] = bq.x; ta[t][5] = bq.y; ta[t][6] = bq.z; ta[t][7] = bq.w;
#pragma unroll
                    for (int q = 0; q < 8; ++q) tg[t][q] = 0.0f;
                }
                pkey = c.key;
            }
            const float w[4] = {c.w00, c.w01, c.w10, c.w11};
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float g = gs[q / M::CPG];
                const float warped = w[0] * ta[0][q] + w[1] * ta[1][q] + w[2] * ta[2][q] + w[3] * ta[3][q];
                dref[q] = fmaf(g, warped, dref[q]);
                const float gr = g * r[q];
#pragma unroll
                for (int t = 0; t < 4; ++t) tg[t][q] = fmaf(gr, w[t], tg[t][q]);
            }
        }
        if (pkey != pm::kKeyNone) flush(pkey);
    }
    float4 *dp = reinterpret_cast<float4 *>(p.dref + ((size_t)b * HW + n) * C) + li * 2;
    dp[0] = make_float4(dref[0], dref[1], dref[2], dref[3]);
    dp[1] = make_float4(dref[4], dref[5], dref[6], dref[7]);
}

template <int C, int G>
__global__ void __launch_bounds__(128) warp_corr_backward_kernel(const WarpCorrBwdParams p) {
    warp_corr_backward_body<C, G, false>(p, nullptr);
}

// per-view source extents (pmb200_warp_corr_views_backward)
template <int C, int G>
__global__ void __launch_bounds__(128) warp_corr_backward_views_kernel(const WarpCorrBwdParams p, const BwdViewTable vt) {
    warp_corr_backward_body<C, G, true>(p, &vt);
}

// ------------------------------------------------------------------------------------------
// aggregate_views backward (first stage-3 iteration: the weights come from PixelwiseNet and carry gradient)
// ------------------------------------------------------------------------------------------

__global__ void aggregate_views_backward_kernel(const float *__restrict__ sims, const float *__restrict__ vw,
                                                const float *__restrict__ gout, float *__restrict__ dsims,
                                                float *__restrict__ dvw, int V, int B, int GD, int HW) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HW) return;
    float w[PMB200_MAX_VIEWS], dw[PMB200_MAX_VIEWS];
    float wsum = 1e-5f;
    for (int v = 0; v < V; ++v) {
        w[v] = __ldg(vw + ((size_t)b * V + v) * HW + n);
        wsum += w[v];
        dw[v] = 0.0f;
    }
    const size_t vstride = (size_t)B * GD * HW;
    for (int k = 0; k < GD; ++k) {
        const size_t o = ((size_t)b * GD + k) * HW + n;
        const float g = __ldg(gout + o);
        float S = 0.0f;
        for (int v = 0; v < V; ++v) S = fmaf(__ldg(sims + v * vstride + o), w[v], S);
        S /= wsum;
        for (int v = 0; v < V; ++v) {
            const float sv = __ldg(sims + v * vstride + o);
            dsims[v * vstride + o] = g * w[v] / wsum;
            dw[v] = fmaf(g, (sv - S) / wsum, dw[v]);
        }
    }
    for (int v = 0; v < V; ++v) dvw[((size_t)b * V + v) * HW + n] = dw[v];
}

// ------------------------------------------------------------------------------------------
// K-A' backward: gradient of the neighbour self-correlation w.r.t. the learned evaluation offsets
// ------------------------------------------------------------------------------------------

struct OffsetCorrBwdParams {
    const float *ref, *offsets, *gout;
    float *doff;
    int B, H, W, K, dilation;
};

template <int C, int G>
__global__ void __launch_bounds__(128) offset_corr_backward_kernel(const OffsetCorrBwdParams p) {
    using M = BwdMap<C, G>;
    constexpr int V4 = C / 4;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int HW = p.H * p.W;
    const int b = blockIdx.y;
    const int grp = lane / M::LPP, li = lane % M::LPP;
    const int n = warp * M::PPW + grp;
    const bool live = n < HW;
    const int nc = live ? n : HW - 1;
    const int g0 = li * M::GPL;
    constexpr float inv_cpg = 1.0f / (float)M::CPG;
    float r[8];
    {
        const float4 *rp = reinterpret_cast<const float4 *>(p.ref + ((size_t)b * HW + nc) * C) + li * 2;
        const float4 q0 = __ldg(rp), q1 = __ldg(rp + 1);
        r[0] = q0.x; r[1] = q0.y; r[2] = q0.z; r[3] = q0.w;
        r[4] = q1.x; r[5] = q1.y; r[6] = q1.z; r[7] = q1.w;
    }
    const float4 *sv = reinterpret_cast<const float4 *>(p.ref + (size_t)b * HW * C) + li * 2;
    for (int k = 0; k < p.K; ++k) {
        int dy = 0, dx = 0;
        pm::neighbour_offset(true, p.K, p.dilation, k, &dy, &dx);
        const float ox = (float)dx + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k) * HW + nc);
        const float oy = (float)dy + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k + 1) * HW + nc);
        const BorderTap t = border_tap((float)(nc % p.W) + ox, (float)(nc / p.W) + oy, p.H, p.W);
        const float4 *t0 = sv + (size_t)t.r0 * V4;
        const float4 *tq[4] = {t0, t0 + t.dx * V4, t0 + (size_t)t.dy * p.W * V4, t0 + (size_t)t.dy * p.W * V4 + t.dx * V4};
        float ta[4][8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float4 a = __ldg(tq[q]), bq = __ldg(tq[q] + 1);
            ta[q][0] = a.x; ta[q][1] = a.y; ta[q][2] = a.z; ta[q][3] = a.w;
            ta[q][4] = bq.x; ta[q][5] = bq.y; ta[q][6] = bq.z; ta[q][7] = bq.w;
        }
        float gx = 0.0f, gy = 0.0f;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float g = __ldg(p.gout + (((size_t)b * G + g0 + q / M::CPG) * p.K + k) * HW + nc) * inv_cpg * r[q];
            float gix, giy;
            bilinear_grad(t, ta[0][q], ta[1][q], ta[2][q], ta[3][q], &gix, &giy);
            gx = fmaf(g, gix, gx);
            gy = fmaf(g, giy, gy);
        }
#pragma unroll
        for (int off = 1; off < M::LPP; off <<= 1) {
            gx += __shfl_xor_sync(0xffffffffu, gx, off);
            gy += __shfl_xor_sync(0xffffffffu, gy, off);
        }
        if (li == 0 && live) {
            p.doff[((size_t)b * 2 * p.K + 2 * k) * HW + n] = gx * t.gmx;
            p.doff[((size_t)b * 2 * p.K + 2 * k + 1) * HW + n] = gy * t.gmy;
        }
    }
}

// ------------------------------------------------------------------------------------------
// K-C backward: gradient of the sorted hypotheses w.r.t. the learned propagation offsets
// ------------------------------------------------------------------------------------------

struct PropBwdParams {
    const float *seed, *offsets, *dmin, *dmax, *gout;
    float *doff;
    int mode, B, H, W, Ns, Kp, dilation;
    float interval_scale;
};

__device__ __forceinline__ float centre_value(const PropBwdParams &p, int b, int q, int HW, float inv_min, float inv_max) {
    if (p.mode == 0) return pm::random_hypothesis(__ldg(p.seed + ((size_t)b * 48 + 24) * HW + q), 24, inv_min, inv_max);
    const float d = __ldg(p.seed + (size_t)b * HW + q);
    if (p.mode == 1) return pm::perturbed_hypothesis(d, pm::floor_div2_neg(p.Ns) + p.Ns / 2, inv_min, inv_max, p.interval_scale);
    return d;
}

__device__ __forceinline__ float own_value(const PropBwdParams &p, int b, int n, int k, int HW, float inv_min, float inv_max) {
    if (p.mode == 0) return pm::random_hypothesis(__ldg(p.seed + ((size_t)b * 48 + k) * HW + n), k, inv_min, inv_max);
    const float d = __ldg(p.seed + (size_t)b * HW + n);
    if (p.mode == 1) return pm::perturbed_hypothesis(d, pm::floor_div2_neg(p.Ns) + k, inv_min, inv_max, p.interval_scale);
    return d;
}

// One thread per pixel (training path; D <= PMB200_MAX_HYPOTHESES): recompute the hypotheses, find where the
// sort put every propagated one (rank = number of smaller values, ties broken by slot as a stable sort would),
// and push the incoming gradient through the bilinear gather of the centre hypothesis map.
__global__ void init_propagate_backward_kernel(const PropBwdParams p) {
    const int HW = p.H * p.W;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HW) return;
    const float inv_min = 1.0f / __ldg(p.dmin + b), inv_max = 1.0f / __ldg(p.dmax + b);
    const int D = p.Ns + p.Kp;
    const float x = (float)(n % p.W), y = (float)(n / p.W);
    for (int kk = 0; kk < p.Kp; ++kk) {
        int dy = 0, dx = 0;
        pm::neighbour_offset(false, p.Kp, p.dilation, kk, &dy, &dx);
        const float ox = (float)dx + __ldg(p.offsets + ((size_t)b * 2 * p.Kp + 2 * kk) * HW + n);
        const float oy = (float)dy + __ldg(p.offsets + ((size_t)b * 2 * p.Kp + 2 * kk + 1) * HW + n);
        const BorderTap t = border_tap(x + ox, y + oy, p.H, p.W);
        const float v00 = centre_value(p, b, t.r0, HW, inv_min, inv_max);
        const float v01 = centre_value(p, b, t.r0 + t.dx, HW, inv_min, inv_max);
        const float v10 = centre_value(p, b, t.r0 + t.dy * p.W, HW, inv_min, inv_max);
        const float v11 = centre_value(p, b, t.r0 + t.dy * p.W + t.dx, HW, inv_min, inv_max);
        const float hx = 1.0f - t.fx, hy = 1.0f - t.fy;
        float val = v00 * (hx * hy);
        val = fmaf(v01, t.dx ? t.fx * hy : 0.0f, val);
        val = fmaf(v10, t.dy ? hx * t.fy : 0.0f, val);
        val = fmaf(v11, (t.dx && t.dy) ? t.fx * t.fy : 0.0f, val);
        // rank of this propagated hypothesis among all Ns + Kp (stable order: own samples first, then neighbours)
        int rank = 0;
        for (int k = 0; k < p.Ns; ++k) rank += own_value(p, b, n, k, HW, inv_min, inv_max) <= val ? 1 : 0;
        for (int k2 = 0; k2 < p.Kp; ++k2) {
            if (k2 == kk) continue;
            int dy2 = 0, dx2 = 0;
            pm::neighbour_offset(false, p.Kp, p.dilation, k2, &dy2, &dx2);
            const float ox2 = (float)dx2 + __ldg(p.offsets + ((size_t)b * 2 * p.Kp + 2 * k2) * HW + n);
            const float oy2 = (float)dy2 + __ldg(p.offsets + ((size_t)b * 2 * p.Kp + 2 * k2 + 1) * HW + n);
            const pm::Cell c2 = pm::border_cell(x + ox2, y + oy2, p.H, p.W);
            const int r0 = pm::cell_r0(c2.key), ddx = pm::cell_dx(c2.key), ddy = pm::cell_dy(c2.key);
            float o = centre_value(p, b, r0, HW, inv_min, inv_max) * c2.w00;
            o = fmaf(centre_value(p, b, r0 + ddx, HW, inv_min, inv_max), c2.w01, o);
            o = fmaf(centre_value(p, b, r0 + ddy * p.W, HW, inv_min, inv_max), c2.w10, o);
            o = fmaf(centre_value(p, b, r0 + ddy * p.W + ddx, HW, inv_min, inv_max), c2.w11, o);
            rank += (o < val || (o == val && k2 < kk)) ? 1 : 0;
        }
        const float g = __ldg(p.gout + ((size_t)b * D + rank) * HW + n);
        float gix, giy;
        bilinear_grad(t, v00, v01, v10, v11, &gix, &giy);
        p.doff[((size_t)b * 2 * p.Kp + 2 * kk) * HW + n] = g * gix * t.gmx;
        p.doff[((size_t)b * 2 * p.Kp + 2 * kk + 1) * HW + n] = g * giy * t.gmy;
    }
}

// ------------------------------------------------------------------------------------------
// K-B backward
// ------------------------------------------------------------------------------------------

struct EvalBwdParams {
    const float *score0, *depth, *xnorm, *offsets, *fw, *dmin, *dmax, *prob, *gdepth, *gprob;
    float *dscore0, *dhyp, *doff, *dfw;
    int B, D, H, W, K, dilation, is_inverse;
    float interval_scale;
};

// One thread per pixel.  d_score0 is scattered with atomics (zero-initialised by the caller); d_hyp, d_offsets
// and d_fw are owned by the pixel.
__global__ void adaptive_eval_backward_kernel(const EvalBwdParams p) {
    const int HW = p.H * p.W;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HW) return;
    const float inv_min = 1.0f / __ldg(p.dmin + b), inv_max = 1.0f / __ldg(p.dmax + b);
    const float x = (float)(n % p.W), y = (float)(n / p.W);
    const float gd = p.gdepth ? __ldg(p.gdepth + (size_t)b * HW + n) : 0.0f;
    const size_t base = (size_t)b * p.D * HW + n;

    // regression: d(depth)/d(prob_d), d(depth)/d(hyp_d)
    float idx = 0.0f, inv_lo = 0.0f, inv_hi = 0.0f, depth_out = 0.0f;
    if (p.is_inverse) {
        for (int d = 0; d < p.D; ++d) idx = fmaf((float)d, __ldg(p.prob + base + (size_t)d * HW), idx);
        inv_hi = 1.0f / __ldg(p.depth + base + (size_t)(p.D - 1) * HW);
        inv_lo = 1.0f / __ldg(p.depth + base);
        depth_out = 1.0f / (inv_lo + idx / (float)(p.D - 1) * (inv_hi - inv_lo));
    }
    float dot = 0.0f;  // sum_j gp_j * prob_j
    for (int d = 0; d < p.D; ++d) {
        const float pr = __ldg(p.prob + base + (size_t)d * HW);
        const float hy = __ldg(p.depth + base + (size_t)d * HW);
        float gp = p.gprob ? __ldg(p.gprob + base + (size_t)d * HW) : 0.0f;
        float dh;
        if (p.is_inverse) {
            const float didx = -depth_out * depth_out * (inv_hi - inv_lo) / (float)(p.D - 1);
            gp += gd * didx * (float)d;
            dh = 0.0f;
            if (d == 0) dh += gd * depth_out * depth_out * (1.0f - idx / (float)(p.D - 1)) / (hy * hy);
            if (d == p.D - 1) dh += gd * depth_out * depth_out * (idx / (float)(p.D - 1)) / (hy * hy);
        } else {
            gp += gd * hy;
            dh = gd * pr;
        }
        p.dhyp[base + (size_t)d * HW] = dh;
        dot = fmaf(gp, pr, dot);
    }

    float doffx[PMB200_MAX_NEIGHBORS], doffy[PMB200_MAX_NEIGHBORS], dfw[PMB200_MAX_NEIGHBORS];
    for (int k = 0; k < p.K; ++k) { doffx[k] = 0.0f; doffy[k] = 0.0f; dfw[k] = 0.0f; }

    for (int d = 0; d < p.D; ++d) {
        const float pr = __ldg(p.prob + base + (size_t)d * HW);
        const float hy = __ldg(p.depth + base + (size_t)d * HW);
        float gp = p.gprob ? __ldg(p.gprob + base + (size_t)d * HW) : 0.0f;
        if (p.is_inverse) gp += gd * (-depth_out * depth_out * (inv_hi - inv_lo) / (float)(p.D - 1)) * (float)d;
        else gp += gd * hy;
        const float ds = pr * (gp - dot);  // gradient w.r.t. the aggregated score of this hypothesis
        const float *smap = p.score0 + ((size_t)b * p.D + d) * HW;
        const float *dmap = p.depth + ((size_t)b * p.D + d) * HW;
        const float *xmap = p.xnorm ? p.xnorm + ((size_t)b * p.D + d) * HW : nullptr;
        float *gsmap = p.dscore0 + ((size_t)b * p.D + d) * HW;
        const float xc = xmap ? __ldg(xmap + n) : pm::normalised_inverse_depth(__ldg(dmap + n), inv_min, inv_max);
        // first pass over the neighbours: weights and the aggregated score
        float num = 0.0f, den = 0.0f;
        for (int k = 0; k < p.K; ++k) {
            int dy = 0, dx = 0;
            pm::neighbour_offset(true, p.K, p.dilation, k, &dy, &dx);
            const float ox = (float)dx + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k) * HW + n);
            const float oy = (float)dy + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k + 1) * HW + n);
            const pm::Cell c = pm::border_cell(x + ox, y + oy, p.H, p.W);
            const int r0 = pm::cell_r0(c.key), ddx = pm::cell_dx(c.key), ddy = pm::cell_dy(c.key);
            const int r1 = r0 + ddx, r2 = r0 + ddy * p.W, r3 = r2 + ddx;
            auto xn_at = [&](int q) { return xmap ? __ldg(xmap + q) : pm::normalised_inverse_depth(__ldg(dmap + q), inv_min, inv_max); };
            const float xn = fmaf(xn_at(r3), c.w11, fmaf(xn_at(r2), c.w10, fmaf(xn_at(r1), c.w01, xn_at(r0) * c.w00)));
            const float sn = fmaf(__ldg(smap + r3), c.w11, fmaf(__ldg(smap + r2), c.w10, fmaf(__ldg(smap + r1), c.w01, __ldg(smap + r0) * c.w00)));
            const float wk = pm::depth_similarity(xc, xn, p.interval_scale) * __ldg(p.fw + ((size_t)b * p.K + k) * HW + n);
            num = fmaf(sn, wk, num);
            den += wk;
        }
        const float s = num / den;
        // second pass: distribute ds
        for (int k = 0; k < p.K; ++k) {
            int dy = 0, dx = 0;
            pm::neighbour_offset(true, p.K, p.dilation, k, &dy, &dx);
            const float ox = (float)dx + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k) * HW + n);
            const float oy = (float)dy + __ldg(p.offsets + ((size_t)b * 2 * p.K + 2 * k + 1) * HW + n);
            const BorderTap t = border_tap(x + ox, y + oy, p.H, p.W);
            const int r0 = t.r0, r1 = r0 + t.dx, r2 = r0 + t.dy * p.W, r3 = r2 + t.dx;
            const float hx = 1.0f - t.fx, hyw = 1.0f - t.fy;
            const float w00 = hx * hyw, w01 = t.dx ? t.fx * hyw : 0.0f, w10 = t.dy ? hx * t.fy : 0.0f,
                        w11 = (t.dx && t.dy) ? t.fx * t.fy : 0.0f;
            auto xn_at = [&](int q) { return xmap ? __ldg(xmap + q) : pm::normalised_inverse_depth(__ldg(dmap + q), inv_min, inv_max); };
            const float xn = fmaf(xn_at(r3), w11, fmaf(xn_at(r2), w10, fmaf(xn_at(r1), w01, xn_at(r0) * w00)));
            const float s00 = __ldg(smap + r0), s01 = __ldg(smap + r1), s10 = __ldg(smap + r2), s11 = __ldg(smap + r3);
            const float sn = fmaf(s11, w11, fmaf(s10, w10, fmaf(s01, w01, s00 * w00)));
            const float dwk = pm::depth_similarity(xc, xn, p.interval_scale);
            const float fwk = __ldg(p.fw + ((size_t)b * p.K + k) * HW + n);
            const float dsn = ds * dwk * fwk / den;  // d L / d (gathered score of neighbour k)
            atomicAdd(gsmap + r0, dsn * w00);
            if (w01 != 0.0f) atomicAdd(gsmap + r1, dsn * w01);
            if (w10 != 0.0f) atomicAdd(gsmap + r2, dsn * w10);
            if (w11 != 0.0f) atomicAdd(gsmap + r3, dsn * w11);
            float gix, giy;
            bilinear_grad(t, s00, s01, s10, s11, &gix, &giy);
            doffx[k] = fmaf(dsn, gix * t.gmx, doffx[k]);
            doffy[k] = fmaf(dsn, giy * t.gmy, doffy[k]);
            dfw[k] = fmaf(ds, dwk * (sn - s) / den, dfw[k]);
        }
    }
    for (int k = 0; k < p.K; ++k) {
        p.doff[((size_t)b * 2 * p.K + 2 * k) * HW + n] = doffx[k];
        p.doff[((size_t)b * 2 * p.K + 2 * k + 1) * HW + n] = doffy[k];
        p.dfw[((size_t)b * p.K + k) * HW + n] = dfw[k];
    }
}

}  // namespace

#if !defined(PM_EMU)  // the emulation build stops here: the launchers below need the CUDA runtime
// ==========================================================================================
// C ABI
// ==========================================================================================

extern "C" {

int pmb200_warp_corr_backward(const float *ref_nhwc, const float *src_nhwc, const float *rt, const float *depth,
                              const float *view_weights, const float *grad_out, float *d_ref_nhwc, float *d_src_nhwc,
                              int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D, void *stream) {
    if (!ref_nhwc || !src_nhwc || !rt || !depth || !grad_out || !d_ref_nhwc || !d_src_nhwc)
        return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_backward: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || H < 1 || W < 1 || Hs < 1 || Ws < 1 || D < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_backward: bad size");
    // every check runs before anything is written: the tap keys hold a 29-bit texel index (pm::Cell)
    if ((long long)Hs * Ws >= (1LL << pm::kKeyDxShift))
        return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_backward: source map too large");
    if (!((C == 64 && G == 8) || (C == 32 && G == 8) || (C == 16 && G == 4)))
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "warp_corr_backward: (C,G) must be (64,8), (32,8) or (16,4)");
    WarpCorrBwdParams p;
    p.ref = ref_nhwc; p.src = src_nhwc; p.rt = rt; p.depth = depth; p.vw = view_weights; p.gout = grad_out;
    p.dref = d_ref_nhwc; p.dsrc = d_src_nhwc;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = Hs; p.Ws = Ws; p.D = D;
    p.sx = (W > 1) ? (float)(Ws - 1) / (float)(W - 1) : 1.0f;
    p.sy = (H > 1) ? (float)(Hs - 1) / (float)(H - 1) : 1.0f;
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(d_src_nhwc, 0, (size_t)V * B * Hs * Ws * C * sizeof(float), st);
    if (e != cudaSuccess) return pmb200_internal_fail((int)e, "warp_corr_backward: memset failed");
    const int HW = H * W;
#define PMB200_LAUNCH_WB(CC, GG)                                                         \
    do {                                                                                 \
        const int pix_per_block = 4 * BwdMap<CC, GG>::PPW;                               \
        dim3 grid((HW + pix_per_block - 1) / pix_per_block, B);                          \
        warp_corr_backward_kernel<CC, GG><<<grid, 128, 0, st>>>(p);                      \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_WB(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_WB(32, 8);
    else PMB200_LAUNCH_WB(16, 4);
#undef PMB200_LAUNCH_WB
    return pmb200_internal_launch_status("warp_corr_backward");
}

int pmb200_warp_corr_views_backward(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                    const float *rt, const float *depth, const float *view_weights, const float *grad_out,
                                    float *d_ref_nhwc, float *d_src_flat, int V, int B, int C, int G, int H, int W, int D,
                                    void *stream) {
    if (!ref_nhwc || !src_flat || !views_host || !rt || !depth || !grad_out || !d_ref_nhwc || !d_src_flat)
        return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || H < 1 || W < 1 || D < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: bad size");
    if (!((C == 64 && G == 8) || (C == 32 && G == 8) || (C == 16 && G == 4)))
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "warp_corr_views_backward: (C,G) must be (64,8), (32,8) or (16,4)");
    // every check runs before anything is written: a rejected call leaves d_ref / d_src untouched
    BwdViewTable vt;
    long long end = 0;  // floats of the pack: the zero fill covers every view and the padding between views
    for (int v = 0; v < V; ++v) {
        const pmb200_view_extent &e = views_host[v];
        if (e.height < 1 || e.width < 1)
            return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: a view has a non-positive size");
        if ((long long)e.height * e.width >= (1LL << pm::kKeyDxShift))
            return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: source map too large");
        if (e.offset < 0 || e.offset % 4 != 0)
            return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: offsets must be non-negative multiples of 4 floats");
        const long long view_end = e.offset + (long long)B * e.height * e.width * C;
        if (e.offset / 4 >= (1LL << 31) || view_end / 4 >= (1LL << 31))
            return pmb200_internal_fail(PMB200_EINVAL, "warp_corr_views_backward: source pack too large (2^31 float4 elements)");
        end = view_end > end ? view_end : end;
        vt.base[v] = e.offset;
        vt.hs[v] = e.height;
        vt.ws[v] = e.width;
        // F.grid_sample(align_corners=True) maps the normalised coordinate onto each source's own extent
        vt.sx[v] = (W > 1) ? (float)(e.width - 1) / (float)(W - 1) : 1.0f;
        vt.sy[v] = (H > 1) ? (float)(e.height - 1) / (float)(H - 1) : 1.0f;
    }
    WarpCorrBwdParams p;
    p.ref = ref_nhwc; p.src = src_flat; p.rt = rt; p.depth = depth; p.vw = view_weights; p.gout = grad_out;
    p.dref = d_ref_nhwc; p.dsrc = d_src_flat;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = vt.hs[0]; p.Ws = vt.ws[0]; p.D = D;
    p.sx = vt.sx[0]; p.sy = vt.sy[0];
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(d_src_flat, 0, (size_t)end * sizeof(float), st);
    if (e != cudaSuccess) return pmb200_internal_fail((int)e, "warp_corr_views_backward: memset failed");
    const int HW = H * W;
#define PMB200_LAUNCH_WBV(CC, GG)                                                        \
    do {                                                                                 \
        const int pix_per_block = 4 * BwdMap<CC, GG>::PPW;                               \
        dim3 grid((HW + pix_per_block - 1) / pix_per_block, B);                          \
        warp_corr_backward_views_kernel<CC, GG><<<grid, 128, 0, st>>>(p, vt);            \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_WBV(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_WBV(32, 8);
    else PMB200_LAUNCH_WBV(16, 4);
#undef PMB200_LAUNCH_WBV
    return pmb200_internal_launch_status("warp_corr_views_backward");
}

int pmb200_aggregate_views_backward(const float *sims, const float *view_weights, const float *grad_out, float *d_sims,
                                    float *d_view_weights, int V, int B, int G, int D, int H, int W, void *stream) {
    if (!sims || !view_weights || !grad_out || !d_sims || !d_view_weights)
        return pmb200_internal_fail(PMB200_EINVAL, "aggregate_views_backward: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || G < 1 || D < 1 || H < 1 || W < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "aggregate_views_backward: bad size");
    const int HW = H * W;
    dim3 grid((HW + 127) / 128, B);
    aggregate_views_backward_kernel<<<grid, 128, 0, as_stream(stream)>>>(sims, view_weights, grad_out, d_sims,
                                                                         d_view_weights, V, B, G * D, HW);
    return pmb200_internal_launch_status("aggregate_views_backward");
}

int pmb200_offset_corr_backward(const float *ref_nhwc, const float *offsets, const float *grad_out, float *d_offsets, int B,
                                int C, int G, int H, int W, int K, int dilation, void *stream) {
    if (!ref_nhwc || !offsets || !grad_out || !d_offsets)
        return pmb200_internal_fail(PMB200_EINVAL, "offset_corr_backward: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2) return pmb200_internal_fail(PMB200_EINVAL, "offset_corr_backward: bad size");
    if (K != 9 && K != 17) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "offset_corr_backward: evaluate_neighbors must be 9 or 17");
    OffsetCorrBwdParams p;
    p.ref = ref_nhwc; p.offsets = offsets; p.gout = grad_out; p.doff = d_offsets;
    p.B = B; p.H = H; p.W = W; p.K = K; p.dilation = dilation;
    const int HW = H * W;
    cudaStream_t st = as_stream(stream);
#define PMB200_LAUNCH_OB(CC, GG)                                                         \
    do {                                                                                 \
        const int pix_per_block = 4 * BwdMap<CC, GG>::PPW;                               \
        dim3 grid((HW + pix_per_block - 1) / pix_per_block, B);                          \
        offset_corr_backward_kernel<CC, GG><<<grid, 128, 0, st>>>(p);                    \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_OB(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_OB(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_OB(16, 4);
    else return pmb200_internal_fail(PMB200_EUNSUPPORTED, "offset_corr_backward: (C,G) must be (64,8), (32,8) or (16,4)");
#undef PMB200_LAUNCH_OB
    return pmb200_internal_launch_status("offset_corr_backward");
}

int pmb200_init_propagate_backward(const float *seed_map, const float *offsets, const float *depth_min, const float *depth_max,
                                   const float *grad_out, float *d_offsets, int mode, int B, int H, int W, int Ns, int Kp,
                                   int dilation, float interval_scale, void *stream) {
    if (!seed_map || !offsets || !depth_min || !depth_max || !grad_out || !d_offsets)
        return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2 || Ns < 1 || mode < 0 || mode > 2)
        return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: bad size");
    if (Kp != 4 && Kp != 8 && Kp != 16)
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "init_propagate_backward: propagate_neighbors must be 4, 8 or 16");
    // what pmb200_init_propagate rejects: the kernel reads seed[(b*48 + k)*HW] for every k < Ns in random mode, one
    // seed plane otherwise, and packs 29-bit texel indices (pm::border_cell)
    if (mode == 0 && Ns != 48)
        return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: random init has 48 samples");
    if (mode == 2 && Ns != 1) return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: passthrough needs Ns == 1");
    if (Ns + Kp > PMB200_MAX_HYPOTHESES) return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: too many hypotheses");
    if ((long long)H * W >= (1LL << pm::kKeyDxShift)) return pmb200_internal_fail(PMB200_EINVAL, "init_propagate_backward: map too large");
    PropBwdParams p;
    p.seed = seed_map; p.offsets = offsets; p.dmin = depth_min; p.dmax = depth_max; p.gout = grad_out; p.doff = d_offsets;
    p.mode = mode; p.B = B; p.H = H; p.W = W; p.Ns = Ns; p.Kp = Kp; p.dilation = dilation; p.interval_scale = interval_scale;
    dim3 grid((H * W + 127) / 128, B);
    init_propagate_backward_kernel<<<grid, 128, 0, as_stream(stream)>>>(p);
    return pmb200_internal_launch_status("init_propagate_backward");
}

int pmb200_adaptive_eval_backward(const float *score0, const float *depth_sample, const float *xnorm, const float *offsets,
                                  const float *feature_weight, const float *depth_min, const float *depth_max,
                                  const float *prob, const float *grad_depth, const float *grad_prob, float *d_score0,
                                  float *d_depth_sample, float *d_offsets, float *d_feature_weight, int B, int D, int H, int W,
                                  int K, int dilation, float interval_scale, int is_inverse, void *stream) {
    if (!score0 || !depth_sample || !offsets || !feature_weight || !depth_min || !depth_max || !prob || !d_score0 ||
        !d_depth_sample || !d_offsets || !d_feature_weight)
        return pmb200_internal_fail(PMB200_EINVAL, "adaptive_eval_backward: null pointer");
    if (!grad_depth && !grad_prob) return pmb200_internal_fail(PMB200_EINVAL, "adaptive_eval_backward: no incoming gradient");
    if (B < 1 || B > 65535 || H < 2 || W < 2 || D < 1 || D > PMB200_MAX_HYPOTHESES)
        return pmb200_internal_fail(PMB200_EINVAL, "adaptive_eval_backward: bad size");
    if (K != 9 && K != 17) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "adaptive_eval_backward: evaluate_neighbors must be 9 or 17");
    // what pmb200_adaptive_eval rejects, before the zero fill: the inverse regression divides by D - 1, and the gathers
    // pack 29-bit texel indices (pm::border_cell)
    if (is_inverse && D < 2) return pmb200_internal_fail(PMB200_EINVAL, "adaptive_eval_backward: inverse regression needs D >= 2");
    if ((long long)H * W >= (1LL << pm::kKeyDxShift)) return pmb200_internal_fail(PMB200_EINVAL, "adaptive_eval_backward: map too large");
    EvalBwdParams p;
    p.score0 = score0; p.depth = depth_sample; p.xnorm = xnorm; p.offsets = offsets; p.fw = feature_weight;
    p.dmin = depth_min; p.dmax = depth_max; p.prob = prob; p.gdepth = grad_depth; p.gprob = grad_prob;
    p.dscore0 = d_score0; p.dhyp = d_depth_sample; p.doff = d_offsets; p.dfw = d_feature_weight;
    p.B = B; p.D = D; p.H = H; p.W = W; p.K = K; p.dilation = dilation; p.is_inverse = is_inverse;
    p.interval_scale = interval_scale;
    cudaStream_t st = as_stream(stream);
    cudaError_t e = cudaMemsetAsync(d_score0, 0, (size_t)B * D * H * W * sizeof(float), st);
    if (e != cudaSuccess) return pmb200_internal_fail((int)e, "adaptive_eval_backward: memset failed");
    dim3 grid((H * W + 63) / 64, B);
    adaptive_eval_backward_kernel<<<grid, 64, 0, st>>>(p);
    return pmb200_internal_launch_status("adaptive_eval_backward");
}

}  // extern "C"
#endif  // !PM_EMU
