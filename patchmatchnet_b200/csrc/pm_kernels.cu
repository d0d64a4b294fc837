// pm_kernels.cu -- sm_90a forward kernels of the learned-PatchMatch hot path + their C ABI
// (backward kernels: pm_backward.cu; per-element formulas shared with the CPU formula tests: pm_math.cuh).
//
// Kernel map (DESIGN.md has the byte/flop budgets and the measured numbers):
//   wc4::warp_corr4_kernel<C,G,EPI,NW,MINB>  K-A, fourth generation (default, pm_warpcorr4.cuh): homography warp + bilinear
//                                  gather + group-wise correlation + view-weighted aggregation + (eval) 1x1x1 head epilogue
//                                  as a persistent producer/consumer pipeline over TMA-staged shared-memory windows
//                                  pmb200_warp_corr / _score / _view_weights
//   warp_corr3_kernel<C,G,EPI,DC,PIPE,MINB>  K-A, third generation: register/L1 gather; taken for shapes generation 4
//                                  declines and selectable for A/B measurements (pmb200_set_tuning("ka_gen", 3));
//                                  warp_corr_generic_kernel: any C % G == 0
//   warp_corr3_views_kernel / warp_corr_generic_views_kernel   the same bodies with a size per source view (ragged pack)
//                                  pmb200_warp_corr_views / _score_views / _view_weights_views
//   aggregate_views_kernel / aggregate_score_kernel   weighted view average of stored similarities (+ head)
//   offset_corr_kernel<C,G,HEAD>   K-A': reference self-correlation at the learned evaluation neighbours (+ head)
//   init_propagate_kernel<NPAD>    K-C: hypothesis init + neighbour gather + warp-shuffle bitonic sort
//   adaptive_eval_kernel<K>        K-B: depth/feature weights + neighbour aggregation + softmax + regression
//   relative_projection_kernel, pack_nhwc_kernel, upsample2x_add_nhwc_kernel, photometric_confidence_kernel   helpers
//
// Lane mapping of the gather (K-A, K-A'): features are channels-last, each lane owns 8 consecutive channels of one
// pixel, C/8 lanes share a pixel, a warp covers 32/(C/8) consecutive pixels.  One bilinear tap of one pixel is one
// contiguous C*4-byte read split over C/8 lanes as 2 x 16-byte loads (a full 128-byte line per pixel at C=32, two at
// C=64).  PatchMatch hypotheses of one pixel are sorted and clustered, so consecutive hypotheses mostly land in the
// same source cell; every generation of K-A exploits that differently (see the comments above each kernel).
#include <atomic>

#if !defined(PM_EMU)  // host emulation build (tests/warp_emu.h) brings its own CUDA vocabulary
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/patchmatch_b200.h"
#include "pm_math.cuh"

namespace {

thread_local char g_err[256] = "";

int fail(int code, const char *msg) {
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}

#if !defined(PM_EMU)
int launch_status(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}
#endif

// Learned 2-D offset (x, y) of neighbour k at pixel n.  The offset convs' output is consumed in place in either
// layout: planar [B,2K,H,W] (NCHW-contiguous) or channels-last [B,H,W,2K] (what cuDNN emits for a channels-last
// input; then (x, y) is one aligned 8-byte load).
__device__ __forceinline__ float2 load_offset(const float *__restrict__ off, int nhwc, int b, int k, int n, int K, int HW) {
    if (nhwc) return __ldg(reinterpret_cast<const float2 *>(off + ((size_t)b * HW + n) * 2 * K) + k);
    const float *q = off + ((size_t)b * 2 * K + 2 * k) * HW + n;
    return make_float2(__ldg(q), __ldg(q + HW));
}

// A lane's 8 channels of a texel: 32 contiguous bytes as two 128-bit read-only loads (LDG.E.128.CONSTANT; Hopper has
// no 256-bit load).  The entry points keep the 32-byte alignment check so a lane's pair never straddles a sector.
__device__ __forceinline__ void ldg256(const float4 *__restrict__ p, float4 &lo, float4 &hi) {
#if defined(PM_EMU)
    assert((reinterpret_cast<uintptr_t>(p) & 31u) == 0);
#endif
    lo = __ldg(p);
    hi = __ldg(p + 1);
}

inline bool misaligned32(const void *q) { return (reinterpret_cast<uintptr_t>(q) & 31u) != 0; }

constexpr int kWarpsPerBlock = 8;
constexpr int kChunk = 8;  // hypotheses (or neighbours) handled per warp pass

template <int C, int G>
struct LaneMap {
    static_assert(C % 8 == 0 && (32 % (C / 8)) == 0, "C must be 8,16,32,64,128 or 256");
    static constexpr int CPL = 8;               // channels per lane
    static constexpr int LPP = C / CPL;         // lanes per pixel
    static constexpr int PPW = 32 / LPP;        // pixels per warp
    static constexpr int CPG = C / G;           // channels per group
    static_assert(CPG == 4 || CPG == 8, "fast path needs 4 or 8 channels per group");
    static constexpr int GPL = CPL / CPG;       // groups per lane (1 or 2)
    static constexpr int EPW = PPW * kChunk;    // footprints per warp pass
};

// ------------------------------------------------------------------------------------------
// gather/correlate core
// ------------------------------------------------------------------------------------------

template <int C, int G>
__device__ __forceinline__ void gather_dot(const float4 *__restrict__ map_lane, int key, int cols,
                                           const float (&r)[8], float (&T)[4][LaneMap<C, G>::GPL]) {
    constexpr int V4 = C / 4;  // float4 per texel
    const int r0 = pm::cell_r0(key), dx = pm::cell_dx(key), dy = pm::cell_dy(key);
    const float4 *t0 = map_lane + (size_t)r0 * V4;
    const float4 *t1 = t0 + dx * V4;
    const float4 *t2 = t0 + (size_t)dy * cols * V4;
    const float4 *t3 = t2 + dx * V4;
    float4 a0, a1, b0, b1, c0, c1, d0, d1;
    ldg256(t0, a0, a1);
    ldg256(t1, b0, b1);
    ldg256(t2, c0, c1);
    ldg256(t3, d0, d1);
    auto lo = [&](const float4 &q) { return r[0] * q.x + r[1] * q.y + r[2] * q.z + r[3] * q.w; };
    auto hi = [&](const float4 &q) { return r[4] * q.x + r[5] * q.y + r[6] * q.z + r[7] * q.w; };
    if constexpr (LaneMap<C, G>::GPL == 1) {
        T[0][0] = lo(a0) + hi(a1);
        T[1][0] = lo(b0) + hi(b1);
        T[2][0] = lo(c0) + hi(c1);
        T[3][0] = lo(d0) + hi(d1);
    } else {
        T[0][0] = lo(a0); T[0][1] = hi(a1);
        T[1][0] = lo(b0); T[1][1] = hi(b1);
        T[2][0] = lo(c0); T[2][1] = hi(c1);
        T[3][0] = lo(d0); T[3][1] = hi(d1);
    }
}

template <int C, int G>
__device__ __forceinline__ void load_reference(const float *__restrict__ ref_nhwc, size_t pixel, int lane_in_pixel,
                                               float (&r)[8]) {
    const float4 *rp = reinterpret_cast<const float4 *>(ref_nhwc + pixel * C) + lane_in_pixel * 2;
    float4 q0, q1;
    ldg256(rp, q0, q1);
    constexpr float s = 1.0f / (float)LaneMap<C, G>::CPG;  // the group mean; exact (power of two)
    r[0] = q0.x * s; r[1] = q0.y * s; r[2] = q0.z * s; r[3] = q0.w * s;
    r[4] = q1.x * s; r[5] = q1.y * s; r[6] = q1.z * s; r[7] = q1.w * s;
}

// Two IEEE fp32 fused multiply-adds on a pair of lanes of the head MLP, the blend and the gather dot products.  Hopper
// has no packed fp32x2 FMA, so this is two FFMAs; the pairing keeps the input-major weight layout of MlpParams.
__device__ __forceinline__ float2 ffma2(const float2 a, const float2 b, const float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// Folded (conv3d 1x1x1 + eval-mode BatchNorm) weights of one G -> 16 -> 8 -> 1 head in the layout the device code
// wants: input-major ("transposed") so that the weights of two adjacent outputs are one 64-bit constant operand.
// Passed by value inside the kernel parameter block, i.e. it lives in the constant bank.
struct alignas(16) MlpParams {
    float w0t[8][16];  // [input g (padded to 8)][output j]
    float b0[16];
    float w1t[16][8];  // [input j][output i]
    float b1[8];
    float w2[8];
    float b2;
};

// public layout (pmb200_mlp: output-major, as the convolutions store them) -> device layout
inline MlpParams to_device_layout(const pmb200_mlp *h) {
    static_assert(sizeof(MlpParams) >= sizeof(pmb200_mlp), "pmb200_mlp layout");
    MlpParams m;
    for (int j = 0; j < 16; ++j)
        for (int g = 0; g < 8; ++g) m.w0t[g][j] = h->w0[j * 8 + g];
    for (int j = 0; j < 16; ++j) m.b0[j] = h->b0[j];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 16; ++j) m.w1t[j][i] = h->w1[i * 16 + j];
    for (int i = 0; i < 8; ++i) { m.b1[i] = h->b1[i]; m.w2[i] = h->w2[i]; }
    m.b2 = h->b2;
    return m;
}

template <int G>
__device__ __forceinline__ float mlp_eval(const MlpParams &m, const float (&x)[G]) {
    float2 h0[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) h0[q] = make_float2(m.b0[2 * q], m.b0[2 * q + 1]);
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const float2 xx = make_float2(x[g], x[g]);
#pragma unroll
        for (int q = 0; q < 8; ++q) h0[q] = ffma2(make_float2(m.w0t[g][2 * q], m.w0t[g][2 * q + 1]), xx, h0[q]);
    }
    float2 h1[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) h1[q] = make_float2(m.b1[2 * q], m.b1[2 * q + 1]);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float hj = fmaxf((j & 1) ? h0[j >> 1].y : h0[j >> 1].x, 0.0f);
        const float2 hh = make_float2(hj, hj);
#pragma unroll
        for (int q = 0; q < 4; ++q) h1[q] = ffma2(make_float2(m.w1t[j][2 * q], m.w1t[j][2 * q + 1]), hh, h1[q]);
    }
    float2 acc = make_float2(m.b2, 0.0f);
#pragma unroll
    for (int q = 0; q < 4; ++q)
        acc = ffma2(make_float2(m.w2[2 * q], m.w2[2 * q + 1]), make_float2(fmaxf(h1[q].x, 0.0f), fmaxf(h1[q].y, 0.0f)), acc);
    return acc.x + acc.y;
}

struct WarpCorrParams {
    const float *ref, *src, *rt, *depth, *vw;
    float *out;
    int V, B, H, W, Hs, Ws, D;
    float sx, sy;
    int ostride = 1;  // element stride of the score epilogue's output (2: the .y lane of an (xnorm, score) buffer)
};

// Per-view source extents of a ragged source pack (the *_views entry points): view v, batch b starts at float4 index
// base4[v] + b * hs[v] * ws[v] * C / 4 of p.src; sx / sy are that view's align_corners=True scales.  Passed as a kernel
// parameter of its own so that the uniform instantiations keep the parameter block (and the code) they always had; the
// per-view instantiations read p.Hs / p.Ws / p.sx / p.sy from here instead.
struct ViewTable {
    unsigned base4[PMB200_MAX_VIEWS];
    int hs[PMB200_MAX_VIEWS], ws[PMB200_MAX_VIEWS];
    float sx[PMB200_MAX_VIEWS], sy[PMB200_MAX_VIEWS];
};

// Epilogue of the fused warp+correlation kernel
constexpr int kEpiSims = 0;    // per-view similarities                 out [V,B,G,D,H,W]
constexpr int kEpiAgg = 1;     // view-weighted average                 out [B,G,D,H,W]
constexpr int kEpiScore = 2;   // view-weighted average -> MLP          out [B,D,H,W]      (SimilarityNet head, eval mode)
constexpr int kEpiViewW = 3;   // per-view -> MLP -> max_d -> sigmoid   out [B,V,H,W]      (PixelwiseNet, eval mode)

#include "pm_warpcorr4.cuh"  // K-A generation 4 (default): persistent, warp-specialised, TMA-staged shared-memory windows

constexpr int kWarps2 = 4;  // warps per CTA of the third-generation kernel


// ------------------------------------------------------------------------------------------
// K-A, third generation.  Same three phases as the second, with the profile-driven changes
// (phase 1 was a third of the issued instructions, the gather loop took most of the stall samples):
//   * unique cells are numbered PER PIXEL in "layers" (slot = layer * PPW + pixel) straight from the
//     ballot mask with one popc -- no shuffle prefix scan; every lane group then gathers the cells of
//     its OWN pixel, so the reference vector stays in registers (no shared-memory copy of it);
//   * the gather loop is software pipelined two deep: the taps of layer j+1 are in flight while layer j
//     is being dotted with the reference vector;
//   * projection with MUFU.RCP instead of two IEEE divisions, footprint routine with an interior fast path.
// ------------------------------------------------------------------------------------------
template <int PPW>
__device__ __forceinline__ unsigned pixel_lane_mask(int pixel) {
    constexpr unsigned base = PPW == 4 ? 0x11111111u : (PPW == 8 ? 0x01010101u : 0x00010001u);
    return base << pixel;
}

// The four taps of one unique cell for this lane: 4 x LDG.256.  Addresses are formed from ONE 64-bit base (the feature
// pack, a kernel parameter = uniform register) and 32-bit float4 indices: `lane_idx` (view / batch / lane offset, computed
// once per view) + the texel offsets decoded from the key.  The first version added 64-bit pointers per tap; under the
// 128-register cap of the pipelined variant ptxas rematerialised the 64-bit view base and the row stride inside the
// gather loop (~35 of the ~95 instructions per lane and layer, tools/sass_lines.py); with 32-bit indices it is ~13.
// The C entry points reject packs with more than 2^31 float4 elements.
template <int C, int G>
__device__ __forceinline__ void load_taps(const float4 *__restrict__ pack, unsigned lane_idx, int key, unsigned row_stride,
                                          float4 (&t)[8]) {
    constexpr unsigned V4 = C / 4;  // float4 per texel (4, 8 or 16)
    constexpr int kLog2V4 = V4 == 4 ? 2 : (V4 == 8 ? 3 : 4);
    static_assert(V4 == 4 || V4 == 8 || V4 == 16, "load_taps: C must be 16, 32 or 64");
    const unsigned ukey = (unsigned)key;
    const unsigned ox = (ukey >> (pm::kKeyDxShift - kLog2V4)) & V4;            // dx ? V4 : 0
    const unsigned oy = ((ukey >> pm::kKeyDyShift) & 1u) * row_stride;         // dy ? cols * V4 : 0
    const unsigned i0 = lane_idx + (ukey & (unsigned)pm::kKeyIndexMask) * V4;
    const unsigned i2 = i0 + oy;
    ldg256(pack + i0, t[0], t[1]);
    ldg256(pack + (i0 + ox), t[2], t[3]);
    ldg256(pack + i2, t[4], t[5]);
    ldg256(pack + (i2 + ox), t[6], t[7]);
}

template <int C, int G>
__device__ __forceinline__ void dot_store(const float4 (&t)[8], const float (&r)[8], float *__restrict__ tp) {
    using M = LaneMap<C, G>;
    const float2 r01 = make_float2(r[0], r[1]), r23 = make_float2(r[2], r[3]);
    const float2 r45 = make_float2(r[4], r[5]), r67 = make_float2(r[6], r[7]);
    const float2 zero = make_float2(0.0f, 0.0f);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float4 a = t[2 * k], bq = t[2 * k + 1];
        const float2 lo = ffma2(r23, make_float2(a.z, a.w), ffma2(r01, make_float2(a.x, a.y), zero));
        if constexpr (M::GPL == 1) {
            const float2 s = ffma2(r67, make_float2(bq.z, bq.w), ffma2(r45, make_float2(bq.x, bq.y), lo));
            tp[k * G] = s.x + s.y;
        } else {
            const float2 hi = ffma2(r67, make_float2(bq.z, bq.w), ffma2(r45, make_float2(bq.x, bq.y), zero));
            *reinterpret_cast<float2 *>(tp + k * G) = make_float2(lo.x + lo.y, hi.x + hi.y);
        }
    }
}

// The body of both third-generation kernels.  VIEWS = false: one (Hs, Ws) for every source view, read from p (the uniform
// entry points; vt is null).  VIEWS = true: view v's extent and scales come from vt (the *_views entry points).
template <int C, int G, int EPI, int DC, int PIPE, bool VIEWS>
__device__ __forceinline__ void warp_corr3_body(const WarpCorrParams &p, const ViewTable *vt, const MlpParams &mlp,
                                                float *__restrict__ sims_out) {
    using M = LaneMap<C, G>;
    constexpr int EPW = M::PPW * DC;   // footprints per warp pass
    static_assert(EPW % 32 == 0, "PPW * DC must be a multiple of the warp size");
    constexpr int NE = EPW / 32;       // footprints per lane
    constexpr int RPK = 32 / M::PPW;   // hypothesis rows covered by one k
    constexpr int TS = 4 * G + 4;      // floats per slot in s_T
    constexpr bool kWeighted = (EPI == kEpiAgg || EPI == kEpiScore);
    __shared__ int s_key[kWarps2][EPW];
    __shared__ __align__(16) float s_T[kWarps2][EPW * TS];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int HW = p.H * p.W;
    const int n0 = (blockIdx.x * kWarps2 + warp) * M::PPW;
    if (n0 >= HW) return;  // warp-level barriers only below
    const int b = blockIdx.z, d0 = blockIdx.y * DC;
    const unsigned full = 0xffffffffu;

    // gather mapping: lane group `grp` works on pixel n0+grp, lane `li` of the group owns channels 8*li..8*li+7
    const int li = lane % M::LPP, grp = lane / M::LPP;
    float r[8];
    load_reference<C, G>(p.ref, (size_t)b * HW + min(n0 + grp, HW - 1), li, r);
    const unsigned gmask = pixel_lane_mask<M::PPW>(grp);

    // footprint mapping: all footprints of a lane belong to pixel n0+pi, rows row0 + k*RPK
    const int pi = lane % M::PPW, row0 = lane / M::PPW;
    const unsigned fmask = pixel_lane_mask<M::PPW>(pi);
    const unsigned le_mask = 0xffffffffu >> (31 - lane);
    const int n = n0 + pi;
    const bool live = n < HW;
    const int nc = live ? n : HW - 1;
    const float px_x = (float)(nc % p.W), px_y = (float)(nc / p.W);
    float dep[NE];
    bool ev[NE];
#pragma unroll
    for (int k = 0; k < NE; ++k) {
        const int d = d0 + row0 + k * RPK;
        ev[k] = live && d < p.D;
        dep[k] = ev[k] ? __ldg(p.depth + ((size_t)b * p.D + d) * HW + n) : 1.0f;
    }
    float acc[NE][G];
#pragma unroll
    for (int k = 0; k < NE; ++k)
#pragma unroll
        for (int g = 0; g < G; ++g) acc[k][g] = 0.0f;
    float wsum = 1e-5f;  // reference models/patchmatch.py:192

    for (int v = 0; v < p.V; ++v) {
        float rt[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) rt[i] = __ldg(p.rt + ((size_t)v * p.B + b) * 12 + i);
        const pm::Ray ray = pm::pixel_ray(rt, px_x, px_y);
        // issued here so that its latency hides behind phase 1 (it was 10 % of the stall samples right before its use)
        const float wv = kWeighted ? __ldg(p.vw + ((size_t)b * p.V + v) * HW + nc) : 1.0f;
        const int Hs = VIEWS ? vt->hs[v] : p.Hs, Ws = VIEWS ? vt->ws[v] : p.Ws;
        const float sx = VIEWS ? vt->sx[v] : p.sx, sy = VIEWS ? vt->sy[v] : p.sy;

        // ---- phase 1: footprints, per-pixel layered numbering of the unique cells ----
        float4 w[NE];
        int key[NE], slot[NE];
        int mine_before = 0;   // unique cells of my footprint pixel found in earlier k
        int cg = 0;            // unique cells of my gather pixel
#pragma unroll
        for (int k = 0; k < NE; ++k) {
            pm::Cell c;
            c.w00 = c.w01 = c.w10 = c.w11 = 0.0f;
            c.key = pm::kKeyNone;
            if (ev[k]) {
                float uu, vv;
                pm::project_fast(ray, rt, dep[k], p.W, p.H, sx, sy, &uu, &vv);
                c = pm::zero_pad_cell_fast(uu, vv, Hs, Ws);
            }
            w[k] = make_float4(c.w00, c.w01, c.w10, c.w11);
            key[k] = c.key;
            int pk = __shfl_up_sync(full, key[k], M::PPW);  // previous hypothesis row, same pixel
            if (k > 0) {
                const int ck = __shfl_sync(full, key[k > 0 ? k - 1 : 0], 32 - M::PPW + pi);
                if (lane < M::PPW) pk = ck;
            } else if (lane < M::PPW) {
                pk = pm::kKeyNone;
            }
            const bool isnew = key[k] != pm::kKeyNone && key[k] != pk;
            const unsigned m = __ballot_sync(full, isnew);
            const int c_incl = mine_before + __popc(m & fmask & le_mask);  // unique cells of my pixel up to my row
            slot[k] = (c_incl - 1) * M::PPW + pi;                          // >= 0 whenever key != none
            if (isnew) s_key[warp][slot[k]] = key[k];
            mine_before += __popc(m & fmask);
            cg += __popc(m & gmask);
        }
        __syncwarp();
        if (kWeighted) wsum += wv;

        // ---- phase 2a: gather layer by layer, two layers in flight ----
        const float4 *pack = reinterpret_cast<const float4 *>(p.src);
        const unsigned row_stride = (unsigned)Ws * (C / 4);
        const unsigned sv = (VIEWS ? vt->base4[v] + (unsigned)b * ((unsigned)Hs * row_stride)
                                   : (unsigned)(v * p.B + b) * ((unsigned)Hs * row_stride)) + li * 2;  // float4 index of this lane's channels
        const int maxc = __reduce_max_sync(full, cg);
        if constexpr (PIPE) {
            float4 ta[8], tb[8];
            float *tbase = s_T[warp] + grp * TS + li * M::GPL;
            if (cg > 0) load_taps<C, G>(pack, sv, s_key[warp][grp], row_stride, ta);
            for (int j = 0; j < maxc; j += 2) {
                if (j + 1 < cg) load_taps<C, G>(pack, sv, s_key[warp][(j + 1) * M::PPW + grp], row_stride, tb);
                if (j < cg) dot_store<C, G>(ta, r, tbase + j * M::PPW * TS);
                if (j + 2 < cg) load_taps<C, G>(pack, sv, s_key[warp][(j + 2) * M::PPW + grp], row_stride, ta);
                if (j + 1 < cg) dot_store<C, G>(tb, r, tbase + (j + 1) * M::PPW * TS);
            }
        } else {
            float *tbase = s_T[warp] + grp * TS + li * M::GPL;
            for (int j = 0; j < maxc; ++j) {
                if (j < cg) {
                    float4 ta[8];
                    load_taps<C, G>(pack, sv, s_key[warp][j * M::PPW + grp], row_stride, ta);
                    dot_store<C, G>(ta, r, tbase + j * M::PPW * TS);
                }
            }
        }
        __syncwarp();

        // ---- phase 2b: one footprint per lane ----
        float best = -INFINITY;  // kEpiViewW only
#pragma unroll
        for (int k = 0; k < NE; ++k) {
            float sim[G];
#pragma unroll
            for (int g = 0; g < G; ++g) sim[g] = 0.0f;
            if (key[k] != pm::kKeyNone) {
                const float4 *tp = reinterpret_cast<const float4 *>(s_T[warp] + slot[k] * TS);
                const float2 wx = make_float2(w[k].x, w[k].x), wy = make_float2(w[k].y, w[k].y);
                const float2 wz = make_float2(w[k].z, w[k].z), ww = make_float2(w[k].w, w[k].w);
                const float2 zero = make_float2(0.0f, 0.0f);
#pragma unroll
                for (int q = 0; q < G / 4; ++q) {
                    const float4 t0 = tp[q], t1 = tp[G / 4 + q], t2 = tp[2 * (G / 4) + q], t3 = tp[3 * (G / 4) + q];
                    const float2 lo = ffma2(ww, make_float2(t3.x, t3.y), ffma2(wz, make_float2(t2.x, t2.y),
                                      ffma2(wy, make_float2(t1.x, t1.y), ffma2(wx, make_float2(t0.x, t0.y), zero))));
                    const float2 hi = ffma2(ww, make_float2(t3.z, t3.w), ffma2(wz, make_float2(t2.z, t2.w),
                                      ffma2(wy, make_float2(t1.z, t1.w), ffma2(wx, make_float2(t0.z, t0.w), zero))));
                    sim[4 * q + 0] = lo.x; sim[4 * q + 1] = lo.y; sim[4 * q + 2] = hi.x; sim[4 * q + 3] = hi.y;
                }
            }
            if (kWeighted) {
                const float2 wv2 = make_float2(wv, wv);
#pragma unroll
                for (int g = 0; g < G; g += 2) {
                    const float2 a2 = ffma2(make_float2(sim[g], sim[g + 1]), wv2, make_float2(acc[k][g], acc[k][g + 1]));
                    acc[k][g] = a2.x;
                    acc[k][g + 1] = a2.y;
                }
            } else {
                const int d = d0 + row0 + k * RPK;
                if ((EPI == kEpiSims || sims_out != nullptr) && ev[k]) {
                    float *o = (EPI == kEpiSims ? p.out : sims_out) + ((((size_t)v * p.B + b) * G) * p.D + d) * HW + n;
#pragma unroll
                    for (int g = 0; g < G; ++g) o[(size_t)g * p.D * HW] = sim[g];
                }
                if (EPI == kEpiViewW && ev[k]) best = fmaxf(best, mlp_eval<G>(mlp, sim));
            }
        }
        if (EPI == kEpiViewW) {
#pragma unroll
            for (int off = M::PPW; off < 32; off <<= 1) best = fmaxf(best, __shfl_xor_sync(full, best, off));
            if (lane < M::PPW && live && best > -INFINITY) {
                const float sg = 1.0f / (1.0f + expf(-best));
                atomicMax(reinterpret_cast<int *>(p.out + ((size_t)b * p.V + v) * HW + n), __float_as_int(sg));
            }
        }
        __syncwarp();  // s_key / s_T are rewritten by the next view
    }

    // One IEEE division per thread, then multiplies: the NE*G divisions that stood here were 13 instructions each
    // (221 of this kernel's 1608 SASS instructions at C32 D16, tools/sass_lines.py); a * (1/b) is within 1.5 ulp of a / b.
    const float inv_wsum = 1.0f / wsum;
    if (EPI == kEpiAgg) {
#pragma unroll
        for (int k = 0; k < NE; ++k) {
            const int d = d0 + row0 + k * RPK;
            if (ev[k]) {
                float *o = p.out + (((size_t)b * G) * p.D + d) * HW + n;
#pragma unroll
                for (int g = 0; g < G; ++g) o[(size_t)g * p.D * HW] = acc[k][g] * inv_wsum;
            }
        }
    } else if (EPI == kEpiScore) {
#pragma unroll
        for (int k = 0; k < NE; ++k) {
            const int d = d0 + row0 + k * RPK;
            float x[G];
#pragma unroll
            for (int g = 0; g < G; ++g) x[g] = acc[k][g] * inv_wsum;
            const float y = mlp_eval<G>(mlp, x);
            if (ev[k]) p.out[(((size_t)b * p.D + d) * HW + n) * p.ostride] = y;
        }
    }
}

template <int C, int G, int EPI, int DC, int PIPE, int MINB>
__global__ void __launch_bounds__(kWarps2 * 32, MINB) warp_corr3_kernel(const WarpCorrParams p, const MlpParams mlp,
                                                                  float *__restrict__ sims_out) {
    warp_corr3_body<C, G, EPI, DC, PIPE, false>(p, nullptr, mlp, sims_out);
}

// per-view source extents (pmb200_warp_corr*_views)
template <int C, int G, int EPI, int DC, int PIPE, int MINB>
__global__ void __launch_bounds__(kWarps2 * 32, MINB) warp_corr3_views_kernel(const WarpCorrParams p, const ViewTable vt,
                                                                        const MlpParams mlp, float *__restrict__ sims_out) {
    warp_corr3_body<C, G, EPI, DC, PIPE, true>(p, &vt, mlp, sims_out);
}

// sum_v sims[v]*w_v / (1e-5 + sum_v w_v) -> SimilarityNet head -> score [B,D,H,W]   (first stage-3 iteration, eval)
template <int G>
__global__ void aggregate_score_kernel(const float *__restrict__ sims, const float *__restrict__ vw,
                                       float *__restrict__ score, const MlpParams mlp, int V, int B, int D, int HW,
                                       int ostride) {
    const size_t total = (size_t)B * D * HW;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int n = (int)(idx % HW);
    const int d = (int)((idx / HW) % D);
    const int b = (int)(idx / ((size_t)HW * D));
    float x[G];
#pragma unroll
    for (int g = 0; g < G; ++g) x[g] = 0.0f;
    float wsum = 1e-5f;
    for (int v = 0; v < V; ++v) {
        const float w = __ldg(vw + ((size_t)b * V + v) * HW + n);
        wsum += w;
        const float *sp = sims + ((((size_t)v * B + b) * G) * D + d) * HW + n;
#pragma unroll
        for (int g = 0; g < G; ++g) x[g] = fmaf(__ldg(sp + (size_t)g * D * HW), w, x[g]);
    }
    const float inv_wsum = 1.0f / wsum;
#pragma unroll
    for (int g = 0; g < G; ++g) x[g] *= inv_wsum;
    score[idx * ostride] = mlp_eval<G>(mlp, x);
}

// Any C % G == 0: one thread per (batch, hypothesis, pixel), scalar channel loop.  Slow path.  VIEWS as in warp_corr3_body.
template <bool VIEWS>
__device__ __forceinline__ void warp_corr_generic_body(const WarpCorrParams &p, const ViewTable *vt, int C, int G) {
    const int HW = p.H * p.W;
    const size_t total = (size_t)p.B * p.D * HW;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int n = (int)(idx % HW);
    const int d = (int)((idx / HW) % p.D);
    const int b = (int)(idx / ((size_t)HW * p.D));
    const float x = (float)(n % p.W), y = (float)(n / p.W);
    const float dep = p.depth[((size_t)b * p.D + d) * HW + n];
    const float *ref = p.ref + ((size_t)b * HW + n) * C;
    const int cpg = C / G;
    const bool fused = p.vw != nullptr;
    for (int g = 0; g < G; ++g) {
        float acc = 0.0f, wsum = 1e-5f;
        for (int v = 0; v < p.V; ++v) {
            float rt[12];
            for (int i = 0; i < 12; ++i) rt[i] = p.rt[((size_t)v * p.B + b) * 12 + i];
            const int Hs = VIEWS ? vt->hs[v] : p.Hs, Ws = VIEWS ? vt->ws[v] : p.Ws;
            float u, w;
            pm::project(pm::pixel_ray(rt, x, y), rt, dep, p.W, p.H, VIEWS ? vt->sx[v] : p.sx, VIEWS ? vt->sy[v] : p.sy, &u, &w);
            const pm::Cell c = pm::zero_pad_cell(u, w, Hs, Ws);
            float sim = 0.0f;
            if (c.key != pm::kKeyNone) {
                const float *base = VIEWS ? p.src + (size_t)vt->base4[v] * 4 + (size_t)b * Hs * Ws * C
                                          : p.src + ((size_t)v * p.B + b) * Hs * Ws * C;
                const float *t0 = base + (size_t)pm::cell_r0(c.key) * C;
                const float *t1 = t0 + pm::cell_dx(c.key) * C;
                const float *t2 = t0 + (size_t)pm::cell_dy(c.key) * Ws * C;
                const float *t3 = t2 + pm::cell_dx(c.key) * C;
                for (int k = g * cpg; k < (g + 1) * cpg; ++k)
                    sim += ref[k] * (c.w00 * t0[k] + c.w01 * t1[k] + c.w10 * t2[k] + c.w11 * t3[k]);
                sim /= (float)cpg;
            }
            if (fused) {
                const float wv = p.vw[((size_t)b * p.V + v) * HW + n];
                acc += sim * wv;
                wsum += wv;
            } else {
                p.out[((((size_t)v * p.B + b) * G + g) * p.D + d) * HW + n] = sim;
            }
        }
        if (fused) p.out[(((size_t)b * G + g) * p.D + d) * HW + n] = acc / wsum;
    }
}

__global__ void warp_corr_generic_kernel(const WarpCorrParams p, int C, int G) { warp_corr_generic_body<false>(p, nullptr, C, G); }

__global__ void warp_corr_generic_views_kernel(const WarpCorrParams p, const ViewTable vt, int C, int G) {
    warp_corr_generic_body<true>(p, &vt, C, G);
}

struct OffsetCorrParams {
    const float *ref, *offsets;
    float *out;
    int B, H, W, K, dilation;
    int off_nhwc = 0;
};

template <int C, int G, bool HEAD>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) offset_corr_kernel(const OffsetCorrParams p, const MlpParams mlp) {
    using M = LaneMap<C, G>;
    __shared__ float4 s_w[kWarpsPerBlock][M::EPW];
    __shared__ int s_key[kWarpsPerBlock][M::EPW];
    __shared__ float s_sim[HEAD ? kWarpsPerBlock : 1][HEAD ? M::EPW * G : 1];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int HW = p.H * p.W;
    const int n0 = (blockIdx.x * kWarpsPerBlock + warp) * M::PPW;
    if (n0 >= HW) return;
    const int b = blockIdx.z, k0 = blockIdx.y * kChunk;
    const int pi = lane / M::LPP, li = lane % M::LPP;
    const int n = n0 + pi;
    const bool live = n < HW;
    const int nc = live ? n : HW - 1;
    const int g0 = li * M::GPL;

    float r[8];
    load_reference<C, G>(p.ref, (size_t)b * HW + nc, li, r);

    for (int e = lane; e < M::EPW; e += 32) {
        const int epi = e % M::PPW, ekj = e / M::PPW;
        const int en = n0 + epi, ek = k0 + ekj;
        pm::Cell c;
        c.w00 = c.w01 = c.w10 = c.w11 = 0.0f;
        c.key = pm::kKeyNone;
        if (en < HW && ek < p.K) {
            int dy = 0, dx = 0;
            pm::neighbour_offset(true, p.K, p.dilation, ek, &dy, &dx);
            const float2 lo = load_offset(p.offsets, p.off_nhwc, b, ek, en, p.K, HW);
            const float ox = (float)dx + lo.x, oy = (float)dy + lo.y;
            c = pm::border_cell((float)(en % p.W) + ox, (float)(en / p.W) + oy, p.H, p.W);
        }
        s_w[warp][e] = make_float4(c.w00, c.w01, c.w10, c.w11);
        s_key[warp][e] = c.key;
    }
    __syncwarp();

    const float4 *sv = reinterpret_cast<const float4 *>(p.ref + (size_t)b * HW * C) + li * 2;
    int pkey = pm::kKeyNone;
    float T[4][M::GPL];
#pragma unroll
    for (int t = 0; t < 4; ++t)
#pragma unroll
        for (int g = 0; g < M::GPL; ++g) T[t][g] = 0.0f;
#pragma unroll
    for (int kj = 0; kj < kChunk; ++kj) {
        const float4 w = s_w[warp][kj * M::PPW + pi];
        const int key = s_key[warp][kj * M::PPW + pi];
        float sim[M::GPL];
#pragma unroll
        for (int g = 0; g < M::GPL; ++g) sim[g] = 0.0f;
        if (key != pm::kKeyNone) {  // none only for k >= K or dead pixels
            if (key != pkey) {
                gather_dot<C, G>(sv, key, p.W, r, T);
                pkey = key;
            }
#pragma unroll
            for (int g = 0; g < M::GPL; ++g) sim[g] = w.x * T[0][g] + w.y * T[1][g] + w.z * T[2][g] + w.w * T[3][g];
        }
        if (HEAD) {
#pragma unroll
            for (int g = 0; g < M::GPL; ++g) s_sim[warp][(kj * M::PPW + pi) * G + g0 + g] = sim[g];
        } else if (live && k0 + kj < p.K) {
#pragma unroll
            for (int g = 0; g < M::GPL; ++g) p.out[(((size_t)b * G + g0 + g) * p.K + k0 + kj) * HW + n] = sim[g];
        }
    }
    if (HEAD) {  // FeatureWeightNet head (reference models/patchmatch.py:624): sigmoid(MLP(correlation)) -> [B,K,H,W]
        __syncwarp();
        for (int e = lane; e < M::EPW; e += 32) {
            float x[G];
#pragma unroll
            for (int g = 0; g < G; ++g) x[g] = s_sim[warp][e * G + g];
            const float y = mlp_eval<G>(mlp, x);
            const int en = n0 + e % M::PPW, ek = k0 + e / M::PPW;
            if (en < HW && ek < p.K) p.out[((size_t)b * p.K + ek) * HW + en] = 1.0f / (1.0f + expf(-y));
        }
    }
}

__global__ void offset_corr_generic_kernel(const OffsetCorrParams p, int C, int G) {
    const int HW = p.H * p.W;
    const size_t total = (size_t)p.B * p.K * HW;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int n = (int)(idx % HW);
    const int k = (int)((idx / HW) % p.K);
    const int b = (int)(idx / ((size_t)HW * p.K));
    int dy = 0, dx = 0;
    pm::neighbour_offset(true, p.K, p.dilation, k, &dy, &dx);
    const float2 lo = load_offset(p.offsets, p.off_nhwc, b, k, n, p.K, HW);
    const float ox = (float)dx + lo.x, oy = (float)dy + lo.y;
    const pm::Cell c = pm::border_cell((float)(n % p.W) + ox, (float)(n / p.W) + oy, p.H, p.W);
    const float *ref = p.ref + ((size_t)b * HW + n) * C;
    const float *t0 = p.ref + ((size_t)b * HW + pm::cell_r0(c.key)) * C;
    const float *t1 = t0 + pm::cell_dx(c.key) * C;
    const float *t2 = t0 + (size_t)pm::cell_dy(c.key) * p.W * C;
    const float *t3 = t2 + pm::cell_dx(c.key) * C;
    const int cpg = C / G;
    for (int g = 0; g < G; ++g) {
        float sim = 0.0f;
        for (int q = g * cpg; q < (g + 1) * cpg; ++q)
            sim += ref[q] * (c.w00 * t0[q] + c.w01 * t1[q] + c.w10 * t2[q] + c.w11 * t3[q]);
        p.out[(((size_t)b * G + g) * p.K + k) * HW + n] = sim / (float)cpg;
    }
}

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------

__global__ void aggregate_views_kernel(const float *__restrict__ sims, const float *__restrict__ vw,
                                       float *__restrict__ out, int V, int B, int GD, int HW) {
    // one thread per (b, g*d, pixel); sims [V,B,GD,HW], vw [B,V,HW]
    const size_t total = (size_t)B * GD * HW;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const int n = (int)(idx % HW);
        const int b = (int)(idx / ((size_t)GD * HW));
        float acc = 0.0f, wsum = 1e-5f;
        for (int v = 0; v < V; ++v) {
            const float w = __ldg(vw + ((size_t)b * V + v) * HW + n);
            acc = fmaf(__ldg(sims + (size_t)v * total + idx), w, acc);
            wsum += w;
        }
        out[idx] = acc / wsum;
    }
}

struct PtrList {
    const float *p[PMB200_MAX_VIEWS + 1];
};

struct PackParams {
    PtrList maps;
    float *out;
    int n, B, C, HW;
};

__global__ void pack_nhwc_kernel(const PackParams p) {
    __shared__ float tile[32][33];
    const int m = blockIdx.z / p.B, b = blockIdx.z % p.B;
    const float *in = p.maps.p[m] + (size_t)b * p.C * p.HW;
    float *out = p.out + ((size_t)m * p.B + b) * p.HW * p.C;
    const int hw0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int c = c0 + j, hw = hw0 + threadIdx.x;
        tile[j][threadIdx.x] = (c < p.C && hw < p.HW) ? __ldg(in + (size_t)c * p.HW + hw) : 0.0f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int hw = hw0 + j, c = c0 + threadIdx.x;
        if (c < p.C && hw < p.HW) out[(size_t)hw * p.C + c] = tile[threadIdx.x][j];
    }
}

// out[n,oy,ox,:] = bilinear_up2(x)[n,oy,ox,:] + y[n,oy,ox,:], channels-last, float4 over channels.
// Same sampling as F.interpolate(scale_factor=2, mode="bilinear", align_corners=False).
__global__ void upsample2x_add_nhwc_kernel(const float4 *__restrict__ x, const float4 *__restrict__ y,
                                           const float4 *__restrict__ bias, float4 *__restrict__ out, int N, int h,
                                           int w, int C4) {
    const int H = 2 * h, W = 2 * w;
    const size_t total = (size_t)N * H * W * C4;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % C4);
    const int ox = (int)((idx / C4) % W);
    const int oy = (int)((idx / ((size_t)C4 * W)) % H);
    const int n = (int)(idx / ((size_t)C4 * W * H));
    const float sy = fmaxf(0.5f * ((float)oy + 0.5f) - 0.5f, 0.0f), sx = fmaxf(0.5f * ((float)ox + 0.5f) - 0.5f, 0.0f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float ly = sy - (float)y0, lx = sx - (float)x0;
    const float hy = 1.0f - ly, hx = 1.0f - lx;
    const float4 *b = x + (size_t)n * h * w * C4 + c;
    const float4 a00 = __ldg(b + ((size_t)y0 * w + x0) * C4), a01 = __ldg(b + ((size_t)y0 * w + x1) * C4);
    const float4 a10 = __ldg(b + ((size_t)y1 * w + x0) * C4), a11 = __ldg(b + ((size_t)y1 * w + x1) * C4);
    float4 r = __ldg(y + idx);
    if (bias) {  // per-channel bias of the lateral 1x1 conv, folded in here instead of a separate elementwise pass
        const float4 bb = __ldg(bias + c);
        r.x += bb.x; r.y += bb.y; r.z += bb.z; r.w += bb.w;
    }
    float4 o;
    o.x = hy * (hx * a00.x + lx * a01.x) + ly * (hx * a10.x + lx * a11.x) + r.x;
    o.y = hy * (hx * a00.y + lx * a01.y) + ly * (hx * a10.y + lx * a11.y) + r.y;
    o.z = hy * (hx * a00.z + lx * a01.z) + ly * (hx * a10.z + lx * a11.z) + r.z;
    o.w = hy * (hx * a00.w + lx * a01.w) + ly * (hx * a10.w + lx * a11.w) + r.w;
    out[idx] = o;
}

// Photometric confidence (caller side, reference models/net.py:289-299): probability mass of the four
// hypotheses around the regressed index, nearest-upsampled to the output size -- one launch instead of
// pad + avg_pool3d + mul + arange + mul + sum + long + clamp + gather + interpolate.
__global__ void photometric_confidence_kernel(const float *__restrict__ prob, float *__restrict__ out, int B, int D,
                                              int h, int w, int H, int W) {
    const size_t total = (size_t)B * H * W;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int X = (int)(idx % W), Y = (int)((idx / W) % H), b = (int)(idx / ((size_t)W * H));
    const float sy = (float)h / (float)H, sx = (float)w / (float)W;
    const int y = min((int)floorf((float)Y * sy), h - 1), x = min((int)floorf((float)X * sx), w - 1);
    const float *pp = prob + (size_t)b * D * h * w + (size_t)y * w + x;
    const size_t plane = (size_t)h * w;
    float e = 0.0f;
    for (int d = 0; d < D; ++d) e += __ldg(pp + d * plane) * (float)d;
    int k = (int)e;  // .long(): truncation
    k = max(0, min(k, D - 1));
    float sum = 0.0f;
#pragma unroll
    for (int j = -1; j <= 2; ++j) {
        const int d = k + j;
        sum += (d >= 0 && d < D) ? __ldg(pp + d * plane) : 0.0f;
    }
    out[idx] = 4.0f * (sum * 0.25f);
}

struct ProjParams {
    const float *ref;
    PtrList src;
    float *out;
    long long ref_stride, src_stride;
    int V, B;
};

__global__ void relative_projection_kernel(const ProjParams p) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= p.V * p.B) return;
    const int v = idx / p.B, b = idx % p.B;
    double a[4][8];
    const float *R = p.ref + (size_t)b * p.ref_stride;
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            a[i][j] = (double)R[i * 4 + j];
            a[i][4 + j] = (i == j) ? 1.0 : 0.0;
        }
    // Gauss-Jordan with partial pivoting, fp64
    for (int col = 0; col < 4; ++col) {
        int piv = col;
        double best = fabs(a[col][col]);
        for (int i = col + 1; i < 4; ++i)
            if (fabs(a[i][col]) > best) { best = fabs(a[i][col]); piv = i; }
        if (piv != col)
            for (int j = 0; j < 8; ++j) { const double t = a[col][j]; a[col][j] = a[piv][j]; a[piv][j] = t; }
        const double inv = 1.0 / a[col][col];  // singular input -> inf/nan, as torch.inverse would error; caller's contract
        for (int j = 0; j < 8; ++j) a[col][j] *= inv;
        for (int i = 0; i < 4; ++i) {
            if (i == col) continue;
            const double f = a[i][col];
            for (int j = 0; j < 8; ++j) a[i][j] -= f * a[col][j];
        }
    }
    const float *S = p.src.p[v] + (size_t)b * p.src_stride;
    float *o = p.out + ((size_t)v * p.B + b) * 12;
    for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 4; ++j) {
            double s = 0.0;
            for (int k = 0; k < 4; ++k) s += (double)S[i * 4 + k] * a[k][4 + j];
            if (j < 3) o[i * 3 + j] = (float)s;
            else o[9 + i] = (float)s;
        }
    }
}

// ------------------------------------------------------------------------------------------
// K-C: init + propagate + sort
// ------------------------------------------------------------------------------------------

struct PropParams {
    const float *seed, *offsets, *dmin, *dmax;
    float *out, *xnorm;
    int xstride;  // element stride of xnorm (2 when it is the .x lane of an interleaved (xnorm, score) buffer)
    int off_nhwc;
    int mode, B, H, W, Ns, Kp, dilation;
    float interval_scale;
};

__device__ __forceinline__ float centre_hypothesis(const PropParams &p, int b, int q, int HW, float inv_min,
                                                   float inv_max) {
    if (p.mode == 0) return pm::random_hypothesis(__ldg(p.seed + ((size_t)b * 48 + 24) * HW + q), 24, inv_min, inv_max);
    const float d = __ldg(p.seed + (size_t)b * HW + q);
    if (p.mode == 1)
        return pm::perturbed_hypothesis(d, pm::floor_div2_neg(p.Ns) + p.Ns / 2, inv_min, inv_max, p.interval_scale);
    return d;
}

__device__ __forceinline__ float own_hypothesis(const PropParams &p, int b, int n, int k, int HW, float inv_min,
                                                float inv_max) {
    if (p.mode == 0) return pm::random_hypothesis(__ldg(p.seed + ((size_t)b * 48 + k) * HW + n), k, inv_min, inv_max);
    const float d = __ldg(p.seed + (size_t)b * HW + n);
    if (p.mode == 1) return pm::perturbed_hypothesis(d, pm::floor_div2_neg(p.Ns) + k, inv_min, inv_max, p.interval_scale);
    return d;
}

__device__ __forceinline__ float propagated_hypothesis(const PropParams &p, int b, int n, int kk, int HW,
                                                       float inv_min, float inv_max) {
    int dy = 0, dx = 0;
    pm::neighbour_offset(false, p.Kp, p.dilation, kk, &dy, &dx);
    const float2 lo = load_offset(p.offsets, p.off_nhwc, b, kk, n, p.Kp, HW);
    const float ox = (float)dx + lo.x, oy = (float)dy + lo.y;
    const pm::Cell c = pm::border_cell((float)(n % p.W) + ox, (float)(n / p.W) + oy, p.H, p.W);
    const int r0 = pm::cell_r0(c.key), ddx = pm::cell_dx(c.key), ddy = pm::cell_dy(c.key);
    float s = centre_hypothesis(p, b, r0, HW, inv_min, inv_max) * c.w00;
    s = fmaf(centre_hypothesis(p, b, r0 + ddx, HW, inv_min, inv_max), c.w01, s);
    s = fmaf(centre_hypothesis(p, b, r0 + ddy * p.W, HW, inv_min, inv_max), c.w10, s);
    s = fmaf(centre_hypothesis(p, b, r0 + ddy * p.W + ddx, HW, inv_min, inv_max), c.w11, s);
    return s;
}

// Sorting version (Kp > 0): min(NPAD,32) lanes per pixel, each lane owns hypothesis slot `lane` (and
// `lane + 32` when NPAD == 64); the ascending sort over the hypothesis axis is a bitonic network run
// with warp shuffles, so a 64x80 map is 5120 warps of parallel work instead of 5120 serial threads.
template <int NPAD>
__global__ void __launch_bounds__(128) init_propagate_kernel(const PropParams p) {
    constexpr int LPX = NPAD < 32 ? NPAD : 32;  // lanes per pixel
    constexpr int PPW = 32 / LPX;               // pixels per warp
    constexpr int VPL = NPAD / LPX;             // values per lane
    const int HW = p.H * p.W;
    const int lane = threadIdx.x & 31;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int b = blockIdx.y;
    const int slot = lane % LPX;
    const int n = warp * PPW + lane / LPX;
    const bool live = n < HW;
    const int nc = live ? n : HW - 1;
    const float inv_min = 1.0f / __ldg(p.dmin + b), inv_max = 1.0f / __ldg(p.dmax + b);
    const int D = p.Ns + p.Kp;
    const float kInf = __int_as_float(0x7f800000);

    float v[VPL];
#pragma unroll
    for (int r = 0; r < VPL; ++r) {
        const int k = slot + 32 * r;
        if (k < p.Ns) v[r] = own_hypothesis(p, b, nc, k, HW, inv_min, inv_max);
        else if (k < D) v[r] = propagated_hypothesis(p, b, nc, k - p.Ns, HW, inv_min, inv_max);
        else v[r] = kInf;  // padding sorts to the end
    }
#pragma unroll
    for (int k2 = 2; k2 <= NPAD; k2 <<= 1) {
#pragma unroll
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            if (j >= 32) {  // NPAD == 64, final merge: partner lives in the same lane
                const float lo = fminf(v[0], v[VPL - 1]), hi = fmaxf(v[0], v[VPL - 1]);
                v[0] = lo;
                v[VPL - 1] = hi;
            } else {
#pragma unroll
                for (int r = 0; r < VPL; ++r) {
                    const int idx = slot + 32 * r;
                    const float other = __shfl_xor_sync(0xffffffffu, v[r], j);
                    const bool up = (idx & k2) == 0, lower = (idx & j) == 0;
                    v[r] = (lower == up) ? fminf(v[r], other) : fmaxf(v[r], other);
                }
            }
        }
    }
    if (live) {
#pragma unroll
        for (int r = 0; r < VPL; ++r) {
            const int k = slot + 32 * r;
            if (k < D) {
                p.out[((size_t)b * D + k) * HW + n] = v[r];
                if (p.xnorm) p.xnorm[(((size_t)b * D + k) * HW + n) * p.xstride] = pm::normalised_inverse_depth(v[r], inv_min, inv_max);
            }
        }
    }
}

// No propagation (Kp == 0): initialisation order is kept (descending depth), nothing to sort.
__global__ void __launch_bounds__(128) init_only_kernel(const PropParams p) {
    const int HW = p.H * p.W;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HW) return;
    const float inv_min = 1.0f / __ldg(p.dmin + b), inv_max = 1.0f / __ldg(p.dmax + b);
    for (int k = 0; k < p.Ns; ++k) {
        const float v = own_hypothesis(p, b, n, k, HW, inv_min, inv_max);
        p.out[((size_t)b * p.Ns + k) * HW + n] = v;
        if (p.xnorm) p.xnorm[(((size_t)b * p.Ns + k) * HW + n) * p.xstride] = pm::normalised_inverse_depth(v, inv_min, inv_max);
    }
}

// D > 64: write unsorted, then insertion-sort each pixel's column in place.  Slow path.
__global__ void init_propagate_generic_kernel(const PropParams p) {
    const int HW = p.H * p.W;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int b = blockIdx.y;
    if (n >= HW) return;
    const float inv_min = 1.0f / p.dmin[b], inv_max = 1.0f / p.dmax[b];
    const int D = p.Ns + p.Kp;
    float *col = p.out + (size_t)b * D * HW + n;
    for (int k = 0; k < D; ++k)
        col[(size_t)k * HW] = k < p.Ns ? own_hypothesis(p, b, n, k, HW, inv_min, inv_max)
                                       : propagated_hypothesis(p, b, n, k - p.Ns, HW, inv_min, inv_max);
    if (p.Kp > 0) {
        for (int i = 1; i < D; ++i) {
            const float x = col[(size_t)i * HW];
            int j = i - 1;
            while (j >= 0 && col[(size_t)j * HW] > x) {
                col[(size_t)(j + 1) * HW] = col[(size_t)j * HW];
                --j;
            }
            col[(size_t)(j + 1) * HW] = x;
        }
    }
    if (p.xnorm) {
        for (int k = 0; k < D; ++k) p.xnorm[(((size_t)b * D + k) * HW + n) * p.xstride] = pm::normalised_inverse_depth(col[(size_t)k * HW], inv_min, inv_max);
    }
}

// ------------------------------------------------------------------------------------------
// K-B: adaptive evaluation tail
// ------------------------------------------------------------------------------------------

struct EvalParams {
    const float *score0, *depth, *xnorm, *offsets, *fw, *dmin, *dmax;
    const float2 *xs;  // optional interleaved (xnorm, score0): one 8-byte gather per tap instead of two 4-byte ones
    int off_nhwc;
    float *prob, *depth_out;
    int B, D, H, W, K, dilation, is_inverse;
    float interval_scale;
};

// block (TP pixels, DY hypothesis lanes); dynamic smem: float4 cw[K][TP]; int ck[K][TP]; float sc[D][TP]; float pr[D][TP];
// float cf[K][TP]
// KT = number of evaluation neighbours (9 or 17) as a compile-time constant: the neighbour loop is fully unrolled
// so that the 8 gathers of every neighbour are issued back to back instead of one neighbour at a time.
template <int KT>
__global__ void __launch_bounds__(256) adaptive_eval_kernel(const EvalParams p) {
#if defined(PM_EMU)
    float4 *smem4 = static_cast<float4 *>(emu::dyn_smem());
#else
    extern __shared__ float4 smem4[];
#endif
    const int TP = blockDim.x, DY = blockDim.y;
    float4 *cw = smem4;
    int *ck = reinterpret_cast<int *>(cw + (size_t)p.K * TP);
    float *sc = reinterpret_cast<float *>(ck + (size_t)p.K * TP);
    float *pr = sc + (size_t)p.D * TP;
    float *cf = pr + (size_t)p.D * TP;  // feature weight of (neighbour, pixel): independent of the hypothesis, read D times

    const int tp = threadIdx.x, ty = threadIdx.y;
    const int HW = p.H * p.W;
    const int n = blockIdx.x * TP + tp;
    const int b = blockIdx.y;
    const bool live = n < HW;
    const int nc = live ? n : HW - 1;
    const float inv_min = 1.0f / __ldg(p.dmin + b), inv_max = 1.0f / __ldg(p.dmax + b);
    const float inv_interval = 1.0f / p.interval_scale;

    for (int k = ty; k < p.K; k += DY) {
        int dy = 0, dx = 0;
        pm::neighbour_offset(true, p.K, p.dilation, k, &dy, &dx);
        const float2 lo = load_offset(p.offsets, p.off_nhwc, b, k, nc, p.K, HW);
        const float ox = (float)dx + lo.x, oy = (float)dy + lo.y;
        const pm::Cell c = pm::border_cell((float)(nc % p.W) + ox, (float)(nc / p.W) + oy, p.H, p.W);
        cw[k * TP + tp] = make_float4(c.w00, c.w01, c.w10, c.w11);
        ck[k * TP + tp] = c.key;
        cf[k * TP + tp] = __ldg(p.fw + ((size_t)b * p.K + k) * HW + nc);
    }
    __syncthreads();

    for (int d = ty; d < p.D; d += DY) {
        const float *smap = p.score0 + ((size_t)b * p.D + d) * HW;
        float num = 0.0f, den = 0.0f;
        if (p.xs) {
            const float2 *xsm = p.xs + ((size_t)b * p.D + d) * HW;
            const float xc = __ldg(xsm + nc).x;
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                const float4 w = cw[k * TP + tp];
                const int key = ck[k * TP + tp];
                const int r0 = pm::cell_r0(key), ddx = pm::cell_dx(key), ddy = pm::cell_dy(key);
                const float2 *q0 = xsm + r0, *q2 = q0 + ddy * p.W;
                const float2 v0 = __ldg(q0), v1 = __ldg(q0 + ddx), v2 = __ldg(q2), v3 = __ldg(q2 + ddx);
                const float2 acc = ffma2(v3, make_float2(w.w, w.w), ffma2(v2, make_float2(w.z, w.z),
                                   ffma2(v1, make_float2(w.y, w.y), make_float2(v0.x * w.x, v0.y * w.x))));
                const float t = fminf(fabsf(acc.x - xc) * inv_interval, 4.0f);
                const float sg = __fdividef(1.0f, 1.0f + __expf(2.0f * t - 4.0f));
                const float wk = sg * cf[k * TP + tp];
                num = fmaf(acc.y, wk, num);
                den += wk;
            }
        } else if (p.xnorm) {  // normalised inverse depth precomputed by K-C: 8 loads + 8 FMAs per neighbour
            const float *xmap = p.xnorm + ((size_t)b * p.D + d) * HW;
            const float xc = __ldg(xmap + nc);
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                const float4 w = cw[k * TP + tp];
                const int key = ck[k * TP + tp];
                const int r0 = pm::cell_r0(key), ddx = pm::cell_dx(key), ddy = pm::cell_dy(key);
                const int r1 = r0 + ddx, r2 = r0 + ddy * p.W, r3 = r2 + ddx;
                const float x0 = __ldg(xmap + r0), x1 = __ldg(xmap + r1), x2 = __ldg(xmap + r2), x3 = __ldg(xmap + r3);
                const float s0 = __ldg(smap + r0), s1 = __ldg(smap + r1), s2 = __ldg(smap + r2), s3 = __ldg(smap + r3);
                const float xn = fmaf(x3, w.w, fmaf(x2, w.z, fmaf(x1, w.y, x0 * w.x)));
                const float sn = fmaf(s3, w.w, fmaf(s2, w.z, fmaf(s1, w.y, s0 * w.x)));
                // sigmoid(4 - 2*clamp(|dx|/interval, 0, 4)) with the fast exponential / reciprocal
                // (argument in [-4, 4]: relative error ~1e-7, far below the parity tolerance)
                const float t = fminf(fabsf(xn - xc) * inv_interval, 4.0f);
                const float sg = __fdividef(1.0f, 1.0f + __expf(2.0f * t - 4.0f));
                const float wk = sg * cf[k * TP + tp];
                num = fmaf(sn, wk, num);
                den += wk;
            }
        } else {
            const float *dmap = p.depth + ((size_t)b * p.D + d) * HW;
            const float xc = pm::normalised_inverse_depth(__ldg(dmap + nc), inv_min, inv_max);
            for (int k = 0; k < p.K; ++k) {
                const float4 w = cw[k * TP + tp];
                const int key = ck[k * TP + tp];
                const int r0 = pm::cell_r0(key), ddx = pm::cell_dx(key), ddy = pm::cell_dy(key);
                const int r1 = r0 + ddx, r2 = r0 + ddy * p.W, r3 = r2 + ddx;
                float xn = pm::normalised_inverse_depth(__ldg(dmap + r0), inv_min, inv_max) * w.x;
                xn = fmaf(pm::normalised_inverse_depth(__ldg(dmap + r1), inv_min, inv_max), w.y, xn);
                xn = fmaf(pm::normalised_inverse_depth(__ldg(dmap + r2), inv_min, inv_max), w.z, xn);
                xn = fmaf(pm::normalised_inverse_depth(__ldg(dmap + r3), inv_min, inv_max), w.w, xn);
                float sn = __ldg(smap + r0) * w.x;
                sn = fmaf(__ldg(smap + r1), w.y, sn);
                sn = fmaf(__ldg(smap + r2), w.z, sn);
                sn = fmaf(__ldg(smap + r3), w.w, sn);
                const float wk = pm::depth_similarity(xc, xn, p.interval_scale) * cf[k * TP + tp];
                num = fmaf(sn, wk, num);
                den += wk;
            }
        }
        sc[d * TP + tp] = num / den;
    }
    __syncthreads();

    // softmax over the hypotheses of this pixel: one exponential per (pixel, hypothesis) thread
    float m = -INFINITY;
    for (int d = 0; d < p.D; ++d) m = fmaxf(m, sc[d * TP + tp]);
    for (int d = ty; d < p.D; d += DY) pr[d * TP + tp] = expf(sc[d * TP + tp] - m);
    __syncthreads();
    float sum = 0.0f;
    for (int d = 0; d < p.D; ++d) sum += pr[d * TP + tp];
    const float lse = logf(sum);
    __syncthreads();  // everybody has read the un-normalised values
    for (int d = ty; d < p.D; d += DY) {
        const float q = expf(sc[d * TP + tp] - m - lse);  // exp(log_softmax), as the reference writes it
        pr[d * TP + tp] = q;
        if (live) p.prob[((size_t)b * p.D + d) * HW + n] = q;
    }
    __syncthreads();

    if (ty == 0 && live) {
        float out;
        if (p.is_inverse) {  // reference models/patchmatch.py:227-234
            float idx = 0.0f;
            for (int d = 0; d < p.D; ++d) idx = fmaf((float)d, pr[d * TP + tp], idx);
            const float inv_hi = 1.0f / __ldg(p.depth + ((size_t)b * p.D + (p.D - 1)) * HW + n);
            const float inv_lo = 1.0f / __ldg(p.depth + ((size_t)b * p.D) * HW + n);
            out = 1.0f / (inv_lo + idx / (float)(p.D - 1) * (inv_hi - inv_lo));
        } else {
            float e = 0.0f;
            for (int d = 0; d < p.D; ++d) e = fmaf(__ldg(p.depth + ((size_t)b * p.D + d) * HW + n), pr[d * TP + tp], e);
            out = e;
        }
        p.depth_out[(size_t)b * HW + n] = out;
    }
}

#if defined(PM_EMU)
}  // namespace  (the emulation build stops here: launchers and the C ABI below need the CUDA runtime)
#else
cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

// ------------------------------------------------------------------------------------------
// Launch-configuration knobs.  Defaults are the values measured best so far; a measurement tool
// (tools/kbench.py) changes them through pmb200_set_tuning().  Nothing in the launch path reads the environment.
// ------------------------------------------------------------------------------------------
enum Tune { kTuneKaGen, kTuneKa3Dc, kTuneKa3DcVw, kTuneKa3Pipe, kTuneKa3MinB, kTuneKa4Nw, kTuneKa4Ctas, kTuneKa4Cap, kTuneKa4Grid,
            kTuneKa4Stages, kTuneKbTp, kTuneKbDy, kTuneStemPpt, kTuneCount };
const char *const kTuneNames[kTuneCount] = {"ka_gen", "ka3_dc", "ka3_dc_vw", "ka3_pipe", "ka3_minb", "ka4_nw", "ka4_ctas", "ka4_cap",
                                            "ka4_grid", "ka4_stages", "kb_tp", "kb_dy", "stem_ppt"};
// ka_gen: 3.  Generation 4 (TMA-staged windows) is parity-green but was slower at every bench shape (DESIGN.md has the analysis)
// stem_ppt: 2 (4 pixels per thread measured no faster: the LDCU : FFMA ratio is not the limiter)
const int kTuneDefaults[kTuneCount] = {3, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0, 0, 2};
int g_tune[kTuneCount] = {3, 0, 0, -1, 0, 0, 0, 0, 0, 0, 0, 0, 2};
inline int tune(Tune t) { return __atomic_load_n(&g_tune[t], __ATOMIC_RELAXED); }

// Shared memory per CTA (s_T + s_key) decides how many CTAs of the plain-gather kernel fit; asking ptxas for more than
// that only caps the registers for nothing.
template <int C, int G, int DC>
constexpr int wc3_min_blocks() {
    constexpr int kSmem = kWarps2 * LaneMap<C, G>::PPW * DC * ((4 * G + 4) * 4 + 4);
    constexpr int kFit = (227 * 1024) / (kSmem + 1024);
    return kFit >= 6 ? 6 : (kFit >= 5 ? 5 : 4);
}

// Rows per warp pass of the default third-generation launch
template <int C, int G, int EPI>
constexpr int wc3_default_dc() {
    constexpr int PPW = LaneMap<C, G>::PPW;
    constexpr int kDefault = PPW == 4 ? 16 : (PPW == 8 ? 8 : 4);
    return EPI == kEpiScore ? kDefault : (PPW == 4 ? 8 : kDefault);
}

// Third-generation K-A launch (kept for shapes generation 4 does not take and for A/B measurements).
template <int C, int G, int EPI, int DC>
void launch_wc3(const WarpCorrParams &p, const MlpParams &m, float *sims_out, cudaStream_t st) {
    const int HW = p.H * p.W;
    constexpr int pix_per_block = kWarps2 * LaneMap<C, G>::PPW;
    dim3 grid((HW + pix_per_block - 1) / pix_per_block, (p.D + DC - 1) / DC, p.B);
    // the plain gather loop measured faster at every lane map than the two-deep pipeline, whose 128 registers cost a resident CTA
    constexpr int kPipeDefault = 0;
    const int pipe = tune(kTuneKa3Pipe) < 0 ? kPipeDefault : tune(kTuneKa3Pipe);
    if constexpr (EPI == kEpiScore && LaneMap<C, G>::PPW == 8) {
        // sweep candidate (ka3_minb = 5): the pipelined stage-2 kernel holds 128 registers -> 4 resident CTAs per SM; capped
        // at 96 registers 5 fit
        if (pipe && tune(kTuneKa3MinB) == 5) {
            warp_corr3_kernel<C, G, EPI, DC, 1, 5><<<grid, kWarps2 * 32, 0, st>>>(p, m, sims_out);
            return;
        }
    }
    if (pipe) warp_corr3_kernel<C, G, EPI, DC, 1, 4><<<grid, kWarps2 * 32, 0, st>>>(p, m, sims_out);
    else {
        warp_corr3_kernel<C, G, EPI, DC, 0, wc3_min_blocks<C, G, DC>()><<<grid, kWarps2 * 32, 0, st>>>(p, m, sims_out);
    }
}

template <int C, int G, int EPI>
void launch_wc3_auto(const WarpCorrParams &p, const MlpParams &m, float *sims_out, cudaStream_t st) {
    constexpr int PPW = LaneMap<C, G>::PPW;
    if constexpr (EPI == kEpiScore || EPI == kEpiViewW) {
        const int d = tune(EPI == kEpiScore ? kTuneKa3Dc : kTuneKa3DcVw);
#define PMB200_TRY3(DD)                                                                                  \
    if (d == DD) {                                                                                       \
        if constexpr ((PPW * DD) % 32 == 0 && PPW * DD * (4 * G + 4) * 4 * kWarps2 <= 40 * 1024) {       \
            launch_wc3<C, G, EPI, DD>(p, m, sims_out, st);                                               \
            return;                                                                                      \
        }                                                                                                \
    }
        PMB200_TRY3(4) PMB200_TRY3(8) PMB200_TRY3(16)
#undef PMB200_TRY3
    }
    launch_wc3<C, G, EPI, wc3_default_dc<C, G, EPI>()>(p, m, sims_out, st);
}

// Per-view K-A launch (the *_views entry points): generation 3 at its default launch shape.  The ka3_* knobs choose among
// the uniform instantiations only; generation 4 does not take per-view extents.
template <int C, int G, int EPI>
void launch_wc3_views(const WarpCorrParams &p, const ViewTable &vt, const MlpParams &m, float *sims_out, cudaStream_t st) {
    constexpr int DC = wc3_default_dc<C, G, EPI>();
    constexpr int pix_per_block = kWarps2 * LaneMap<C, G>::PPW;
    dim3 grid((p.H * p.W + pix_per_block - 1) / pix_per_block, (p.D + DC - 1) / DC, p.B);
    warp_corr3_views_kernel<C, G, EPI, DC, 0, wc3_min_blocks<C, G, DC>()><<<grid, kWarps2 * 32, 0, st>>>(p, vt, m, sims_out);
}

// ------------------------------------------------------------------------------------------
// Fourth-generation K-A launch: tensor map of the reference pack, ring-slot size from the shared-memory budget,
// persistent grid from the occupancy.
// ------------------------------------------------------------------------------------------
struct DeviceFacts {
    int sms = 0, smem_optin = 0;
};
const DeviceFacts &device_facts() {
    static thread_local int cached_dev = -1;
    static thread_local DeviceFacts f;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev != cached_dev) {
        cudaDeviceGetAttribute(&f.sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&f.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cached_dev = dev;
    }
    return f;
}

PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
    static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
        void *sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            sym = nullptr;
        return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(sym);
    }();
    return fn;
}

// [B][H][W][C] fp32 channels-last tensor, box {C, 8, box_rows, 1}, no swizzle, zero fill outside
bool make_ref_map(CUtensorMap *tm, const float *ref, int B, int H, int W, int C, int box_rows) {
    auto enc = tensor_map_encoder();
    if (!enc) return false;
    const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
    const cuuint32_t box[4] = {(cuuint32_t)C, 8u, (cuuint32_t)box_rows, 1u};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(ref), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

bool wc4_accepts(const WarpCorrParams &p) {
    return p.Ws < (1 << wc4::kXBits) && p.Hs < (1 << 15) && p.V <= 32 && (reinterpret_cast<uintptr_t>(p.ref) & 15u) == 0 &&
           (reinterpret_cast<uintptr_t>(p.src) & 15u) == 0;
}

template <int C, int G, int EPI, int NW, int MINB>
bool launch_wc4_nw(const WarpCorrParams &p, const MlpParams &m, float *sims_out, cudaStream_t st) {
    using L = wc4::Layout<C, G, NW>;
    const DeviceFacts &dev = device_facts();
    auto kern = wc4::warp_corr4_kernel<C, G, EPI, NW, MINB>;
    // ring: `stages` slots of `cap` texels out of what is left of the per-CTA share of shared memory when `ctas` CTAs are to
    // be resident
    const int ctas = tune(kTuneKa4Ctas) > 0 ? tune(kTuneKa4Ctas) : MINB;
    int stages = tune(kTuneKa4Stages) > 0 ? tune(kTuneKa4Stages) : 3;
    stages = stages < 2 ? 2 : (stages > wc4::kMaxStages ? wc4::kMaxStages : stages);
    const int share = (dev.smem_optin + 1024) / ctas - 1024;  // 1 KB per CTA is reserved by the runtime
    int cap = (share - L::fixed_bytes) / (stages * C * 4);
    if (tune(kTuneKa4Cap) > 0) cap = tune(kTuneKa4Cap);
    const int cap_max = (dev.smem_optin - L::fixed_bytes) / (stages * C * 4);
    if (cap > cap_max) cap = cap_max;
    if (cap > 1024) cap = 1024;
    if (cap < 16) return false;
    const int smem = L::fixed_bytes + stages * cap * C * 4;
    // opt in once per (instantiation, device) to the device maximum: the same value from every host thread
    static std::atomic<unsigned long long> optin_done{0};
    int cur_dev = 0;
    cudaGetDevice(&cur_dev);
    if (cur_dev < 0 || cur_dev >= 64 || !((optin_done.load(std::memory_order_relaxed) >> cur_dev) & 1ull)) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dev.smem_optin) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        if (cur_dev >= 0 && cur_dev < 64) optin_done.fetch_or(1ull << cur_dev, std::memory_order_relaxed);
    }
    static thread_local int occ_smem = -1, occ = 0;
    if (occ_smem != smem) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, (NW + 1) * 32, smem) != cudaSuccess || occ < 1) {
            cudaGetLastError();
            return false;
        }
        occ_smem = smem;
    }
    CUtensorMap ref_map;
    if (!make_ref_map(&ref_map, p.ref, p.B, p.H, p.W, C, NW)) return false;
    wc4::Params4 q;
    q.p = p;
    q.ntx = (p.W + wc4::kTW - 1) / wc4::kTW;
    q.nty = (p.H + NW - 1) / NW;
    q.nd = (p.D + wc4::kDItem - 1) / wc4::kDItem;
    const long long items = (long long)q.ntx * q.nty * q.nd * p.B;
    if (items > 0x7fffffffLL) return false;
    q.nitems = (int)items;
    q.cap = cap;
    q.stages = stages;
    long long grid = (long long)dev.sms * occ;
    if (tune(kTuneKa4Grid) > 0) grid = tune(kTuneKa4Grid);
    if (grid > items) grid = items;
    kern<<<(unsigned)grid, (NW + 1) * 32, smem, st>>>(q, m, sims_out, ref_map);
    return true;
}

template <int C, int G, int EPI>
bool launch_wc4(const WarpCorrParams &p, const MlpParams &m, float *sims_out, cudaStream_t st) {
    if (!wc4_accepts(p)) return false;
    const int nw = tune(kTuneKa4Nw) > 0 ? tune(kTuneKa4Nw) : 4;
    if (nw == 8) return launch_wc4_nw<C, G, EPI, 8, 2>(p, m, sims_out, st);
    return launch_wc4_nw<C, G, EPI, 4, 3>(p, m, sims_out, st);
}

// K-A dispatch: generation 4 unless the knob or the shape says otherwise
template <int C, int G, int EPI>
void launch_ka(const WarpCorrParams &p, const MlpParams &m, float *sims_out, cudaStream_t st) {
    if (tune(kTuneKaGen) != 3 && launch_wc4<C, G, EPI>(p, m, sims_out, st)) return;
    launch_wc3_auto<C, G, EPI>(p, m, sims_out, st);
}

}  // namespace

// ==========================================================================================
// C ABI
// ==========================================================================================

extern "C" {

// shared with pm_backward.cu (not part of the public header)
int pmb200_internal_fail(int code, const char *msg) { return fail(code, msg); }
int pmb200_internal_launch_status(const char *what) { return launch_status(what); }
int pmb200_internal_tuning(const char *key) {
    for (int i = 0; i < kTuneCount; ++i)
        if (strcmp(key, kTuneNames[i]) == 0) return tune((Tune)i);
    return 0;
}

int pmb200_abi_version(void) { return PMB200_ABI_VERSION; }

int pmb200_set_tuning(const char *key, int value) {
    if (!key) return fail(PMB200_EINVAL, "set_tuning: null key");
    if (strcmp(key, "reset") == 0) {
        for (int i = 0; i < kTuneCount; ++i) __atomic_store_n(&g_tune[i], kTuneDefaults[i], __ATOMIC_RELAXED);
        return 0;
    }
    for (int i = 0; i < kTuneCount; ++i)
        if (strcmp(key, kTuneNames[i]) == 0) {
            __atomic_store_n(&g_tune[i], value, __ATOMIC_RELAXED);
            return 0;
        }
    return fail(PMB200_EINVAL, "set_tuning: unknown key");
}

const char *pmb200_last_error(void) { return g_err; }

int pmb200_relative_projection(const float *ref_proj, int64_t ref_batch_stride, const float *const *src_projs_host,
                               int64_t src_batch_stride, int V, int B, float *rt_out, void *stream) {
    if (!ref_proj || !src_projs_host || !rt_out) return fail(PMB200_EINVAL, "relative_projection: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1) return fail(PMB200_EINVAL, "relative_projection: bad V or B");
    ProjParams p;
    p.ref = ref_proj;
    for (int v = 0; v < V; ++v) {
        if (!src_projs_host[v]) return fail(PMB200_EINVAL, "relative_projection: null source matrix");
        p.src.p[v] = src_projs_host[v];
    }
    p.out = rt_out;
    p.ref_stride = ref_batch_stride;
    p.src_stride = src_batch_stride;
    p.V = V;
    p.B = B;
    const int total = V * B;
    relative_projection_kernel<<<(total + 63) / 64, 64, 0, as_stream(stream)>>>(p);
    return launch_status("relative_projection");
}

int pmb200_pack_nhwc(const float *const *maps_host, int n, int B, int C, int H, int W, float *out_nhwc,
                     void *stream) {
    if (!maps_host || !out_nhwc) return fail(PMB200_EINVAL, "pack_nhwc: null pointer");
    if (n < 1 || n > PMB200_MAX_VIEWS + 1 || B < 1 || C < 1 || H < 1 || W < 1)
        return fail(PMB200_EINVAL, "pack_nhwc: bad size");
    if ((long long)n * B > 65535) return fail(PMB200_EINVAL, "pack_nhwc: n*B exceeds grid.z");
    PackParams p;
    for (int i = 0; i < n; ++i) {
        if (!maps_host[i]) return fail(PMB200_EINVAL, "pack_nhwc: null map");
        p.maps.p[i] = maps_host[i];
    }
    p.out = out_nhwc;
    p.n = n;
    p.B = B;
    p.C = C;
    p.HW = H * W;
    dim3 grid((p.HW + 31) / 32, (C + 31) / 32, n * B);
    pack_nhwc_kernel<<<grid, dim3(32, 8), 0, as_stream(stream)>>>(p);
    return launch_status("pack_nhwc");
}

int pmb200_photometric_confidence(const float *prob, float *confidence_out, int B, int D, int h, int w, int H_out,
                                  int W_out, void *stream) {
    if (!prob || !confidence_out) return fail(PMB200_EINVAL, "photometric_confidence: null pointer");
    if (B < 1 || D < 1 || h < 1 || w < 1 || H_out < 1 || W_out < 1) return fail(PMB200_EINVAL, "photometric_confidence: bad size");
    const size_t total = (size_t)B * H_out * W_out;
    photometric_confidence_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(prob, confidence_out, B, D, h, w,
                                                                                                H_out, W_out);
    return launch_status("photometric_confidence");
}

int pmb200_upsample2x_add_nhwc(const float *x_nhwc, const float *y_nhwc, const float *bias, float *out_nhwc, int N, int h,
                               int w, int C, void *stream) {
    if (!x_nhwc || !y_nhwc || !out_nhwc) return fail(PMB200_EINVAL, "upsample2x_add_nhwc: null pointer");
    if (N < 1 || h < 1 || w < 1 || C < 4 || C % 4 != 0) return fail(PMB200_EINVAL, "upsample2x_add_nhwc: bad size (C % 4 == 0)");
    const size_t total = (size_t)N * 2 * h * 2 * w * (C / 4);
    upsample2x_add_nhwc_kernel<<<(unsigned)((total + 255) / 256), 256, 0, as_stream(stream)>>>(
        reinterpret_cast<const float4 *>(x_nhwc), reinterpret_cast<const float4 *>(y_nhwc),
        reinterpret_cast<const float4 *>(bias), reinterpret_cast<float4 *>(out_nhwc), N, h, w, C / 4);
    return launch_status("upsample2x_add_nhwc");
}

int pmb200_warp_corr(const float *ref_nhwc, const float *src_nhwc, const float *rt, const float *depth,
                     const float *view_weights, float *out, int V, int B, int C, int G, int H, int W, int Hs,
                     int Ws, int D, void *stream) {
    if (!ref_nhwc || !src_nhwc || !rt || !depth || !out) return fail(PMB200_EINVAL, "warp_corr: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || H < 1 || W < 1 || Hs < 1 || Ws < 1 || D < 1)
        return fail(PMB200_EINVAL, "warp_corr: bad size");
    if (C < 1 || G < 1 || C % G != 0) return fail(PMB200_EINVAL, "warp_corr: C must be a multiple of G");
    if ((long long)Hs * Ws >= (1LL << pm::kKeyDxShift)) return fail(PMB200_EINVAL, "warp_corr: source map too large");
    if (C % 8 == 0 && (misaligned32(ref_nhwc) || misaligned32(src_nhwc)))
        return fail(PMB200_EINVAL, "warp_corr: feature packs must be 32-byte aligned (256-bit loads)");
    if ((long long)V * B * Hs * Ws * C / 4 >= (1LL << 31)) return fail(PMB200_EINVAL, "warp_corr: source pack too large (32-bit tap indices)");
    WarpCorrParams p;
    p.ref = ref_nhwc; p.src = src_nhwc; p.rt = rt; p.depth = depth; p.vw = view_weights; p.out = out;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = Hs; p.Ws = Ws; p.D = D;
    // F.grid_sample(align_corners=True) maps the normalised coordinate onto the *source* extent
    p.sx = (W > 1) ? (float)(Ws - 1) / (float)(W - 1) : 1.0f;
    p.sy = (H > 1) ? (float)(Hs - 1) / (float)(H - 1) : 1.0f;
    const int HW = H * W;
    cudaStream_t st = as_stream(stream);
    const bool fused = view_weights != nullptr;
    if ((D + 3) / 4 > 65535) return fail(PMB200_EINVAL, "warp_corr: too many hypotheses");
#define PMB200_LAUNCH_WC(CC, GG)                                                                   \
    do {                                                                                           \
        if (fused) launch_ka<CC, GG, kEpiAgg>(p, MlpParams(), nullptr, st);                        \
        else launch_ka<CC, GG, kEpiSims>(p, MlpParams(), nullptr, st);                             \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_WC(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_WC(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_WC(16, 4);
    else {
        const size_t total = (size_t)B * D * HW;
        warp_corr_generic_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(p, C, G);
    }
#undef PMB200_LAUNCH_WC
    return launch_status("warp_corr");
}

namespace {
int warp_corr_head(const char *what, int epi, const float *ref_nhwc, const float *src_nhwc, const float *rt,
                   const float *depth, const float *view_weights, const pmb200_mlp *head_host, float *out,
                   float *sims_out, int out_stride, int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D,
                   void *stream) {
    if (!ref_nhwc || !src_nhwc || !rt || !depth || !out || !head_host) return fail(PMB200_EINVAL, "warp_corr head: null pointer");
    if (epi == kEpiScore && !view_weights) return fail(PMB200_EINVAL, "warp_corr_score: view_weights missing");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || H < 1 || W < 1 || Hs < 1 || Ws < 1 || D < 1)
        return fail(PMB200_EINVAL, "warp_corr head: bad size");
    if ((long long)Hs * Ws >= (1LL << pm::kKeyDxShift)) return fail(PMB200_EINVAL, "warp_corr head: source map too large");
    if (misaligned32(ref_nhwc) || misaligned32(src_nhwc))
        return fail(PMB200_EINVAL, "warp_corr head: feature packs must be 32-byte aligned (256-bit loads)");
    if ((long long)V * B * Hs * Ws * C / 4 >= (1LL << 31)) return fail(PMB200_EINVAL, "warp_corr head: source pack too large (32-bit tap indices)");
    WarpCorrParams p;
    p.ref = ref_nhwc; p.src = src_nhwc; p.rt = rt; p.depth = depth; p.vw = view_weights; p.out = out;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = Hs; p.Ws = Ws; p.D = D;
    p.sx = (W > 1) ? (float)(Ws - 1) / (float)(W - 1) : 1.0f;
    p.sy = (H > 1) ? (float)(Hs - 1) / (float)(H - 1) : 1.0f;
    p.ostride = out_stride < 1 ? 1 : out_stride;
    const MlpParams m = to_device_layout(head_host);
    const int HW = H * W;
    cudaStream_t st = as_stream(stream);
    if ((D + 3) / 4 > 65535) return fail(PMB200_EINVAL, "warp_corr head: too many hypotheses");
    if (epi == kEpiViewW) {  // atomic max target starts at 0 (weights are sigmoids, > 0)
        cudaError_t e = cudaMemsetAsync(out, 0, (size_t)B * V * HW * sizeof(float), st);
        if (e != cudaSuccess) return fail((int)e, "warp_corr_view_weights: memset failed");
    }
#define PMB200_LAUNCH_WH(CC, GG)                                                                   \
    do {                                                                                           \
        if (epi == kEpiScore) launch_ka<CC, GG, kEpiScore>(p, m, nullptr, st);                     \
        else launch_ka<CC, GG, kEpiViewW>(p, m, sims_out, st);                                     \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_WH(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_WH(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_WH(16, 4);
    else return fail(PMB200_EUNSUPPORTED, "warp_corr head: fused heads exist for (C,G) in {(64,8),(32,8),(16,4)} only");
#undef PMB200_LAUNCH_WH
    return launch_status(what);
}
}  // namespace

int pmb200_warp_corr_score(const float *ref_nhwc, const float *src_nhwc, const float *rt, const float *depth,
                           const float *view_weights, const pmb200_mlp *head_host, float *score_out, int score_stride,
                           int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D, void *stream) {
    return warp_corr_head("warp_corr_score", kEpiScore, ref_nhwc, src_nhwc, rt, depth, view_weights, head_host, score_out,
                          nullptr, score_stride, V, B, C, G, H, W, Hs, Ws, D, stream);
}

int pmb200_warp_corr_view_weights(const float *ref_nhwc, const float *src_nhwc, const float *rt, const float *depth,
                                  const pmb200_mlp *head_host, float *view_weights_out, float *sims_out, int V, int B,
                                  int C, int G, int H, int W, int Hs, int Ws, int D, void *stream) {
    return warp_corr_head("warp_corr_view_weights", kEpiViewW, ref_nhwc, src_nhwc, rt, depth, nullptr, head_host,
                          view_weights_out, sims_out, 1, V, B, C, G, H, W, Hs, Ws, D, stream);
}

namespace {
// The three *_views entry points: K-A over a ragged source pack, one extent per view.  epi: kEpiSims / kEpiAgg (no head;
// kEpiAgg when view_weights is given), kEpiScore, kEpiViewW.  Every check runs before anything is written.
int warp_corr_views(const char *what, int epi, const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                    const float *rt, const float *depth, const float *view_weights, const pmb200_mlp *head_host, float *out,
                    float *sims_out, int out_stride, int V, int B, int C, int G, int H, int W, int D, void *stream) {
    const bool head = epi == kEpiScore || epi == kEpiViewW;
    if (!ref_nhwc || !src_flat || !views_host || !rt || !depth || !out || (head && !head_host))
        return fail(PMB200_EINVAL, "warp_corr views: null pointer");
    if (epi == kEpiScore && !view_weights) return fail(PMB200_EINVAL, "warp_corr_score_views: view_weights missing");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || B > 65535 || H < 1 || W < 1 || D < 1 || (D + 3) / 4 > 65535)
        return fail(PMB200_EINVAL, "warp_corr views: bad size");
    if (C < 1 || G < 1 || C % G != 0) return fail(PMB200_EINVAL, "warp_corr views: C must be a multiple of G");
    const bool fast = (C == 64 && G == 8) || (C == 32 && G == 8) || (C == 16 && G == 4);
    if (head && !fast) return fail(PMB200_EUNSUPPORTED, "warp_corr views: fused heads exist for (C,G) in {(64,8),(32,8),(16,4)} only");
    if (fast && (misaligned32(ref_nhwc) || misaligned32(src_flat)))
        return fail(PMB200_EINVAL, "warp_corr views: feature packs must be 32-byte aligned (256-bit loads)");
    ViewTable vt;
    for (int v = 0; v < V; ++v) {
        const pmb200_view_extent &e = views_host[v];
        if (e.height < 1 || e.width < 1) return fail(PMB200_EINVAL, "warp_corr views: a view has a non-positive size");
        if ((long long)e.height * e.width >= (1LL << pm::kKeyDxShift)) return fail(PMB200_EINVAL, "warp_corr views: source map too large");
        if (e.offset < 0 || e.offset % 4 != 0) return fail(PMB200_EINVAL, "warp_corr views: offsets must be non-negative multiples of 4 floats");
        if (e.offset / 4 >= (1LL << 31) || (e.offset + (long long)B * e.height * e.width * C) / 4 >= (1LL << 31))
            return fail(PMB200_EINVAL, "warp_corr views: source pack too large (32-bit tap indices)");
        vt.base4[v] = (unsigned)(e.offset / 4);
        vt.hs[v] = e.height;
        vt.ws[v] = e.width;
        // F.grid_sample(align_corners=True) maps the normalised coordinate onto each source's own extent
        vt.sx[v] = (W > 1) ? (float)(e.width - 1) / (float)(W - 1) : 1.0f;
        vt.sy[v] = (H > 1) ? (float)(e.height - 1) / (float)(H - 1) : 1.0f;
    }
    WarpCorrParams p;
    p.ref = ref_nhwc; p.src = src_flat; p.rt = rt; p.depth = depth; p.vw = view_weights; p.out = out;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = vt.hs[0]; p.Ws = vt.ws[0]; p.D = D;
    p.sx = vt.sx[0]; p.sy = vt.sy[0];
    p.ostride = out_stride < 1 ? 1 : out_stride;
    const MlpParams m = head ? to_device_layout(head_host) : MlpParams();
    cudaStream_t st = as_stream(stream);
    if (epi == kEpiViewW) {  // atomic max target starts at 0 (weights are sigmoids, > 0)
        cudaError_t e = cudaMemsetAsync(out, 0, (size_t)B * V * H * W * sizeof(float), st);
        if (e != cudaSuccess) return fail((int)e, "warp_corr_view_weights_views: memset failed");
    }
    if (epi == kEpiSims && view_weights) epi = kEpiAgg;
#define PMB200_LAUNCH_WV(CC, GG)                                                                   \
    do {                                                                                           \
        if (epi == kEpiSims) launch_wc3_views<CC, GG, kEpiSims>(p, vt, m, nullptr, st);            \
        else if (epi == kEpiAgg) launch_wc3_views<CC, GG, kEpiAgg>(p, vt, m, nullptr, st);         \
        else if (epi == kEpiScore) launch_wc3_views<CC, GG, kEpiScore>(p, vt, m, nullptr, st);     \
        else launch_wc3_views<CC, GG, kEpiViewW>(p, vt, m, sims_out, st);                          \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_WV(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_WV(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_WV(16, 4);
    else {
        const size_t total = (size_t)B * D * H * W;
        warp_corr_generic_views_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(p, vt, C, G);
    }
#undef PMB200_LAUNCH_WV
    return launch_status(what);
}
}  // namespace

int pmb200_warp_corr_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host, const float *rt,
                           const float *depth, const float *view_weights, float *out, int V, int B, int C, int G, int H, int W,
                           int D, void *stream) {
    return warp_corr_views("warp_corr_views", kEpiSims, ref_nhwc, src_flat, views_host, rt, depth, view_weights, nullptr, out,
                           nullptr, 1, V, B, C, G, H, W, D, stream);
}

int pmb200_warp_corr_score_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                 const float *rt, const float *depth, const float *view_weights, const pmb200_mlp *head_host,
                                 float *score_out, int score_stride, int V, int B, int C, int G, int H, int W, int D,
                                 void *stream) {
    return warp_corr_views("warp_corr_score_views", kEpiScore, ref_nhwc, src_flat, views_host, rt, depth, view_weights, head_host,
                           score_out, nullptr, score_stride, V, B, C, G, H, W, D, stream);
}

int pmb200_warp_corr_view_weights_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                        const float *rt, const float *depth, const pmb200_mlp *head_host,
                                        float *view_weights_out, float *sims_out, int V, int B, int C, int G, int H, int W,
                                        int D, void *stream) {
    return warp_corr_views("warp_corr_view_weights_views", kEpiViewW, ref_nhwc, src_flat, views_host, rt, depth, nullptr,
                           head_host, view_weights_out, sims_out, 1, V, B, C, G, H, W, D, stream);
}

int pmb200_aggregate_views_score(const float *sims, const float *view_weights, const pmb200_mlp *head_host,
                                 float *score_out, int score_stride, int V, int B, int G, int D, int H, int W,
                                 void *stream) {
    if (!sims || !view_weights || !head_host || !score_out) return fail(PMB200_EINVAL, "aggregate_views_score: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || D < 1 || H < 1 || W < 1)
        return fail(PMB200_EINVAL, "aggregate_views_score: bad size");
    const MlpParams m = to_device_layout(head_host);
    const size_t total = (size_t)B * D * H * W;
    const unsigned blocks = (unsigned)((total + 127) / 128);
    const int os = score_stride < 1 ? 1 : score_stride;
    if (G == 8) aggregate_score_kernel<8><<<blocks, 128, 0, as_stream(stream)>>>(sims, view_weights, score_out, m, V, B, D, H * W, os);
    else if (G == 4) aggregate_score_kernel<4><<<blocks, 128, 0, as_stream(stream)>>>(sims, view_weights, score_out, m, V, B, D, H * W, os);
    else return fail(PMB200_EUNSUPPORTED, "aggregate_views_score: G must be 4 or 8");
    return launch_status("aggregate_views_score");
}

int pmb200_offset_corr_weight(const float *ref_nhwc, const float *offsets, int offsets_channels_last,
                              const pmb200_mlp *head_host, float *weight_out, int B, int C, int G, int H, int W, int K,
                              int dilation, void *stream) {
    if (!ref_nhwc || !offsets || !weight_out || !head_host) return fail(PMB200_EINVAL, "offset_corr_weight: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2) return fail(PMB200_EINVAL, "offset_corr_weight: bad size");
    if (K != 9 && K != 17) return fail(PMB200_EUNSUPPORTED, "offset_corr_weight: evaluate_neighbors must be 9 or 17");
    if ((long long)H * W >= (1LL << pm::kKeyDxShift)) return fail(PMB200_EINVAL, "offset_corr_weight: map too large");
    if (misaligned32(ref_nhwc)) return fail(PMB200_EINVAL, "offset_corr_weight: feature pack must be 32-byte aligned (256-bit loads)");
    OffsetCorrParams p;
    p.ref = ref_nhwc; p.offsets = offsets; p.out = weight_out;
    p.B = B; p.H = H; p.W = W; p.K = K; p.dilation = dilation; p.off_nhwc = offsets_channels_last ? 1 : 0;
    const MlpParams m = to_device_layout(head_host);
    const int HW = H * W;
    cudaStream_t st = as_stream(stream);
    const int nchunk = (K + kChunk - 1) / kChunk;
#define PMB200_LAUNCH_OW(CC, GG)                                                                   \
    do {                                                                                           \
        dim3 grid((HW + kWarpsPerBlock * LaneMap<CC, GG>::PPW - 1) / (kWarpsPerBlock * LaneMap<CC, GG>::PPW), \
                  nchunk, B);                                                                      \
        offset_corr_kernel<CC, GG, true><<<grid, kWarpsPerBlock * 32, 0, st>>>(p, m);              \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_OW(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_OW(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_OW(16, 4);
    else return fail(PMB200_EUNSUPPORTED, "offset_corr_weight: fused head exists for (C,G) in {(64,8),(32,8),(16,4)} only");
#undef PMB200_LAUNCH_OW
    return launch_status("offset_corr_weight");
}

int pmb200_aggregate_views(const float *sims, const float *view_weights, float *out, int V, int B, int G, int D,
                           int H, int W, void *stream) {
    if (!sims || !view_weights || !out) return fail(PMB200_EINVAL, "aggregate_views: null pointer");
    if (V < 1 || V > PMB200_MAX_VIEWS || B < 1 || G < 1 || D < 1 || H < 1 || W < 1)
        return fail(PMB200_EINVAL, "aggregate_views: bad size");
    const size_t total = (size_t)B * G * D * H * W;
    size_t blocks = (total + 255) / 256;
    const size_t max_blocks = (size_t)(device_facts().sms > 0 ? device_facts().sms : 1) * 16;
    if (blocks > max_blocks) blocks = max_blocks;
    aggregate_views_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(sims, view_weights, out, V, B, G * D, H * W);
    return launch_status("aggregate_views");
}

int pmb200_offset_corr(const float *ref_nhwc, const float *offsets, int offsets_channels_last, float *out, int B, int C,
                       int G, int H, int W, int K, int dilation, void *stream) {
    if (!ref_nhwc || !offsets || !out) return fail(PMB200_EINVAL, "offset_corr: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2) return fail(PMB200_EINVAL, "offset_corr: bad size");
    if (C < 1 || G < 1 || C % G != 0) return fail(PMB200_EINVAL, "offset_corr: C must be a multiple of G");
    if (K != 9 && K != 17) return fail(PMB200_EUNSUPPORTED, "offset_corr: evaluate_neighbors must be 9 or 17");
    if ((long long)H * W >= (1LL << pm::kKeyDxShift)) return fail(PMB200_EINVAL, "offset_corr: map too large");
    if (C % 8 == 0 && misaligned32(ref_nhwc)) return fail(PMB200_EINVAL, "offset_corr: feature pack must be 32-byte aligned (256-bit loads)");
    OffsetCorrParams p;
    p.ref = ref_nhwc; p.offsets = offsets; p.out = out;
    p.B = B; p.H = H; p.W = W; p.K = K; p.dilation = dilation; p.off_nhwc = offsets_channels_last ? 1 : 0;
    const int HW = H * W;
    cudaStream_t st = as_stream(stream);
    const int nchunk = (K + kChunk - 1) / kChunk;
#define PMB200_LAUNCH_OC(CC, GG)                                                                   \
    do {                                                                                           \
        dim3 grid((HW + kWarpsPerBlock * LaneMap<CC, GG>::PPW - 1) / (kWarpsPerBlock * LaneMap<CC, GG>::PPW), \
                  nchunk, B);                                                                      \
        offset_corr_kernel<CC, GG, false><<<grid, kWarpsPerBlock * 32, 0, st>>>(p, MlpParams());                       \
    } while (0)
    if (C == 64 && G == 8) PMB200_LAUNCH_OC(64, 8);
    else if (C == 32 && G == 8) PMB200_LAUNCH_OC(32, 8);
    else if (C == 16 && G == 4) PMB200_LAUNCH_OC(16, 4);
    else {
        const size_t total = (size_t)B * K * HW;
        offset_corr_generic_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(p, C, G);
    }
#undef PMB200_LAUNCH_OC
    return launch_status("offset_corr");
}

int pmb200_init_propagate(const float *seed_map, const float *offsets, int offsets_channels_last, const float *depth_min,
                          const float *depth_max, float *out, float *xnorm_out, int xnorm_stride, int mode, int B, int H,
                          int W, int Ns, int Kp, int dilation, float interval_scale, void *stream) {
    if (!seed_map || !depth_min || !depth_max || !out) return fail(PMB200_EINVAL, "init_propagate: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2 || Ns < 1) return fail(PMB200_EINVAL, "init_propagate: bad size");
    if (mode < 0 || mode > 2) return fail(PMB200_EINVAL, "init_propagate: bad mode");
    if (mode == 0 && Ns != 48) return fail(PMB200_EINVAL, "init_propagate: random init has 48 samples");
    if (mode == 2 && Ns != 1) return fail(PMB200_EINVAL, "init_propagate: passthrough needs Ns == 1");
    if (Kp != 0 && Kp != 4 && Kp != 8 && Kp != 16)
        return fail(PMB200_EUNSUPPORTED, "init_propagate: propagate_neighbors must be 0, 4, 8 or 16");
    if (Kp > 0 && !offsets) return fail(PMB200_EINVAL, "init_propagate: offsets missing");
    if (Ns + Kp > PMB200_MAX_HYPOTHESES) return fail(PMB200_EINVAL, "init_propagate: too many hypotheses");
    PropParams p;
    p.seed = seed_map; p.offsets = offsets; p.dmin = depth_min; p.dmax = depth_max; p.out = out; p.xnorm = xnorm_out;
    p.xstride = xnorm_stride < 1 ? 1 : xnorm_stride;
    p.off_nhwc = offsets_channels_last ? 1 : 0;
    p.mode = mode; p.B = B; p.H = H; p.W = W; p.Ns = Ns; p.Kp = Kp; p.dilation = dilation;
    p.interval_scale = interval_scale;
    const int HW = H * W, D = Ns + Kp;
    cudaStream_t st = as_stream(stream);
    dim3 grid((HW + 127) / 128, B);
    auto warp_grid = [&](int lanes_per_pixel) {  // 4 warps per block, 32/lanes_per_pixel pixels per warp
        const int pix_per_block = 4 * (32 / lanes_per_pixel);
        return dim3((HW + pix_per_block - 1) / pix_per_block, B);
    };
    if (Kp == 0 && D <= 64) init_only_kernel<<<grid, 128, 0, st>>>(p);
    else if (D <= 8) init_propagate_kernel<8><<<warp_grid(8), 128, 0, st>>>(p);
    else if (D <= 16) init_propagate_kernel<16><<<warp_grid(16), 128, 0, st>>>(p);
    else if (D <= 32) init_propagate_kernel<32><<<warp_grid(32), 128, 0, st>>>(p);
    else if (D <= 64) init_propagate_kernel<64><<<warp_grid(32), 128, 0, st>>>(p);
    else init_propagate_generic_kernel<<<grid, 128, 0, st>>>(p);
    return launch_status("init_propagate");
}

int pmb200_adaptive_eval(const float *score0, const float *depth_sample, const float *xnorm, const float *xnorm_score,
                         const float *offsets, int offsets_channels_last, const float *feature_weight, const float *depth_min,
                         const float *depth_max, float *prob_out, float *depth_out, int B, int D, int H, int W, int K,
                         int dilation, float interval_scale, int is_inverse, void *stream) {
    if ((!score0 && !xnorm_score) || !depth_sample || !offsets || !feature_weight || !depth_min || !depth_max || !prob_out ||
        !depth_out)
        return fail(PMB200_EINVAL, "adaptive_eval: null pointer");
    if (B < 1 || B > 65535 || H < 2 || W < 2 || D < 1 || D > PMB200_MAX_HYPOTHESES)
        return fail(PMB200_EINVAL, "adaptive_eval: bad size");
    if (K != 9 && K != 17) return fail(PMB200_EUNSUPPORTED, "adaptive_eval: evaluate_neighbors must be 9 or 17");
    if (is_inverse && D < 2) return fail(PMB200_EINVAL, "adaptive_eval: inverse regression needs D >= 2");
    EvalParams p;
    p.score0 = score0; p.depth = depth_sample; p.xnorm = xnorm; p.offsets = offsets; p.fw = feature_weight;
    p.xs = reinterpret_cast<const float2 *>(xnorm_score);
    p.off_nhwc = offsets_channels_last ? 1 : 0;
    p.dmin = depth_min; p.dmax = depth_max; p.prob = prob_out; p.depth_out = depth_out;
    p.B = B; p.D = D; p.H = H; p.W = W; p.K = K; p.dilation = dilation; p.is_inverse = is_inverse;
    p.interval_scale = interval_scale;
    const int HW = H * W;
    // Block shape: large maps want 32 pixels x few hypothesis lanes (each thread then walks D/DY hypotheses with the
    // footprints it already decoded), small maps 16 pixels x 16 lanes so that the grid still covers every SM twice.
    int TP = 32, DY = D <= 16 ? (D < 4 ? D : 4) : 8;
    if ((long long)((HW + 31) / 32) * B < 2LL * device_facts().sms) {
        TP = 16;
        DY = D < 16 ? D : 16;
    }
    auto smem_for = [&](int tp) { return (size_t)K * tp * (sizeof(float4) + sizeof(int) + sizeof(float)) + 2 * (size_t)D * tp * sizeof(float); };
    if (smem_for(TP) > 48 * 1024) {  // many hypotheses: fewer pixels per block keeps the tile under the default 48 KB
        TP = 8;
        DY = D < 32 ? D : 32;
    }
    {   // measurement aid (tools/kbench.py): kb_tp / kb_dy override the block shape
        const int etp = tune(kTuneKbTp), edy = tune(kTuneKbDy);
        if (etp > 0 && edy > 0 && etp * edy <= 256 && smem_for(etp) <= 48 * 1024) {
            TP = etp;
            DY = edy < D ? edy : D;
        }
    }
    const size_t smem = smem_for(TP);
    dim3 grid((HW + TP - 1) / TP, B);
    if (K == 9) adaptive_eval_kernel<9><<<grid, dim3(TP, DY), smem, as_stream(stream)>>>(p);
    else adaptive_eval_kernel<17><<<grid, dim3(TP, DY), smem, as_stream(stream)>>>(p);
    return launch_status("adaptive_eval");
}

}  // extern "C"
#endif  // !PM_EMU
