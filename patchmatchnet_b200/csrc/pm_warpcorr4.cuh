// pm_warpcorr4.cuh -- K-A, fourth generation: the fused warp + correlation kernel as a persistent, warp-specialised
// pipeline over shared-memory windows staged by the TMA engine (sm_90a).  Included by pm_kernels.cu inside its anonymous
// namespace, after MlpParams / WarpCorrParams / mlp_eval / ffma2.
//
// Reference: models/module.py:130-181 (differentiable_warping), models/patchmatch.py:192-217 (group-wise correlation and
// view-weighted aggregation), :547-549 / :690-702 (the 1x1x1 heads, eval mode, BatchNorm folded).
//
// Decomposition (DESIGN.md "K-A generation 4"):
//   item      = 8 x NW reference pixels (one tile row of 8 pixels per consumer warp) x 8 consecutive hypotheses x ALL views;
//               items are dealt round-robin to a persistent grid (blockIdx.x + i * gridDim.x).
//   producer  = one warp per CTA.  Per item it reads the tile's hypotheses (coalesced) into shared memory, takes their
//               min / max, bounds every view's source footprint from the tile's corner rays at those two depths, and asks
//               the TMA engine for (a) the reference-feature tile [NW][8][C] -- ONE tensor-map box, cp.async.bulk.tensor,
//               zero-filled past the map edge -- and (b) per view the source window, h rows of w texels, one bulk copy
//               (cp.async.bulk) per row with run-time extents.  Completion is signalled on mbarriers; the windows live in
//               an S-deep ring, the per-item data in a 2-deep ring, so the copies of item i+1 overlap the arithmetic of i.
//   consumers = NW warps.  Lane = (pixel 0..7 of the warp's tile row, hypothesis row 0..3), two consecutive hypotheses
//               per lane.  Per view: footprints (projection, bilinear weights, zero padding) -> the distinct source cells
//               of the warp pass are numbered densely from two ballots (consecutive hypotheses of a pixel mostly share a
//               cell) -> ONE LANE PER CELL gathers its four taps and the pixel's reference vector from shared memory
//               (LDS.128; chunk order rotated by lane so that the 8 lanes of a quarter-warp hit 8 different bank groups
//               without any swizzle arithmetic) and scatters the 4 x G tap/group dot products into a per-warp table ->
//               every footprint blends its cell's table row with its own weights -> view-weighted accumulation -> epilogue
//               (per-view similarities / weighted average / SimilarityNet head / PixelwiseNet head, as generation 3).
//   fallback  = a cell whose taps are not all inside the staged window (box larger than the ring slot, points behind the
//               camera at a tile corner, ...) is gathered from global memory by the same lane: always correct, only slower.
#pragma once

#if !defined(PM_EMU)
#include <cuda.h>
#include <cudaTypedefs.h>
#endif

namespace wc4 {

// ----------------------------------------------------------------------------------------------------------------------
// mbarrier / bulk-copy vocabulary (PTX on the device, a cooperative-fiber restatement under the CPU emulator)
// ----------------------------------------------------------------------------------------------------------------------
#if defined(PM_EMU)
struct MBar {
    int init, pending;
    long long tx;
    int phase;
};
inline void mbar_settle(MBar *b) {
    if (b->pending == 0 && b->tx == 0) {
        b->phase ^= 1;
        b->pending = b->init;
    }
}
inline void mbar_init(MBar *b, int count) { b->init = b->pending = count; b->tx = 0; b->phase = 0; }
inline void mbar_fence_init() {}
inline void mbar_arrive(MBar *b) { --b->pending; mbar_settle(b); }
inline void mbar_arrive_expect_tx(MBar *b, unsigned bytes) { b->tx += bytes; --b->pending; mbar_settle(b); }
inline void mbar_complete_tx(MBar *b, unsigned bytes) { b->tx -= bytes; mbar_settle(b); }
inline void mbar_wait(MBar *b, unsigned parity) {  // returns once the phase with this parity has completed
    for (long spin = 0; (unsigned)b->phase == parity; ++spin) {
        assert(spin < (1L << 26) && "emulated mbarrier wait never satisfied (pipeline deadlock)");
        emu::yield();
    }
}
inline void mbar_wait_backoff(MBar *b, unsigned parity) { mbar_wait(b, parity); }
inline void bulk_row_g2s(float *dst, const float *src, unsigned bytes, MBar *b) {
    assert(bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && (reinterpret_cast<uintptr_t>(dst) & 15u) == 0);
    memcpy(dst, src, bytes);
    mbar_complete_tx(b, bytes);
}
struct TensorMap {  // what the tiled tensor map describes: a channels-last [B][H][W][C] fp32 tensor, box [1][BH][8][C]
    const float *base;
    int B, H, W, C, BH;
};
inline void tma_ref_tile(float *dst, const TensorMap *tm, int x, int y, int b, MBar *bar) {
    for (int r = 0; r < tm->BH; ++r)
        for (int c = 0; c < 8; ++c)
            for (int k = 0; k < tm->C; ++k) {
                const int yy = y + r, xx = x + c;
                const bool in = yy >= 0 && yy < tm->H && xx >= 0 && xx < tm->W;
                dst[(r * 8 + c) * tm->C + k] = in ? tm->base[(((size_t)b * tm->H + yy) * tm->W + xx) * tm->C + k] : 0.0f;
            }
    mbar_complete_tx(bar, (unsigned)(tm->BH * 8 * tm->C * 4));
}
inline int clz32(unsigned v) { return v ? __builtin_clz(v) : 32; }
inline void trap_now() { abort(); }
#else
struct MBar {
    unsigned long long raw;
};
using TensorMap = CUtensorMap;
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(MBar *b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(MBar *b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(MBar *b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(MBar *b, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(b)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded: a pipeline bug must surface as a launch error (trap), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(MBar *b, unsigned parity) {
    for (int spin = 0; spin < (1 << 22); ++spin)
        if (mbar_try_wait(b, parity)) return;
    __trap();
}
// the producer's waits: it is ahead of the consumers most of the time; sleeping between polls keeps its spinning out of the
// issue slots the consumer warps of the same SM sub-partition need
__device__ __forceinline__ void mbar_wait_backoff(MBar *b, unsigned parity) {
    for (int spin = 0; spin < (1 << 22); ++spin) {
        if (mbar_try_wait(b, parity)) return;
        __nanosleep(100);
    }
    __trap();
}
// one row of a source window: `bytes` contiguous bytes (multiple of 16, 16-byte aligned on both sides)  -> SASS UBLKCP
__device__ __forceinline__ void bulk_row_g2s(float *dst, const float *src, unsigned bytes, MBar *b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(b))
                 : "memory");
}
// the reference-feature tile: one 4-D tensor-map box {C, 8, NW, 1} at (0, x, y, b), zero fill outside the map -> SASS UTMALDG
__device__ __forceinline__ void tma_ref_tile(float *dst, const TensorMap *tm, int x, int y, int b, MBar *bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<unsigned long long>(tm)), "r"(smem_u32(bar)), "r"(0), "r"(x), "r"(y), "r"(b)
        : "memory");
}
__device__ __forceinline__ int clz32(unsigned v) { return __clz((int)v); }
__device__ __forceinline__ void trap_now() { __trap(); }
#endif

// ----------------------------------------------------------------------------------------------------------------------
// shapes
// ----------------------------------------------------------------------------------------------------------------------
constexpr int kTW = 8;        // tile width in reference pixels = pixels per consumer warp
constexpr int kRows = 4;      // hypothesis rows per warp pass (32 lanes / 8 pixels)
constexpr int kNE = 2;        // consecutive hypotheses per lane
constexpr int kDItem = kRows * kNE;  // hypotheses per item (8)
constexpr int kMaxStages = 4;  // source-window ring depth is a launch parameter (2..4)
constexpr int kMaxRows = 64;  // window rows a producer warp will stage (2 bulk copies per lane)

// Footprint key of this generation: x0 | y0 << 14 | dx << 29 | dy << 30 (source maps up to 16383 x 32767).
constexpr int kXBits = 14;
constexpr int kKeyNone = pm::kKeyNone;

// Zero-padded bilinear footprint, same cases as pm::zero_pad_cell (models/module.py:170-181), (x0, y0) kept apart.
__device__ __forceinline__ int footprint(float u, float v, int rows, int cols, float4 &w) {
    const float xf = floorf(u), yf = floorf(v);
    const float fx = u - xf, fy = v - yf;
    const float gx = 1.0f - fx, gy = 1.0f - fy;
    if (xf >= 0.0f && xf < (float)(cols - 1) && yf >= 0.0f && yf < (float)(rows - 1)) {  // interior: all four taps inside
        w = make_float4(gx * gy, fx * gy, gx * fy, fx * fy);
        return (int)xf | ((int)yf << kXBits) | (1 << pm::kKeyDxShift) | (1 << pm::kKeyDyShift);
    }
    if (!(u >= -1.0f && u < (float)cols && v >= -1.0f && v < (float)rows)) {  // NaN fails both tests
        w = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        return kKeyNone;
    }
    const int x0 = (int)xf, y0 = (int)yf;
    const bool x0in = x0 >= 0, x1in = x0 + 1 <= cols - 1;
    const bool y0in = y0 >= 0, y1in = y0 + 1 <= rows - 1;
    w.x = (x0in && y0in) ? gx * gy : 0.0f;
    w.y = (x1in && y0in) ? fx * gy : 0.0f;
    w.z = (x0in && y1in) ? gx * fy : 0.0f;
    w.w = (x1in && y1in) ? fx * fy : 0.0f;
    const int x0c = x0in ? x0 : 0, y0c = y0in ? y0 : 0;
    const int dx = (x0in && x1in) ? 1 : 0, dy = (y0in && y1in) ? 1 : 0;
    return x0c | (y0c << kXBits) | (dx << pm::kKeyDxShift) | (dy << pm::kKeyDyShift);
}

struct alignas(16) WinInfo {  // written by the producer before it arms the window's barrier
    int x0, y0, w, h;  // staged box in source texels; h == 0: nothing staged (every cell takes the global path)
};

struct alignas(16) ItemInfo {
    int b, d0, tx0, ty0;
};

template <int C, int G, int NW>
struct Layout {
    static constexpr int CPG = C / G;                     // channels per group: 4 (one 16-byte chunk) or 8 (two)
    static_assert(CPG == 4 || CPG == 8, "generation 4 handles 4 or 8 channels per group");
    static constexpr int LPC = (C * 4 > 128) ? C * 4 / 128 : 1;  // lanes per cell: a lane gathers at most 32 channels
    static_assert(LPC == 1 || LPC == 2, "C must be 16, 32 or 64");
    static constexpr int NCELL = 32 / LPC;                // cells gathered per round
    static constexpr int TP = 4 * G + 4;                  // table pitch between consecutive slots (floats, 16-byte multiple)
    static constexpr int TA = 8 * TP + (G == 8 ? 8 : 4);  // pitch between groups of 8 slots: makes the scattered 4-byte
                                                          // stores of a gather round hit 32 different banks (see DESIGN.md)
    static constexpr int TABLE = 4 * TA;                  // floats per warp (32 slots)
    static constexpr int PIX = kTW * NW;                  // reference pixels per item
    // dynamic shared memory carve-up (bytes), every block 128-byte aligned
    static constexpr int oBars = 0;                                            // MBar[2*kMaxStages + 4]
    static constexpr int oWin = 384;                                           // WinInfo[kMaxStages]
    static constexpr int oItem = oWin + 16 * kMaxStages;                       // ItemInfo[2]
    static constexpr int oRt = oItem + 64;                                     // float[2][PMB200_MAX_VIEWS * 12]
    static constexpr int oDepth = oRt + 2 * PMB200_MAX_VIEWS * 12 * 4;         // float[2][kDItem * PIX]
    static constexpr int oVw = oDepth + 2 * kDItem * PIX * 4;                  // float[2][PMB200_MAX_VIEWS * PIX]
    static constexpr int oCell = oVw + 2 * PMB200_MAX_VIEWS * PIX * 4;         // int2[NW][kNE * 32]
    static constexpr int oTable = oCell + NW * kNE * 32 * 8;                   // float[NW][TABLE]
    static constexpr int oRef = (oTable + NW * TABLE * 4 + 127) / 128 * 128;   // float[2][PIX * C]
    static constexpr int oWinData = oRef + 2 * PIX * C * 4;                    // float[stages][cap * C]
    static constexpr int fixed_bytes = oWinData;
    static_assert(sizeof(MBar) * (2 * kMaxStages + 4) <= oWin && sizeof(WinInfo) == 16 && sizeof(ItemInfo) == 16, "barrier / info blocks");
    static_assert(oDepth % 128 == 0, "blocks stay 128-byte aligned");
};

struct Params4 {
    WarpCorrParams p;
    int ntx, nty, nd, nitems;
    int cap;     // texels per window slot
    int stages;  // window ring depth, 2..kMaxStages
};

// ----------------------------------------------------------------------------------------------------------------------
// gather of one cell by one lane (LPC == 1) or by one of its two lanes (LPC == 2): 4 taps x the lane's channels against
// the pixel's reference vector, results scattered into the warp's table.  `tap` are float pointers to the four texels
// (lane's channel half already applied), `ref` to the reference vector, `tb` to the slot's table row.
// ----------------------------------------------------------------------------------------------------------------------
template <int C, int G, bool GLOBAL>
__device__ __forceinline__ float4 ld4(const float *p) {
#if defined(PM_EMU)
    return *reinterpret_cast<const float4 *>(p);
#else
    if constexpr (GLOBAL) return __ldg(reinterpret_cast<const float4 *>(p));
    else return *reinterpret_cast<const float4 *>(p);
#endif
}

__device__ __forceinline__ float dot4(const float4 &a, const float4 &b, float acc) {
    const float2 s = ffma2(make_float2(a.z, a.w), make_float2(b.z, b.w), ffma2(make_float2(a.x, a.y), make_float2(b.x, b.y), make_float2(acc, 0.0f)));
    return s.x + s.y;
}

template <int C, int G, bool GLOBAL>
__device__ __forceinline__ void gather_cell(const float *t00, const float *t01, const float *t10, const float *t11,
                                            const float *ref, float *tb, int lane) {
    constexpr int CPG = C / G;
    constexpr float kScale = 1.0f / (float)CPG;  // the group mean; exact (power of two)
    if constexpr (CPG == 4) {
        constexpr int NCH = C / 4;  // 16-byte chunks = groups
        const int rot = lane & (NCH - 1);
#pragma unroll
        for (int s = 0; s < NCH; ++s) {
            const int c = (s + rot) & (NCH - 1);
            const float4 r = *reinterpret_cast<const float4 *>(ref + 4 * c);
            const float4 a = ld4<C, G, GLOBAL>(t00 + 4 * c), b = ld4<C, G, GLOBAL>(t01 + 4 * c);
            const float4 cc = ld4<C, G, GLOBAL>(t10 + 4 * c), d = ld4<C, G, GLOBAL>(t11 + 4 * c);
            tb[0 * G + c] = dot4(r, a, 0.0f) * kScale;
            tb[1 * G + c] = dot4(r, b, 0.0f) * kScale;
            tb[2 * G + c] = dot4(r, cc, 0.0f) * kScale;
            tb[3 * G + c] = dot4(r, d, 0.0f) * kScale;
        }
    } else {
        // C = 64, G = 8: this lane owns 32 channels = 4 groups of two chunks; `ref`, `t..` already point at its half.
        // The two chunks of a pair are read in opposite order by the two lanes of a cell: 8 lanes, 8 bank groups.
        const int hh = lane & 1, rot = (lane >> 1) & 3;
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const int p = (s + rot) & 3;
            const int c0 = 8 * p + 4 * hh, c1 = 8 * p + 4 * (1 - hh);
            const float4 r0 = *reinterpret_cast<const float4 *>(ref + c0), r1 = *reinterpret_cast<const float4 *>(ref + c1);
            const float4 a0 = ld4<C, G, GLOBAL>(t00 + c0), b0 = ld4<C, G, GLOBAL>(t01 + c0);
            const float4 e0 = ld4<C, G, GLOBAL>(t10 + c0), d0 = ld4<C, G, GLOBAL>(t11 + c0);
            const float4 a1 = ld4<C, G, GLOBAL>(t00 + c1), b1 = ld4<C, G, GLOBAL>(t01 + c1);
            const float4 e1 = ld4<C, G, GLOBAL>(t10 + c1), d1 = ld4<C, G, GLOBAL>(t11 + c1);
            const int g = 4 * hh + p;
            tb[0 * G + g] = dot4(r1, a1, dot4(r0, a0, 0.0f)) * kScale;
            tb[1 * G + g] = dot4(r1, b1, dot4(r0, b0, 0.0f)) * kScale;
            tb[2 * G + g] = dot4(r1, e1, dot4(r0, e0, 0.0f)) * kScale;
            tb[3 * G + g] = dot4(r1, d1, dot4(r0, d0, 0.0f)) * kScale;
        }
    }
}

// ----------------------------------------------------------------------------------------------------------------------
// the kernel
// ----------------------------------------------------------------------------------------------------------------------
template <int C, int G, int EPI, int NW, int MINB>
__global__ void __launch_bounds__((NW + 1) * 32, MINB)
warp_corr4_kernel(const Params4 q, const MlpParams mlp, float *__restrict__ sims_out, const __grid_constant__ TensorMap ref_map) {
    using L = Layout<C, G, NW>;
    constexpr bool kWeighted = (EPI == kEpiAgg || EPI == kEpiScore);
    constexpr int PIX = L::PIX;
#if defined(PM_EMU)
    char *smem = static_cast<char *>(emu::dyn_smem());
#else
    extern __shared__ __align__(128) char smem[];
#endif
    MBar *bars = reinterpret_cast<MBar *>(smem + L::oBars);
    MBar *win_full = bars, *win_empty = bars + kMaxStages, *item_full = bars + 2 * kMaxStages, *item_empty = bars + 2 * kMaxStages + 2;
    WinInfo *s_win = reinterpret_cast<WinInfo *>(smem + L::oWin);
    ItemInfo *s_item = reinterpret_cast<ItemInfo *>(smem + L::oItem);
    float *s_rt = reinterpret_cast<float *>(smem + L::oRt);
    float *s_depth = reinterpret_cast<float *>(smem + L::oDepth);
    float *s_vw = reinterpret_cast<float *>(smem + L::oVw);
    float *s_ref = reinterpret_cast<float *>(smem + L::oRef);
    float *s_data = reinterpret_cast<float *>(smem + L::oWinData);

    const WarpCorrParams &p = q.p;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int HW = p.H * p.W;
    const unsigned full = 0xffffffffu;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kMaxStages; ++s) {
            mbar_init(&win_full[s], 1);
            mbar_init(&win_empty[s], NW);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(&item_full[s], 1);
            mbar_init(&item_empty[s], NW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == NW) {
        // ===================================================== producer =====================================================
        // Software pipeline: the hypotheses / view weights of item i+1 are fetched into registers while the windows of item i
        // are being issued, so the global-load latency of the per-item data never sits in front of a TMA request.
        constexpr int ND = kDItem * PIX / 32;            // hypotheses per lane
        constexpr int NV = PMB200_MAX_VIEWS * PIX / 32;  // view weights per lane (at most)
        float dreg[ND], vreg[kWeighted ? NV : 1];
        auto decode = [&](int it, int &b, int &d0, int &tx0, int &ty0) {
            int rem = it;
            const int tx = rem % q.ntx; rem /= q.ntx;
            const int ty = rem % q.nty; rem /= q.nty;
            const int dc = rem % q.nd;
            b = rem / q.nd; d0 = dc * kDItem; tx0 = tx * kTW; ty0 = ty * NW;
        };
        auto prefetch = [&](int it) {
            int b, d0, tx0, ty0;
            decode(it, b, d0, tx0, ty0);
#pragma unroll
            for (int j = 0; j < ND; ++j) {
                const int idx = lane + 32 * j, dl = idx / PIX, pix = idx % PIX;
                const int y = ty0 + pix / kTW, x = tx0 + pix % kTW, d = d0 + dl;
                // NaN marks "no hypothesis here" (outside the map / past D): excluded from the range, stored as 1.0
                dreg[j] = (y < p.H && x < p.W && d < p.D) ? __ldg(p.depth + ((size_t)b * p.D + d) * HW + (size_t)y * p.W + x)
                                                          : __int_as_float(0x7fc00000);
            }
            if (kWeighted) {
#pragma unroll
                for (int j = 0; j < NV; ++j) {
                    const int idx = lane + 32 * j, v = idx / PIX, pix = idx % PIX;
                    const int y = ty0 + pix / kTW, x = tx0 + pix % kTW;
                    vreg[j] = (v < p.V && y < p.H && x < p.W) ? __ldg(p.vw + ((size_t)b * p.V + v) * HW + (size_t)y * p.W + x) : 0.0f;
                }
            }
        };
        int ws = 0;
        unsigned wpar = 0;  // ring position of the next window: slot and phase parity
        int i = 0;
        if ((int)blockIdx.x < q.nitems) prefetch(blockIdx.x);
        for (int it = blockIdx.x; it < q.nitems; it += gridDim.x, ++i) {
            const int is = i & 1;
            int b, d0, tx0, ty0;
            decode(it, b, d0, tx0, ty0);
            mbar_wait_backoff(&item_empty[is], ((unsigned)(i >> 1) & 1u) ^ 1u);  // consumers are done with item i-2
            // per-item data -> shared memory; range of the tile's hypotheses
            float dlo = INFINITY, dhi = -INFINITY;
            float *sd = s_depth + is * (kDItem * PIX);
#pragma unroll
            for (int j = 0; j < ND; ++j) {
                const float val = dreg[j];
                const bool has = val == val;
                if (has) { dlo = fminf(dlo, val); dhi = fmaxf(dhi, val); }
                sd[lane + 32 * j] = has ? val : 1.0f;
            }
            if (kWeighted) {
                float *sv = s_vw + is * (PMB200_MAX_VIEWS * PIX);
#pragma unroll
                for (int j = 0; j < NV; ++j)
                    if (lane + 32 * j < p.V * PIX) sv[lane + 32 * j] = vreg[j];
            }
            for (int idx = lane; idx < p.V * 12; idx += 32)  // the item's relative projections, read by every consumer lane
                s_rt[is * (PMB200_MAX_VIEWS * 12) + idx] = __ldg(p.rt + ((size_t)(idx / 12) * p.B + b) * 12 + idx % 12);
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                dlo = fminf(dlo, __shfl_xor_sync(full, dlo, off));
                dhi = fmaxf(dhi, __shfl_xor_sync(full, dhi, off));
            }
            if (lane == 0) s_item[is] = ItemInfo{b, d0, tx0, ty0};
            __syncwarp();
            if (lane == 0) {
                mbar_arrive_expect_tx(&item_full[is], (unsigned)(PIX * C * 4));
                tma_ref_tile(s_ref + is * (PIX * C), &ref_map, tx0, ty0, b, &item_full[is]);
            }
            // bounding box of the tile's footprints in view `lane`: the four corner rays at the two extreme depths
            int bx0 = 0, by0 = 0, bw = 0, bh = 0;
            if (lane < p.V && dlo <= dhi) {
                float rt[12];
#pragma unroll
                for (int k = 0; k < 12; ++k) rt[k] = __ldg(p.rt + ((size_t)lane * p.B + b) * 12 + k);
                const float xa = (float)tx0, xb = (float)min(tx0 + kTW - 1, p.W - 1);
                const float ya = (float)ty0, yb = (float)min(ty0 + NW - 1, p.H - 1);
                float umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
                bool ok = true;
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const pm::Ray ray = pm::pixel_ray(rt, (c & 1) ? xb : xa, (c & 2) ? yb : ya);
                    const float d = (c & 4) ? dhi : dlo;
                    const float Z = fmaf(ray.az, d, rt[11]);
                    if (!(Z > 1e-3f)) ok = false;
                    float uu, vv;
                    pm::project_fast(ray, rt, d, p.W, p.H, p.sx, p.sy, &uu, &vv);
                    umin = fminf(umin, uu); umax = fmaxf(umax, uu);
                    vmin = fminf(vmin, vv); vmax = fmaxf(vmax, vv);
                }
                // the box exists only if some tap can be inside the map; clamp while still float (huge coordinates must not
                // overflow the conversion); NaN fails the comparisons
                if (ok && umax >= -1.0f && vmax >= -1.0f && umin < (float)p.Ws && vmin < (float)p.Hs) {
                    const float xl = (float)(p.Ws - 1), yl = (float)(p.Hs - 1);
                    const int x0 = (int)fminf(fmaxf(floorf(umin), 0.0f), xl), x1 = (int)fminf(fmaxf(floorf(umax) + 1.0f, 0.0f), xl);
                    const int y0 = (int)fminf(fmaxf(floorf(vmin), 0.0f), yl), y1 = (int)fminf(fmaxf(floorf(vmax) + 1.0f, 0.0f), yl);
                    bx0 = x0; by0 = y0; bw = x1 - x0 + 1; bh = y1 - y0 + 1;
                    if (bh > kMaxRows) { by0 += (bh - kMaxRows) / 2; bh = kMaxRows; }
                    if (bw * bh > q.cap) {  // larger than a ring slot: keep the centre, the rest takes the global path
                        if (bw > q.cap) { bx0 += (bw - q.cap) / 2; bw = q.cap; }
                        const int nh = max(1, q.cap / bw);
                        by0 += (bh - nh) / 2;
                        bh = nh;
                    }
                }
            }
            if (it + (int)gridDim.x < q.nitems) prefetch(it + gridDim.x);  // in flight while this item's windows are issued
            for (int v = 0; v < p.V; ++v) {
                mbar_wait_backoff(&win_empty[ws], wpar ^ 1u);
                const int x0 = __shfl_sync(full, bx0, v), y0 = __shfl_sync(full, by0, v);
                const int w = __shfl_sync(full, bw, v), h = __shfl_sync(full, bh, v);
                const unsigned row_bytes = (unsigned)(w * C * 4);
                if (lane == 0) {
                    s_win[ws] = WinInfo{x0, y0, w, h};
                    mbar_arrive_expect_tx(&win_full[ws], row_bytes * (unsigned)h);
                }
                __syncwarp();
                const float *src_v = p.src + (((size_t)v * p.B + b) * p.Hs) * (size_t)p.Ws * C;
                float *dst = s_data + (size_t)ws * q.cap * C;
                for (int r = lane; r < h; r += 32)
                    bulk_row_g2s(dst + (size_t)r * w * C, src_v + ((size_t)(y0 + r) * p.Ws + x0) * C, row_bytes, &win_full[ws]);
                if (++ws == q.stages) { ws = 0; wpar ^= 1u; }
            }
        }
        return;
    }

    // ======================================================= consumers =======================================================
    int2 *s_cell = reinterpret_cast<int2 *>(smem + L::oCell) + warp * (kNE * 32);
    float *s_tab = reinterpret_cast<float *>(smem + L::oTable) + warp * L::TABLE;
    const int pi = lane & 7, r = lane >> 3;
    const unsigned below = (1u << lane) - 1u;
    const unsigned pmask = 0x01010101u << pi;  // the lanes of my pixel
    int ws = 0;
    unsigned wpar = 0;  // ring position of the next window: slot and phase parity
    int i = 0;
    for (int it = blockIdx.x; it < q.nitems; it += gridDim.x, ++i) {
        const int is = i & 1;
        mbar_wait(&item_full[is], (unsigned)(i >> 1) & 1u);
        const ItemInfo info = s_item[is];
        const int b = info.b;
        const int px = info.tx0 + pi, py = info.ty0 + warp;
        const bool live = px < p.W && py < p.H;
        const int n = py * p.W + px;
        const float *sd = s_depth + is * (kDItem * PIX);
        float dep[kNE];
        bool ev[kNE];
#pragma unroll
        for (int k = 0; k < kNE; ++k) {
            const int dl = r * kNE + k;
            ev[k] = live && info.d0 + dl < p.D;
            dep[k] = sd[dl * PIX + warp * kTW + pi];
        }
        float acc[kNE][G];
#pragma unroll
        for (int k = 0; k < kNE; ++k)
#pragma unroll
            for (int g = 0; g < G; ++g) acc[k][g] = 0.0f;
        float wsum = 1e-5f;  // reference models/patchmatch.py:192
        const float *ref_tile = s_ref + is * (PIX * C) + warp * (kTW * C);

        for (int v = 0; v < p.V; ++v) {
            const int s = ws;
            float rt[12];
#pragma unroll
            for (int k = 0; k < 12; ++k) rt[k] = s_rt[is * (PMB200_MAX_VIEWS * 12) + v * 12 + k];
            mbar_wait(&win_full[s], wpar);
            if (++ws == q.stages) { ws = 0; wpar ^= 1u; }
            const WinInfo wi = s_win[s];
            const int wx0 = wi.x0, wy0 = wi.y0, ww = wi.w, wh = wi.h;
            const float wv = kWeighted ? s_vw[is * (PMB200_MAX_VIEWS * PIX) + v * PIX + warp * kTW + pi] : 1.0f;
            if (kWeighted) wsum += wv;

            // ---- phase A: footprints; the distinct cells of the warp pass numbered from two ballots ----
            const pm::Ray ray = pm::pixel_ray(rt, (float)px, (float)py);
            float4 w[kNE];
            int key[kNE];
#pragma unroll
            for (int k = 0; k < kNE; ++k) {
                key[k] = kKeyNone;
                w[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
                if (ev[k]) {
                    float uu, vv;
                    pm::project_fast(ray, rt, dep[k], p.W, p.H, p.sx, p.sy, &uu, &vv);
                    key[k] = footprint(uu, vv, p.Hs, p.Ws, w[k]);
                }
            }
            int pk = __shfl_up_sync(full, key[1], 8);  // the hypothesis before my first one: last of the previous row
            if (r == 0) pk = kKeyNone;
            const bool new0 = key[0] != kKeyNone && key[0] != pk;
            const bool new1 = key[1] != kKeyNone && key[1] != key[0];
            const unsigned m0 = __ballot_sync(full, new0), m1 = __ballot_sync(full, new1);
            const int c0 = __popc(m0);
            const int ncell = c0 + __popc(m1);
            int slot[kNE];
            if (new0) {
                slot[0] = __popc(m0 & below);
            } else {  // first cell of my run: the latest new cell of my pixel in an earlier row (k = 1 is later than k = 0)
                const unsigned u0 = m0 & pmask & below, u1 = m1 & pmask & below;
                const int h0 = 31 - clz32(u0), h1 = 31 - clz32(u1);
                slot[0] = (h1 >= h0) ? (c0 + __popc(m1 & ((1u << (h1 & 31)) - 1u))) : __popc(m0 & ((1u << (h0 & 31)) - 1u));
            }
            slot[1] = new1 ? (c0 + __popc(m1 & below)) : slot[0];
            if (new0) s_cell[slot[0]] = make_int2(key[0], pi);
            if (new1) s_cell[slot[1]] = make_int2(key[1], pi);
            __syncwarp();

            // ---- phases B / C in rounds of NCELL cells: one lane (or lane pair) per cell gathers; footprints blend ----
            float best = -INFINITY;  // kEpiViewW only
            const float *win = s_data + (size_t)s * q.cap * C;
            const float *src_v = p.src + (((size_t)v * p.B + b) * p.Hs) * (size_t)p.Ws * C;
            for (int base = 0; base == 0 || base < ncell; base += L::NCELL) {
                const int j = base + lane / L::LPC;
                if (j < ncell) {
                    const int2 ck = s_cell[j];
                    const int x0 = ck.x & ((1 << kXBits) - 1), y0 = (ck.x >> kXBits) & 0x7fff;
                    const int dx = (ck.x >> pm::kKeyDxShift) & 1, dy = (ck.x >> pm::kKeyDyShift) & 1;
                    const int ox = x0 - wx0, oy = y0 - wy0;
                    const int half = (L::LPC == 2) ? (lane & 1) * 32 : 0;
                    const float *ref = ref_tile + ck.y * C + half;
                    const int rs = lane / L::LPC;
                    float *tb = s_tab + (rs & 7) * L::TP + (rs >> 3) * L::TA;
                    if (ox >= 0 && oy >= 0 && ox + dx < ww && oy + dy < wh) {
                        const float *t00 = win + (oy * ww + ox) * C + half;
                        const float *t10 = t00 + dy * ww * C;
                        gather_cell<C, G, false>(t00, t00 + dx * C, t10, t10 + dx * C, ref, tb, lane);
                    } else {
                        const float *t00 = src_v + ((size_t)y0 * p.Ws + x0) * C + half;
                        const float *t10 = t00 + (size_t)dy * p.Ws * C;
                        gather_cell<C, G, true>(t00, t00 + dx * C, t10, t10 + dx * C, ref, tb, lane);
                    }
                }
                __syncwarp();
#pragma unroll
                for (int k = 0; k < kNE; ++k) {
                    const int rs = slot[k] - base;
                    const bool mine = key[k] != kKeyNone && rs >= 0 && rs < L::NCELL;
                    const bool empty = key[k] == kKeyNone && base == 0;  // all taps outside: similarity exactly 0
                    if (!(mine || empty)) continue;
                    float sim[G];
#pragma unroll
                    for (int g = 0; g < G; ++g) sim[g] = 0.0f;
                    if (mine) {
                        const float4 *tp = reinterpret_cast<const float4 *>(s_tab + (rs & 7) * L::TP + (rs >> 3) * L::TA);
                        const float2 wx = make_float2(w[k].x, w[k].x), wy = make_float2(w[k].y, w[k].y);
                        const float2 wz = make_float2(w[k].z, w[k].z), wq = make_float2(w[k].w, w[k].w);
                        const float2 zero = make_float2(0.0f, 0.0f);
#pragma unroll
                        for (int qd = 0; qd < G / 4; ++qd) {
                            const float4 t0 = tp[qd], t1 = tp[G / 4 + qd], t2 = tp[2 * (G / 4) + qd], t3 = tp[3 * (G / 4) + qd];
                            const float2 lo = ffma2(wq, make_float2(t3.x, t3.y), ffma2(wz, make_float2(t2.x, t2.y),
                                              ffma2(wy, make_float2(t1.x, t1.y), ffma2(wx, make_float2(t0.x, t0.y), zero))));
                            const float2 hi = ffma2(wq, make_float2(t3.z, t3.w), ffma2(wz, make_float2(t2.z, t2.w),
                                              ffma2(wy, make_float2(t1.z, t1.w), ffma2(wx, make_float2(t0.z, t0.w), zero))));
                            sim[4 * qd + 0] = lo.x; sim[4 * qd + 1] = lo.y; sim[4 * qd + 2] = hi.x; sim[4 * qd + 3] = hi.y;
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
                    } else if (ev[k]) {
                        const int d = info.d0 + r * kNE + k;
                        if (EPI == kEpiSims || sims_out != nullptr) {
                            float *o = (EPI == kEpiSims ? p.out : sims_out) + ((((size_t)v * p.B + b) * G) * p.D + d) * HW + n;
#pragma unroll
                            for (int g = 0; g < G; ++g) o[(size_t)g * p.D * HW] = sim[g];
                        }
                        if (EPI == kEpiViewW) best = fmaxf(best, mlp_eval<G>(mlp, sim));
                    }
                }
                __syncwarp();  // the table is rewritten by the next round / view
            }
            if (lane == 0) mbar_arrive(&win_empty[s]);  // every lane of the warp is past its last read of the window
            if (EPI == kEpiViewW) {
                // PixelwiseNet (models/patchmatch.py:702): max over hypotheses of sigmoid(MLP(sim)); sigmoid is monotonic ->
                // max first, one sigmoid per pixel, atomic max across the items that split the hypothesis axis
                best = fmaxf(best, __shfl_xor_sync(full, best, 8));
                best = fmaxf(best, __shfl_xor_sync(full, best, 16));
                if (r == 0 && live && best > -INFINITY) {
                    const float sg = 1.0f / (1.0f + expf(-best));
                    atomicMax(reinterpret_cast<int *>(p.out + ((size_t)b * p.V + v) * HW + n), __float_as_int(sg));
                }
            }
        }

        const float inv_wsum = 1.0f / wsum;
        if (EPI == kEpiAgg) {
#pragma unroll
            for (int k = 0; k < kNE; ++k) {
                const int d = info.d0 + r * kNE + k;
                if (ev[k]) {
                    float *o = p.out + (((size_t)b * G) * p.D + d) * HW + n;
#pragma unroll
                    for (int g = 0; g < G; ++g) o[(size_t)g * p.D * HW] = acc[k][g] * inv_wsum;
                }
            }
        } else if (EPI == kEpiScore) {
#pragma unroll
            for (int k = 0; k < kNE; ++k) {
                // (inside the branch: an unconditional call makes the head's ~290 constant-bank operands loop invariants of the
                // persistent item loop, which the compiler then hoists into registers and spills -- 1 KB of stack per thread)
                if (ev[k]) {
                    const int d = info.d0 + r * kNE + k;
                    float x[G];
#pragma unroll
                    for (int g = 0; g < G; ++g) x[g] = acc[k][g] * inv_wsum;
                    p.out[(((size_t)b * p.D + d) * HW + n) * p.ostride] = mlp_eval<G>(mlp, x);
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&item_empty[is]);  // the item's hypotheses / weights / reference tile may be overwritten
    }
}

}  // namespace wc4
