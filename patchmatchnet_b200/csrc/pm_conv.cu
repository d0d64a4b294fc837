// pm_conv.cu -- sm_90a channels-last 2-D convolution family for the small learned convs either side of the
// PatchMatch hot path: the offset convs ON the path (propa_conv / eval_conv, reference models/patchmatch.py:288-311),
// the feature pyramid that produces the path's inputs (FeatureNet, reference models/net.py:9-70) and the refinement
// head that consumes its output (Refinement, reference models/net.py:73-122).  SURVEY.md 8(f) rows f1 / f3.
//
// Why hand-written: these layers have 1..64 channels.  The library's implicit-GEMM kernels are tiled for hundreds of
// channels (256x64x8 / 128x128x8 tiles) and run the 23 convs of one 640x512 forward far below HBM speed.  At these widths a
// conv is a
// memory-bound streaming op with a small dense contraction inside, so the design is:
//
//   * activations channels-last (NHWC) end to end -- the layout the fused PatchMatch kernels gather from;
//   * one CTA = 4 warps = an output tile of 16 columns x (4*MT) rows.  The input halo tile (all input channels) is
//     staged ONCE in shared memory with a pixel stride chosen so that the tensor-core fragment loads are bank-conflict
//     free for the layer's stride; zero padding, image borders and the zero-stuffing of a transposed conv are
//     resolved during staging, so the inner loop has no bounds checks;
//   * the contraction runs on the tensor cores as implicit GEMM, M = 16 output pixels of one row, N = 8 output
//     channels, K = 8 input channels of one filter tap (mma.sync.m16n8k8 TF32, fp32 accumulate).  The MMA's k slots
//     (t, t+4) of a lane are mapped to the ADJACENT channels (2t, 2t+1), so an A fragment is two 64-bit shared loads.
//     The filter is pre-arranged ON THE HOST in fragment order ([tap][k-slice][n-tile][lane]), so a warp fetches a B
//     fragment with one coalesced read-only load that stays L1/L2-resident for every CTA of the layer: no shared
//     memory for weights, no per-CTA weight staging; a 3x3 filter of <= 18 fragments lives in registers;
//   * NO conversion instructions in the inner loop (cvt.rna.tf32.f32 expands to a multi-instruction sequence that made
//     the first version issue-bound).
//     `precision == 1` (the library's behaviour under torch.backends.cudnn.allow_tf32 = True, torch's default): the
//     host rounds the filter to TF32 (nearest, ties away) while packing, activations go to the tensor core as fp32
//     bit patterns whose low 13 mantissa bits it ignores -- exactly what wgmma kind tf32 does with the library's
//     shared-memory operands.  `precision == 3` is the error-compensated 3xTF32 split (a_hi*b_hi + a_hi*b_lo +
//     a_lo*b_hi; filter split on the host, activations split in registers), fp32-accurate, used by the parity tests;
//   * bias + ReLU fused in the epilogue; the output may be written into a channel slice of a wider buffer
//     (concat fusion) and a transposed stride-2 conv is the same kernel over a virtually zero-stuffed input.
//
// wgmma is deliberately not used here: with N <= 64 and K <= 64 per tap the operands are far below a warpgroup MMA's
// 64xNx8 tile economy, and the layers are bound by activation traffic, not by MMA issue.
#include <atomic>

#if !defined(PM_EMU)  // host emulation build (tests/warp_emu.h) brings its own CUDA vocabulary
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);  // pm_kernels.cu: sets pmb200_last_error()

namespace {

struct ConvParams {
    const float *x;      // [N,H,W,Cin]
    const float *wf;     // fragment-ordered filter [taps][KCIN/8][NT][32][2 (TF32) or 4 (3xTF32: b0h,b1h,b0l,b1l)]
    const float *bias;   // [Cout] or null
    const float *up;     // optional [N,Ho/2,Wo/2,Cout]: its bilinear x2 upsample is added in the epilogue
    float *y;            // [N,Ho,Wo,ycs] written at channel offset yco
    int N, H, W, Cin, Ho, Wo, Cout;
    int KS, S, pad, dil, relu;
    int ps;              // shared-memory pixel stride (floats)
    int rw, rh;          // staged input region (pixels)
    int buf_floats;      // one halo buffer (multiple of 4 floats)
    int ycs, yco;        // output channel stride / offset
    int stuff;           // 1: the input is virtually zero-stuffed x2 (transposed stride-2 conv)
    int tiles_x, tiles_y, total_tiles;
    int nt_total;        // 8-wide output-channel tiles of the layer (a warp handles NT of them)
    int nbuf;            // 2: halo tiles double-buffered (several tiles per CTA); 1: one buffer, more resident CTAs
    int cpp, cpp_shift;  // cp.async chunks per pixel (Cin/4 16-byte chunks, or Cin 4-byte chunks), log2 or -1
    int row_chunks, tile_chunks;        // chunks per region row / per halo tile
    unsigned magic_row, magic_cpp;      // floor(2^32 / d) + 1: idx / d == umulhi(idx, magic) for idx * d < 2^32
    int step_r[2], step_c[2];           // (128 or 256) / row_chunks and % row_chunks: per-iteration advance of a thread
};

#if defined(PM_EMU)
// Host emulation (tests/warp_emu.h): the PTX below restated in C++ -- cvt.rna (nearest, ties away from zero, 10-bit
// mantissa), the m16n8k8 TF32 MMA as a warp collective with the hardware's fragment layout (operands truncated to TF32 as
// the tensor core does), cp.async as an immediate copy / zero fill.
__device__ __forceinline__ uint32_t to_tf32(float f) { return emu::cvt_rna_tf32(f); }
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) { emu::mma_m16n8k8_tf32(d, a, b0, b1); }
template <int BYTES>
__device__ __forceinline__ void cp_async(float *smem_dst, const float *gmem_src, bool valid) {
    assert((reinterpret_cast<uintptr_t>(smem_dst) % BYTES) == 0 && (!valid || (reinterpret_cast<uintptr_t>(gmem_src) % BYTES) == 0));
    if (valid) memcpy(smem_dst, gmem_src, BYTES);
    else memset(smem_dst, 0, BYTES);
}
__device__ __forceinline__ void cp_async_commit() {}
template <int N>
__device__ __forceinline__ void cp_async_wait() {}
#else
__device__ __forceinline__ uint32_t to_tf32(float f) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(f));
    return r;
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Asynchronous global -> shared copy of BYTES (4, 8 or 16) bytes; `valid` false writes zeros (src-size 0).
template <int BYTES>
__device__ __forceinline__ void cp_async(float *smem_dst, const float *gmem_src, bool valid) {
    const uint32_t dst = (uint32_t)__cvta_generic_to_shared(smem_dst);
    const int n = valid ? BYTES : 0;
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(dst), "l"(gmem_src), "n"(BYTES), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif

// high part of the 3xTF32 activation split: the value with its 13 low mantissa bits cleared
__device__ __forceinline__ uint32_t split_hi(float f) { return __float_as_uint(f) & 0xffffe000u; }

// Stage the halo tile of output tile `tile` into `buf` ([rh][rw][ps]): the CTA's threads stride over the
// tile's copy chunks (16-byte channel vectors when VEC, else single floats: Cin % 4 != 0).  Out-of-image pixels and
// (STUFF) the odd positions of a zero-stuffed input are written as zeros by the copy engine itself (src-size 0);
// channels >= Cin are never written and stay zero from the kernel prologue.  Index decomposition by multiply-high
// with host-made reciprocals (exact for the ranges used here); 32-bit offsets (the host checks the image fits).
template <bool VEC, bool STUFF, int THREADS>
__device__ __forceinline__ void stage_tile(const ConvParams &p, int tile, float *buf, int rows_per_tile) {
    const int per_img = p.tiles_x * p.tiles_y;
    const int n = tile / per_img, tt = tile - n * per_img;
    const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
    const int ix0 = tx * 16 * p.S - p.pad, iy0 = ty * rows_per_tile * p.S - p.pad;
    const unsigned Hv = STUFF ? 2 * p.H : p.H, Wv = STUFF ? 2 * p.W : p.W;
    const float *img = p.x + (size_t)n * p.H * p.W * p.Cin;
    // this thread's first chunk, then THREADS chunks further each iteration: (row, chunk-in-row) advance by a constant
    int r = (int)__umulhi(threadIdx.x, p.magic_row);
    int c = (int)threadIdx.x - r * p.row_chunks;
#pragma unroll 2
    for (int idx = threadIdx.x; idx < p.tile_chunks; idx += THREADS) {
        const int rx = p.cpp_shift >= 0 ? (c >> p.cpp_shift) : (int)__umulhi((unsigned)c, p.magic_cpp);
        const int v = c - rx * p.cpp;
        int iy = iy0 + r, ix = ix0 + rx;
        bool inside = (unsigned)iy < Hv && (unsigned)ix < Wv;
        if (STUFF) {
            inside = inside && ((iy | ix) & 1) == 0;
            iy >>= 1;
            ix >>= 1;
        }
        const unsigned goff = inside ? (unsigned)((iy * p.W + ix) * p.Cin) : 0u;
        const int soff = (r * p.rw + rx) * p.ps;
        if (VEC) cp_async<16>(buf + soff + v * 4, img + goff + v * 4, inside);  // ps % 4 == 0: 16-byte aligned
        else cp_async<4>(buf + soff + v, img + goff + v, inside);
        r += p.step_r[THREADS / 256];
        c += p.step_c[THREADS / 256];
        if (c >= p.row_chunks) {
            c -= p.row_chunks;
            ++r;
        }
    }
}

// The same copy with a FIXED column per thread, for halo rows of at most THREADS chunks (every layer the policy runs
// natively except the 64-channel ones): thread -> (first row r0, chunk-in-row c) once, then it walks down the rows in steps
// of THREADS / row_chunks.  Everything that depends on the column -- the pixel, the channel vector, the x bounds test, the
// zero-stuffing parity, the shared and global column offsets -- leaves the loop; per chunk there remain the row bounds test,
// one multiply-add for the global row and the copy (~8 instructions instead of ~22: staging was ~45 % of the issued
// instructions of the 8-channel full-resolution layers, tools/sass_lines.py).
template <bool VEC, bool STUFF, int THREADS>
__device__ __forceinline__ void stage_tile_cols(const ConvParams &p, int tile, float *buf, int rows_per_tile) {
    const int rows_per_iter = p.step_r[THREADS / 256];  // THREADS / row_chunks >= 1
    const int r0 = (int)__umulhi(threadIdx.x, p.magic_row);
    if (r0 >= rows_per_iter) return;  // the remainder threads of the last partial row group have no column
    const int per_img = p.tiles_x * p.tiles_y;
    const int n = tile / per_img, tt = tile - n * per_img;
    const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
    const int ix0 = tx * 16 * p.S - p.pad, iy0 = ty * rows_per_tile * p.S - p.pad;
    const unsigned Hv = STUFF ? 2 * p.H : p.H, Wv = STUFF ? 2 * p.W : p.W;
    const float *img = p.x + (size_t)n * p.H * p.W * p.Cin;
    const int c = (int)threadIdx.x - r0 * p.row_chunks;
    const int rx = p.cpp_shift >= 0 ? (c >> p.cpp_shift) : (int)__umulhi((unsigned)c, p.magic_cpp);
    const int v = (c - rx * p.cpp) * (VEC ? 4 : 1);  // first channel of this thread's chunk
    int ix = ix0 + rx;
    bool in_x = (unsigned)ix < Wv;
    if (STUFF) {
        in_x = in_x && (ix & 1) == 0;
        ix >>= 1;
    }
    const unsigned gcol = in_x ? (unsigned)(ix * p.Cin + v) : 0u;
    const unsigned grow = (unsigned)(p.W * p.Cin);
    float *dst = buf + (r0 * p.rw + rx) * p.ps + v;
    const int dstep = rows_per_iter * p.rw * p.ps;
#pragma unroll 2
    for (int r = r0; r < p.rh; r += rows_per_iter, dst += dstep) {
        int iy = iy0 + r;
        bool inside = in_x && (unsigned)iy < Hv;
        if (STUFF) {
            inside = inside && (iy & 1) == 0;
            iy >>= 1;
        }
        const unsigned goff = inside ? (unsigned)iy * grow + gcol : 0u;
        if (VEC) cp_async<16>(dst, img + goff, inside);
        else cp_async<4>(dst, img + goff, inside);
    }
}

// Not inlined: one copy of the eight staging variants per kernel instead of three (prologue, prefetch, single-buffer
// path), and their address arithmetic does not inflate the register allocation of the MMA loop (the planner counts on
// <= ~100 registers for 5 resident CTAs; inlined, the 8-channel register-filter kernel went from 96 to 118).  The kernel
// takes its parameter block as __grid_constant__, so the reference handed to this function points into the parameter
// space itself and no per-thread stack copy of the 176-byte block is made.
template <int THREADS>
__device__ __noinline__ void stage_any(const ConvParams &p, int tile, float *buf, int rows_per_tile) {
    const bool cols = p.step_r[THREADS / 256] >= 1;  // a halo row has at most THREADS chunks
    if (p.stuff) {
        if ((p.Cin & 3) == 0) {
            if (cols) stage_tile_cols<true, true, THREADS>(p, tile, buf, rows_per_tile);
            else stage_tile<true, true, THREADS>(p, tile, buf, rows_per_tile);
        } else {
            if (cols) stage_tile_cols<false, true, THREADS>(p, tile, buf, rows_per_tile);
            else stage_tile<false, true, THREADS>(p, tile, buf, rows_per_tile);
        }
    } else if ((p.Cin & 3) == 0) {
        if (cols) stage_tile_cols<true, false, THREADS>(p, tile, buf, rows_per_tile);
        else stage_tile<true, false, THREADS>(p, tile, buf, rows_per_tile);
    } else {
        if (cols) stage_tile_cols<false, false, THREADS>(p, tile, buf, rows_per_tile);
        else stage_tile<false, false, THREADS>(p, tile, buf, rows_per_tile);
    }
}

// KCIN: input channels rounded up to 8/16/32/64 (the padding channels are zero in shared memory); NT: 8-wide
// output-channel tiles PER WARP; MT: 16-pixel output rows per warp; PREC: 1 = TF32, 3 = 3xTF32; WREG: 3x3 filter
// with KCIN/8 * NT <= 2 -- the whole filter lives in registers for the lifetime of the persistent CTA; NSPLIT: warp
// groups per CTA that share one halo tile and split the output channels (NSPLIT * NT tiles in all): the layers with
// few pixels and many channels get twice the warps per tile without staging the halo twice.
template <int KCIN, int NT, int MT, int PREC, bool WREG, int NSPLIT>
__global__ void __launch_bounds__(128 * NSPLIT) conv_nhwc_mma_kernel(const __grid_constant__ ConvParams p) {
#if defined(PM_EMU)
    float *s_in = static_cast<float *>(emu::dyn_smem());
#else
    extern __shared__ __align__(16) float s_in[];
#endif
    constexpr int KK = KCIN / 8;
    constexpr int ROWS = 4 * MT;
    constexpr int THREADS = 128 * NSPLIT;
    // WREG kernels serve 3x3 / stride 1 / dilation 1 only: the halo row is 18 pixels and the pixel stride is known at
    // compile time, so every A-fragment address is the lane's base plus an immediate offset
    constexpr int kPsW = KCIN == 8 ? 8 : 24, kRwW = 18;
    const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int nbase = (threadIdx.x >> 7) * NT;  // first output-channel tile of this warp group

    // prologue: zero the halo buffers once (the channel padding is never rewritten)
    for (int i = threadIdx.x; i < p.nbuf * p.buf_floats / 4; i += THREADS) reinterpret_cast<float4 *>(s_in)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();

    int tile = blockIdx.x;
    if (p.nbuf == 2) {
        if (tile < p.total_tiles) stage_any<THREADS>(p, tile, s_in, ROWS);
        cp_async_commit();
    }

    // register-resident filter (3x3, at most two fragments per tap)
    uint32_t wh[WREG ? 9 * KK * NT : 1][2], wlo[(WREG && PREC == 3) ? 9 * KK * NT : 1][2];
    if constexpr (WREG) {
#pragma unroll
        for (int q = 0; q < 9 * KK * NT; ++q) {
            if constexpr (PREC == 1) {
                const float2 b = __ldg(reinterpret_cast<const float2 *>(p.wf) + (size_t)q * 32 + lane);
                wh[q][0] = __float_as_uint(b.x);
                wh[q][1] = __float_as_uint(b.y);
            } else {
                const float4 b = __ldg(reinterpret_cast<const float4 *>(p.wf) + (size_t)q * 32 + lane);
                wh[q][0] = __float_as_uint(b.x);
                wh[q][1] = __float_as_uint(b.y);
                wlo[q][0] = __float_as_uint(b.z);
                wlo[q][1] = __float_as_uint(b.w);
            }
        }
    }

    // this lane's two output channels of every n-tile and their bias, fixed for the lifetime of the CTA
    float bi0[NT], bi1[NT];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const int co = (nbase + j) * 8 + 2 * t;
        bi0[j] = (p.bias && co < p.Cout) ? __ldg(p.bias + co) : 0.f;
        bi1[j] = (p.bias && co + 1 < p.Cout) ? __ldg(p.bias + co + 1) : 0.f;
    }
    const int arow = g * p.S * p.ps + 2 * t;  // lane part of the A-fragment address: channels 2t, 2t+1 of pixel g
    const int astep8 = 8 * p.S * p.ps;    // 8 output pixels further right
    const bool vec2 = ((p.ycs | p.yco) & 1) == 0;
    const int per_img = p.tiles_x * p.tiles_y;

    for (int it = 0; tile < p.total_tiles; tile += gridDim.x, ++it) {
        const float *cur = s_in;
        if (p.nbuf == 2) {  // prefetch the next tile of this CTA into the other buffer while this one is computed
            cur = s_in + (size_t)(it & 1) * p.buf_floats;
            const int next = tile + gridDim.x;
            if (next < p.total_tiles) stage_any<THREADS>(p, next, s_in + (size_t)((it + 1) & 1) * p.buf_floats, ROWS);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            stage_any<THREADS>(p, tile, s_in, ROWS);
            cp_async_commit();
            cp_async_wait<0>();
        }
        __syncthreads();

        float acc[MT][NT][4];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int j = 0; j < NT; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) acc[m][j][i] = 0.f;

        auto mma_step = [&](const float *ap0, const uint32_t (&bh)[NT][2], const uint32_t (&bl)[NT][2]) {
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const float *ap = ap0 + (WREG ? m * kRwW * kPsW : m * p.S * p.rw * p.ps);
                const float2 lo = *reinterpret_cast<const float2 *>(ap);           // pixel g:   k slots t, t+4
                const float2 hi = *reinterpret_cast<const float2 *>(ap + (WREG ? 8 * kPsW : astep8));  // pixel g+8
                uint32_t ah[4];
                if constexpr (PREC == 1) {  // the tensor core ignores the low 13 mantissa bits
                    ah[0] = __float_as_uint(lo.x); ah[1] = __float_as_uint(hi.x);
                    ah[2] = __float_as_uint(lo.y); ah[3] = __float_as_uint(hi.y);
#pragma unroll
                    for (int j = 0; j < NT; ++j) mma_tf32(acc[m][j], ah, bh[j][0], bh[j][1]);
                } else {
                    uint32_t al[4];
                    // split without conversion instructions: a_hi = the TF32 the tensor core would read anyway (low 13 mantissa
                    // bits cleared), a_lo = a - a_hi, exact in fp32 (Sterbenz) and handed over as raw bits -- the hardware keeps
                    // its 11 leading bits, so a_hi + tf32(a_lo) carries >= 22 bits of a.  cvt.rna here was ~10 issue slots per
                    // register; this is one LOP3 and one FADD.
                    ah[0] = split_hi(lo.x); ah[1] = split_hi(hi.x); ah[2] = split_hi(lo.y); ah[3] = split_hi(hi.y);
                    al[0] = __float_as_uint(lo.x - __uint_as_float(ah[0]));
                    al[1] = __float_as_uint(hi.x - __uint_as_float(ah[1]));
                    al[2] = __float_as_uint(lo.y - __uint_as_float(ah[2]));
                    al[3] = __float_as_uint(hi.y - __uint_as_float(ah[3]));
#pragma unroll
                    for (int j = 0; j < NT; ++j) {  // small terms first
                        mma_tf32(acc[m][j], al, bh[j][0], bh[j][1]);
                        mma_tf32(acc[m][j], ah, bl[j][0], bl[j][1]);
                        mma_tf32(acc[m][j], ah, bh[j][0], bh[j][1]);
                    }
                }
            }
        };

        const float *abase = WREG ? cur + (warp * MT) * (kRwW * kPsW) + g * kPsW + 2 * t
                                  : cur + (warp * MT * p.S) * p.rw * p.ps + arow;
        if constexpr (WREG) {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx)
#pragma unroll
                    for (int kk = 0; kk < KK; ++kk) {
                        uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
                        for (int j = 0; j < NT; ++j) {
                            const int q = ((ky * 3 + kx) * KK + kk) * NT + j;
                            bh[j][0] = wh[q][0]; bh[j][1] = wh[q][1];
                            bl[j][0] = wlo[(PREC == 3) ? q : 0][0]; bl[j][1] = wlo[(PREC == 3) ? q : 0][1];
                        }
                        mma_step(abase + (ky * kRwW + kx) * kPsW + kk * 8, bh, bl);
                    }
        } else {
            // filter fragments streamed through L1, one (tap, k-slice) ahead of the MMAs that use them
            using Frag = typename std::conditional<PREC == 1, float2, float4>::type;
            const Frag *wp = reinterpret_cast<const Frag *>(p.wf) + nbase * 32 + lane;
            const int wstep = p.nt_total * 32;  // fragments of one (tap, k-slice)
            Frag bn[NT];
#pragma unroll
            for (int j = 0; j < NT; ++j) bn[j] = __ldg(wp + j * 32);
            const int steps = p.KS * p.KS * KK;
            int q = 0;
#pragma unroll 1
            for (int ky = 0; ky < p.KS; ++ky) {
#pragma unroll 1
                for (int kx = 0; kx < p.KS; ++kx) {
                    const float *atap = abase + (ky * p.dil * p.rw + kx * p.dil) * p.ps;
#pragma unroll
                    for (int kk = 0; kk < KK; ++kk) {
                        uint32_t bh[NT][2], bl[NT][2];
#pragma unroll
                        for (int j = 0; j < NT; ++j) {
                            bh[j][0] = __float_as_uint(bn[j].x);
                            bh[j][1] = __float_as_uint(bn[j].y);
                            if constexpr (PREC == 3) {
                                bl[j][0] = __float_as_uint(bn[j].z);
                                bl[j][1] = __float_as_uint(bn[j].w);
                            } else {
                                bl[j][0] = bl[j][1] = 0u;
                            }
                        }
                        ++q;
                        wp += wstep;
                        if (q < steps) {
#pragma unroll
                            for (int j = 0; j < NT; ++j) bn[j] = __ldg(wp + j * 32);
                        }
                        mma_step(atap + kk * 8, bh, bl);
                    }
                }
            }
        }

        // ---- epilogue: bias, ReLU, channels-last store (c0,c1 -> pixel g; c2,c3 -> pixel g+8; channels 2t, 2t+1) ----
        const int n = tile / per_img, tt = tile - n * per_img;
        const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
        const int ox0 = tx * 16, oy0 = ty * ROWS;
        const int oyw = oy0 + warp * MT;
        float *const dst0 = p.y + (((size_t)n * p.Ho + oyw) * p.Wo + ox0 + g) * p.ycs + p.yco + nbase * 8 + 2 * t;
        const int row_step = p.Wo * p.ycs, half_step = 8 * p.ycs;
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const int oy = oyw + m;
            if (oy >= p.Ho) continue;
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const int co = (nbase + j) * 8 + 2 * t;
                if (co >= p.Cout) continue;
                const bool pair = co + 1 < p.Cout;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ox = ox0 + g + 8 * h;
                    if (ox >= p.Wo) continue;
                    float v0 = acc[m][j][2 * h] + bi0[j], v1 = acc[m][j][2 * h + 1] + bi1[j];
                    if (p.up) {  // + bilinear x2 upsample of the coarser map (F.interpolate, align_corners=False); Cout even
                        const int hc = p.Ho >> 1, wc = p.Wo >> 1;
                        const float sy = fmaxf(0.5f * ((float)oy + 0.5f) - 0.5f, 0.0f), sx = fmaxf(0.5f * ((float)ox + 0.5f) - 0.5f, 0.0f);
                        const int y0 = (int)sy, x0 = (int)sx;
                        const int y1 = min(y0 + 1, hc - 1), x1 = min(x0 + 1, wc - 1);
                        const float ly = sy - (float)y0, lx = sx - (float)x0, hy = 1.0f - ly, hx = 1.0f - lx;
                        const float *ub = p.up + (size_t)n * hc * wc * p.Cout + co;
                        const float2 a00 = __ldg(reinterpret_cast<const float2 *>(ub + ((size_t)y0 * wc + x0) * p.Cout));
                        const float2 a01 = __ldg(reinterpret_cast<const float2 *>(ub + ((size_t)y0 * wc + x1) * p.Cout));
                        const float2 a10 = __ldg(reinterpret_cast<const float2 *>(ub + ((size_t)y1 * wc + x0) * p.Cout));
                        const float2 a11 = __ldg(reinterpret_cast<const float2 *>(ub + ((size_t)y1 * wc + x1) * p.Cout));
                        v0 += hy * (hx * a00.x + lx * a01.x) + ly * (hx * a10.x + lx * a11.x);
                        v1 += hy * (hx * a00.y + lx * a01.y) + ly * (hx * a10.y + lx * a11.y);
                    }
                    if (p.relu) {
                        v0 = fmaxf(v0, 0.f);
                        v1 = fmaxf(v1, 0.f);
                    }
                    float *dst = dst0 + (m * row_step + h * half_step + j * 8);
                    if (pair && vec2) {
                        *reinterpret_cast<float2 *>(dst) = make_float2(v0, v1);
                    } else {
                        dst[0] = v0;
                        if (pair) dst[1] = v1;
                    }
                }
            }
        }
        __syncthreads();  // every warp is done with `cur` before the next iteration's prefetch overwrites it
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------------------------------

int conv_fail(int code, const char *msg) { return pmb200_internal_fail(code, msg); }

// Shared-memory pixel stride (floats) >= kcin such that the 64-bit A-fragment loads are bank-conflict free: a
// half-warp reads 4 pixels x 8 consecutive floats, so (stride_in_pixels * ps) mod 32 must be 8 or 24; ps % 4 == 0 keeps
// every 16-byte cp.async destination aligned.
int pixel_stride(int kcin, int S) {
    for (int ps = kcin;; ps += 4) {
        const int r = (S * ps) % 32;
        if (r == 8 || r == 24) return ps;
    }
}

struct DeviceInfo {
    int sms = 0;
};

// SM count of the current device (cached per device; benign race: every writer stores the same value)
int sm_count(int dev) {
    static DeviceInfo info[64];
#if !defined(PM_EMU)  // (the emulation build re-reads its pretend SM count every call)
    if (dev >= 0 && dev < 64 && info[dev].sms > 0) return info[dev].sms;
#endif
    int n = 132;  // H100 SXM
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
    if (dev >= 0 && dev < 64) info[dev].sms = n;
    return n;
}

struct LaunchPlan {
    size_t smem;
    int ctas;
};

template <int KCIN, int NT, int MT, int PREC, bool WREG, int NSPLIT>
int launch_conv(const ConvParams &p, const LaunchPlan &plan, cudaStream_t st) {
    auto kern = conv_nhwc_mma_kernel<KCIN, NT, MT, PREC, WREG, NSPLIT>;
    if (plan.smem > 48 * 1024) {
        // opt in to the device's maximum dynamic shared memory once per (instantiation, device): always the same value, so
        // concurrent callers (one host thread per GPU, several streams) can only repeat an idempotent call
        static std::atomic<unsigned long long> optin_done{0};
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64 || !((optin_done.load(std::memory_order_relaxed) >> dev) & 1ull)) {
            int optin = 0;
            cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
            if (optin < (int)plan.smem) optin = (int)plan.smem;
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
            if (e != cudaSuccess) {
                char msg[200];
                snprintf(msg, sizeof(msg), "conv2d_nhwc: cudaFuncSetAttribute(%d B): %s", optin, cudaGetErrorString(e));
                return pmb200_internal_fail((int)e, msg);
            }
            if (dev >= 0 && dev < 64) optin_done.fetch_or(1ull << dev, std::memory_order_relaxed);
        }
    }
#if defined(PM_EMU)
    (void)st;
    emu::launch(dim3((unsigned)plan.ctas), dim3(128 * NSPLIT), plan.smem, [&] { kern(p); });
#else
    kern<<<(unsigned)plan.ctas, 128 * NSPLIT, plan.smem, st>>>(p);
#endif
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        char msg[200];
        snprintf(msg, sizeof(msg), "conv2d_nhwc launch: %s", cudaGetErrorString(e));
        return pmb200_internal_fail((int)e, msg);
    }
    return 0;
}

template <int KCIN, int NT, int MT, int NSPLIT>
int launch_prec(const ConvParams &p, const LaunchPlan &plan, int prec, cudaStream_t st) {
    constexpr bool kCanHold = NSPLIT == 1 && (KCIN / 8) * NT <= 2;  // <= 18 fragments of a 3x3 filter in registers
    if constexpr (kCanHold) {
        if (p.KS == 3 && p.S == 1 && p.dil == 1)  // the register-resident form hard-codes the 18-pixel halo row
            return prec == 1 ? launch_conv<KCIN, NT, MT, 1, true, 1>(p, plan, st) : launch_conv<KCIN, NT, MT, 3, true, 1>(p, plan, st);
    }
    return prec == 1 ? launch_conv<KCIN, NT, MT, 1, false, NSPLIT>(p, plan, st) : launch_conv<KCIN, NT, MT, 3, false, NSPLIT>(p, plan, st);
}

// (nt per warp, nsplit, mt) combinations that are instantiated:
//   nsplit 1: nt 1, 2 with mt 1/2/4; nt 3, 4 with mt 1/2; nt 8 with mt 1      nsplit 2: nt 2 (4 tiles) and 4 (8 tiles), mt 1/2
template <int KCIN>
int launch_shape(const ConvParams &p, const LaunchPlan &plan, int nt, int nsplit, int mt, int prec, cudaStream_t st) {
    if (nsplit == 2) {
        if (nt == 2) return mt >= 2 ? launch_prec<KCIN, 2, 2, 2>(p, plan, prec, st) : launch_prec<KCIN, 2, 1, 2>(p, plan, prec, st);
        return mt >= 2 ? launch_prec<KCIN, 4, 2, 2>(p, plan, prec, st) : launch_prec<KCIN, 4, 1, 2>(p, plan, prec, st);
    }
    switch (nt) {
        case 1:
            return mt == 4 ? launch_prec<KCIN, 1, 4, 1>(p, plan, prec, st)
                           : (mt == 2 ? launch_prec<KCIN, 1, 2, 1>(p, plan, prec, st) : launch_prec<KCIN, 1, 1, 1>(p, plan, prec, st));
        case 2:
            return mt == 4 ? launch_prec<KCIN, 2, 4, 1>(p, plan, prec, st)
                           : (mt == 2 ? launch_prec<KCIN, 2, 2, 1>(p, plan, prec, st) : launch_prec<KCIN, 2, 1, 1>(p, plan, prec, st));
        case 3: return mt >= 2 ? launch_prec<KCIN, 3, 2, 1>(p, plan, prec, st) : launch_prec<KCIN, 3, 1, 1>(p, plan, prec, st);
        case 4: return mt >= 2 ? launch_prec<KCIN, 4, 2, 1>(p, plan, prec, st) : launch_prec<KCIN, 4, 1, 1>(p, plan, prec, st);
        default: return launch_prec<KCIN, 8, 1, 1>(p, plan, prec, st);
    }
}

inline int round_kcin(int cin) { return cin <= 8 ? 8 : (cin <= 16 ? 16 : (cin <= 32 ? 32 : 64)); }
inline int round_nt(int cout) {
    const int nt = (cout + 7) / 8;
    return nt <= 4 ? nt : 8;
}

// rows per warp actually instantiated for this (n-tiles per warp, warp groups, requested mt)
inline int effective_mt(int nt, int nsplit, int mt) {
    if (nsplit == 1 && nt <= 2 && mt == 4) return 4;
    if (nt <= 4 && mt >= 2) return 2;
    return 1;
}

}  // namespace

extern "C" {

int pmb200_conv2d_filter_floats(int Cin, int Cout, int KS, int precision) {
    if (Cin < 1 || Cin > 64 || Cout < 1 || Cout > 64 || KS < 1 || (precision != 1 && precision != 3)) return PMB200_EINVAL;
    return KS * KS * (round_kcin(Cin) / 8) * round_nt(Cout) * 32 * (precision == 1 ? 2 : 4);
}

int pmb200_conv2d_nhwc(const float *x, const float *filter_frag, const float *bias, const float *add_up2x, float *y, int N,
                       int H, int W, int Cin, int Cout, int KS, int stride, int pad, int dil, int relu, int precision,
                       int transposed2x, int y_channel_stride, int y_channel_offset, int rows_per_warp, void *stream) {
    if (!x || !filter_frag || !y) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: null pointer");
    if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || Cin > 64 || Cout > 64)
        return conv_fail(PMB200_EINVAL, "conv2d_nhwc: sizes out of range (1 <= Cin, Cout <= 64)");
    if (KS < 1 || KS > 7 || stride < 1 || stride > 2 || dil < 1 || pad < 0)
        return conv_fail(PMB200_EINVAL, "conv2d_nhwc: kernel size 1..7, stride 1..2, dilation >= 1");
    if (precision != 1 && precision != 3) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: precision must be 1 (TF32) or 3 (3xTF32)");
    if (transposed2x && stride != 1) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: the zero-stuffed (transposed) form runs at stride 1");
    if ((Cin % 4) == 0 && (reinterpret_cast<uintptr_t>(x) & 15u)) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: x must be 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(x) & 3u) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: x must be 4-byte aligned");
    if (reinterpret_cast<uintptr_t>(filter_frag) & 15u) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: filter must be 16-byte aligned");
    const int Hv = transposed2x ? 2 * H : H, Wv = transposed2x ? 2 * W : W;
    const int Ho = (Hv + 2 * pad - dil * (KS - 1) - 1) / stride + 1;
    const int Wo = (Wv + 2 * pad - dil * (KS - 1) - 1) / stride + 1;
    if (Ho < 1 || Wo < 1) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: empty output");
    if ((long long)H * W * Cin >= (1ll << 31)) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: one image must be smaller than 2^31 elements");
    const int ycs = y_channel_stride > 0 ? y_channel_stride : Cout;
    if (y_channel_offset < 0 || y_channel_offset + Cout > ycs) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: channel slice outside the output");
    if (((ycs | y_channel_offset) & 1) == 0 && (reinterpret_cast<uintptr_t>(y) & 7u))
        return conv_fail(PMB200_EINVAL, "conv2d_nhwc: y must be 8-byte aligned");

    if (add_up2x) {
        if ((Ho & 1) || (Wo & 1) || (Cout & 1)) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: add_up2x needs even Ho, Wo and Cout");
        if (reinterpret_cast<uintptr_t>(add_up2x) & 7u) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: add_up2x must be 8-byte aligned");
    }
    const int kcin = round_kcin(Cin), nt = round_nt(Cout);
    ConvParams p;
    p.up = add_up2x;
    p.x = x; p.wf = filter_frag; p.bias = bias; p.y = y;
    p.N = N; p.H = H; p.W = W; p.Cin = Cin; p.Ho = Ho; p.Wo = Wo; p.Cout = Cout;
    p.KS = KS; p.S = stride; p.pad = pad; p.dil = dil; p.relu = relu ? 1 : 0;
    p.ps = pixel_stride(kcin, stride);
    p.ycs = ycs; p.yco = y_channel_offset; p.stuff = transposed2x ? 1 : 0;
    p.tiles_x = (Wo + 15) / 16;
    p.rw = 15 * stride + dil * (KS - 1) + 1;
    p.cpp = (Cin % 4) == 0 ? Cin / 4 : Cin;
    p.cpp_shift = -1;
    for (int sft = 0; sft < 7; ++sft)
        if ((1 << sft) == p.cpp) p.cpp_shift = sft;

    // Work decomposition.  8 (and, when the map is small, 4) output-channel tiles are split over two warp groups that
    // share one halo tile: twice the warps per tile for the layers with few pixels and many channels.
    int dev = 0;
    cudaGetDevice(&dev);
    const int sms = sm_count(dev);
    const long px_tiles16x8 = (long)p.tiles_x * ((Ho + 7) / 8) * N;
    int nsplit = 1, ntw = nt;
    if (nt == 8 || (nt == 4 && px_tiles16x8 < 8L * sms)) {
        nsplit = 2;
        ntw = nt / 2;
    }
    if (rows_per_warp < 0) {  // negative: force rows_per_warp = -value with ONE warp group (measurement aid)
        nsplit = 1;
        ntw = nt;
        rows_per_warp = -rows_per_warp;
    }
    p.nt_total = nt;

    // rows per warp: as many as the accumulator budget allows while there are still several tiles per SM; two halo
    // buffers (prefetch of the CTA's next tile) only when a CTA will see more than ~2 tiles anyway
    int mt = rows_per_warp > 0 ? rows_per_warp : 4;
    LaunchPlan plan{0, 0};
    for (;;) {
        mt = effective_mt(ntw, nsplit, mt);
        const int rows = 4 * mt;
        p.tiles_y = (Ho + rows - 1) / rows;
        p.rh = (rows - 1) * stride + dil * (KS - 1) + 1;
        p.buf_floats = ((p.rh * p.rw * p.ps + 3) / 4) * 4;
        const size_t one = (size_t)p.buf_floats * sizeof(float);
        const long tiles = (long)p.tiles_x * p.tiles_y * N;
        const bool fits = one <= 200 * 1024;
        const bool enough = rows_per_warp > 0 || tiles >= 6L * sms || mt == 1;
        const bool roomy = rows_per_warp > 0 || one <= 56 * 1024 || mt == 1;  // >= 4 single-buffered CTAs per SM
        if (fits && enough && roomy) {
            p.total_tiles = (int)tiles;
            const long reg_cap = nsplit == 2 ? 3 : 5;  // resident CTAs per SM the register file allows (<= ~100 regs/thread)
            long cap1 = (long)(224 * 1024) / (long)(one + 1024);
            if (cap1 > reg_cap) cap1 = reg_cap;
            if (cap1 < 1) cap1 = 1;
            long cap2 = (long)(224 * 1024) / (long)(2 * one + 1024);
            if (cap2 > reg_cap) cap2 = reg_cap;
            if (tiles > 2 * cap1 * sms && cap2 >= 1 && 2 * one <= 200 * 1024) {
                p.nbuf = 2;
                plan.smem = 2 * one;
                plan.ctas = (int)(cap2 * sms < tiles ? cap2 * sms : tiles);
            } else {
                p.nbuf = 1;
                plan.smem = one;
                plan.ctas = (int)(cap1 * sms < tiles ? cap1 * sms : tiles);
            }
            break;
        }
        if (mt == 1) return conv_fail(PMB200_EINVAL, "conv2d_nhwc: halo tile does not fit in shared memory (dilation too large)");
        mt /= 2;
    }
    p.row_chunks = p.rw * p.cpp;
    p.tile_chunks = p.rh * p.row_chunks;
    p.magic_row = (unsigned)((1ull << 32) / (unsigned)p.row_chunks + 1ull);
    p.magic_cpp = (unsigned)((1ull << 32) / (unsigned)p.cpp + 1ull);
    for (int i = 0; i < 2; ++i) {
        p.step_r[i] = (128 << i) / p.row_chunks;
        p.step_c[i] = (128 << i) % p.row_chunks;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    switch (kcin) {
        case 8: return launch_shape<8>(p, plan, ntw, nsplit, mt, precision, st);
        case 16: return launch_shape<16>(p, plan, ntw, nsplit, mt, precision, st);
        case 32: return launch_shape<32>(p, plan, ntw, nsplit, mt, precision, st);
        default: return launch_shape<64>(p, plan, ntw, nsplit, mt, precision, st);
    }
}

}  // extern "C"
