// pm_conv5.cu -- K-D5: channels-last 2-D convolution as an implicit GEMM on Hopper's warpgroup tensor cores
// (wgmma.mma_async kind tf32, fp32 accumulators in registers, operands staged by TMA behind mbarriers), fp32-accurate
// through the error-compensated 3xTF32 split.  Serves the FLOP-bound layers of the cascade in the fp32-accurate (timed,
// parity) mode: FeatureNet conv2..10 (reference models/net.py:9-70), the stage-2/3 offset convs (models/patchmatch.py:288-311),
// Refinement's 16->8 conv (models/net.py:73-122).  The memory-bound layers and everything with a fused epilogue stay on
// pm_conv.cu (mma.sync).
//
// GEMM view: D[128 output pixels, Cout] = sum over filter taps of A_tap[128, Cin] . W_tap[Cin, Cout].
//   * A_tap is ONE TMA box per tap: tensor map over the channels-last input {Cin, W, H, N}, box {<=32 channels, 16*s, 8*s, 1}
//     with element strides {1, s, s, 1} (s = conv stride), placed at (x0*s + kx*dil - pad, y0*s + ky*dil - pad): the
//     padding border and the map edge come back as zeros from the copy engine, the 128 pixels of the 16 x 8 output tile
//     land as 128 rows of a K-major operand in the shared-memory swizzle (32 / 64 / 128 B = row bytes) wgmma reads.
//   * W_tap (hi and lo parts, Cout padded to a multiple of 16) is pre-packed by the host IN that shared-memory image
//     (ops.pack_conv_filter_tc5) and fetched with one bulk copy per tap.
//   * 3xTF32: every landed A tile is split in place into A_hi (13 low mantissa bits cleared -- what the tensor core would
//     read anyway) and A_lo = A - A_hi (exact); per 8-channel slice two wgmmas accumulate a_hi x [w_hi | w_lo] (N = 2 Npad)
//     and a_lo x w_hi (N = Npad) into the same fp32 registers: >= 21 bits of every product.  The accumulator fragment of
//     N = Npad is the first half of the one of N = 2 Npad, so column c holds a_hi.w_hi + a_lo.w_hi and column Npad + c holds
//     a_hi.w_lo; the epilogue adds the two.
// Roles per CTA (288 threads): warps 0..3 and 4..7 are two consumer warpgroups, each owning 64 of the tile's 128 pixels
// (split its rows, issue its wgmmas, run its epilogue); warp 8 is the TMA producer.  A consumer splits stage t+1 while
// the wgmmas of stage t are still in flight (wgmma.wait_group 1).  Persistent CTAs walk tiles blockIdx.x, +gridDim.x, ...;
// an S-deep ring of (A, A_lo, W) stages decouples producer and consumers; every mbarrier wait is bounded (a pipeline bug
// traps instead of hanging the GPU).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kTW = 16, kTH = 8;  // output tile: 128 pixels = two wgmma M = 64 halves
constexpr int kThreads = 288;     // two consumer warpgroups + one producer warp
constexpr int kProducerWarp = 8;

struct Conv5Params {
    const float *wpack;  // [tap][kblock][w_hi rows Npad | w_lo rows Npad][RB bytes], swizzled image
    const float *bias;
    float *y;
    int N, H, W, Ho, Wo, Cin, Cout, Npad, KS, S, pad, dil, relu, ycs, yco;
    int tiles_x, tiles_y, total_tiles;
    int RB;        // row bytes of one K block: min(Cin, 32) * 4
    int KB;        // K blocks: Cin / 32 (1 when Cin <= 32)
    int stages;
    int a_bytes;   // 128 * RB * KB
    int w_bytes;   // Npad * RB * KB (one of hi / lo)
    int stage_bytes;
    uint32_t layout_type;  // wgmma smem-descriptor swizzle code (bits 62-63): 1 = 128B, 2 = 64B, 3 = 32B
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *b, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(smem_u32(b)), "r"(parity)
                 : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity) {
    for (int spin = 0; spin < (1 << 22); ++spin)
        if (mbar_try_wait(b, parity)) return;
    __trap();
}
__device__ __forceinline__ void tma_box_4d(void *dst, const CUtensorMap *tm, int c0, int c1, int c2, int c3, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<unsigned long long>(tm)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void proxy_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier over `threads` threads (a multiple of 32); id 0 is __syncthreads
__device__ __forceinline__ void bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// wgmma bookkeeping: fence before the first wgmma that reads registers other code wrote, commit the issued wgmmas as one group,
// wait until at most N groups of this warp are pending
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator registers across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64, N] (+)= A[64, 8] . B[8, N]^T, tf32 operands from shared memory (both K-major), fp32 accumulators: thread (warp w, lane l)
// holds for every 8-column chunk i the registers 4i..4i+3 = (row 16w + l/4, cols 8i + 2(l%4) + {0,1}), (row + 8, same cols).
// scale_d == 0 overwrites the accumulators.
template <int N>
struct Wgmma;
template <> struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
template <> struct Wgmma<48> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
template <> struct Wgmma<96> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float *d, uint64_t a, uint64_t b, uint32_t scale_d) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(a), "l"(b), "r"(scale_d));
    }
};
// Shared-memory matrix descriptor: bits 0-13 start address >> 4, 16-29 leading byte offset >> 4 (distance of the K-adjacent
// core matrix; unused by the swizzled K-major layouts), 32-45 stride byte offset >> 4 (distance of the next 8-row group),
// 62-63 swizzle (0 none, 1 = 128B, 2 = 64B, 3 = 32B).  The kernels carry it as (lo, hi) words and only add 16-byte offsets
// to lo (shared-memory addresses stay below 2^18, so the 14-bit field never carries).
__device__ __forceinline__ uint64_t desc_of(uint32_t lo, uint32_t hi) { return ((uint64_t)hi << 32) | lo; }

// the epilogue of one consumer warpgroup: its 64 accumulator rows -> bias, ReLU -> channels-last stores (channel slice of a
// wider tensor allowed).  pix(m) maps the tile row m (0..127) to the output pixel; rows outside the map are dropped.
template <int NPAD, typename PixOf>
__device__ __forceinline__ void store_tile(const float (&acc)[NPAD], const float *bias, float *y, int n, int Ho, int Wo, int Cout,
                                           int relu, int ycs, int yco, int row0, PixOf pix) {
    const int lane = threadIdx.x & 31, w4 = (threadIdx.x >> 5) & 3;
    const bool vec2 = ((ycs | yco) & 1) == 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = row0 + 16 * w4 + (lane >> 2) + 8 * h;
        int oy, ox;
        pix(m, oy, ox);
        if (oy >= Ho || ox >= Wo) continue;
        float *dst = y + (((size_t)n * Ho + oy) * Wo + ox) * ycs + yco;
#pragma unroll
        for (int i = 0; i < NPAD / 8; ++i) {
            const int co = 8 * i + 2 * (lane & 3);
            float v0 = acc[4 * i + 2 * h] + acc[4 * (i + NPAD / 8) + 2 * h];
            float v1 = acc[4 * i + 2 * h + 1] + acc[4 * (i + NPAD / 8) + 2 * h + 1];
            if (bias) {
                v0 += co < Cout ? __ldg(bias + co) : 0.0f;
                v1 += co + 1 < Cout ? __ldg(bias + co + 1) : 0.0f;
            }
            if (relu) { v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f); }
            if (co + 1 < Cout && vec2) {
                *reinterpret_cast<float2 *>(dst + co) = make_float2(v0, v1);
            } else {
                if (co < Cout) dst[co] = v0;
                if (co + 1 < Cout) dst[co + 1] = v1;
            }
        }
    }
}

__device__ __forceinline__ float4 tf32_hi(const float4 v) {
    return make_float4(__uint_as_float(__float_as_uint(v.x) & 0xffffe000u), __uint_as_float(__float_as_uint(v.y) & 0xffffe000u),
                       __uint_as_float(__float_as_uint(v.z) & 0xffffe000u), __uint_as_float(__float_as_uint(v.w) & 0xffffe000u));
}

template <int NPAD>
__global__ void __launch_bounds__(kThreads) conv5_kernel(const Conv5Params p, const __grid_constant__ CUtensorMap xmap) {
    extern __shared__ unsigned char smem_raw[];
    // the swizzled operand tiles need 1024-byte alignment: align the dynamic segment by hand (the launch adds the slack)
    unsigned char *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    // [0, 256): barriers; stages start at 1024
    uint64_t *full = reinterpret_cast<uint64_t *>(smem);  // [stages]  TMA landed
    uint64_t *empty = full + 8;                            // [stages]  the wgmmas that read the stage have completed (8 warps)
    unsigned char *stage0 = smem + 1024;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < p.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int T = p.KS * p.KS;
    const int per_img = p.tiles_x * p.tiles_y;

    if (warp == kProducerWarp) {
        // ------------------------------------------------ TMA producer ------------------------------------------------
        if (lane == 0) {
            int s = 0;
            uint32_t par = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                const int n = tile / per_img, tt = tile - n * per_img;
                const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
                const int x_in0 = tx * kTW * p.S - p.pad, y_in0 = ty * kTH * p.S - p.pad;
                for (int t = 0; t < T; ++t) {
                    mbar_wait(&empty[s], par ^ 1u);
                    unsigned char *st = stage0 + (size_t)s * p.stage_bytes;
                    mbar_arrive_expect_tx(&full[s], (uint32_t)(p.a_bytes + 2 * p.w_bytes));
                    const int ky = t / p.KS, kx = t - ky * p.KS;
                    for (int kb = 0; kb < p.KB; ++kb)
                        tma_box_4d(st + (size_t)kb * 128 * p.RB, &xmap, kb * 32, x_in0 + kx * p.dil, y_in0 + ky * p.dil, n, &full[s]);
                    bulk_g2s(st + 2 * (size_t)p.a_bytes, reinterpret_cast<const unsigned char *>(p.wpack) + (size_t)t * 2 * p.w_bytes,
                             (uint32_t)(2 * p.w_bytes), &full[s]);
                    if (++s == p.stages) { s = 0; par ^= 1u; }
                }
            }
        }
        return;
    }
    // ------------------------------------------------- consumers -------------------------------------------------
    const int wg = warp >> 2, wt = threadIdx.x & 127;
    float acc[NPAD];
    int s = 0, pend = -1;  // pend: stage whose wgmmas may still be in flight
    uint32_t par = 0;
    const int per_row = p.RB / 32;  // 8-channel slices per operand row
    const uint32_t hiword = ((8u * (uint32_t)p.RB) >> 4) | (p.layout_type << 30);  // SBO = 8 rows
    const uint32_t stage_u32 = smem_u32(stage0);
    const uint32_t a_kb16 = (128u * (uint32_t)p.RB) >> 4, w_kb16 = (2u * (uint32_t)NPAD * (uint32_t)p.RB) >> 4;
    const uint32_t half16 = (uint32_t)wg * ((64u * (uint32_t)p.RB) >> 4);  // this warpgroup's 64 rows
    const int chunks = 4 * p.RB;                           // 16-byte chunks of 64 rows of one K block
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        for (int t = 0; t < T; ++t) {
            mbar_wait(&full[s], par);
            unsigned char *a = stage0 + (size_t)s * p.stage_bytes;
            for (int kb = 0; kb < p.KB; ++kb) {
                unsigned char *rows = a + (size_t)kb * 128 * p.RB + (size_t)wg * 64 * p.RB;
                for (int c = wt; c < chunks; c += 128) {
                    float4 *q = reinterpret_cast<float4 *>(rows + (size_t)c * 16);
                    const float4 v = *q, h = tf32_hi(v);
                    *q = h;
                    *reinterpret_cast<float4 *>(reinterpret_cast<unsigned char *>(q) + p.a_bytes) =
                        make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
                }
            }
            proxy_fence_async();  // generic-proxy writes above -> visible to the tensor core's async-proxy reads
            bar_sync(1 + wg, 128);
            const uint32_t a_hi = ((stage_u32 + (uint32_t)(s * p.stage_bytes)) >> 4) + half16;
            const uint32_t a_lo = a_hi + ((uint32_t)p.a_bytes >> 4), w0 = ((stage_u32 + (uint32_t)(s * p.stage_bytes)) >> 4) +
                                                                           2u * ((uint32_t)p.a_bytes >> 4);
            acc_fence(acc);
            wg_fence();
            for (int kb = 0; kb < p.KB; ++kb) {
                for (int kin = 0; kin < per_row; ++kin) {
                    const uint32_t ao = (uint32_t)kb * a_kb16 + 2u * kin, wo = (uint32_t)kb * w_kb16 + 2u * kin;  // 32 bytes per slice
                    const uint64_t dw = desc_of((w0 + wo) | (1u << 16), hiword);
                    Wgmma<2 * NPAD>::mma(acc, desc_of((a_hi + ao) | (1u << 16), hiword), dw, (t | kb | kin) ? 1u : 0u);
                    Wgmma<NPAD>::mma(acc, desc_of((a_lo + ao) | (1u << 16), hiword), dw, 1u);
                }
            }
            wg_commit();
            acc_fence(acc);
            wg_wait<1>();  // the wgmmas of the previous stage have completed: hand it back to the producer
            if (pend >= 0 && lane == 0) mbar_arrive(&empty[pend]);
            pend = s;
            if (++s == p.stages) { s = 0; par ^= 1u; }
        }
        wg_wait<0>();
        acc_fence(acc);
        if (lane == 0) mbar_arrive(&empty[pend]);
        pend = -1;
        const int n = tile / per_img, tt = tile - n * per_img;
        const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
        store_tile<NPAD>(acc, p.bias, p.y, n, p.Ho, p.Wo, p.Cout, p.relu, p.ycs, p.yco, 64 * wg,
                         [&](int m, int &oy, int &ox) { oy = ty * kTH + m / kTW; ox = tx * kTW + m % kTW; });
    }
}

// ----------------------------------------------------------------------------------------------------------------------
// K-D5h: the stride-1 form.  conv5_kernel above re-reads (and re-splits) the input once per filter tap; for stride 1 every
// tap's A operand is just a SHIFTED view of one halo tile, if that tile is stored so that a shift keeps the tensor core's
// canonical layout intact.  The no-swizzle K-major layout does: its core matrix is 8 rows x 16 bytes stored contiguously,
// so with the halo tile kept as channel-chunk PLANES [Cin/4][rows][cols][4 floats] (16 bytes per pixel and plane)
//   * 8 consecutive pixels of one plane ARE a core matrix (128 contiguous bytes),
//   * the next 8-row group of the operand = the next output row = + (halo cols * 16) bytes      (descriptor SBO),
//   * the second half of an 8-channel K slice = the next plane = + (halo rows * cols * 16) bytes (descriptor LBO),
//   * filter tap (ky, kx) = start address + ((ky*dil) * cols + kx*dil) * 16 bytes -- always 16-byte aligned, no swizzle phase,
// The halo tile arrives as ONE dense TMA box {Cin, cols, rows, 1} (rows of Cin*4 bytes, zero fill for the padding) in a staging
// buffer; the consumer warpgroup that owns it, which touches every element anyway, writes A_hi / A_lo TRANSPOSED into its
// planes (chunk order rotated by pixel: conflict-free reads and writes).
// Work unit: the 8 x 8 output block one warpgroup's M = 64 covers.  Each consumer warpgroup walks its OWN units (worker
// blockIdx.x + wg * gridDim.x of 2 * gridDim.x) with its own plane set: it splits, issues its wgmmas and runs its epilogue
// without meeting the other warpgroup, so one warpgroup's split and epilogue run under the other's wgmmas.  Load and split
// happen ONCE per unit; the filter taps stay resident in shared memory when they fit, else stream through a small ring that
// both warpgroups read in step (a warpgroup out of units passes over the ring's taps until the other one is done).
// The filter tap is stored as ONE operand [chunk][w_hi rows | w_lo rows][4 floats] (ops.pack_conv_filter_tc5h): a_hi x
// [w_hi | w_lo] is one wgmma of N = 2 Npad, a_lo x w_hi one of N = Npad -- 2 wgmmas per K slice instead of 3.
// ----------------------------------------------------------------------------------------------------------------------
constexpr int kHT = 8;  // output unit: 8 x 8 pixels = one warpgroup's M = 64

struct Conv5hParams {
    const float *wpack;  // [tap][Cin/4 chunks][hi rows Npad | lo rows Npad][4]
    const float *bias;
    float *y;
    int N, H, W, Ho, Wo, Cin, Cout, Npad, KS, pad, dil, relu, ycs, yco;
    int tiles_x, tiles_y, total_tiles;  // 8 x 8 units
    int hcols, hrows;     // halo tile: 8 + dil*(KS-1) columns and rows
    int plane_bytes;      // hrows * hcols * 16
    int a_bytes;          // plane_bytes * Cin/4 (one of hi / lo) = what one TMA box delivers into a staging buffer
    int a_stride;         // a_bytes rounded up to 128: distance between staging buffers, hi -> lo, plane sets (2 * a_stride)
    int sbufs;            // staging buffers shared by both warpgroups in request order: 2 when they fit (one per warpgroup), else 1
    int psets;            // plane sets: 2 (one per consumer warpgroup), or 1 when there are no more units than CTAs (warpgroup 1
                          // then never owns a unit and the space goes to the filter ring)
    int w_bytes;          // Npad * Cin * 4 (one of hi / lo)
    int wstages;
    int w_resident;       // 1: wstages == KS*KS, every tap loaded once per CTA; 0: taps stream through the ring per unit
    // Debugging aid (pmb200_debug_conv5h_trace): clock64 stamps of CTA 0, [role][unit 0..15 of warpgroup 0][event 0..3]:
    // role 0 producer (ev 0: halo requested), 1 wgmmas (ev 0: all completed), 2 split (ev 0: halo landed, ev 1: planes
    // written), 3 epilogue (ev 0: stored).  Only warpgroup 0's units are stamped.
    long long *trace;
};

__device__ __forceinline__ void stamp(const Conv5hParams &p, int role, int it, int ev) {
    if (p.trace && blockIdx.x == 0 && it < 16) p.trace[(role * 16 + it) * 4 + ev] = clock64();
}

// the wgmmas of one filter tap: per 8-channel slice a_hi x [w_hi | w_lo] (N = 2 Npad) and a_lo x w_hi (N = Npad)
template <int NPAD, int KSL>
__device__ __forceinline__ void issue_tap(float (&acc)[NPAD], uint32_t ah, uint32_t al, uint32_t w, uint32_t a_kstep, uint32_t w_kstep,
                                          uint32_t a_hiword, uint32_t w_hiword, uint32_t first) {
#pragma unroll
    for (int k = 0; k < KSL; ++k) {
        const uint64_t dw = desc_of(w + k * w_kstep, w_hiword);
        Wgmma<2 * NPAD>::mma(acc, desc_of(ah + k * a_kstep, a_hiword), dw, k == 0 ? first : 1u);
        Wgmma<NPAD>::mma(acc, desc_of(al + k * a_kstep, a_hiword), dw, 1u);
    }
}

template <int NPAD>
__global__ void __launch_bounds__(kThreads) conv5h_kernel(const Conv5hParams p, const __grid_constant__ CUtensorMap xmap) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
    uint64_t *h_full = reinterpret_cast<uint64_t *>(smem);  // [warpgroup] this warpgroup's next halo tile has landed
    uint64_t *s_free = h_full + 2;                           // [sbufs] the split has read the staging buffer
    uint64_t *w_full = s_free + 2;                           // [25] filter tap landed
    uint64_t *w_empty = w_full + 25;                         // [25] its wgmmas have completed (8 consumer warps)
    unsigned char *stage0 = smem + 640;                                     // [sbufs][a_stride]  dense [rows][cols][Cin]
    unsigned char *halo0 = stage0 + (size_t)p.sbufs * p.a_stride;           // [psets][hi, lo][a_stride]  planes of warpgroup 0, 1
    unsigned char *wring = halo0 + (size_t)p.psets * 2 * p.a_stride;        // [wstages][hi, lo][w_bytes]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int a = 0; a < 2; ++a) {
            mbar_init(&h_full[a], 1);
            mbar_init(&s_free[a], 1);
        }
        for (int s = 0; s < p.wstages; ++s) {
            mbar_init(&w_full[s], 1);
            mbar_init(&w_empty[s], 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int T = p.KS * p.KS;
    const int per_img = p.tiles_x * p.tiles_y;
    // unit k of warpgroup g is blockIdx.x + (2k + g) * gridDim.x; warpgroup 0 has n0 units, warpgroup 1 n0 or n0 - 1
    const int G = gridDim.x, U = p.total_tiles;
    const int n0 = ((int)blockIdx.x < U) ? (U - (int)blockIdx.x + 2 * G - 1) / (2 * G) : 0;
    auto unit_of = [&](int g, int k) { return (int)blockIdx.x + (2 * k + g) * G; };

    if (warp == kProducerWarp) {
        // ------------------------------------------------ TMA producer ------------------------------------------------
        // Halo requests are numbered r = 2k + g and take staging buffer r % sbufs: request r waits for the split of r - sbufs
        // (only this thread waits on s_free, in request order).  Each warpgroup has its own h_full, so it waits on every phase
        // of it in turn even when the two share one staging buffer.
        if (lane == 0) {
            auto load_halo = [&](int g, int k) {
                const int u = unit_of(g, k);
                if (k >= n0 || u >= U) return;
                const int r = 2 * k + g, sb = r % p.sbufs;
                const int n = u / per_img, tt = u - n * per_img;
                const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
                mbar_wait(&s_free[sb], ((uint32_t)(r / p.sbufs) & 1u) ^ 1u);
                if (g == 0) stamp(p, 0, k, 0);
                mbar_arrive_expect_tx(&h_full[g], (uint32_t)p.a_bytes);
                tma_box_4d(stage0 + (size_t)sb * p.a_stride, &xmap, 0, tx * kHT - p.pad, ty * kHT - p.pad, n, &h_full[g]);
            };
            auto load_tap = [&](int t, int s) {
                mbar_arrive_expect_tx(&w_full[s], (uint32_t)(2 * p.w_bytes));
                bulk_g2s(wring + (size_t)s * 2 * p.w_bytes, reinterpret_cast<const unsigned char *>(p.wpack) + (size_t)t * 2 * p.w_bytes,
                         (uint32_t)(2 * p.w_bytes), &w_full[s]);
            };
            load_halo(0, 0);
            load_halo(1, 0);
            if (p.w_resident)
                for (int t = 0; t < T; ++t) load_tap(t, t);  // the whole filter stays in shared memory: loaded once per CTA
            int s = 0;
            uint32_t wpar = 0;
            for (int k = 0; k < n0; ++k) {
                // the NEXT units' halos first: their latency (and their splits) hide under this unit's wgmmas.  With one
                // staging buffer, warpgroup 1's request waits for warpgroup 0's split of unit k + 1, which needs the taps of
                // unit k: issue those first.
                load_halo(0, k + 1);
                if (p.w_resident || p.sbufs > 1) load_halo(1, k + 1);
                if (p.w_resident) continue;
                for (int t = 0; t < T; ++t) {
                    mbar_wait(&w_empty[s], wpar ^ 1u);
                    load_tap(t, s);
                    if (++s == p.wstages) { s = 0; wpar ^= 1u; }
                }
                if (p.sbufs == 1) load_halo(1, k + 1);
            }
        }
        return;
    }
    // ------------------------------------------------- consumers -------------------------------------------------
    const int wg = warp >> 2, wt = threadIdx.x & 127;  // wt: 0..127 within this warpgroup
    float acc[NPAD];
    int s = 0;
    uint32_t wpar = 0;
    const int kslices = p.Cin / 8;
    const int P = p.hcols * p.hrows, NC = p.Cin / 4;  // pixels of the halo tile, 16-byte channel chunks per pixel
    const uint32_t a_hiword = (uint32_t)p.hcols;          // SBO = hcols * 16 bytes, no swizzle
    const uint32_t w_hiword = 128u >> 4;                  // SBO = 128 bytes
    const uint32_t a_lbo16 = (uint32_t)p.plane_bytes >> 4, w_lbo16 = 2u * (uint32_t)NPAD;  // next chunk: plane / 2 Npad rows
    const uint32_t a_kstep = 2u * a_lbo16, w_kstep = 2u * w_lbo16;                        // one K slice = two chunks
    const uint32_t ring_u32 = smem_u32(wring);
    unsigned char *planes = halo0 + (size_t)wg * 2 * p.a_stride;  // this warpgroup's A_hi, A_lo
    const uint32_t ahi_lo = (smem_u32(planes) >> 4) | (a_lbo16 << 16);
    const uint32_t alo_lo = ahi_lo + ((uint32_t)p.a_stride >> 4);
    const bool stamps = wg == 0 && wt == 0;
    // With a streamed filter both warpgroups read every tap of the ring, so both walk n0 units; a warpgroup whose unit lies
    // past the end only passes over the taps.  A resident filter needs no such pass.
    const int iters = wg == 0 || !p.w_resident ? n0 : (n0 > 0 && unit_of(1, n0 - 1) < U ? n0 : n0 - 1);
    for (int k = 0; k < iters; ++k) {
        const int unit = unit_of(wg, k);
        if (unit >= U) {
            for (int t = 0; t < T; ++t) {
                mbar_wait(&w_full[s], wpar);
                if (lane == 0) mbar_arrive(&w_empty[s]);
                if (++s == p.wstages) { s = 0; wpar ^= 1u; }
            }
            continue;
        }
        // ---- split: dense staging tile -> this warpgroup's A_hi / A_lo planes.  The barrier first: every warp of the
        // warpgroup has waited for its wgmmas of unit k - 1, which read the planes.
        const int r = 2 * k + wg, sb = r % p.sbufs;
        mbar_wait(&h_full[wg], (uint32_t)k & 1u);
        if (stamps) stamp(p, 2, k, 0);
        bar_sync(1 + wg, 128);
        {
            const float4 *src = reinterpret_cast<const float4 *>(stage0 + (size_t)sb * p.a_stride);
            float4 *ahi = reinterpret_cast<float4 *>(planes);
            float4 *alo = reinterpret_cast<float4 *>(planes + p.a_stride);
            for (int px = wt; px < P; px += 128) {
                for (int j = 0; j < NC; ++j) {
                    const int c = (j + px) & (NC - 1);  // rotated by pixel: the 8 lanes of a quarter-warp read 8 bank groups
                    const float4 v = src[px * NC + c], h = tf32_hi(v);
                    ahi[c * P + px] = h;  // plane c: 16 bytes per pixel; consecutive lanes, consecutive pixels
                    alo[c * P + px] = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
                }
            }
        }
        proxy_fence_async();
        bar_sync(1 + wg, 128);
        if (wt == 0) mbar_arrive(&s_free[sb]);
        if (stamps) stamp(p, 2, k, 1);
        // ---- wgmmas of this unit's 64 pixels
        int pend = -1;  // ring slot whose wgmmas may still be in flight
        acc_fence(acc);
        for (int ky = 0; ky < p.KS; ++ky) {
            for (int kx = 0; kx < p.KS; ++kx) {
                if (!p.w_resident || k == 0) mbar_wait(&w_full[s], wpar);  // a resident filter is waited for once
                const uint32_t shift = (uint32_t)((ky * p.dil) * p.hcols + kx * p.dil);
                const uint32_t ah = ahi_lo + shift, al = alo_lo + shift;
                const uint32_t w = ((ring_u32 + (uint32_t)(s * 2 * p.w_bytes)) >> 4) | (w_lbo16 << 16);
                const uint32_t first = (ky | kx) ? 1u : 0u;  // 0 for the very first wgmma of the unit (overwrites the accumulators)
                wg_fence();
                switch (kslices) {  // unrolled: the per-slice descriptor steps become immediates
                case 1: issue_tap<NPAD, 1>(acc, ah, al, w, a_kstep, w_kstep, a_hiword, w_hiword, first); break;
                case 2: issue_tap<NPAD, 2>(acc, ah, al, w, a_kstep, w_kstep, a_hiword, w_hiword, first); break;
                case 4: issue_tap<NPAD, 4>(acc, ah, al, w, a_kstep, w_kstep, a_hiword, w_hiword, first); break;
                default: issue_tap<NPAD, 8>(acc, ah, al, w, a_kstep, w_kstep, a_hiword, w_hiword, first); break;
                }
                wg_commit();
                acc_fence(acc);
                if (p.w_resident) {
                    if (++s == p.wstages) s = 0;  // phase 0 of every w_full completed once and stays complete
                } else {
                    wg_wait<1>();  // the previous tap's wgmmas have completed: its ring slot goes back to the producer
                    if (pend >= 0 && lane == 0) mbar_arrive(&w_empty[pend]);
                    pend = s;
                    if (++s == p.wstages) { s = 0; wpar ^= 1u; }
                }
            }
        }
        wg_wait<0>();
        acc_fence(acc);
        if (pend >= 0 && lane == 0) mbar_arrive(&w_empty[pend]);
        if (stamps) stamp(p, 1, k, 0);
        const int n = unit / per_img, tt = unit - n * per_img;
        const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
        store_tile<NPAD>(acc, p.bias, p.y, n, p.Ho, p.Wo, p.Cout, p.relu, p.ycs, p.yco, 0,
                         [&](int m, int &oy, int &ox) { oy = ty * kHT + m / kHT; ox = tx * kHT + m % kHT; });
        if (stamps) stamp(p, 3, k, 0);
    }
}

long long *g_conv5h_trace = nullptr;

PFN_cuTensorMapEncodeTiled_v12000 encoder() {
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

// Opt a kernel in to the device's maximum dynamic shared memory, once per (kernel, device).  Always the SAME value, so
// concurrent host threads (one per GPU, or several streams of one GPU) can only repeat an idempotent call -- a per-thread or
// per-size high-water mark let one thread lower the attribute under another thread's larger launch.
template <typename Kern>
bool optin_max_smem(Kern kern, std::atomic<unsigned long long> &done, int dev, int smem_optin) {
    if (dev >= 0 && dev < 64 && ((done.load(std::memory_order_relaxed) >> dev) & 1ull)) return true;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_optin) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    if (dev >= 0 && dev < 64) done.fetch_or(1ull << dev, std::memory_order_relaxed);
    return true;
}

// CTAs per SM the kernel's registers allow at this shared-memory size (at least 1, at most `want`)
template <typename Kern>
int resident_ctas(Kern kern, int smem, int want) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kThreads, smem) != cudaSuccess) {
        cudaGetLastError();
        return 1;
    }
    return n < 1 ? 1 : (n > want ? want : n);
}

int npad_of(int cout) { return (cout + 15) / 16 * 16; }

// one instantiation per padded Cout: the accumulator fragment is a register array of Npad floats per thread
template <template <int> class Launch, typename... Args>
int by_npad(int npad, Args &&...args) {
    switch (npad) {
    case 16: return Launch<16>::run(args...);
    case 32: return Launch<32>::run(args...);
    case 48: return Launch<48>::run(args...);
    default: return Launch<64>::run(args...);
    }
}

template <int NPAD>
struct LaunchConv5 {
    static int run(const Conv5Params &p, const CUtensorMap &xmap, int dev, int sms, int smem_optin, cudaStream_t st) {
        static std::atomic<unsigned long long> optin_done{0};
        if (!optin_max_smem(conv5_kernel<NPAD>, optin_done, dev, smem_optin))
            return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5: shared-memory opt-in failed");
        const int smem = 1024 + p.stages * p.stage_bytes + 1024;  // + slack for the 1024-byte alignment of the dynamic segment
        const int two = (2 * smem <= smem_optin + 1024) ? 2 : 1;
        long long grid = (long long)sms * resident_ctas(conv5_kernel<NPAD>, smem, two);
        if (grid > p.total_tiles) grid = p.total_tiles;
        conv5_kernel<NPAD><<<(unsigned)grid, kThreads, smem, st>>>(p, xmap);
        return pmb200_internal_launch_status("conv2d_tc5");
    }
};

template <int NPAD>
struct LaunchConv5h {
    static int run(const Conv5hParams &p, const CUtensorMap &xmap, int smem, int ctas, int dev, int sms, int smem_optin, cudaStream_t st) {
        static std::atomic<unsigned long long> optin_done{0};
        if (!optin_max_smem(conv5h_kernel<NPAD>, optin_done, dev, smem_optin))
            return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: shared-memory opt-in failed");
        long long grid = (long long)sms * resident_ctas(conv5h_kernel<NPAD>, smem, ctas);
        if (grid > p.total_tiles) grid = p.total_tiles;
        conv5h_kernel<NPAD><<<(unsigned)grid, kThreads, smem, st>>>(p, xmap);
        return pmb200_internal_launch_status("conv2d_tc5h");
    }
};

}  // namespace

extern "C" {

// 1 when pmb200_conv2d_tc5 takes this layer
int pmb200_conv2d_tc5_supported(int Cin, int Cout, int KS, int stride) {
    const bool cin_ok = Cin == 8 || Cin == 16 || Cin == 32 || Cin == 64;
    return (cin_ok && Cout >= 1 && Cout <= 64 && (KS == 1 || KS == 3 || KS == 5) && (stride == 1 || stride == 2)) ? 1 : 0;
}

// floats of the packed filter: [tap][Cin/32 blocks][hi rows Npad | lo rows Npad][min(Cin,32)] (ops.pack_conv_filter_tc5)
int pmb200_conv2d_tc5_filter_floats(int Cin, int Cout, int KS) {
    if (!pmb200_conv2d_tc5_supported(Cin, Cout, KS, 1)) return -1;
    return KS * KS * 2 * npad_of(Cout) * Cin;
}

int pmb200_conv2d_tc5(const float *x_nhwc, const float *filter_tc5, const float *bias, float *y_nhwc, int N, int H, int W, int Cin,
                      int Cout, int KS, int stride, int pad, int dil, int relu, int y_channel_stride, int y_channel_offset,
                      void *stream) {
    if (!x_nhwc || !filter_tc5 || !y_nhwc) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: null pointer");
    if (!pmb200_conv2d_tc5_supported(Cin, Cout, KS, stride))
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5: Cin in {8,16,32,64}, Cout <= 64, KS in {1,3,5}, stride 1 or 2");
    if (N < 1 || H < 1 || W < 1 || pad < 0 || dil < 1) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: bad size");
    if ((reinterpret_cast<uintptr_t>(x_nhwc) & 15u) || (reinterpret_cast<uintptr_t>(filter_tc5) & 15u))
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: input and filter must be 16-byte aligned");
    const int Ho = (H + 2 * pad - dil * (KS - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (KS - 1) - 1) / stride + 1;
    if (Ho < 1 || Wo < 1) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: empty output");
    if (y_channel_stride < Cout + y_channel_offset || y_channel_offset < 0)
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: output channel slice out of range");
    auto enc = encoder();
    if (!enc) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5: cuTensorMapEncodeTiled unavailable");

    Conv5Params p;
    p.wpack = filter_tc5; p.bias = bias; p.y = y_nhwc;
    p.N = N; p.H = H; p.W = W; p.Ho = Ho; p.Wo = Wo; p.Cin = Cin; p.Cout = Cout; p.Npad = npad_of(Cout);
    p.KS = KS; p.S = stride; p.pad = pad; p.dil = dil; p.relu = relu; p.ycs = y_channel_stride; p.yco = y_channel_offset;
    p.tiles_x = (Wo + kTW - 1) / kTW; p.tiles_y = (Ho + kTH - 1) / kTH;
    const long long tiles = (long long)p.tiles_x * p.tiles_y * N;
    if (tiles > 0x7fffffffLL) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: too many tiles");
    p.total_tiles = (int)tiles;
    const int cblk = Cin < 32 ? Cin : 32;
    p.RB = cblk * 4;
    p.KB = Cin / cblk;
    p.a_bytes = 128 * p.RB * p.KB;
    p.w_bytes = p.Npad * p.RB * p.KB;
    p.stage_bytes = 2 * p.a_bytes + 2 * p.w_bytes;  // multiples of 1024 except tiny layers: keep every stage 1024-aligned
    p.stage_bytes = (p.stage_bytes + 1023) / 1024 * 1024;
    p.layout_type = p.RB == 128 ? 1u : (p.RB == 64 ? 2u : 3u);

    int dev = 0, sms = 0, smem_optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    // two CTAs per SM when the ring allows at least 3 stages each, else one CTA with as many stages as fit (<= 8)
    int stages = ((smem_optin + 1024) / 2 - 1024 - 2048) / p.stage_bytes;
    if (stages < 3) stages = (smem_optin - 2048) / p.stage_bytes;
    if (stages > 8) stages = 8;
    if (stages < 2) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5: a ring of two stages does not fit in shared memory");
    p.stages = stages;
    CUtensorMap xmap;
    const cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t strides[3] = {(cuuint64_t)Cin * 4, (cuuint64_t)W * Cin * 4, (cuuint64_t)H * W * Cin * 4};
    const cuuint32_t box[4] = {(cuuint32_t)cblk, (cuuint32_t)(kTW * stride), (cuuint32_t)(kTH * stride), 1u};
    const cuuint32_t estr[4] = {1u, (cuuint32_t)stride, (cuuint32_t)stride, 1u};
    const CUtensorMapSwizzle sw = p.RB == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : (p.RB == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    if (enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(x_nhwc), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5: tensor map rejected (alignment / size)");
    return by_npad<LaunchConv5>(p.Npad, p, xmap, dev, sms, smem_optin, reinterpret_cast<cudaStream_t>(stream));
}

// Debugging aid: device buffer of 4 roles x 16 units x 4 events (256 int64) that the next K-D5h launches stamp with clock64
// for warpgroup 0 of CTA 0 (Conv5hParams::trace: producer / wgmmas done / split / epilogue done); nullptr switches it off.  Not part of the reference-facing surface.
int pmb200_debug_conv5h_trace(long long *device_buffer_256) {
    g_conv5h_trace = device_buffer_256;
    return 0;
}

// K-D5h shared-memory plan (see include/patchmatch_b200.h).  Barriers (640 B), staging buffers, one plane set (hi, lo) per
// consumer warpgroup, filter stages, 128 B alignment slack.  Preference order: whole filter resident with a staging buffer per
// warpgroup; resident with one shared staging buffer; else a ring as deep as fits (>= 2 stages; the staging buffer per
// warpgroup is kept when 4 stages fit with it).  As many CTAs per SM (up to 4) as the SM's shared memory holds; the launch
// lowers that to what the registers allow.  With no more units than SMs
// every CTA gets one unit, run by warpgroup 0: one plane set and one staging buffer, the rest for the ring (the stage-3
// offset convs, whose two-slot ring otherwise leaves every tap's filter load exposed).
int pmb200_conv2d_tc5h_plan(int Cin, int Cout, int KS, int dil, int units, int sms, int smem_optin, int *plan) {
    if (!plan || !pmb200_conv2d_tc5_supported(Cin, Cout, KS, 1) || dil < 1 || units < 1 || sms < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h_plan: unsupported layer");
    const int side = kHT + dil * (KS - 1);
    if (side > 256) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: dilation too large for one TMA box");
    const long long a_stride = ((long long)side * side * 16 * (Cin / 4) + 127) / 128 * 128;
    const long long w2 = 2LL * npad_of(Cout) * Cin * 4;  // one filter stage: hi + lo
    const int T = KS * KS;
    const int psets = units <= sms ? 1 : 2;
    auto fixed_of = [&](int sb) { return 640 + sb * a_stride + psets * 2 * a_stride + 128; };
    int sbufs = psets, wst = 0, resident = 0;
    if (fixed_of(sbufs) + T * w2 <= smem_optin) { resident = 1; wst = T; }
    else if (fixed_of(1) + T * w2 <= smem_optin) { sbufs = 1; resident = 1; wst = T; }
    else {
        const int want_w = T < 4 ? T : 4;
        if (fixed_of(sbufs) + want_w * w2 > smem_optin) sbufs = 1;
        const long long fit = (smem_optin - fixed_of(sbufs)) / w2;
        wst = fit > 8 ? 8 : (int)(fit < 0 ? 0 : fit);
        if (wst > T) wst = T;
        // a ring slot is released one tap after its wgmmas were issued, so a streamed filter needs two slots
        if (wst < 2) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: halo tiles + filter ring do not fit in shared memory");
    }
    const long long per_sm = smem_optin + 1024;  // an SM's shared memory: the per-block limit + the 1 KB the driver reserves per block
    // A resident filter that leaves room for one CTA only (conv6/7): a ring of >= 4 stages that lets two CTAs share the SM
    // measured faster, alone and beside the other requests' kernels.
    if (resident && psets == 2 && 2 * (fixed_of(sbufs) + wst * w2 + 1024) > per_sm) {
        const long long budget = per_sm / 2 - 1024;
        for (int sb = 2; sb >= 1; --sb) {
            long long fit = (budget - fixed_of(sb)) / w2;
            if (fit > 8) fit = 8;
            if (fit > T) fit = T;
            if (fit >= 4) { sbufs = sb; wst = (int)fit; resident = wst == T; break; }
        }
    }
    const long long smem = fixed_of(sbufs) + wst * w2;
    long long ctas = per_sm / (smem + 1024);
    plan[0] = sbufs;
    plan[1] = wst;
    plan[2] = resident;
    plan[3] = (int)smem;
    plan[4] = (int)(ctas > 4 ? 4 : (ctas < 1 ? 1 : ctas));
    plan[5] = psets;
    return 0;
}

// Stride-1 form (K-D5h): one halo tile per 8 x 8 output unit, filter taps as shifted views.  Filter image:
// [tap][Cin/4 chunks][hi rows Npad | lo rows Npad][4 floats] (ops.pack_conv_filter_tc5h), same float count as the per-tap form.
int pmb200_conv2d_tc5h(const float *x_nhwc, const float *filter_tc5h, const float *bias, float *y_nhwc, int N, int H, int W, int Cin,
                       int Cout, int KS, int pad, int dil, int relu, int y_channel_stride, int y_channel_offset, void *stream) {
    if (!x_nhwc || !filter_tc5h || !y_nhwc) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: null pointer");
    if (!pmb200_conv2d_tc5_supported(Cin, Cout, KS, 1))
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: Cin in {8,16,32,64}, Cout <= 64, KS in {1,3,5}");
    if (N < 1 || H < 1 || W < 1 || pad < 0 || dil < 1) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: bad size");
    if ((reinterpret_cast<uintptr_t>(x_nhwc) & 15u) || (reinterpret_cast<uintptr_t>(filter_tc5h) & 15u))
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: input and filter must be 16-byte aligned");
    const int Ho = H + 2 * pad - dil * (KS - 1), Wo = W + 2 * pad - dil * (KS - 1);
    if (Ho < 1 || Wo < 1) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: empty output");
    if (y_channel_stride < Cout + y_channel_offset || y_channel_offset < 0)
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: output channel slice out of range");
    auto enc = encoder();
    if (!enc) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: cuTensorMapEncodeTiled unavailable");
    Conv5hParams p;
    p.wpack = filter_tc5h; p.bias = bias; p.y = y_nhwc;
    p.N = N; p.H = H; p.W = W; p.Ho = Ho; p.Wo = Wo; p.Cin = Cin; p.Cout = Cout; p.Npad = npad_of(Cout);
    p.KS = KS; p.pad = pad; p.dil = dil; p.relu = relu; p.ycs = y_channel_stride; p.yco = y_channel_offset;
    p.trace = g_conv5h_trace;
    p.tiles_x = (Wo + kHT - 1) / kHT; p.tiles_y = (Ho + kHT - 1) / kHT;
    const long long tiles = (long long)p.tiles_x * p.tiles_y * N;
    if (tiles > 0x7fffffffLL) return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: too many tiles");
    p.total_tiles = (int)tiles;
    p.hcols = kHT + dil * (KS - 1); p.hrows = kHT + dil * (KS - 1);
    if (p.hcols > 256 || p.hrows > 256) return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: dilation too large for one TMA box");
    p.plane_bytes = p.hrows * p.hcols * 16;
    p.a_bytes = p.plane_bytes * (Cin / 4);
    p.w_bytes = p.Npad * Cin * 4;
    if ((unsigned)p.plane_bytes >= (1u << 18) || p.hcols * 16 >= (1 << 18))
        return pmb200_internal_fail(PMB200_EUNSUPPORTED, "conv2d_tc5h: halo tile exceeds the descriptor's 14-bit offsets");
    int dev = 0, sms = 0, smem_optin = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    p.a_stride = (p.a_bytes + 127) / 128 * 128;
    int plan[6];
    const int rc = pmb200_conv2d_tc5h_plan(Cin, Cout, KS, dil, p.total_tiles, sms, smem_optin, plan);
    if (rc != 0) return rc;
    p.sbufs = plan[0]; p.wstages = plan[1]; p.w_resident = plan[2]; p.psets = plan[5];
    const int smem = plan[3], ctas = plan[4];
    CUtensorMap xmap;
    const cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t strides[3] = {(cuuint64_t)Cin * 4, (cuuint64_t)W * Cin * 4, (cuuint64_t)H * W * Cin * 4};
    const cuuint32_t box[4] = {(cuuint32_t)Cin, (cuuint32_t)p.hcols, (cuuint32_t)p.hrows, 1u};
    const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
    if (enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float *>(x_nhwc), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return pmb200_internal_fail(PMB200_EINVAL, "conv2d_tc5h: tensor map rejected (alignment / size)");
    return by_npad<LaunchConv5h>(p.Npad, p, xmap, smem, ctas, dev, sms, smem_optin, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
