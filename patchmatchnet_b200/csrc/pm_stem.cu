// pm_stem.cu -- K-S: the two full-resolution layers of FeatureNet fused into one launch.
//
//   y = relu(conv1(relu(conv0(x))))     conv0: 3 -> 8, 3x3, pad 1;  conv1: 8 -> 8, 3x3, pad 1;  BatchNorm folded (eval mode)
//   (reference models/net.py:18-19 `self.conv0 = ConvBnReLU(3, 8)`, `self.conv1 = ConvBnReLU(8, 8)`, :44 `conv1 = self.conv1(self.conv0(x))`)
//
// Why its own kernel.  At 640x512 x 5 views these two layers were 141 us of a 0.9 ms step on the tensor-core conv family
// (K-D, 3xTF32): with 3 / 8 input and 8 output channels an m16n8k8 MMA is mostly padding and the 3x split triples it, and the
// 8-channel full-resolution map between them (52 MB) was written and read back through HBM.  The arithmetic is tiny --
// 216 + 576 multiply-adds per pixel -- so plain fp32 FFMA is both exact (no operand rounding at all) and faster:
//   * the 808 folded weights ride in the KERNEL PARAMETER BLOCK (3.3 KB of the 4 KB limit), i.e. the constant bank: every
//     FFMA takes its weight as a c[0x0][imm] operand -- no weight loads, no weight registers, thread-safe and graph-safe
//     (the values are baked into the launch), which is why the entry point takes the weights from HOST memory;
//   * one CTA = one 32 x 16 output tile: the planar NCHW image halo (36 x 20 x 3) is staged in shared memory, conv0 is
//     evaluated once on the 34 x 18 halo of the tile (1.2x recompute, zero outside the image: that IS conv1's padding) into
//     two float4 planes [ch 0-3 | ch 4-7][pixel] (consecutive lanes -> consecutive 16-byte slots: conflict-free LDS.128),
//     conv1 reads 9 taps x 2 LDS.128 per pixel and writes channels-last [N,H,W,8];
//   * the input is read as the caller's NCHW planes (coalesced along W): no NCHW -> NHWC conversion pass for the views.
// Bound: fp32 FFMA issue -- (576 + 1.2 * 216) FFMA per pixel x 1.64 M pixels / (132 SMs x 128 lanes x 1.98 GHz, H100 SXM)
// = 41 us at 100 % issue; HBM traffic 20 MB in + 52 MB out = 21 us at the data sheet's 3.35 TB/s.
#if !defined(PM_EMU)  // host emulation build (tests/warp_emu.h) brings its own CUDA vocabulary
#include <cuda_runtime.h>
#endif
#include <stdint.h>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);  // pm_kernels.cu: sets pmb200_last_error()
#if !defined(PM_EMU)
extern "C" int pmb200_internal_launch_status(const char *what);
extern "C" int pmb200_internal_tuning(const char *key);  // pm_kernels.cu: current value of a pmb200_set_tuning knob
#else
static int g_emu_stem_ppt = 2;
extern "C" void emu_conv_set_stem_ppt(int v) { g_emu_stem_ppt = v; }
#endif

namespace {

constexpr int kSTW = 32, kSTH = 16;                    // output tile
constexpr int kHW = kSTW + 2, kHH = kSTH + 2;          // conv0 outputs needed by the tile (conv1's halo)
constexpr int kIW = kSTW + 4, kIH = kSTH + 4;          // image pixels needed by those
// Output pixels per thread (PPT): 2 -> 256 threads per CTA, 4 -> 128.  Every weight reaches the FFMA through a uniform register
// loaded by LDCU.128 (4 weights per load); a thread's PPT pixels share the load, so PPT
// sets the LDCU : FFMA ratio of the conv1 phase (1 : 4 PPT).  pmb200_set_tuning("stem_ppt", 2 | 4) for A/B runs.

struct StemParams {
    const float *x;  // [N,CIN0,H,W]
    float *y;        // [N,H,W,8]
    const float *lo, *hi;  // NORM: per-image [N] range; the input is (x - lo) / (hi - lo) (Refinement's depth normalisation)
    int N, H, W, tiles_x, tiles_y;
    float w0[27 * 8];  // [(ci*9 + ky*3 + kx)][co]
    float b0[8];
    float w1[72 * 8];  // [((ky*3 + kx)*8 + ci)][co]
    float b1[8];
};
static_assert(sizeof(StemParams) <= 4096, "the weights must fit the kernel parameter block");

template <int CIN0, bool NORM, int PPT>
__global__ void __launch_bounds__(32 * (kSTH / PPT)) conv_stem_kernel(const __grid_constant__ StemParams p) {
    constexpr int kStemThreads = 32 * (kSTH / PPT), kWarps = kStemThreads / 32, kRowStep = kSTH / PPT;
    __shared__ float img[CIN0][kIH][kIW];
    __shared__ float4 mid[2][kHH * kHW];  // conv0 output: plane 0 = channels 0-3, plane 1 = channels 4-7
    const int tile = blockIdx.x;
    const int per_img = p.tiles_x * p.tiles_y;
    const int n = tile / per_img, tt = tile - n * per_img;
    const int ty = tt / p.tiles_x, tx = tt - ty * p.tiles_x;
    const int y0 = ty * kSTH, x0 = tx * kSTW;
    const int tid = threadIdx.x;

    // ---- image halo (rows y0-2 .., cols x0-2 ..), zero outside the image = conv0's padding.  One warp per halo row (3 planes x
    // 20 rows = 60 rows over 8 warps), lanes along the row (32 + 4 columns): no per-element index arithmetic, and the loads of a
    // warp's rows are all issued before the first store so their latencies overlap.
    const float *xin = p.x + (size_t)n * CIN0 * p.H * p.W;
    float nlo = 0.0f, nspan = 1.0f;
    if (NORM) {
        nlo = p.lo[n];
        nspan = p.hi[n] - nlo;
    }
    {
        const int warp = tid >> 5, lane = tid & 31;
        constexpr int kRowsPerWarp = (CIN0 * kIH + kWarps - 1) / kWarps;
        float v0[kRowsPerWarp], v1[kRowsPerWarp];
        const int gx0 = x0 - 2 + lane, gx1 = gx0 + 32;
        const bool in0 = gx0 >= 0 && gx0 < p.W, in1 = lane < kIW - 32 && gx1 < p.W;
#pragma unroll
        for (int k = 0; k < kRowsPerWarp; ++k) {
            const int row = warp + kWarps * k;  // plane * kIH + r
            const int ci = row / kIH, r = row - ci * kIH;
            const int gy = y0 - 2 + r;
            const bool rin = row < CIN0 * kIH && gy >= 0 && gy < p.H;
            const float *src = xin + ((size_t)ci * p.H + (rin ? gy : 0)) * p.W;
            v0[k] = (rin && in0) ? src[gx0] : 0.0f;
            v1[k] = (rin && in1) ? src[gx1] : 0.0f;
            if (NORM) {  // IEEE division like the reference's (depth - lo) / span; the zero padding stays zero
                v0[k] = (rin && in0) ? (v0[k] - nlo) / nspan : 0.0f;
                v1[k] = (rin && in1) ? (v1[k] - nlo) / nspan : 0.0f;
            }
        }
#pragma unroll
        for (int k = 0; k < kRowsPerWarp; ++k) {
            const int row = warp + kWarps * k;
            if (row < CIN0 * kIH) {
                const int ci = row / kIH, r = row - ci * kIH;
                img[ci][r][lane] = v0[k];
                if (lane < kIW - 32) img[ci][r][32 + lane] = v1[k];
            }
        }
    }
    __syncthreads();

    // ---- conv0 + ReLU on the 34 x 18 halo of the tile; outside the image the value is conv1's zero padding
    for (int pos = tid; pos < kHH * kHW; pos += kStemThreads) {
        const int r = pos / kHW, c = pos - r * kHW;
        const int gy = y0 - 1 + r, gx = x0 - 1 + c;
        float a[8];
#pragma unroll
        for (int co = 0; co < 8; ++co) a[co] = p.b0[co];
#pragma unroll
        for (int ci = 0; ci < CIN0; ++ci)
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float v = img[ci][r + ky][c + kx];
#pragma unroll
                    for (int co = 0; co < 8; ++co) a[co] = fmaf(v, p.w0[(ci * 9 + ky * 3 + kx) * 8 + co], a[co]);
                }
        const bool inside = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W;
#pragma unroll
        for (int co = 0; co < 8; ++co) a[co] = inside ? fmaxf(a[co], 0.0f) : 0.0f;
        mid[0][pos] = make_float4(a[0], a[1], a[2], a[3]);
        mid[1][pos] = make_float4(a[4], a[5], a[6], a[7]);
    }
    __syncthreads();

    // ---- conv1 + ReLU: PPT output pixels per thread (rows oy + kRowStep * q of the tile, same column)
    const int ox = tid & (kSTW - 1), oy = tid >> 5;  // 32 columns x kRowStep rows of threads
    float acc[PPT][8];
#pragma unroll
    for (int q = 0; q < PPT; ++q)
#pragma unroll
        for (int co = 0; co < 8; ++co) acc[q][co] = p.b1[co];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
#pragma unroll
            for (int q = 0; q < PPT; ++q) {
                const int pos = (oy + kRowStep * q + ky) * kHW + ox + kx;
                const float4 lo = mid[0][pos], hi = mid[1][pos];
                const float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int ci = 0; ci < 8; ++ci)
#pragma unroll
                    for (int co = 0; co < 8; ++co) acc[q][co] = fmaf(v[ci], p.w1[((ky * 3 + kx) * 8 + ci) * 8 + co], acc[q][co]);
            }
        }
#pragma unroll
    for (int q = 0; q < PPT; ++q) {
        const int gy = y0 + oy + kRowStep * q, gx = x0 + ox;
        if (gy < p.H && gx < p.W) {
            float4 *dst = reinterpret_cast<float4 *>(p.y + (((size_t)n * p.H + gy) * p.W + gx) * 8);
            dst[0] = make_float4(fmaxf(acc[q][0], 0.0f), fmaxf(acc[q][1], 0.0f), fmaxf(acc[q][2], 0.0f), fmaxf(acc[q][3], 0.0f));
            dst[1] = make_float4(fmaxf(acc[q][4], 0.0f), fmaxf(acc[q][5], 0.0f), fmaxf(acc[q][6], 0.0f), fmaxf(acc[q][7], 0.0f));
        }
    }
}

// fills the parameter block from PyTorch-layout host weights and launches
template <int CIN0, bool NORM>
int launch_stem(const char *what, const float *x, const float *lo, const float *hi, const float *host_w0, const float *host_b0,
                const float *host_w1, const float *host_b1, float *y_nhwc, int N, int H, int W, void *stream) {
    if (!x || !host_w0 || !host_b0 || !host_w1 || !host_b1 || !y_nhwc || (NORM && (!lo || !hi))) return pmb200_internal_fail(PMB200_EINVAL, "conv_stem / refine_low: null pointer");
    if (N < 1 || H < 1 || W < 1) return pmb200_internal_fail(PMB200_EINVAL, "conv_stem / refine_low: bad size");
    if (reinterpret_cast<uintptr_t>(y_nhwc) & 15u) return pmb200_internal_fail(PMB200_EINVAL, "conv_stem / refine_low: output must be 16-byte aligned");
    StemParams p;
    p.x = x; p.y = y_nhwc; p.lo = lo; p.hi = hi; p.N = N; p.H = H; p.W = W;
    p.tiles_x = (W + kSTW - 1) / kSTW; p.tiles_y = (H + kSTH - 1) / kSTH;
    const long long tiles = (long long)p.tiles_x * p.tiles_y * N;
    if (tiles > 0x7fffffffLL) return pmb200_internal_fail(PMB200_EINVAL, "conv_stem / refine_low: too many tiles");
    for (int i = 0; i < 27 * 8; ++i) p.w0[i] = 0.0f;
    for (int co = 0; co < 8; ++co) {
        p.b0[co] = host_b0[co];
        p.b1[co] = host_b1[co];
        for (int ci = 0; ci < CIN0; ++ci)
            for (int t = 0; t < 9; ++t) p.w0[(ci * 9 + t) * 8 + co] = host_w0[(co * CIN0 + ci) * 9 + t];
        for (int ci = 0; ci < 8; ++ci)
            for (int t = 0; t < 9; ++t) p.w1[(t * 8 + ci) * 8 + co] = host_w1[(co * 8 + ci) * 9 + t];
    }
#if defined(PM_EMU)
    (void)stream; (void)what;
    if (g_emu_stem_ppt == 2)
        emu::launch(dim3((unsigned)tiles), dim3(256), 0, [&] { conv_stem_kernel<CIN0, NORM, 2>(p); });
    else
        emu::launch(dim3((unsigned)tiles), dim3(128), 0, [&] { conv_stem_kernel<CIN0, NORM, 4>(p); });
    return 0;
#else
    if (pmb200_internal_tuning("stem_ppt") != 4)
        conv_stem_kernel<CIN0, NORM, 2><<<(unsigned)tiles, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    else
        conv_stem_kernel<CIN0, NORM, 4><<<(unsigned)tiles, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return pmb200_internal_launch_status(what);
#endif
}

}  // namespace

extern "C" {

// Fused conv0 -> conv1 of FeatureNet (3 -> 8 -> 8 channels, 3x3, pad 1, BatchNorm folded, ReLU after each).
//   x_nchw   device, [N,3,H,W] contiguous        y_nhwc   device, [N,H,W,8], 16-byte aligned
//   host_w0  HOST memory, [8][3][3][3] (PyTorch conv weight layout, BatchNorm folded), host_b0 [8]
//   host_w1  HOST memory, [8][8][3][3], host_b1 [8]
// The weights are copied into the kernel's parameter block (constant bank) at launch: later changes to the host arrays do not
// affect launches already enqueued or captured in a CUDA graph.
int pmb200_conv_stem(const float *x_nchw, const float *host_w0, const float *host_b0, const float *host_w1, const float *host_b1,
                     float *y_nhwc, int N, int H, int W, void *stream) {
    return launch_stem<3, false>("conv_stem", x_nchw, nullptr, nullptr, host_w0, host_b0, host_w1, host_b1, y_nhwc, N, H, W, stream);
}

// The half-resolution head of Refinement (reference models/net.py:104-110): d = (depth - depth_min) / (depth_max - depth_min),
// relu(conv2(relu(conv1(d)))) with conv1 1 -> 8, conv2 8 -> 8, 3x3, pad 1, BatchNorm folded -- the same kernel with one input
// plane and the normalisation applied as the plane is staged (zero padding applies to the NORMALISED map, as in the reference).
//   depth_half  device [N,1,h,w] contiguous;  depth_min / depth_max  device [N]
int pmb200_refine_low(const float *depth_half, const float *depth_min, const float *depth_max, const float *host_w1, const float *host_b1,
                      const float *host_w2, const float *host_b2, float *low_nhwc, int N, int h, int w, void *stream) {
    return launch_stem<1, true>("refine_low", depth_half, depth_min, depth_max, host_w1, host_b1, host_w2, host_b2, low_nhwc, N, h, w, stream);
}

}  // extern "C"
