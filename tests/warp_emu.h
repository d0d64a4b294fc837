// warp_emu.h -- host-side lockstep emulator for the warp-level CUDA kernels of this repo.
//
// TEST INFRASTRUCTURE ONLY (never part of the product): it lets the CPU build box, which has no GPU, execute the *kernel
// source itself* -- shuffles, ballots, warp / block barriers, shared memory, the grid loop -- and compare the result with
// the oracle, so that a restructured kernel is functionally checked before any GPU time is spent on it.  The kernels'
// .cu file is compiled by g++ with -DPM_EMU (tests/emu_kernels.cpp includes it after this header); the few places where
// the device code uses inline PTX carry a plain-C++ alternative under `#if defined(PM_EMU)`.
//
// Execution model: one thread block at a time; every CUDA thread of the block is a fiber (ucontext) on ONE OS thread.
// A fiber runs until it reaches a collective (__shfl*_sync, __ballot_sync, __reduce_*_sync, __syncwarp, __syncthreads),
// posts its operand, and yields; it continues once every participating lane has arrived.  Values are double buffered by
// collective generation, so a fast lane can be at most one collective ahead.  Exited lanes count as arrived.
// What this checks: indexing, lane mappings, data flow through shuffles / shared memory, barrier placement (a missing
// __syncwarp shows up only as far as the fiber order exposes it), argument plumbing.  What it cannot check: timing,
// memory-model races, alignment faults of vector loads (the shims assert the alignment the PTX would need).
#pragma once

#include <assert.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <algorithm>
#include <functional>
#include <vector>

#include <vector_functions.h>
#include <vector_types.h>

#undef __global__
#undef __device__
#undef __host__
#undef __forceinline__
#undef __noinline__
#undef __grid_constant__
#undef __shared__
#undef __launch_bounds__
#undef __align__
#define __global__ static
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __grid_constant__
#define __shared__ static
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

namespace emu {

constexpr int kSlotWords = 4;  // 64-bit operand words a lane can post per collective (the MMA posts its A and B fragments at once)

struct Fiber {
    ucontext_t ctx;
    std::vector<char> stack;
    bool done = false;
    uint3 tid{0, 0, 0};
    int linear = 0;
    unsigned long long warp_gen = 0;   // collectives of my warp I have arrived at
    unsigned long long block_gen = 0;  // __syncthreads I have arrived at
};

struct Block {
    std::vector<Fiber> fibers;
    std::vector<uint64_t> slot[2];  // [generation parity][linear thread id * kSlotWords + word]
    dim3 block_dim{1, 1, 1}, grid_dim{1, 1, 1};
    uint3 block_idx{0, 0, 0};
    ucontext_t sched;
    const std::function<void()> *body = nullptr;
};

inline Block *&blk() {
    static Block *b = nullptr;
    return b;
}
inline Fiber *&cur() {
    static Fiber *f = nullptr;
    return f;
}
inline std::vector<char> &dyn_smem_storage() {
    static std::vector<char> s;
    return s;
}
inline void *dyn_smem() { return dyn_smem_storage().data(); }

inline void yield() {
    Fiber *f = cur();
    swapcontext(&f->ctx, &blk()->sched);
}

inline void fiber_main() {
    (*blk()->body)();
    cur()->done = true;
    yield();  // never resumed
}

// Run `body` once per CUDA thread of a grid x block launch (blocks sequentially, threads of a block in lockstep at collectives).
inline void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()> &body) {
    const int nthreads = (int)(block.x * block.y * block.z);
    assert(nthreads >= 1 && nthreads <= 1024);
    dyn_smem_storage().assign(smem_bytes + 64, 0);
    Block b;
    b.block_dim = block;
    b.grid_dim = grid;
    b.body = &body;
    b.fibers.resize((size_t)nthreads);
    b.slot[0].assign((size_t)nthreads * kSlotWords, 0);
    b.slot[1].assign((size_t)nthreads * kSlotWords, 0);
    for (auto &f : b.fibers) f.stack.resize(256 * 1024);
    blk() = &b;
    for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
            for (unsigned bx = 0; bx < grid.x; ++bx) {
                b.block_idx = uint3{bx, by, bz};
                int lin = 0;
                for (unsigned tz = 0; tz < block.z; ++tz)
                    for (unsigned ty = 0; ty < block.y; ++ty)
                        for (unsigned tx = 0; tx < block.x; ++tx, ++lin) {
                            Fiber &f = b.fibers[(size_t)lin];
                            f.done = false;
                            f.tid = uint3{tx, ty, tz};
                            f.linear = lin;
                            f.warp_gen = f.block_gen = 0;
                            getcontext(&f.ctx);
                            f.ctx.uc_stack.ss_sp = f.stack.data();
                            f.ctx.uc_stack.ss_size = f.stack.size();
                            f.ctx.uc_link = nullptr;
                            makecontext(&f.ctx, (void (*)())fiber_main, 0);
                        }
                for (;;) {
                    bool any = false;
                    for (auto &f : b.fibers) {
                        if (f.done) continue;
                        any = true;
                        cur() = &f;
                        swapcontext(&b.sched, &f.ctx);
                    }
                    if (!any) break;
                }
            }
    blk() = nullptr;
    cur() = nullptr;
}

inline int lane_id() { return cur()->linear & 31; }
inline int warp_base() { return cur()->linear & ~31; }

// Arrive at a warp collective with NW operand words; returns once every live lane named in `mask` has arrived.
// `out[w][l]` then holds word w of lane l (only meaningful for lanes in the mask that are alive).
template <int NW>
inline void warp_exchange_n(unsigned mask, const uint64_t (&v)[NW], uint64_t (&out)[NW][32]) {
    static_assert(NW >= 1 && NW <= kSlotWords, "too many operand words");
    Block *b = blk();
    Fiber *me = cur();
    const int base = warp_base();
    const int nthreads = (int)b->fibers.size();
    assert((mask >> lane_id()) & 1u);  // the calling lane must be named in the mask
    const unsigned long long g = ++me->warp_gen;
    for (int w = 0; w < NW; ++w) b->slot[g & 1][(size_t)me->linear * kSlotWords + w] = v[w];
    for (;;) {
        bool all = true;
        for (int l = 0; l < 32; ++l) {
            if (!((mask >> l) & 1u) || base + l >= nthreads) continue;
            const Fiber &o = b->fibers[(size_t)(base + l)];
            if (!o.done && o.warp_gen < g) { all = false; break; }
        }
        if (all) break;
        yield();
    }
    for (int w = 0; w < NW; ++w)
        for (int l = 0; l < 32; ++l) out[w][l] = (base + l < nthreads) ? b->slot[g & 1][(size_t)(base + l) * kSlotWords + w] : 0;
}

inline void warp_exchange(unsigned mask, uint64_t v, uint64_t (&out)[32]) {
    const uint64_t in[1] = {v};
    uint64_t all[1][32];
    warp_exchange_n<1>(mask, in, all);
    for (int l = 0; l < 32; ++l) out[l] = all[0][l];
}

inline void block_barrier() {
    Block *b = blk();
    Fiber *me = cur();
    const unsigned long long g = ++me->block_gen;
    for (;;) {
        bool all = true;
        for (const Fiber &o : b->fibers)
            if (!o.done && o.block_gen < g) { all = false; break; }
        if (all) break;
        yield();
    }
}

template <typename T>
inline uint64_t bits_of(T v) {
    static_assert(sizeof(T) <= 8, "operand too wide");
    uint64_t u = 0;
    memcpy(&u, &v, sizeof(T));
    return u;
}
template <typename T>
inline T from_bits(uint64_t u) {
    T v;
    memcpy(&v, &u, sizeof(T));
    return v;
}

}  // namespace emu

// ---- built-in variables -------------------------------------------------------------------------------------------
#define threadIdx (emu::cur()->tid)
#define blockIdx (emu::blk()->block_idx)
#define blockDim (emu::blk()->block_dim)
#define gridDim (emu::blk()->grid_dim)
#define warpSize 32

// ---- barriers and warp collectives ----------------------------------------------------------------------------------
inline void __syncthreads() { emu::block_barrier(); }
inline void __syncwarp(unsigned mask = 0xffffffffu) {
    uint64_t tmp[32];
    emu::warp_exchange(mask, 0, tmp);
}
template <typename T>
inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    const int lane = emu::lane_id(), seg = lane & ~(width - 1);
    return emu::from_bits<T>(all[seg + (src & (width - 1))]);
}
template <typename T>
inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    const int lane = emu::lane_id(), seg = lane & ~(width - 1);
    const int src = lane - (int)delta;
    return src >= seg ? emu::from_bits<T>(all[src]) : v;
}
template <typename T>
inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    const int lane = emu::lane_id(), seg = lane & ~(width - 1);
    const int src = lane + (int)delta;
    return src < seg + width ? emu::from_bits<T>(all[src]) : v;
}
template <typename T>
inline T __shfl_xor_sync(unsigned mask, T v, int lane_mask, int width = 32) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    const int lane = emu::lane_id(), seg = lane & ~(width - 1);
    const int src = lane ^ lane_mask;
    return (src >= seg && src < seg + width) ? emu::from_bits<T>(all[src]) : v;
}
inline unsigned __ballot_sync(unsigned mask, int pred) {
    uint64_t all[32];
    emu::warp_exchange(mask, pred ? 1u : 0u, all);
    const int base = emu::warp_base();
    unsigned r = 0;
    for (int l = 0; l < 32; ++l) {
        const bool alive = base + l < (int)emu::blk()->fibers.size() && !emu::blk()->fibers[(size_t)(base + l)].done;
        if (((mask >> l) & 1u) && alive && all[l]) r |= 1u << l;
    }
    return r;
}
inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, !pred) == 0; }
inline int __reduce_max_sync(unsigned mask, int v) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    int r = v;
    for (int l = 0; l < 32; ++l)
        if ((mask >> l) & 1u) r = std::max(r, emu::from_bits<int>(all[l]));
    return r;
}
inline int __reduce_add_sync(unsigned mask, int v) {
    uint64_t all[32];
    emu::warp_exchange(mask, emu::bits_of(v), all);
    int r = 0;
    for (int l = 0; l < 32; ++l)
        if ((mask >> l) & 1u) r += emu::from_bits<int>(all[l]);
    return r;
}

// ---- scalar intrinsics ----------------------------------------------------------------------------------------------
template <typename T>
inline T __ldg(const T *p) { return *p; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline void __nanosleep(unsigned) {}
inline int __float_as_int(float f) { return emu::from_bits<int>(emu::bits_of(f)); }
inline float __int_as_float(int i) { return emu::from_bits<float>(emu::bits_of(i)); }
inline float __fdividef(float a, float b) { return a / b; }
inline float __expf(float x) { return expf(x); }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline int atomicMax(int *p, int v) { const int o = *p; *p = std::max(o, v); return o; }
inline int atomicMin(int *p, int v) { const int o = *p; *p = std::min(o, v); return o; }
inline float atomicAdd(float *p, float v) { const float o = *p; *p = o + v; return o; }
inline int atomicAdd(int *p, int v) { const int o = *p; *p = o + v; return o; }
inline float4 atomicAdd(float4 *p, float4 v) {  // sm_90+ 128-bit vector atomic (needs a 16-byte aligned address)
    assert((reinterpret_cast<uintptr_t>(p) & 15u) == 0);
    const float4 o = *p;
    p->x += v.x; p->y += v.y; p->z += v.z; p->w += v.w;
    return o;
}
inline float2 atomicAdd(float2 *p, float2 v) {
    assert((reinterpret_cast<uintptr_t>(p) & 7u) == 0);
    const float2 o = *p;
    p->x += v.x; p->y += v.y;
    return o;
}
inline unsigned __float_as_uint(float f) { return emu::from_bits<unsigned>(emu::bits_of(f)); }
inline float __uint_as_float(unsigned u) { return emu::from_bits<float>(emu::bits_of(u)); }
inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
using std::max;
using std::min;

// ---- the slice of the CUDA runtime API the launch-planning host code touches (pm_conv.cu) ---------------------------
// (types and enumerators come from the toolkit's driver_types.h, which vector_types.h includes; only the calls are stubbed)
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline const char *cudaGetErrorString(cudaError_t) { return "emulated"; }
inline cudaError_t cudaGetDevice(int *dev) { *dev = 0; return cudaSuccess; }
// the launch planner sizes persistent grids from the SM count: 132 (H100) unless PM_EMU_SMS says otherwise -- a tiny "GPU"
// makes small test maps run the multi-tile, double-buffered paths
inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int) {
    const char *e = getenv("PM_EMU_SMS");
    *v = (e && atoi(e) > 0) ? atoi(e) : 132;
    return cudaSuccess;
}
template <typename F>
inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }

namespace emu {

// cvt.rna.tf32.f32: round to nearest, ties away from zero, keep 10 mantissa bits
inline uint32_t cvt_rna_tf32(float f) {
    uint32_t u = from_bits<uint32_t>(bits_of(f));
    if ((u & 0x7f800000u) == 0x7f800000u) return u;  // inf / nan pass through
    return (u + 0x1000u) & 0xffffe000u;
}

// mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 as a warp collective.  Fragments (PTX ISA): g = lane / 4, t = lane % 4;
// A 16x8: a0 (g, t)  a1 (g+8, t)  a2 (g, t+4)  a3 (g+8, t+4);  B 8x8: b0 (k = t, n = g)  b1 (k = t+4, n = g);
// C/D 16x8: c0 (g, 2t)  c1 (g, 2t+1)  c2 (g+8, 2t)  c3 (g+8, 2t+1).  Operands are read as TF32 (low 13 mantissa bits ignored).
inline void mma_m16n8k8_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    uint64_t x[3][32];
    const uint64_t mine[3] = {((uint64_t)a[1] << 32) | a[0], ((uint64_t)a[3] << 32) | a[2], ((uint64_t)b1 << 32) | b0};
    warp_exchange_n<3>(0xffffffffu, mine, x);
    auto tf = [](uint32_t u) { return from_bits<float>(bits_of((uint32_t)(u & 0xffffe000u))); };
    const int lane = lane_id(), g = lane >> 2, t = lane & 3;
    auto A = [&](int row, int k) {  // row 0..15, k 0..7
        const int src = (row & 7) * 4 + (k & 3);
        const uint64_t w = x[k >> 2][src];
        return tf((row >> 3) ? (uint32_t)(w >> 32) : (uint32_t)w);
    };
    auto B = [&](int k, int n) {
        const uint64_t w = x[2][n * 4 + (k & 3)];
        return tf((k >> 2) ? (uint32_t)(w >> 32) : (uint32_t)w);
    };
    for (int i = 0; i < 4; ++i) {
        const int row = g + ((i >> 1) ? 8 : 0), col = 2 * t + (i & 1);
        float acc = d[i];
        for (int k = 0; k < 8; ++k) acc = fmaf(A(row, k), B(k, col), acc);
        d[i] = acc;
    }
}

}  // namespace emu
