// pm_sample.cu -- surface sampling of triangle meshes on a regular barycentric lattice per face (beyond the reference;
// definition in include/patchmatch_b200.h, INTEGRATION.md "Surface sampling of meshes (beyond the reference)").
//
// Count pass: one thread per face computes its lattice size and sample count (int64) and flags the finite vertices it
// references; CUB exclusive scans turn both into output offsets, and the two totals are read back once.  Emit pass: one
// thread per referenced vertex copies it to its slot; the face samples are split into chunks of kChunk consecutive samples,
// each CTA finds its chunk's first and last face by binary search over the int64 offsets, and each thread finds its sample's
// face within that range, recovers n from the face's count and (i, j) from its index by exact integer row inversion
// (pm_sample_math.cuh).  So a face with millions of samples spreads over thousands of CTAs.  The only floating-point work is
// per thread, in a fixed order: no atomics touch a float, and reruns give the same bits.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cub/device/device_scan.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_sample_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmsample;

constexpr int kBlock = 256;
constexpr int kPerThread = 4;                       // face samples per thread and chunk
constexpr long long kChunk = (long long)kBlock * kPerThread;
constexpr long long kMaxItems = (1ll << 31) - 1;    // nv + 1 and nf + 1 stay CUB int item counts
constexpr int kMaxGrid = 65535;
constexpr unsigned long long kNoFace = ~0ull;

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct Carver {  // bump allocator over the caller's workspace; a NULL base only measures
    char *base;
    size_t used = 0;
    template <typename T>
    T *take(size_t count) {
        T *p = base ? reinterpret_cast<T *>(base + used) : nullptr;
        used += align256((count < 1 ? 1 : count) * sizeof(T));
        return p;
    }
};

// workspace: face offsets int64 [nf + 1], vertex flags uint8 [nv + 1], vertex offsets int64 [nv + 1], counters, CUB storage
struct Layout {
    long long *foff, *voff;
    unsigned char *vflag;
    unsigned long long *ctr;  // [0] first face with n >= 2^31 (kNoFace: none), [1] sum over faces of count >> 32
    void *cub;
    size_t cub_bytes;
};

bool layout(Carver &c, long long nv, long long nf, Layout &l) {
    l.foff = c.take<long long>(nf + 1);
    l.vflag = c.take<unsigned char>(nv + 1);
    l.voff = c.take<long long>(nv + 1);
    l.ctr = c.take<unsigned long long>(2);
    size_t a = 0, b = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, a, (long long *)nullptr, (long long *)nullptr, (int)(nf + 1)) != cudaSuccess) return false;
    if (cub::DeviceScan::ExclusiveScan(nullptr, b, (const unsigned char *)nullptr, (long long *)nullptr, cuda::std::plus<long long>(),
                                       0ll, (int)(nv + 1)) != cudaSuccess)
        return false;
    l.cub_bytes = a > b ? a : b;
    l.cub = c.take<char>(l.cub_bytes);
    return true;
}

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > kMaxGrid ? kMaxGrid : b));
}

#define GRID_LOOP(i, n) for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < (n); i += (long long)gridDim.x * kBlock)

__device__ __forceinline__ bool face_ok(const int *f, long long nv) {
    return f[0] >= 0 && f[0] < nv && f[1] >= 0 && f[1] < nv && f[2] >= 0 && f[2] < nv;
}

__global__ void __launch_bounds__(kBlock) count_kernel(const float *__restrict__ xyz, long long nv, const int *__restrict__ faces,
                                                       long long nf, double s, long long *__restrict__ foff,
                                                       unsigned char *__restrict__ vflag, unsigned long long *__restrict__ ctr) {
    GRID_LOOP(f, nf) {
        const int *fv = faces + 3 * f;
        long long cnt = 0;
        if (face_ok(fv, nv)) {
            const float *a = xyz + 3ll * fv[0], *b = xyz + 3ll * fv[1], *c = xyz + 3ll * fv[2];
            if (finite3(a)) vflag[fv[0]] = 1;  // plain stores of the same value: no atomic needed
            if (finite3(b)) vflag[fv[1]] = 1;
            if (finite3(c)) vflag[fv[2]] = 1;
            const long long n = lattice_size(a, b, c, s);
            if (n >= kMaxLattice) {
                atomicMin(ctr, (unsigned long long)f);
            } else {
                cnt = face_samples(n);
                if (cnt >> 32) atomicAdd(ctr + 1, (unsigned long long)(cnt >> 32));
            }
        }
        foff[f] = cnt;
    }
}

__global__ void __launch_bounds__(kBlock) vertex_kernel(const float *__restrict__ xyz, const unsigned char *__restrict__ rgb, long long nv,
                                                        const unsigned char *__restrict__ vflag, const long long *__restrict__ voff,
                                                        double *__restrict__ out, unsigned char *__restrict__ out_rgb) {
    GRID_LOOP(v, nv) {
        if (!vflag[v]) continue;
        const long long o = voff[v];
        for (int k = 0; k < 3; ++k) out[3 * o + k] = (double)xyz[3 * v + k];
        if (out_rgb)
            for (int k = 0; k < 3; ++k) out_rgb[3 * o + k] = rgb ? rgb[3 * v + k] : 0;
    }
}

// the face f in [lo, hi] with foff[f] <= o < foff[f + 1] (foff ascending, foff[lo] <= o)
__device__ __forceinline__ long long find_face(const long long *__restrict__ foff, long long lo, long long hi, long long o) {
    while (lo < hi) {
        const long long mid = lo + (hi - lo + 1) / 2;
        if (foff[mid] <= o) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kBlock) face_kernel(const float *__restrict__ xyz, const unsigned char *__restrict__ rgb,
                                                      const int *__restrict__ faces, long long nf, const long long *__restrict__ foff,
                                                      long long n_face_samples, long long base, double *__restrict__ out,
                                                      unsigned char *__restrict__ out_rgb) {
    __shared__ long long range[2];
    const long long chunks = (n_face_samples + kChunk - 1) / kChunk;
    for (long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        const long long s0 = ch * kChunk;
        const long long s1 = (s0 + kChunk < n_face_samples ? s0 + kChunk : n_face_samples) - 1;
        __syncthreads();  // range of the previous chunk is no longer read
        if (threadIdx.x < 2) range[threadIdx.x] = find_face(foff, 0, nf - 1, threadIdx.x ? s1 : s0);
        __syncthreads();
        const long long f0 = range[0], f1 = range[1];
        for (int r = 0; r < kPerThread; ++r) {
            const long long o = s0 + (long long)r * kBlock + threadIdx.x;
            if (o > s1) break;
            const long long f = find_face(foff, f0, f1, o);
            const long long k = o - foff[f];
            const long long n = lattice_of_count(foff[f + 1] - foff[f]);
            long long i, j;
            lattice_point(n, k, i, j);
            const int *fv = faces + 3 * f;
            const long long q = base + o;
            double p[3];
            unsigned char col[3];
            const unsigned char *ra = nullptr, *rb = nullptr, *rc = nullptr;
            if (out_rgb && rgb) ra = rgb + 3ll * fv[0], rb = rgb + 3ll * fv[1], rc = rgb + 3ll * fv[2];
            lattice_sample(xyz + 3ll * fv[0], xyz + 3ll * fv[1], xyz + 3ll * fv[2], ra, rb, rc, n, i, j, p, col);
            for (int c = 0; c < 3; ++c) out[3 * q + c] = p[c];
            if (out_rgb)
                for (int c = 0; c < 3; ++c) out_rgb[3 * q + c] = ra ? col[c] : 0;
        }
    }
}

int check_sizes(const char *what, int64_t nv, int64_t nf) {
    if (nv < 0 || nv >= kMaxItems || nf < 0 || nf >= kMaxItems) {
        char msg[160];
        snprintf(msg, sizeof msg, "%s: 0 <= n_vertices, n_faces < 2^31 - 1", what);
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    return 0;
}

}  // namespace

extern "C" int64_t pmb200_mesh_sample_workspace_bytes(int64_t n_vertices, int64_t n_faces) {
    if (const int rc = check_sizes("mesh_sample_workspace_bytes", n_vertices, n_faces)) return rc;
    Carver c{nullptr};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l))
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample_workspace_bytes: no CUDA device to size the CUB scans for");
    return (int64_t)c.used;
}

extern "C" int pmb200_mesh_sample_count(const float *xyz, int64_t n_vertices, const int *faces, int64_t n_faces, double spacing,
                                        int64_t *counts_host, void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || !counts_host || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample_count: null pointer");
    if (const int rc = check_sizes("mesh_sample_count", n_vertices, n_faces)) return rc;
    if (!(spacing > 0.0) || !isfinite(spacing))
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample_count: spacing must be finite and > 0");
    Carver c{static_cast<char *>(workspace)};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample_count: workspace smaller than mesh_sample_workspace_bytes(nv, nf)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaMemsetAsync(l.vflag, 0, n_vertices + 1, st);
    cudaMemsetAsync(l.foff + n_faces, 0, sizeof(long long), st);
    cudaMemsetAsync(l.ctr, 0xff, sizeof(unsigned long long), st);  // kNoFace
    cudaMemsetAsync(l.ctr + 1, 0, sizeof(unsigned long long), st);
    if (n_faces > 0)
        count_kernel<<<grid_blocks(n_faces), kBlock, 0, st>>>(xyz, n_vertices, faces, n_faces, spacing, l.foff, l.vflag, l.ctr);
    size_t bytes = l.cub_bytes;
    if (cub::DeviceScan::ExclusiveSum(l.cub, bytes, l.foff, l.foff, (int)(n_faces + 1), st) != cudaSuccess)
        return pmb200_internal_launch_status("mesh_sample_count (face scan)");
    bytes = l.cub_bytes;
    if (cub::DeviceScan::ExclusiveScan(l.cub, bytes, (const unsigned char *)l.vflag, l.voff, cuda::std::plus<long long>(), 0ll,
                                       (int)(n_vertices + 1), st) != cudaSuccess)
        return pmb200_internal_launch_status("mesh_sample_count (vertex scan)");
    long long host[2];
    unsigned long long hctr[2];
    if (cudaMemcpyAsync(host, l.voff + n_vertices, sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(host + 1, l.foff + n_faces, sizeof(long long), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(hctr, l.ctr, sizeof hctr, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status("mesh_sample_count");
    counts_host[0] = host[0];
    counts_host[1] = host[1];
    counts_host[2] = hctr[0] == kNoFace ? -1 : (int64_t)hctr[0];
    // sum(count) < (sum(count >> 32) + nf) 2^32: below 2^62 when the high parts sum below 2^29 (nf < 2^31 - 1)
    counts_host[3] = hctr[1] >= (1ull << 29) ? 1 : 0;
    return 0;
}

extern "C" int pmb200_mesh_sample(const float *xyz, const unsigned char *rgb, int64_t n_vertices, const int *faces, int64_t n_faces,
                                  int64_t n_vertex_samples, int64_t n_face_samples, double *xyz_out, unsigned char *rgb_out,
                                  void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_vertices > 0) || (!faces && n_faces > 0) || (!xyz_out && n_vertex_samples + n_face_samples > 0) || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample: null pointer");
    if (const int rc = check_sizes("mesh_sample", n_vertices, n_faces)) return rc;
    if (n_vertex_samples < 0 || n_vertex_samples > n_vertices || n_face_samples < 0 || (n_face_samples > 0 && n_faces == 0))
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample: sample counts are not those of mesh_sample_count");
    Carver c{static_cast<char *>(workspace)};
    Layout l;
    if (!layout(c, n_vertices, n_faces, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "mesh_sample: workspace smaller than mesh_sample_workspace_bytes(nv, nf)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (n_vertex_samples > 0)
        vertex_kernel<<<grid_blocks(n_vertices), kBlock, 0, st>>>(xyz, rgb, n_vertices, l.vflag, l.voff, xyz_out, rgb_out);
    if (n_face_samples > 0) {
        const long long chunks = (n_face_samples + kChunk - 1) / kChunk;
        const int grid = (int)(chunks > kMaxGrid ? kMaxGrid : chunks);
        face_kernel<<<grid, kBlock, 0, st>>>(xyz, rgb, faces, n_faces, l.foff, n_face_samples, n_vertex_samples, xyz_out, rgb_out);
    }
    return pmb200_internal_launch_status("mesh_sample");
}
