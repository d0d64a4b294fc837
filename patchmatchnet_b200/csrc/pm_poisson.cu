// pm_poisson.cu -- Poisson surface reconstruction of oriented points on a dense grid (beyond the reference; definition in
// include/patchmatch_b200.h, INTEGRATION.md "Poisson surface reconstruction (beyond the reference)").
//
//   setup     keep test per point, per axis a CUB radix sort of the coordinates for the box quantiles, grid placement on the
//             host, the node-box test and a stable compaction of the points that stay (two host synchronisations);
//   density   rho splatted with 64-bit fixed-point atomics (2^-32), then w_p = 1 / rho(p) per point;
//   rhs       b splatted the same way and rounded to float32 per node;
//   solve     V(2,2) multigrid cycles in float32: damped Jacobi smoothing (weight 1) and residuals as one memory-bound
//             27-point stencil kernel that marches along z and keeps three 3 x 3 planes in registers, full-weighting
//             restriction (P^T), trilinear prolongation, and the coarsest level (N = 2, one unknown) solved exactly by one
//             Jacobi sweep; level l uses the fine stencil times 2^l.  Residual norms and the iso-value are float64 sums over
//             a fixed grid of CTAs, reduced by one CTA in a fixed order.  One host read per cycle;
//   band      tsdf = chi - iso and weight 1 at the interior nodes of the blocks pmb200_tsdf_alloc allocated, 0 elsewhere;
//   colours   per vertex the nearest kept point: points sorted by grid cell, rings of cells searched outwards until the
//             best distance is certified by the ring's radius.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cub/block/block_reduce.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "../../include/patchmatch_b200.h"
#include "pm_poisson_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using namespace pmpoisson;

constexpr int kBlock = 256;
constexpr int kTX = 32, kTY = 8, kTZ = 16;  // stencil CTA: 32 x 8 columns, 16 planes each
constexpr int kRedBlocks = 1024;            // CTAs of the per-point float64 sums
constexpr int kSweeps = 2;                  // pre- and post-smoothing sweeps (even: chi ends in the level's x buffer)

__host__ __device__ inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

struct Carver {  // bump allocator over the caller's workspace; a NULL base only measures
    char *base;
    size_t used = 0;
    template <typename T>
    T *take(size_t count) {
        T *p = base ? reinterpret_cast<T *>(base + used) : nullptr;
        used += align256(count * sizeof(T));
        return p;
    }
};

inline int grid_for(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 * 4 ? 65535 * 4 : b));
}

inline long long nodes_of(int n) { return (long long)(n + 1) * (n + 1) * (n + 1); }

inline dim3 stencil_grid(int n) {
    const int m = n - 1;  // interior nodes per axis
    return dim3((m + kTX - 1) / kTX, (m + kTY - 1) / kTY, (m + kTZ - 1) / kTZ);
}

struct Level {
    int n;                 // N_l: nodes 0..n per axis, interior 1..n-1
    float *x, *t, *b;      // solution, scratch (smoother output / residual), right-hand side
};

struct Layout {
    // points
    unsigned char *flag;
    float *keys_in, *keys_out;
    int *idx, *perm_in, *perm_out;
    float *xyz, *nrm;
    unsigned char *rgb;
    double *w;
    unsigned long long *counts;  // [0] kept, [1] inside
    double *box;                 // lo[3], hi[3]
    double *partials;            // [2 * max partials]
    double *sums;                // [2]
    void *cub;
    size_t cub_bytes;
    // nodes
    unsigned long long *accum;   // level 0: the fixed-point sums, aliasing x and t of level 0
    Level levels[kMaxDepth];
    int n_levels;
    long long max_partials;
};

bool layout(Carver &c, int depth, long long n, Layout &l) {
    const long long m = n < 1 ? 1 : n;
    l.flag = c.take<unsigned char>(m);
    l.keys_in = c.take<float>(m);
    l.keys_out = c.take<float>(m);
    l.idx = c.take<int>(m);
    l.perm_in = c.take<int>(m);
    l.perm_out = c.take<int>(m);
    l.xyz = c.take<float>(3 * m);
    l.nrm = c.take<float>(3 * m);
    l.rgb = c.take<unsigned char>(3 * m);
    l.w = c.take<double>(m);
    l.counts = c.take<unsigned long long>(4);
    l.box = c.take<double>(6);
    const dim3 g = stencil_grid(1 << depth);
    l.max_partials = (long long)g.x * g.y * g.z;
    if (l.max_partials < kRedBlocks) l.max_partials = kRedBlocks;
    l.partials = c.take<double>(2 * l.max_partials);
    l.sums = c.take<double>(2);
    size_t a = 0, b = 0, d = 0;
    if (cub::DeviceRadixSort::SortKeys(nullptr, a, (float *)nullptr, (float *)nullptr, (int)m) != cudaSuccess) return false;
    if (cub::DeviceSelect::Flagged(nullptr, b, cub::CountingInputIterator<int>(0), (unsigned char *)nullptr, (int *)nullptr,
                                   (unsigned long long *)nullptr, (int)m) != cudaSuccess)
        return false;
    if (cub::DeviceRadixSort::SortPairs(nullptr, d, (unsigned *)nullptr, (unsigned *)nullptr, (int *)nullptr, (int *)nullptr, (int)m) !=
        cudaSuccess)
        return false;
    l.cub_bytes = a > b ? a : b;
    if (d > l.cub_bytes) l.cub_bytes = d;
    l.cub = c.take<char>(l.cub_bytes);
    l.n_levels = depth;  // N = 2^depth down to N = 2
    for (int k = 0; k < depth; ++k) {
        const int nl = (1 << depth) >> k;
        const long long M = nodes_of(nl);
        Level &L = l.levels[k];
        L.n = nl;
        if (k == 0) {
            l.accum = c.take<unsigned long long>(M);
            L.x = reinterpret_cast<float *>(l.accum);
            L.t = L.x ? L.x + M : nullptr;
        } else {
            L.x = c.take<float>(M);
            L.t = c.take<float>(M);
        }
        L.b = c.take<float>(M);
    }
    return true;
}

// ---- setup -----------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) keep_kernel(const float *xyz, const float *nrm, long long n, unsigned char *flag,
                                                      unsigned long long *counts) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock) {
        double nn[3];
        const bool k = keep_point(xyz + 3 * i, nrm + 3 * i, nn);
        flag[i] = k;
        if (k) atomicAdd(counts, 1ull);
    }
}

__global__ void __launch_bounds__(kBlock) axis_kernel(const float *xyz, const unsigned char *flag, long long n, int a, float *keys) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock)
        keys[i] = flag[i] ? xyz[3 * i + a] : INFINITY;
}

__global__ void quantile_kernel(const float *sorted, const unsigned long long *counts, double q, int a, double *box) {
    const long long m = (long long)counts[0];
    if (m < 1) return;
    for (int side = 0; side < 2; ++side) {
        const double qq = side ? sub64(1.0, q) : q;
        long long g = quantile_index(qq, m);
        if (g > m - 1) g = m - 1;
        const long long g1 = g + 1 < m ? g + 1 : m - 1;
        box[3 * side + a] = quantile(qq, m, (double)sorted[g], (double)sorted[g1]);
    }
}

struct GridArgs {
    int N;
    double h;
    long long I0[3];
};

GridArgs grid_args(const pmb200_poisson_grid &g) {
    GridArgs a;
    a.N = g.N;
    a.h = g.h;
    for (int k = 0; k < 3; ++k) a.I0[k] = g.I0[k];
    return a;
}

__global__ void __launch_bounds__(kBlock) inbox_kernel(const float *xyz, long long n, GridArgs g, unsigned char *flag) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock) {
        if (!flag[i]) continue;
        bool in = true;
        for (int a = 0; a < 3; ++a) {
            const double u = grid_coord(xyz[3 * i + a], g.h, g.I0[a]);
            in = in && u >= 0.0 && u <= (double)g.N;
        }
        flag[i] = in;
    }
}

__global__ void __launch_bounds__(kBlock) gather_kernel(const float *xyz, const float *nrm, const unsigned char *rgb, const int *idx,
                                                        long long m, float *xyz_out, float *nrm_out, unsigned char *rgb_out) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const long long s = idx[i];
        for (int a = 0; a < 3; ++a) {
            xyz_out[3 * i + a] = xyz[3 * s + a];
            nrm_out[3 * i + a] = nrm[3 * s + a];
            if (rgb) rgb_out[3 * i + a] = rgb[3 * s + a];
        }
    }
}

// ---- density, weights, right-hand side -------------------------------------------------------------------------------------

// the cell and fractions of point i; node index of corner k
struct PointCell {
    int base[3];
    double f[3];
};

__device__ inline PointCell point_cell(const float *xyz, long long i, const GridArgs &g) {
    PointCell pc;
    for (int a = 0; a < 3; ++a) {
        const double u = grid_coord(xyz[3 * i + a], g.h, g.I0[a]);
        pc.base[a] = cell_of(u, g.N);
        pc.f[a] = sub64(u, (double)pc.base[a]);
    }
    return pc;
}

__device__ inline size_t corner_node(const PointCell &pc, int k, int N) {
    const size_t s = (size_t)N + 1;
    return (size_t)(pc.base[0] + (k & 1)) + s * ((size_t)(pc.base[1] + ((k >> 1) & 1)) + s * (size_t)(pc.base[2] + (k >> 2)));
}

__device__ inline unsigned long long to_fixed(double v) { return (unsigned long long)llrint(mul64(v, kFixedScale)); }
__device__ inline double from_fixed(unsigned long long v) { return mul64((double)(long long)v, 1.0 / kFixedScale); }

__global__ void __launch_bounds__(kBlock) density_kernel(const float *xyz, long long m, GridArgs g, unsigned long long *accum) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const PointCell pc = point_cell(xyz, i, g);
        for (int k = 0; k < 8; ++k) atomicAdd(accum + corner_node(pc, k, g.N), to_fixed(corner_weight(pc.f, k)));
    }
}

__global__ void __launch_bounds__(kBlock) weight_kernel(const float *xyz, long long m, GridArgs g, const unsigned long long *accum,
                                                        double *w, double *w_out) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const PointCell pc = point_cell(xyz, i, g);
        double rho = 0.0;
        for (int k = 0; k < 8; ++k) rho = add64(rho, mul64(corner_weight(pc.f, k), from_fixed(accum[corner_node(pc, k, g.N)])));
        const double wi = div64(1.0, rho);
        w[i] = wi;
        if (w_out) w_out[i] = wi;
    }
}

__global__ void __launch_bounds__(kBlock) fixed_to_double_kernel(const unsigned long long *accum, long long M, double *out) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < M; i += (long long)gridDim.x * kBlock) out[i] = from_fixed(accum[i]);
}

__global__ void __launch_bounds__(kBlock) rhs_kernel(const float *xyz, const float *nrm, const double *w, long long m, GridArgs g,
                                                     unsigned long long *accum) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const PointCell pc = point_cell(xyz, i, g);
        double nn[3];
        keep_point(xyz + 3 * i, nrm + 3 * i, nn);
        for (int k = 0; k < 8; ++k) {
            double gr[3];
            corner_gradient(pc.f, k, gr);
            const double dot = add64(add64(mul64(nn[0], gr[0]), mul64(nn[1], gr[1])), mul64(nn[2], gr[2]));
            atomicAdd(accum + corner_node(pc, k, g.N), to_fixed(mul64(w[i], dot)));
        }
    }
}

// b per node as float32, 0 on the boundary
__global__ void __launch_bounds__(kBlock) rhs_round_kernel(const unsigned long long *accum, int N, float *b, float *b_out) {
    const long long s = N + 1, M = s * s * s;
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < M; i += (long long)gridDim.x * kBlock) {
        const long long x = i % s, y = (i / s) % s, z = i / (s * s);
        const bool interior = x > 0 && x < N && y > 0 && y < N && z > 0 && z < N;
        const float v = interior ? (float)from_fixed(accum[i]) : 0.0f;
        b[i] = v;
        if (b_out) b_out[i] = v;
    }
}

// ---- multigrid -------------------------------------------------------------------------------------------------------------

// fixed-order sum of one double per thread over a 2-D CTA (the y dimension must be declared: CUB indexes its storage by
// the linear thread id)
__device__ double block_sum_2d(double v) {
    using Reduce = cub::BlockReduce<double, kTX, cub::BLOCK_REDUCE_WARP_REDUCTIONS, kTY>;
    __shared__ typename Reduce::TempStorage tmp;
    return Reduce(tmp).Sum(v);
}

struct StencilArgs {
    int n;
    float scale;     // 2^level
    float omega;     // smoother weight over the diagonal 8/3 * 2^level
    const float *x;  // null: x = 0 (the first sweep of a coarse level)
    const float *b;
    float *out;
    double *partials;  // residual kernel only: per CTA the sum of r^2, or null
};

// A x at one node from the 3 x 3 neighbourhoods of the planes below (p0), at (p1) and above (p2), as sums of differences
// to the centre (the stencil's rows sum to zero): no cancellation where chi is flat, which is most of the grid.
__device__ inline float apply_stencil(const float *p0, const float *p1, const float *p2) {
    const float c = p1[4];
    const float edges = (((c - p1[0]) + (c - p1[2])) + ((c - p1[6]) + (c - p1[8]))) +
                        ((((c - p0[1]) + (c - p0[3])) + ((c - p0[5]) + (c - p0[7]))) +
                         (((c - p2[1]) + (c - p2[3])) + ((c - p2[5]) + (c - p2[7]))));
    const float corners = (((c - p0[0]) + (c - p0[2])) + ((c - p0[6]) + (c - p0[8]))) +
                          (((c - p2[0]) + (c - p2[2])) + ((c - p2[6]) + (c - p2[8])));
    return edges * (1.0f / 6.0f) + corners * (1.0f / 12.0f);
}

__device__ inline void load_plane(const float *x, size_t centre, size_t sy, float *p) {
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) p[3 * (dy + 1) + dx + 1] = __ldg(x + centre + dy * (long long)sy + dx);
}

// kResidual: out = b - s A x (and per CTA sum of squares); otherwise out = x + omega (b - s A x) / (s 8/3), a Jacobi sweep.
template <bool kResidual>
__global__ void __launch_bounds__(kTX * kTY) stencil_kernel(const StencilArgs a) {
    const int i = blockIdx.x * kTX + threadIdx.x + 1, j = blockIdx.y * kTY + threadIdx.y + 1;
    const int k0 = blockIdx.z * kTZ + 1, k1 = min(k0 + kTZ, a.n);
    const size_t sy = (size_t)a.n + 1, sz = sy * sy;
    double sq = 0.0;
    if (i < a.n && j < a.n) {
        float p0[9], p1[9], p2[9];
        const size_t col = (size_t)i + sy * j;
        if (a.x) {
            load_plane(a.x, col + (k0 - 1) * sz, sy, p0);
            load_plane(a.x, col + k0 * sz, sy, p1);
        }
        for (int k = k0; k < k1; ++k) {
            const size_t g = col + k * sz;
            float ax = 0.0f, xc = 0.0f;
            if (a.x) {
                load_plane(a.x, g + sz, sy, p2);
                ax = a.scale * apply_stencil(p0, p1, p2);
                xc = p1[4];
            }
            const float r = __ldg(a.b + g) - ax;
            if (kResidual) {
                a.out[g] = r;
                sq += (double)r * (double)r;
            } else {
                a.out[g] = xc + a.omega * r;
            }
            if (a.x) {
#pragma unroll
                for (int q = 0; q < 9; ++q) {
                    p0[q] = p1[q];
                    p1[q] = p2[q];
                }
            }
        }
    }
    if (kResidual && a.partials) {
        const double s = block_sum_2d(sq);
        if (threadIdx.x == 0 && threadIdx.y == 0) a.partials[blockIdx.x + gridDim.x * (blockIdx.y + gridDim.y * blockIdx.z)] = s;
    }
}

// b_c = P^T r_f over the coarse interior: weight 1, 1/2, 1/4, 1/8 by the number of non-zero offsets
__global__ void __launch_bounds__(kBlock) restrict_kernel(const float *r, int nf, float *bc, int nc) {
    const long long m = nc - 1, total = m * m * m;
    const size_t sf = (size_t)nf + 1, sc = (size_t)nc + 1;
    for (long long q = blockIdx.x * (long long)kBlock + threadIdx.x; q < total; q += (long long)gridDim.x * kBlock) {
        const int I = (int)(q % m) + 1, J = (int)((q / m) % m) + 1, K = (int)(q / (m * m)) + 1;
        float acc = 0.0f;
        for (int dz = -1; dz <= 1; ++dz)
            for (int dy = -1; dy <= 1; ++dy) {
                float row = 0.0f;
                const size_t base = (size_t)(2 * I) + sf * ((size_t)(2 * J + dy) + sf * (size_t)(2 * K + dz));
                row = 0.5f * __ldg(r + base - 1) + __ldg(r + base) + 0.5f * __ldg(r + base + 1);
                acc += row * ((dy ? 0.5f : 1.0f) * (dz ? 0.5f : 1.0f));
            }
        bc[(size_t)I + sc * ((size_t)J + sc * (size_t)K)] = acc;
    }
}

// x_f += P x_c over the fine interior (the coarse boundary holds 0)
__global__ void __launch_bounds__(kBlock) prolong_kernel(float *xf, int nf, const float *xc, int nc) {
    const long long m = nf - 1, total = m * m * m;
    const size_t sf = (size_t)nf + 1, sc = (size_t)nc + 1;
    for (long long q = blockIdx.x * (long long)kBlock + threadIdx.x; q < total; q += (long long)gridDim.x * kBlock) {
        const int i = (int)(q % m) + 1, j = (int)((q / m) % m) + 1, k = (int)(q / (m * m)) + 1;
        const int ci[3] = {i, j, k};
        int lo[3], hi[3];
        for (int a = 0; a < 3; ++a) {
            lo[a] = ci[a] >> 1;
            hi[a] = (ci[a] + 1) >> 1;
        }
        float acc = 0.0f;
        for (int c = 0; c < 8; ++c) {
            const int X = (c & 1) ? hi[0] : lo[0], Y = (c & 2) ? hi[1] : lo[1], Z = (c & 4) ? hi[2] : lo[2];
            // an even index has lo == hi: count that node once with weight 1
            if (((c & 1) && lo[0] == hi[0]) || ((c & 2) && lo[1] == hi[1]) || ((c & 4) && lo[2] == hi[2])) continue;
            const float wgt = ((lo[0] == hi[0]) ? 1.0f : 0.5f) * ((lo[1] == hi[1]) ? 1.0f : 0.5f) * ((lo[2] == hi[2]) ? 1.0f : 0.5f);
            acc += wgt * __ldg(xc + (size_t)X + sc * ((size_t)Y + sc * (size_t)Z));
        }
        xf[(size_t)i + sf * ((size_t)j + sf * (size_t)k)] += acc;
    }
}

// per CTA partial sums of two values over kRedBlocks CTAs -> one CTA reduces them in a fixed order
__global__ void __launch_bounds__(kBlock) final_sum_kernel(const double *partials, long long n, int pairs, double *out) {
    double a = 0.0, b = 0.0;
    for (long long i = threadIdx.x; i < n; i += kBlock) {
        a += partials[pairs * i];
        if (pairs == 2) b += partials[2 * i + 1];
    }
    using Reduce = cub::BlockReduce<double, kBlock>;
    __shared__ typename Reduce::TempStorage tmp;
    const double sa = Reduce(tmp).Sum(a);
    __syncthreads();
    const double sb = Reduce(tmp).Sum(b);
    if (threadIdx.x == 0) {
        out[0] = sa;
        out[1] = sb;
    }
}

// iso partials: per CTA sum of w_p chi(u_p) and of w_p
__global__ void __launch_bounds__(kBlock) iso_kernel(const float *xyz, const double *w, long long m, GridArgs g, const float *chi,
                                                     double *partials) {
    double a = 0.0, b = 0.0;
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const PointCell pc = point_cell(xyz, i, g);
        double c = 0.0;
        for (int k = 0; k < 8; ++k) c = add64(c, mul64(corner_weight(pc.f, k), (double)chi[corner_node(pc, k, g.N)]));
        a = add64(a, mul64(w[i], c));
        b = add64(b, w[i]);
    }
    using Reduce = cub::BlockReduce<double, kBlock>;
    __shared__ typename Reduce::TempStorage tmp;
    const double sa = Reduce(tmp).Sum(a);
    __syncthreads();
    const double sb = Reduce(tmp).Sum(b);
    if (threadIdx.x == 0) {
        partials[2 * blockIdx.x] = sa;
        partials[2 * blockIdx.x + 1] = sb;
    }
}

// ---- band field and colours ------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) band_kernel(const unsigned long long *keys, long long n_blocks, GridArgs g, const float *chi,
                                                      double iso, float *tsdf, float *weight) {
    const long long total = n_blocks * pmmesh::kBlockVoxels;
    const size_t s = (size_t)g.N + 1;
    for (long long q = blockIdx.x * (long long)kBlock + threadIdx.x; q < total; q += (long long)gridDim.x * kBlock) {
        int b[3];
        pmmesh::key_block(keys[q >> 9], b[0], b[1], b[2]);
        const int v = (int)(q & 511);
        const long long node[3] = {8ll * b[0] + (v & 7) - g.I0[0], 8ll * b[1] + ((v >> 3) & 7) - g.I0[1], 8ll * b[2] + (v >> 6) - g.I0[2]};
        bool interior = true;
        for (int a = 0; a < 3; ++a) interior = interior && node[a] >= 1 && node[a] <= g.N - 1;
        if (interior) {
            const double c = chi[(size_t)node[0] + s * ((size_t)node[1] + s * (size_t)node[2])];
            tsdf[q] = (float)sub64(c, iso);
            weight[q] = 1.0f;
        } else {
            tsdf[q] = 1.0f;
            weight[q] = 0.0f;
        }
    }
}

__global__ void __launch_bounds__(kBlock) cell_key_kernel(const float *xyz, long long m, GridArgs g, unsigned *keys, int *perm) {
    for (long long i = blockIdx.x * (long long)kBlock + threadIdx.x; i < m; i += (long long)gridDim.x * kBlock) {
        const PointCell pc = point_cell(xyz, i, g);
        keys[i] = (unsigned)pc.base[0] + (unsigned)g.N * ((unsigned)pc.base[1] + (unsigned)g.N * (unsigned)pc.base[2]);
        perm[i] = (int)i;
    }
}

__device__ inline long long lower_bound(const unsigned *keys, long long m, unsigned key) {
    long long lo = 0, hi = m;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ inline float get_f32(const unsigned char *p) {
    return __uint_as_float((unsigned)p[0] | ((unsigned)p[1] << 8) | ((unsigned)p[2] << 16) | ((unsigned)p[3] << 24));
}

__global__ void __launch_bounds__(kBlock) colour_kernel(unsigned char *verts, long long nv, const unsigned *keys, const int *perm,
                                                        long long m, const float *xyz, const unsigned char *rgb, GridArgs g) {
    for (long long q = blockIdx.x * (long long)kBlock + threadIdx.x; q < nv; q += (long long)gridDim.x * kBlock) {
        unsigned char *rec = verts + 15 * q;
        const float v[3] = {get_f32(rec), get_f32(rec + 4), get_f32(rec + 8)};
        int c[3];
        for (int a = 0; a < 3; ++a) c[a] = cell_of(grid_coord(v[a], g.h, g.I0[a]), g.N);
        double best = INFINITY;
        long long best_i = -1;
        for (int R = 0; R <= g.N; ++R) {
            for (int dz = -R; dz <= R; ++dz) {
                const int z = c[2] + dz;
                if (z < 0 || z >= g.N) continue;
                for (int dy = -R; dy <= R; ++dy) {
                    const int y = c[1] + dy;
                    if (y < 0 || y >= g.N) continue;
                    const bool face = dz == -R || dz == R || dy == -R || dy == R;
                    // a full row of the ring's face, or its two end cells
                    for (int part = 0; part < (face ? 1 : 2); ++part) {
                        int x0 = face ? c[0] - R : (part ? c[0] + R : c[0] - R), x1 = face ? c[0] + R : x0;
                        if (x0 < 0) x0 = 0;
                        if (x1 > g.N - 1) x1 = g.N - 1;
                        if (x0 > x1) continue;
                        const unsigned row = (unsigned)g.N * ((unsigned)y + (unsigned)g.N * (unsigned)z);
                        const long long e = lower_bound(keys, m, row + (unsigned)x1 + 1u);
                        for (long long s = lower_bound(keys, m, row + (unsigned)x0); s < e; ++s) {
                            const long long p = perm[s];
                            const double dx = sub64((double)xyz[3 * p], (double)v[0]), dy2 = sub64((double)xyz[3 * p + 1], (double)v[1]),
                                         dz2 = sub64((double)xyz[3 * p + 2], (double)v[2]);
                            const double d = add64(add64(mul64(dx, dx), mul64(dy2, dy2)), mul64(dz2, dz2));
                            if (d < best || (d == best && p < best_i)) {
                                best = d;
                                best_i = p;
                            }
                        }
                    }
                }
            }
            // every point not yet seen lies at least R cells away along some axis
            const double reach = mul64((double)R, g.h);
            if (best_i >= 0 && best < mul64(mul64(reach, reach), 1.0 - 1e-9)) break;
        }
        if (best_i >= 0) {
            rec[12] = rgb[3 * best_i];
            rec[13] = rgb[3 * best_i + 1];
            rec[14] = rgb[3 * best_i + 2];
        }
    }
}

int fail(const char *what, const char *msg) {
    static thread_local char buf[200];
    snprintf(buf, sizeof buf, "%s: %s", what, msg);
    return pmb200_internal_fail(PMB200_EINVAL, buf);
}

// the layout of a workspace for `grid`, or an error
int grid_layout(const char *what, const pmb200_poisson_grid *grid, void *workspace, int64_t workspace_bytes, Layout &l) {
    if (!grid || !workspace) return fail(what, "null pointer");
    if (grid->depth < kMinDepth || grid->depth > kMaxDepth || grid->N != (1 << grid->depth) || !(grid->h > 0.0) || !isfinite(grid->h) ||
        grid->n_inside < 1 || grid->n_inside > grid->n_points || grid->n_points >= kMaxPoints)
        return fail(what, "the grid is not one pmb200_poisson_setup returned for a cloud with points inside the node box");
    Carver c{static_cast<char *>(workspace)};
    if (!layout(c, grid->depth, grid->n_points, l) || workspace_bytes < (int64_t)c.used)
        return fail(what, "workspace smaller than poisson_workspace_bytes(depth, n_points)");
    return 0;
}

void run_stencil(bool residual, const Level &L, int level, const float *x, float omega, double *partials, cudaStream_t st) {
    StencilArgs a;
    a.n = L.n;
    a.scale = (float)(1 << level);
    a.omega = omega / (a.scale * (8.0f / 3.0f));
    a.x = x;
    a.b = L.b;
    a.out = L.t;
    a.partials = partials;
    const dim3 block(kTX, kTY);
    if (residual) stencil_kernel<true><<<stencil_grid(L.n), block, 0, st>>>(a);
    else stencil_kernel<false><<<stencil_grid(L.n), block, 0, st>>>(a);
}

// Jacobi sweeps at level k; `zero` when x is 0 (the first sweep needs no read of x)
void smooth(Level &L, int k, int sweeps, bool zero, cudaStream_t st) {
    for (int s = 0; s < sweeps; ++s) {
        run_stencil(false, L, k, (zero && s == 0) ? nullptr : L.x, 1.0f, nullptr, st);
        float *tmp = L.x;
        L.x = L.t;
        L.t = tmp;
    }
}

// ||b - A x||^2 of level 0 into l.sums[0] (residual written to the level's t)
void residual_norm(Layout &l, cudaStream_t st) {
    Level &L = l.levels[0];
    run_stencil(true, L, 0, L.x, 0.0f, l.partials, st);
    const dim3 g = stencil_grid(L.n);
    final_sum_kernel<<<1, kBlock, 0, st>>>(l.partials, (long long)g.x * g.y * g.z, 1, l.sums);
}

void v_cycle(Layout &l, cudaStream_t st) {
    const int top = l.n_levels - 1;
    for (int k = 0; k < top; ++k) {
        Level &L = l.levels[k];
        smooth(L, k, kSweeps, k > 0, st);
        run_stencil(true, L, k, L.x, 0.0f, nullptr, st);
        Level &C = l.levels[k + 1];
        const long long mc = (long long)(C.n - 1) * (C.n - 1) * (C.n - 1);
        restrict_kernel<<<grid_for(mc), kBlock, 0, st>>>(L.t, L.n, C.b, C.n);
    }
    smooth(l.levels[top], top, 1, true, st);  // N = 2: one unknown, exact in one sweep of weight 1
    for (int k = top - 1; k >= 0; --k) {
        Level &L = l.levels[k];
        const long long mf = (long long)(L.n - 1) * (L.n - 1) * (L.n - 1);
        prolong_kernel<<<grid_for(mf), kBlock, 0, st>>>(L.x, L.n, l.levels[k + 1].x, l.levels[k + 1].n);
        smooth(L, k, kSweeps, false, st);
    }
}

}  // namespace

extern "C" int64_t pmb200_poisson_workspace_bytes(int depth, int64_t n_points) {
    if (depth < kMinDepth || depth > kMaxDepth) return fail("poisson_workspace_bytes", "depth must be 5..10");
    if (n_points < 0 || n_points >= kMaxPoints) return fail("poisson_workspace_bytes", "0 <= n < 2^28");
    Carver c{nullptr};
    Layout l;
    if (!layout(c, depth, n_points, l)) return fail("poisson_workspace_bytes", "no CUDA device to size the CUB passes for");
    return (int64_t)c.used;
}

extern "C" int pmb200_poisson_setup(const float *xyz, const float *normals, const unsigned char *rgb, int64_t n_points, int depth,
                                    double scale, double bbox_quantile, pmb200_poisson_grid *grid_out, void *workspace,
                                    int64_t workspace_bytes, void *stream) {
    const char *what = "poisson_setup";
    if ((n_points > 0 && (!xyz || !normals)) || !grid_out || !workspace) return fail(what, "null pointer");
    if (n_points < 0 || n_points >= kMaxPoints) return fail(what, "0 <= n < 2^28");
    if (depth < kMinDepth || depth > kMaxDepth) return fail(what, "depth must be 5..10");
    if (!(scale >= 1.0) || !isfinite(scale)) return fail(what, "scale must be finite and >= 1");
    if (!(bbox_quantile >= 0.0) || !(bbox_quantile < 0.5)) return fail(what, "bbox_quantile must be in [0, 0.5)");
    Carver c{static_cast<char *>(workspace)};
    Layout l;
    if (!layout(c, depth, n_points, l) || workspace_bytes < (int64_t)c.used)
        return fail(what, "workspace smaller than poisson_workspace_bytes(depth, n_points)");
    pmb200_poisson_grid &g = *grid_out;
    g = pmb200_poisson_grid{};
    g.depth = depth;
    g.N = 1 << depth;
    g.n_points = n_points;
    g.has_rgb = rgb != nullptr;
    g.points_offset = (int64_t)(reinterpret_cast<char *>(l.xyz) - static_cast<char *>(workspace));
    if (n_points == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int n = (int)n_points;
    cudaMemsetAsync(l.counts, 0, 4 * sizeof(unsigned long long), st);
    cudaMemsetAsync(l.box, 0, 6 * sizeof(double), st);
    keep_kernel<<<grid_for(n), kBlock, 0, st>>>(xyz, normals, n, l.flag, l.counts);
    for (int a = 0; a < 3; ++a) {
        axis_kernel<<<grid_for(n), kBlock, 0, st>>>(xyz, l.flag, n, a, l.keys_in);
        size_t bytes = l.cub_bytes;
        if (cub::DeviceRadixSort::SortKeys(l.cub, bytes, l.keys_in, l.keys_out, n, 0, 32, st) != cudaSuccess)
            return pmb200_internal_launch_status("poisson_setup (sort)");
        quantile_kernel<<<1, 1, 0, st>>>(l.keys_out, l.counts, bbox_quantile, a, l.box);
    }
    unsigned long long kept = 0;
    if (cudaMemcpyAsync(&kept, l.counts, sizeof kept, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(g.lo, l.box, 3 * sizeof(double), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(g.hi, l.box + 3, 3 * sizeof(double), cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status(what);
    g.n_kept = (int64_t)kept;
    long long I0[3];
    if (kept == 0 || !place_grid(g.lo, g.hi, depth, scale, g.h, I0)) {
        g.h = 0.0;
        return pmb200_internal_launch_status(what);
    }
    for (int a = 0; a < 3; ++a) g.I0[a] = I0[a];
    inbox_kernel<<<grid_for(n), kBlock, 0, st>>>(xyz, n, grid_args(g), l.flag);
    size_t bytes = l.cub_bytes;
    if (cub::DeviceSelect::Flagged(l.cub, bytes, cub::CountingInputIterator<int>(0), l.flag, l.idx, l.counts + 1, n, st) != cudaSuccess)
        return pmb200_internal_launch_status("poisson_setup (select)");
    unsigned long long inside = 0;
    if (cudaMemcpyAsync(&inside, l.counts + 1, sizeof inside, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status(what);
    g.n_inside = (int64_t)inside;
    if (inside > 0) gather_kernel<<<grid_for((long long)inside), kBlock, 0, st>>>(xyz, normals, rgb, l.idx, (long long)inside, l.xyz, l.nrm, l.rgb);
    return pmb200_internal_launch_status(what);
}

extern "C" int pmb200_poisson_density(const pmb200_poisson_grid *grid, double *rho_out, double *w_out, void *workspace,
                                      int64_t workspace_bytes, void *stream) {
    Layout l;
    if (const int rc = grid_layout("poisson_density", grid, workspace, workspace_bytes, l)) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long m = grid->n_inside, M = nodes_of(grid->N);
    const GridArgs g = grid_args(*grid);
    cudaMemsetAsync(l.accum, 0, M * sizeof(unsigned long long), st);
    density_kernel<<<grid_for(m), kBlock, 0, st>>>(l.xyz, m, g, l.accum);
    weight_kernel<<<grid_for(m), kBlock, 0, st>>>(l.xyz, m, g, l.accum, l.w, w_out);
    if (rho_out) fixed_to_double_kernel<<<grid_for(M), kBlock, 0, st>>>(l.accum, M, rho_out);
    return pmb200_internal_launch_status("poisson_density");
}

extern "C" int pmb200_poisson_rhs(const pmb200_poisson_grid *grid, float *b_out, void *workspace, int64_t workspace_bytes, void *stream) {
    Layout l;
    if (const int rc = grid_layout("poisson_rhs", grid, workspace, workspace_bytes, l)) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long m = grid->n_inside, M = nodes_of(grid->N);
    const GridArgs g = grid_args(*grid);
    cudaMemsetAsync(l.accum, 0, M * sizeof(unsigned long long), st);
    rhs_kernel<<<grid_for(m), kBlock, 0, st>>>(l.xyz, l.nrm, l.w, m, g, l.accum);
    rhs_round_kernel<<<grid_for(M), kBlock, 0, st>>>(l.accum, grid->N, l.levels[0].b, b_out);
    cudaMemsetAsync(l.accum, 0, M * sizeof(unsigned long long), st);  // x and t of level 0
    for (int k = 1; k < l.n_levels; ++k) {
        const long long Mk = nodes_of(l.levels[k].n);
        cudaMemsetAsync(l.levels[k].x, 0, Mk * sizeof(float), st);
        cudaMemsetAsync(l.levels[k].t, 0, Mk * sizeof(float), st);
        cudaMemsetAsync(l.levels[k].b, 0, Mk * sizeof(float), st);
    }
    return pmb200_internal_launch_status("poisson_rhs");
}

extern "C" int pmb200_poisson_solve(const pmb200_poisson_grid *grid, double tol, int max_cycles, pmb200_poisson_result *result_out,
                                    float *chi_out, void *workspace, int64_t workspace_bytes, void *stream) {
    const char *what = "poisson_solve";
    Layout l;
    if (const int rc = grid_layout(what, grid, workspace, workspace_bytes, l)) return rc;
    if (!result_out) return fail(what, "null pointer");
    if (!(tol >= 0.0) || !isfinite(tol)) return fail(what, "tol must be finite and >= 0");
    if (max_cycles < 0) return fail(what, "max_cycles must be >= 0");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    pmb200_poisson_result &r = *result_out;
    r = pmb200_poisson_result{};
    double sums[2] = {0.0, 0.0};
    residual_norm(l, st);  // x = 0: ||b||^2
    if (cudaMemcpyAsync(sums, l.sums, sizeof sums, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return pmb200_internal_launch_status(what);
    const double bnorm = sqrt(sums[0]);
    r.residual = bnorm > 0.0 ? 1.0 : 0.0;
    while (r.residual > tol && r.cycles < max_cycles) {
        v_cycle(l, st);
        residual_norm(l, st);
        if (cudaMemcpyAsync(sums, l.sums, sizeof sums, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return pmb200_internal_launch_status(what);
        ++r.cycles;
        r.residual = sqrt(sums[0]) / bnorm;
    }
    r.converged = r.residual <= tol;
    const Level &L = l.levels[0];
    const long long m = grid->n_inside, M = nodes_of(grid->N);
    if (bnorm > 0.0) {
        iso_kernel<<<kRedBlocks, kBlock, 0, st>>>(l.xyz, l.w, m, grid_args(*grid), L.x, l.partials);
        final_sum_kernel<<<1, kBlock, 0, st>>>(l.partials, kRedBlocks, 2, l.sums);
        if (cudaMemcpyAsync(sums, l.sums, sizeof sums, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
            return pmb200_internal_launch_status(what);
        r.iso = sums[0] / sums[1];
    }
    if (chi_out) cudaMemcpyAsync(chi_out, L.x, M * sizeof(float), cudaMemcpyDeviceToDevice, st);
    return pmb200_internal_launch_status(what);
}

extern "C" int pmb200_poisson_band(const pmb200_poisson_grid *grid, double iso, const uint64_t *block_keys, int64_t n_blocks,
                                   float *tsdf_out, float *weight_out, void *workspace, int64_t workspace_bytes, void *stream) {
    const char *what = "poisson_band";
    Layout l;
    if (const int rc = grid_layout(what, grid, workspace, workspace_bytes, l)) return rc;
    if (!block_keys || !tsdf_out || !weight_out) return fail(what, "null pointer");
    if (n_blocks < 1 || n_blocks >= (1ll << 22)) return fail(what, "1 <= n_blocks < 2^22");
    if (!isfinite(iso)) return fail(what, "iso must be finite");
    band_kernel<<<grid_for(n_blocks * pmmesh::kBlockVoxels), kBlock, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const unsigned long long *>(block_keys), n_blocks, grid_args(*grid), l.levels[0].x, iso, tsdf_out, weight_out);
    return pmb200_internal_launch_status(what);
}

extern "C" int pmb200_poisson_colours(const pmb200_poisson_grid *grid, unsigned char *vertices, int64_t n_vertices, void *workspace,
                                      int64_t workspace_bytes, void *stream) {
    const char *what = "poisson_colours";
    Layout l;
    if (const int rc = grid_layout(what, grid, workspace, workspace_bytes, l)) return rc;
    if (!grid->has_rgb) return fail(what, "the cloud has no colours");
    if (n_vertices < 0 || n_vertices >= (1ll << 31)) return fail(what, "0 <= n_vertices < 2^31");
    if (n_vertices > 0 && !vertices) return fail(what, "null pointer");
    if (n_vertices == 0) return 0;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long m = grid->n_inside;
    const GridArgs g = grid_args(*grid);
    unsigned *keys_in = reinterpret_cast<unsigned *>(l.keys_in), *keys_out = reinterpret_cast<unsigned *>(l.keys_out);
    cell_key_kernel<<<grid_for(m), kBlock, 0, st>>>(l.xyz, m, g, keys_in, l.perm_in);
    size_t bytes = l.cub_bytes;
    if (cub::DeviceRadixSort::SortPairs(l.cub, bytes, keys_in, keys_out, l.perm_in, l.perm_out, (int)m, 0, 3 * grid->depth, st) != cudaSuccess)
        return pmb200_internal_launch_status("poisson_colours (sort)");
    colour_kernel<<<grid_for(n_vertices), kBlock, 0, st>>>(vertices, n_vertices, keys_out, l.perm_out, m, l.xyz, l.rgb, g);
    return pmb200_internal_launch_status(what);
}
