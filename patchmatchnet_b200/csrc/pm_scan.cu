// pm_scan.cu -- the laser-beam visibility test and the per-voxel scores of the ETH3D evaluation (beyond the reference;
// INTEGRATION.md "ETH3D evaluation (beyond the reference)", contract in include/patchmatch_b200.h).  float64 throughout.
//
// Beam index of one scan, around its origin o: every scene-frame point p with a = p - o finite and non-zero, binned by the
// direction of a on an equirectangular grid (rows of elevation, columns of azimuth), and within a bin sorted by range r = |a|
// rounded up to float, farthest first.  A record is (a, r).  Per bin only the start of its run is stored.
//
// Query q, b = q - o, rho = |b|: if q lies in p's free beam then (exactly) theta < pi/2, sin(theta - delta) <= r0 cos(delta) / rho,
// with theta the angle between a and b and delta = atan(T), and rho cos(theta) < r.  So the candidates are the points within
// theta_c = min(delta + asin(r0 cos(delta) / rho), pi/2) + margin of b's direction (pi/2 + margin when r0 cos(delta) >= rho)
// whose range exceeds rho (cos(theta_c) - slack).  The cap's latitude / longitude box bounds the bins, a bin whose centre lies
// farther from b than theta_c plus the bin's own radius is skipped, and the bins are visited outward from b's own; a bin's run
// stops at the first record at or under the range bound.  The margins are orders of magnitude above the rounding of the float64 predicate and of
// the angles, so the culling is conservative; the predicate itself is evaluated on every candidate exactly as defined, with
// every operation rounded on its own (no fused multiply-add).
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kBlock = 256;
constexpr int kMaxRows = 1024;             // elevation rows of a beam index; columns of azimuth are twice as many
constexpr double kPointsPerBin = 32.0;     // target mean occupancy of a bin
constexpr double kAngleMargin = 1e-6;      // radians added to every angular bound of the culling
constexpr double kRangeSlack = 1e-9;       // subtracted from cos(theta_c) in the range bound
constexpr double kPi = 3.141592653589793;
constexpr long long kVoxelRange = 1ll << 20;  // voxel indices in [-2^20, 2^20): 21 bits per axis
constexpr unsigned long long kExcluded = 1ull << 63;  // score key of a point that counts for no voxel (above every voxel key)

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

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 ? 65535 : b));
}

inline int bit_width(long long v) {
    int b = 0;
    while (b < 63 && (v >> b) != 0) ++b;
    return b;
}

__device__ inline double dot3(double x0, double x1, double x2, double y0, double y1, double y2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(x0, y0), __dmul_rn(x1, y1)), __dmul_rn(x2, y2));
}

// ---- beam index -----------------------------------------------------------------------------------------------------------

struct BeamGrid {
    int rows, cols;
};

BeamGrid beam_grid(long long n) {
    long long rows = (long long)std::ceil(std::sqrt((double)n / (2.0 * kPointsPerBin)));
    rows = rows < 1 ? 1 : (rows > kMaxRows ? kMaxRows : rows);
    return BeamGrid{(int)rows, (int)(2 * rows)};
}

struct BeamLayout {
    double4 *rec;                  // [n] (a, r), sorted: the index proper, read by beam_observed
    int *starts;                   // [bins + 1]
    unsigned long long *keys_in, *keys_sorted;
    int *idx_in, *idx_sorted;
    void *cub_temp;
    size_t cub_bytes;
};

// The index lies at the start of the workspace, so beam_observed needs only n to find it.
long long beam_layout(Carver &c, long long n, const BeamGrid &g, BeamLayout &w) {
    const int m = (int)(n < 1 ? 1 : n);
    w.rec = c.take<double4>(n);
    w.starts = c.take<int>((size_t)g.rows * g.cols + 1);
    w.keys_in = c.take<unsigned long long>(n);
    w.keys_sorted = c.take<unsigned long long>(n);
    w.idx_in = c.take<int>(n);
    w.idx_sorted = c.take<int>(n);
    size_t bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int *)nullptr,
                                        (int *)nullptr, m, 0, 64) != cudaSuccess)
        return -1;
    w.cub_bytes = bytes;
    w.cub_temp = c.take<char>(bytes);
    return (long long)c.used;
}

__device__ inline double fclamp(double v, double lo, double hi) { return fmin(fmax(v, lo), hi); }

__device__ inline int bin_of(double a0, double a1, double a2, int rows, int cols) {
    const double el = atan2(a2, hypot(a0, a1)), az = atan2(a1, a0);
    const int r = (int)fclamp(floor((el + 0.5 * kPi) * (rows / kPi)), 0.0, rows - 1.0);
    const int c = (int)fclamp(floor((az + kPi) * (cols / (2.0 * kPi))), 0.0, cols - 1.0);
    return r * cols + c;
}

// a = p - o and r = sqrt(a . a), the same operations in the build and in the gather
__device__ inline double4 beam_record(const double *p, long long i, const double *o) {
    const double a0 = __dsub_rn(p[3 * i], o[0]), a1 = __dsub_rn(p[3 * i + 1], o[1]), a2 = __dsub_rn(p[3 * i + 2], o[2]);
    return make_double4(a0, a1, a2, __dsqrt_rn(dot3(a0, a1, a2, a0, a1, a2)));
}

struct Origin {
    double v[3];
};

__global__ void __launch_bounds__(kBlock) beam_keys_kernel(const double *p, int n, const Origin o, int rows, int cols,
                                                           unsigned long long *keys, int *idx) {
    const unsigned long long sentinel = (unsigned long long)rows * cols << 32;
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const double4 a = beam_record(p, i, o.v);
        unsigned long long k = sentinel;
        if (a.w > 0.0 && a.w < INFINITY) {  // a = 0 is never a beam; a non-finite point never passes the predicate
            const unsigned rbits = __float_as_uint(__double2float_ru(a.w));
            k = ((unsigned long long)bin_of(a.x, a.y, a.z, rows, cols) << 32) | (unsigned long long)(0xffffffffu - rbits);
        }
        keys[i] = k;
        idx[i] = i;
    }
}

__global__ void __launch_bounds__(kBlock) beam_gather_kernel(const double *p, int n, const Origin o, const int *idx, double4 *rec) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) rec[i] = beam_record(p, idx[i], o.v);
}

// starts[b] = the first sorted position whose bin is >= b, for b = 0 .. bins (the sentinel bin `bins` holds the excluded points)
__global__ void __launch_bounds__(kBlock) beam_starts_kernel(const unsigned long long *keys, int n, int bins, int *starts) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        const int b = (int)(keys[i] >> 32);
        const int prev = i == 0 ? -1 : (int)(keys[i - 1] >> 32);
        for (int k = prev + 1; k <= b; ++k) starts[k] = i;
        if (i == n - 1)
            for (int k = b + 1; k <= bins; ++k) starts[k] = n;
    }
}

// ---- beam query -----------------------------------------------------------------------------------------------------------

struct BeamParams {
    const double4 *rec;
    const int *starts;
    int rows, cols;
    double o[3];
    double r0, tan_delta, delta, r0_cos_delta;
    const double *q;
    int n_q;
    const unsigned char *mask;
    unsigned char *observed;
};

// q (b = q - o) in the free beam of the record (a, r): 0 < t' < a.a and |a x b|^2 <= (r0 r + t' T)^2
__device__ inline bool in_free_beam(const double4 a, double b0, double b1, double b2, double r0, double T) {
    const double t = dot3(a.x, a.y, a.z, b0, b1, b2);
    if (!(0.0 < t) || !(t < dot3(a.x, a.y, a.z, a.x, a.y, a.z))) return false;
    const double c0 = __dsub_rn(__dmul_rn(a.y, b2), __dmul_rn(a.z, b1));
    const double c1 = __dsub_rn(__dmul_rn(a.z, b0), __dmul_rn(a.x, b2));
    const double c2 = __dsub_rn(__dmul_rn(a.x, b1), __dmul_rn(a.y, b0));
    const double w = __dadd_rn(__dmul_rn(r0, a.w), __dmul_rn(t, T));
    return dot3(c0, c1, c2, c0, c1, c2) <= __dmul_rn(w, w);
}

// the candidate records of one bin, farthest first, until the range bound
__device__ inline bool scan_bin(const BeamParams &p, int bin, double b0, double b1, double b2, double r_bound) {
    const int e = __ldg(p.starts + bin + 1);
    for (int j = __ldg(p.starts + bin); j < e; ++j) {
        const double4 a = p.rec[j];
        if ((double)__double2float_ru(a.w) <= r_bound) return false;  // sorted by this key, descending
        if (in_free_beam(a, b0, b1, b2, p.r0, p.tan_delta)) return true;
    }
    return false;
}

// 0, +1, -1, +2, -2, ...: bins are visited outward from the query's own row and column, so a hit usually ends the search early
__device__ inline int outward(int j) { return (j & 1) ? (j + 1) >> 1 : -(j >> 1); }

__global__ void __launch_bounds__(kBlock) beam_observed_kernel(const BeamParams p) {
    const double row_h = kPi / p.rows, col_w = 2.0 * kPi / p.cols;
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < p.n_q; i += gridDim.x * kBlock) {
        if (p.observed[i] || (p.mask && !p.mask[i])) continue;
        const double b0 = __dsub_rn(p.q[3 * (size_t)i], p.o[0]), b1 = __dsub_rn(p.q[3 * (size_t)i + 1], p.o[1]),
                     b2 = __dsub_rn(p.q[3 * (size_t)i + 2], p.o[2]);
        const double rho = __dsqrt_rn(dot3(b0, b1, b2, b0, b1, b2));
        if (!(rho > 0.0 && rho < INFINITY)) continue;  // b = 0 gives t' = 0; a non-finite b never passes the predicate
        // t' > 0 needs theta < pi/2: the cap is at most a hemisphere (every direction of it when rho <= r0 cos(delta))
        const double s = p.r0_cos_delta / rho;
        const double theta = fmin(s < 1.0 ? p.delta + asin(s) : 0.5 * kPi, 0.5 * kPi) + kAngleMargin;
        const double r_bound = theta < 0.5 * kPi ? rho * (cos(theta) - kRangeSlack) : -1.0;
        const double el = atan2(b2, hypot(b0, b1)), az = atan2(b1, b0);
        const double u0 = b0 / rho, u1 = b1 / rho, u2 = b2 / rho;
        const int row_lo = (int)fclamp(floor((el - theta + 0.5 * kPi) / row_h), 0.0, p.rows - 1.0);
        const int row_hi = (int)fclamp(floor((el + theta + 0.5 * kPi) / row_h), 0.0, p.rows - 1.0);
        const int row_c = (int)fclamp(floor((el + 0.5 * kPi) / row_h), 0.0, p.rows - 1.0);
        const int col_c = (int)floor((az + kPi) / col_w);  // in [0, cols]: the seam wraps below
        int col_lo = col_c - p.cols / 2 + 1, col_hi = col_c + p.cols / 2;  // every column once
        if (fabs(el) + theta < 0.5 * kPi) {  // the cap holds no pole: its longitudes lie within asin(sin theta / cos el) of az
            const double half = asin(fmin(sin(theta) / cos(el), 1.0)) + kAngleMargin;
            const double lo = floor((az - half + kPi) / col_w), hi = floor((az + half + kPi) / col_w);
            if (hi - lo + 1.0 < p.cols) { col_lo = (int)lo; col_hi = (int)hi; }
        }
        const int n_rows = 2 * (row_hi - row_lo) + 1, n_cols = 2 * (col_hi - col_lo) + 1;
        bool hit = false;
        for (int jr = 0; jr < n_rows && !hit; ++jr) {
            const int r = row_c + outward(jr);
            if (r < row_lo || r > row_hi) continue;
            // a bin's directions lie within h of its centre: half its height plus half its width at its widest parallel
            const double el_c = (r + 0.5) * row_h - 0.5 * kPi;
            const double widest = fabs(el_c) <= 0.5 * row_h ? 1.0 : cos(fabs(el_c) - 0.5 * row_h);
            const double reach = theta + 0.5 * row_h + 0.5 * col_w * widest + kAngleMargin;
            const double cos_reach = reach < kPi ? cos(reach) : -2.0;
            double se, ce;
            sincos(el_c, &se, &ce);
            for (int jc = 0; jc < n_cols && !hit; ++jc) {
                const int c = col_c + outward(jc);
                if (c < col_lo || c > col_hi) continue;
                const int cc = c < 0 ? c + p.cols : (c >= p.cols ? c - p.cols : c);  // the azimuth seam
                double sa, ca;
                sincos((cc + 0.5) * col_w - kPi, &sa, &ca);
                if (__dadd_rn(__dadd_rn(u0 * ce * ca, u1 * ce * sa), u2 * se) < cos_reach) continue;  // bin outside the cap
                hit = scan_bin(p, r * p.cols + cc, b0, b1, b2, r_bound);
            }
        }
        if (hit) p.observed[i] = 1;
    }
}

// ---- per-voxel scores -----------------------------------------------------------------------------------------------------

struct ScoreLayout {
    unsigned long long *keys_in, *keys_sorted;
    int *bad_in, *bad_sorted, *heads, *vid, *bad_cum, *starts, *n_vox;
    long long *class_partials;  // [blocks][3]
    double *frac_partials;      // [blocks]
    void *cub_temp;
    size_t cub_bytes;
};

long long score_layout(Carver &c, long long n, ScoreLayout &w) {
    const int m = (int)(n < 1 ? 1 : n);
    const int blocks = grid_blocks(n);
    w.keys_in = c.take<unsigned long long>(n);
    w.keys_sorted = c.take<unsigned long long>(n);
    w.bad_in = c.take<int>(n);
    w.bad_sorted = c.take<int>(n);
    w.heads = c.take<int>(n);
    w.vid = c.take<int>(n);
    w.bad_cum = c.take<int>(n);
    w.starts = c.take<int>(n + 1);
    w.n_vox = c.take<int>(1);
    w.class_partials = c.take<long long>(3 * (size_t)blocks);
    w.frac_partials = c.take<double>(blocks);
    size_t a = 0, s = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, a, (unsigned long long *)nullptr, (unsigned long long *)nullptr, (int *)nullptr,
                                        (int *)nullptr, m, 0, 64) != cudaSuccess ||
        cub::DeviceScan::InclusiveSum(nullptr, s, (int *)nullptr, (int *)nullptr, m) != cudaSuccess)
        return -1;
    w.cub_bytes = a > s ? a : s;
    w.cub_temp = c.take<char>(w.cub_bytes);
    return (long long)c.used;
}

struct ScoreParams {
    const double *p, *d;
    const unsigned char *observed;
    int n;
    double tau;
};

__device__ inline unsigned long long voxel_field(double x, double tau) {
    const double f = fclamp(floor(__ddiv_rn(x, tau)), (double)-kVoxelRange, (double)(kVoxelRange - 1));  // the host checked the bounds
    return (unsigned long long)((long long)f + kVoxelRange);
}

// the block's fixed-tree sum of one value per thread (thread 0 gets the result)
template <typename T>
__device__ inline T block_sum(T v, T *s) {
    s[threadIdx.x] = v;
    __syncthreads();
    for (int o = kBlock / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] = s[threadIdx.x] + s[threadIdx.x + o];
        __syncthreads();
    }
    const T r = s[0];
    __syncthreads();
    return r;
}

// class of each point (accurate / covered = good, inaccurate / missed = bad, else excluded), its voxel key and bad flag
__global__ void __launch_bounds__(kBlock) score_keys_kernel(const ScoreParams sp, unsigned long long *keys, int *bad,
                                                            long long *class_partials) {
    __shared__ long long s[kBlock];
    long long n_good = 0, n_bad = 0, n_excluded = 0;
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < sp.n; i += gridDim.x * kBlock) {
        const bool good = sp.d[i] <= sp.tau;
        const bool is_bad = !good && (!sp.observed || sp.observed[i]);
        n_good += good; n_bad += is_bad; n_excluded += !good && !is_bad;
        keys[i] = !good && !is_bad ? kExcluded
                           : (voxel_field(sp.p[3 * (size_t)i], sp.tau) << 42) | (voxel_field(sp.p[3 * (size_t)i + 1], sp.tau) << 21) |
                                 voxel_field(sp.p[3 * (size_t)i + 2], sp.tau);
        bad[i] = is_bad ? 1 : 0;
    }
    n_good = block_sum(n_good, s);
    n_bad = block_sum(n_bad, s);
    n_excluded = block_sum(n_excluded, s);
    if (threadIdx.x == 0) {
        class_partials[3 * (size_t)blockIdx.x] = n_good;
        class_partials[3 * (size_t)blockIdx.x + 1] = n_bad;
        class_partials[3 * (size_t)blockIdx.x + 2] = n_excluded;
    }
}

__global__ void __launch_bounds__(kBlock) score_heads_kernel(const unsigned long long *keys, int n, int *heads) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock)
        heads[i] = keys[i] != kExcluded && (i == 0 || keys[i - 1] != keys[i]) ? 1 : 0;
}

// starts[v] = sorted position of voxel v's first point, starts[n_vox] = the number of counted points
__global__ void __launch_bounds__(kBlock) score_starts_kernel(const unsigned long long *keys, const int *heads, const int *vid, int n,
                                                              int *starts, int *n_vox) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n; i += gridDim.x * kBlock) {
        if (heads[i]) starts[vid[i] - 1] = i;
        if (keys[i] != kExcluded && (i == n - 1 || keys[i + 1] == kExcluded)) {
            starts[vid[i]] = i + 1;
            *n_vox = vid[i];
        }
    }
}

// per voxel good / (good + bad); each thread sums its voxels in order, then the block's fixed tree
__global__ void __launch_bounds__(kBlock) score_fraction_kernel(const int *starts, const int *bad_cum, const int *n_vox, double *partials) {
    __shared__ double s[kBlock];
    const int nv = *n_vox;
    double acc = 0.0;
    for (int v = blockIdx.x * kBlock + threadIdx.x; v < nv; v += gridDim.x * kBlock) {
        const int b = starts[v], e = starts[v + 1];
        const int bad = bad_cum[e - 1] - (b > 0 ? bad_cum[b - 1] : 0);
        acc = __dadd_rn(acc, __ddiv_rn((double)(e - b - bad), (double)(e - b)));
    }
    const double v = block_sum(acc, s);
    if (threadIdx.x == 0) partials[blockIdx.x] = v;
}

// one CTA: the partials summed by a fixed stride of blocks per thread, in order, then the fixed tree
__global__ void __launch_bounds__(kBlock) score_finish_kernel(const long long *class_partials, const double *frac_partials, int blocks,
                                                              const int *n_vox, long long *counts_out, double *sum_out) {
    __shared__ long long si[kBlock];
    __shared__ double sd[kBlock];
    for (int k = 0; k < 3; ++k) {
        long long v = 0;
        for (int b = threadIdx.x; b < blocks; b += kBlock) v += class_partials[3 * (size_t)b + k];
        v = block_sum(v, si);
        if (threadIdx.x == 0) counts_out[k] = v;
    }
    double f = 0.0;
    for (int b = threadIdx.x; b < blocks; b += kBlock) f = __dadd_rn(f, frac_partials[b]);
    f = block_sum(f, sd);
    if (threadIdx.x == 0) {
        counts_out[3] = *n_vox;
        *sum_out = f;
    }
}

bool finite_vec(const double *v, int k) {
    for (int a = 0; a < k; ++a)
        if (!(v[a] > -INFINITY && v[a] < INFINITY)) return false;
    return true;
}

}  // namespace

extern "C" int64_t pmb200_beam_index_workspace_bytes(int64_t n_scan) {
    if (n_scan < 0 || n_scan >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "beam_index_workspace_bytes: 0 <= n_scan < 2^31");
    Carver c{nullptr};
    BeamLayout w;
    const long long b = beam_layout(c, n_scan, beam_grid(n_scan), w);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "beam_index_workspace_bytes: no CUDA device to size the CUB sort for") : b;
}

extern "C" int pmb200_beam_index(const double *scan_points, int64_t n_scan, const double *origin_host, void *workspace,
                                 int64_t workspace_bytes, void *stream) {
    if ((!scan_points && n_scan > 0) || !origin_host || !workspace) return pmb200_internal_fail(PMB200_EINVAL, "beam_index: null pointer");
    if (n_scan < 0 || n_scan >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "beam_index: 0 <= n_scan < 2^31");
    if (!finite_vec(origin_host, 3)) return pmb200_internal_fail(PMB200_EINVAL, "beam_index: the origin must be finite");
    const BeamGrid g = beam_grid(n_scan);
    Carver c{static_cast<char *>(workspace)};
    BeamLayout w;
    const long long need = beam_layout(c, n_scan, g, w);
    if (need < 0 || workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "beam_index: workspace smaller than beam_index_workspace_bytes(n_scan)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int bins = g.rows * g.cols;
    if (n_scan == 0) {
        cudaMemsetAsync(w.starts, 0, (size_t)(bins + 1) * sizeof(int), st);
        return pmb200_internal_launch_status("beam_index");
    }
    const Origin o{{origin_host[0], origin_host[1], origin_host[2]}};
    const int n = (int)n_scan, blocks = grid_blocks(n);
    beam_keys_kernel<<<blocks, kBlock, 0, st>>>(scan_points, n, o, g.rows, g.cols, w.keys_in, w.idx_in);
    size_t bytes = w.cub_bytes;
    if (cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, w.keys_in, w.keys_sorted, w.idx_in, w.idx_sorted, n, 0,
                                        32 + bit_width(bins), st) != cudaSuccess)
        return pmb200_internal_launch_status("beam_index (sort)");
    beam_gather_kernel<<<blocks, kBlock, 0, st>>>(scan_points, n, o, w.idx_sorted, w.rec);
    beam_starts_kernel<<<blocks, kBlock, 0, st>>>(w.keys_sorted, n, bins, w.starts);
    return pmb200_internal_launch_status("beam_index");
}

extern "C" int pmb200_beam_observed(const double *queries, int64_t n_queries, const unsigned char *mask, const void *index_workspace,
                                    int64_t n_scan, const double *origin_host, double beam_start_radius, double tan_half_angle,
                                    unsigned char *observed, void *stream) {
    if ((!queries || !observed) && n_queries > 0) return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: null pointer");
    if (!index_workspace || !origin_host) return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: null pointer");
    if (n_queries < 0 || n_queries >= (1ll << 31) || n_scan < 0 || n_scan >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: 0 <= n_queries, n_scan < 2^31");
    if (!finite_vec(origin_host, 3)) return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: the origin must be finite");
    if (!(beam_start_radius >= 0.0) || !(beam_start_radius < INFINITY) || !(tan_half_angle >= 0.0) || !(tan_half_angle < INFINITY))
        return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: beam_start_radius and tan_half_angle must be finite and >= 0");
    if (n_queries == 0 || n_scan == 0) return 0;
    const BeamGrid g = beam_grid(n_scan);
    Carver c{const_cast<char *>(static_cast<const char *>(index_workspace))};
    BeamLayout w;
    if (beam_layout(c, n_scan, g, w) < 0) return pmb200_internal_fail(PMB200_EINVAL, "beam_observed: no CUDA device to size the CUB sort for");
    BeamParams p;
    p.rec = w.rec; p.starts = w.starts; p.rows = g.rows; p.cols = g.cols;
    for (int a = 0; a < 3; ++a) p.o[a] = origin_host[a];
    const double delta = std::atan(tan_half_angle);
    p.r0 = beam_start_radius; p.tan_delta = tan_half_angle; p.delta = delta; p.r0_cos_delta = beam_start_radius * std::cos(delta);
    p.q = queries; p.n_q = (int)n_queries; p.mask = mask; p.observed = observed;
    beam_observed_kernel<<<grid_blocks(n_queries), kBlock, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return pmb200_internal_launch_status("beam_observed");
}

extern "C" int64_t pmb200_voxel_score_workspace_bytes(int64_t n) {
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_score_workspace_bytes: 0 <= n < 2^31");
    Carver c{nullptr};
    ScoreLayout w;
    const long long b = score_layout(c, n, w);
    return b < 0 ? pmb200_internal_fail(PMB200_EINVAL, "voxel_score_workspace_bytes: no CUDA device to size the CUB calls for") : b;
}

extern "C" int pmb200_voxel_score(const double *points, const double *dist, int64_t n, double tau, const unsigned char *observed,
                                  const double *bounds_host, int64_t *counts_out, double *fraction_sum_out, void *workspace,
                                  int64_t workspace_bytes, void *stream) {
    if (((!points || !dist) && n > 0) || !bounds_host || !counts_out || !fraction_sum_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: null pointer");
    if (n < 0 || n >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: 0 <= n < 2^31");
    if (!(tau > 0.0) || !(tau < INFINITY)) return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: tau must be positive and finite");
    for (int a = 0; a < 3; ++a) {
        const double lo = bounds_host[a], hi = bounds_host[3 + a];
        if (!(lo <= hi) || !finite_vec(bounds_host + a, 1) || !finite_vec(bounds_host + 3 + a, 1))
            return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: bounds must be finite with min <= max");
        // floor(x / tau) is monotone in x: the bounds' indices bound every counted point's
        if (!(std::floor(lo / tau) >= (double)-kVoxelRange) || !(std::floor(hi / tau) < (double)kVoxelRange))
            return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: a voxel index floor(x / tau) lies outside [-2^20, 2^20)");
    }
    Carver c{static_cast<char *>(workspace)};
    ScoreLayout w;
    const long long need = score_layout(c, n, w);
    if (need < 0 || workspace_bytes < need)
        return pmb200_internal_fail(PMB200_EINVAL, "voxel_score: workspace smaller than voxel_score_workspace_bytes(n)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int m = (int)n, blocks = grid_blocks(n);
    cudaMemsetAsync(w.n_vox, 0, sizeof(int), st);
    const ScoreParams sp{points, dist, observed, m, tau};
    score_keys_kernel<<<blocks, kBlock, 0, st>>>(sp, w.keys_in, w.bad_in, w.class_partials);
    if (m > 0) {
        size_t bytes = w.cub_bytes;
        if (cub::DeviceRadixSort::SortPairs(w.cub_temp, bytes, w.keys_in, w.keys_sorted, w.bad_in, w.bad_sorted, m, 0, 64, st) != cudaSuccess)
            return pmb200_internal_launch_status("voxel_score (sort)");
        score_heads_kernel<<<blocks, kBlock, 0, st>>>(w.keys_sorted, m, w.heads);
        bytes = w.cub_bytes;
        if (cub::DeviceScan::InclusiveSum(w.cub_temp, bytes, w.heads, w.vid, m, st) != cudaSuccess)
            return pmb200_internal_launch_status("voxel_score (scan)");
        bytes = w.cub_bytes;
        if (cub::DeviceScan::InclusiveSum(w.cub_temp, bytes, w.bad_sorted, w.bad_cum, m, st) != cudaSuccess)
            return pmb200_internal_launch_status("voxel_score (scan)");
        score_starts_kernel<<<blocks, kBlock, 0, st>>>(w.keys_sorted, w.heads, w.vid, m, w.starts, w.n_vox);
    }
    score_fraction_kernel<<<blocks, kBlock, 0, st>>>(w.starts, w.bad_cum, w.n_vox, w.frac_partials);
    score_finish_kernel<<<1, kBlock, 0, st>>>(w.class_partials, w.frac_partials, blocks, w.n_vox,
                                              reinterpret_cast<long long *>(counts_out), fraction_sum_out);
    return pmb200_internal_launch_status("voxel_score");
}
