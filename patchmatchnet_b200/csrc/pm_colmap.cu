// pm_colmap.cu -- view selection scores and depth ranges of a COLMAP sparse model (reference colmap_input.py:318-373;
// semantics restated in INTEGRATION.md "COLMAP interop").
//
// The model is held as: points xyz [P,3] float64; per-image observations in CSR form, obs_offsets [N+1] and obs_points [M]
// (int32 dense point indices in each image's own 2D-point order, no -1 entries); camera centres [N,3] and extrinsics [N,4,4],
// float64, composed on the host.
//
// View scores (work O(M log M + T log T), T = the number of (observation, co-observing image) contributions):
//   1. sort the observations by point (stable radix sort of the point index, carrying the global observation index g), so
//      each point's run lists its observations in (image, position) order;
//   2. per sorted observation a in image i: the number of distinct images j > i later in its run; exclusive scan -> offsets;
//      the caller reads the total once to size the second phase;
//   3. emit (key = pair(i,j) << bits(M) | position of a in obs_i, g(theta)) for every such j;
//   4. radix sort the keys; each pair's run is then in obs_i order and is summed by one thread from 0.0, left to right --
//      the order of the reference's loop, so no floating-point atomics and bit-identical results from run to run.
// Every float64 operation is written out (__dmul_rn / __dadd_rn ...): no fused multiply-add, numpy's evaluation order.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kBlock = 256;
constexpr long long kMaxImages = 65536;
constexpr long long kMaxItems = 1ll << 31;  // CUB item counts are int

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

inline int bits_for(long long n) {  // bits to hold 0 .. n-1 (at least 1)
    int b = 1;
    while (b < 62 && (1ll << b) < n) ++b;
    return b;
}

inline int grid_blocks(long long n) {
    const long long b = (n + kBlock - 1) / kBlock;
    return (int)(b < 1 ? 1 : (b > 65535 ? 65535 : b));
}

// image of global observation g: the last i with offsets[i] <= g
__device__ inline int image_of(const int *offsets, int n_images, int g) {
    int lo = 0, hi = n_images;  // offsets[lo] <= g < offsets[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(offsets + mid) <= g) lo = mid; else hi = mid;
    }
    return lo;
}

// ---- view scores ----------------------------------------------------------------------------------------------------------

struct ScoreLayout {
    // phase 1 (sizes depend on N and M only, so the same prefix whatever T is)
    unsigned *pt_in, *pt_sorted;
    int *g_in, *g_sorted, *img_sorted;
    long long *count, *offs;  // offs [M+1]
    void *cub1;
    size_t cub1_bytes;
    // phase 2
    unsigned long long *key_in, *key_sorted;
    double *val_in, *val_sorted;
    void *cub2;
    size_t cub2_bytes;
};

bool score_layout(Carver &c, long long n_obs, long long n_contrib, int pt_bits, int key_bits, ScoreLayout &l) {
    const long long m = n_obs < 1 ? 1 : n_obs;
    l.pt_in = c.take<unsigned>(m); l.pt_sorted = c.take<unsigned>(m);
    l.g_in = c.take<int>(m); l.g_sorted = c.take<int>(m); l.img_sorted = c.take<int>(m);
    l.count = c.take<long long>(m); l.offs = c.take<long long>(m + 1);
    size_t a = 0, b = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, a, (unsigned *)nullptr, (unsigned *)nullptr, (int *)nullptr, (int *)nullptr, (int)m, 0,
                                        pt_bits) != cudaSuccess)
        return false;
    if (cub::DeviceScan::InclusiveSum(nullptr, b, (long long *)nullptr, (long long *)nullptr, (int)m) != cudaSuccess) return false;
    l.cub1_bytes = a > b ? a : b;
    l.cub1 = c.take<char>(l.cub1_bytes);
    const long long t = n_contrib < 1 ? 1 : n_contrib;
    l.key_in = c.take<unsigned long long>(n_contrib > 0 ? t : 0); l.key_sorted = c.take<unsigned long long>(n_contrib > 0 ? t : 0);
    l.val_in = c.take<double>(n_contrib > 0 ? t : 0); l.val_sorted = c.take<double>(n_contrib > 0 ? t : 0);
    l.cub2_bytes = 0;
    if (n_contrib > 0 && cub::DeviceRadixSort::SortPairs(nullptr, l.cub2_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                                         (double *)nullptr, (double *)nullptr, (int)t, 0, key_bits) != cudaSuccess)
        return false;
    l.cub2 = c.take<char>(l.cub2_bytes);
    return true;
}

__global__ void __launch_bounds__(kBlock) obs_keys_kernel(const int *obs_points, int m, unsigned *pt, int *g) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < m; i += gridDim.x * kBlock) {
        pt[i] = (unsigned)obs_points[i];
        g[i] = i;
    }
}

// per sorted observation: its image, and the number of distinct images after its own one in the point's run
__global__ void __launch_bounds__(kBlock) obs_count_kernel(const unsigned *pt, const int *g, const int *offsets, int n_images, int m,
                                                           int *img, long long *count) {
    for (int k = blockIdx.x * kBlock + threadIdx.x; k < m; k += gridDim.x * kBlock) {
        const unsigned p = pt[k];
        const int i = image_of(offsets, n_images, g[k]);
        img[k] = i;
        long long n = 0;
        int last = i;
        for (int q = k + 1; q < m && pt[q] == p; ++q) {
            const int j = image_of(offsets, n_images, g[q]);
            if (j != last) { ++n; last = j; }
        }
        count[k] = n;
    }
}

struct EmitParams {
    const unsigned *pt;
    const int *g, *img;
    const long long *offs;
    const int *offsets;
    const double *xyz, *centers;
    int n_images, m, pos_bits;
    double theta0, sigma1, sigma2;
    unsigned long long *key;
    double *val;
};

// the reference's per-point term for cameras c_i, c_j and point x, written out in numpy's order:
//   theta = (180 / pi) * arccos(dot(ci - x, cj - x) / |ci - x| / |cj - x|),  g = exp(-(theta - t0)^2 / (2 sigma^2))
// with the cosine clamped to [-1, 1] and 0 for a point on either centre (the reference gets NaN in both cases)
__device__ inline double view_term(const double *ci, const double *cj, const double *x, double t0, double s1, double s2) {
    const double ax = __dsub_rn(ci[0], x[0]), ay = __dsub_rn(ci[1], x[1]), az = __dsub_rn(ci[2], x[2]);
    const double bx = __dsub_rn(cj[0], x[0]), by = __dsub_rn(cj[1], x[1]), bz = __dsub_rn(cj[2], x[2]);
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by)), __dmul_rn(az, bz));
    const double na = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay)), __dmul_rn(az, az)));
    const double nb = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(bx, bx), __dmul_rn(by, by)), __dmul_rn(bz, bz)));
    if (na == 0.0 || nb == 0.0) return 0.0;
    const double c = fmin(fmax(__ddiv_rn(__ddiv_rn(dot, na), nb), -1.0), 1.0);
    const double theta = __dmul_rn(180.0 / 3.141592653589793, acos(c));
    const double d = __dsub_rn(theta, t0);
    const double s = theta <= t0 ? s1 : s2;
    return exp(__ddiv_rn(__dmul_rn(-d, d), __dmul_rn(2.0, __dmul_rn(s, s))));
}

__global__ void __launch_bounds__(kBlock) obs_emit_kernel(const EmitParams p) {
    for (int k = blockIdx.x * kBlock + threadIdx.x; k < p.m; k += gridDim.x * kBlock) {
        long long o = p.offs[k];
        if (o == p.offs[k + 1]) continue;
        const unsigned pt = p.pt[k];
        const int i = p.img[k];
        const unsigned long long pos = (unsigned long long)(p.g[k] - __ldg(p.offsets + i));
        double x[3] = {p.xyz[3 * (size_t)pt], p.xyz[3 * (size_t)pt + 1], p.xyz[3 * (size_t)pt + 2]};
        const double ci[3] = {p.centers[3 * i], p.centers[3 * i + 1], p.centers[3 * i + 2]};
        int last = i;
        for (int q = k + 1; q < p.m && p.pt[q] == pt; ++q) {
            const int j = p.img[q];
            if (j == last) continue;
            last = j;
            const double cj[3] = {p.centers[3 * j], p.centers[3 * j + 1], p.centers[3 * j + 2]};
            const unsigned long long pair = (unsigned long long)i * (unsigned long long)p.n_images + (unsigned long long)j;
            p.key[o] = (pair << p.pos_bits) | pos;
            p.val[o] = view_term(ci, cj, x, p.theta0, p.sigma1, p.sigma2);
            ++o;
        }
    }
}

// one thread per pair run: the sum in key (= obs_i) order, from 0.0
__global__ void __launch_bounds__(kBlock) pair_sum_kernel(const unsigned long long *key, const double *val, int t, int pos_bits,
                                                          int n_images, double *score) {
    for (int k = blockIdx.x * kBlock + threadIdx.x; k < t; k += gridDim.x * kBlock) {
        const unsigned long long pair = key[k] >> pos_bits;
        if (k > 0 && (key[k - 1] >> pos_bits) == pair) continue;
        double s = 0.0;
        for (int q = k; q < t && (key[q] >> pos_bits) == pair; ++q) s = __dadd_rn(s, val[q]);
        const long long i = (long long)(pair / (unsigned long long)n_images), j = (long long)(pair % (unsigned long long)n_images);
        score[i * n_images + j] = s;
        score[j * n_images + i] = s;
    }
}

int check_model(int n_images, long long n_obs, long long n_points) {
    if (n_images < 1 || n_images >= kMaxImages) return 1;
    if (n_obs < 0 || n_obs >= kMaxItems) return 2;
    if (n_points < 0 || n_points >= kMaxItems) return 3;
    return 0;
}

const char *model_message(int which) {
    switch (which) {
        case 1: return "1 <= n_images < 65536";
        case 2: return "0 <= n_obs < 2^31";
        default: return "0 <= n_points < 2^31";
    }
}

// ---- depth ranges --------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kBlock) obs_depth_kernel(const int *obs_points, const int *offsets, int n_images, int m,
                                                           const double *xyz, const double *extrinsics, double *z) {
    for (int g = blockIdx.x * kBlock + threadIdx.x; g < m; g += gridDim.x * kBlock) {
        const int i = image_of(offsets, n_images, g);
        const size_t p = (size_t)obs_points[g];
        const double *e = extrinsics + 16 * (size_t)i + 8;  // row 2
        z[g] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], xyz[3 * p]), __dmul_rn(e[1], xyz[3 * p + 1])), __dmul_rn(e[2], xyz[3 * p + 2])), e[3]);
    }
}

// zs_sorted[int(n * 0.01)] and zs_sorted[int(n * 0.99)] per image (NaN for an image without observations)
__global__ void __launch_bounds__(kBlock) depth_pick_kernel(const double *zs, const int *offsets, int n_images, double *ranges) {
    for (int i = blockIdx.x * kBlock + threadIdx.x; i < n_images; i += gridDim.x * kBlock) {
        const int a = offsets[i], n = offsets[i + 1] - a;
        if (n <= 0) {
            ranges[2 * i] = ranges[2 * i + 1] = __longlong_as_double(0x7ff8000000000000ll);
            continue;
        }
        ranges[2 * i] = zs[a + (long long)__dmul_rn((double)n, 0.01)];
        ranges[2 * i + 1] = zs[a + (long long)__dmul_rn((double)n, 0.99)];
    }
}

bool range_layout(Carver &c, int n_images, long long n_obs, double *&z_in, double *&z_sorted, void *&temp, size_t &temp_bytes) {
    const long long m = n_obs < 1 ? 1 : n_obs;
    z_in = c.take<double>(m);
    z_sorted = c.take<double>(m);
    temp_bytes = 0;
    if (cub::DeviceSegmentedSort::SortKeys(nullptr, temp_bytes, (const double *)nullptr, (double *)nullptr, (int)m, n_images,
                                           (const int *)nullptr, (const int *)nullptr) != cudaSuccess)
        return false;
    temp = c.take<char>(temp_bytes);
    return true;
}

}  // namespace

extern "C" int64_t pmb200_view_scores_workspace_bytes(int n_images, int64_t n_obs, int64_t n_contrib) {
    const int bad = check_model(n_images, n_obs, 0);
    if (bad) return pmb200_internal_fail(PMB200_EINVAL, bad == 1 ? "view_scores_workspace_bytes: 1 <= n_images < 65536"
                                                                 : "view_scores_workspace_bytes: 0 <= n_obs < 2^31");
    if (n_contrib < 0 || n_contrib >= kMaxItems)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores_workspace_bytes: the model has 2^31 or more co-visible observation "
                                                   "pairs (n_contrib); split it into smaller models");
    const int pos_bits = bits_for(n_obs + 1);
    const int key_bits = bits_for((long long)n_images * n_images) + pos_bits;
    Carver c{nullptr};
    ScoreLayout l;
    if (!score_layout(c, n_obs, n_contrib, 31, key_bits, l))
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores_workspace_bytes: no CUDA device to size the CUB sort for");
    return (int64_t)c.used;
}

extern "C" int pmb200_view_scores_count(const int *obs_offsets, const int *obs_points, int n_images, int64_t n_obs, int64_t *total_out,
                                        void *workspace, int64_t workspace_bytes, void *stream) {
    if (!obs_offsets || (!obs_points && n_obs > 0) || !total_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores_count: null pointer");
    const int bad = check_model(n_images, n_obs, 0);
    if (bad) return pmb200_internal_fail(PMB200_EINVAL, bad == 1 ? "view_scores_count: 1 <= n_images < 65536" : "view_scores_count: 0 <= n_obs < 2^31");
    Carver c{static_cast<char *>(workspace)};
    ScoreLayout l;
    const int pt_bits = 31;
    if (!score_layout(c, n_obs, 0, pt_bits, 1, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores_count: workspace smaller than view_scores_workspace_bytes(n_images, n_obs, 0)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int m = (int)n_obs;
    cudaMemsetAsync(l.offs, 0, sizeof(long long), st);
    if (m == 0) {
        cudaMemsetAsync(total_out, 0, sizeof(int64_t), st);
        return pmb200_internal_launch_status("view_scores_count");
    }
    const int blocks = grid_blocks(m);
    obs_keys_kernel<<<blocks, kBlock, 0, st>>>(obs_points, m, l.pt_in, l.g_in);
    size_t bytes = l.cub1_bytes;
    if (cub::DeviceRadixSort::SortPairs(l.cub1, bytes, l.pt_in, l.pt_sorted, l.g_in, l.g_sorted, m, 0, pt_bits, st) != cudaSuccess)
        return pmb200_internal_launch_status("view_scores_count (sort)");
    obs_count_kernel<<<blocks, kBlock, 0, st>>>(l.pt_sorted, l.g_sorted, obs_offsets, n_images, m, l.img_sorted, l.count);
    bytes = l.cub1_bytes;
    if (cub::DeviceScan::InclusiveSum(l.cub1, bytes, l.count, l.offs + 1, m, st) != cudaSuccess)
        return pmb200_internal_launch_status("view_scores_count (scan)");
    cudaMemcpyAsync(total_out, l.offs + m, sizeof(int64_t), cudaMemcpyDeviceToDevice, st);
    return pmb200_internal_launch_status("view_scores_count");
}

extern "C" int pmb200_view_scores(const double *xyz, int64_t n_points, const int *obs_offsets, const int *obs_points,
                                  const double *centers, int n_images, int64_t n_obs, int64_t n_contrib, double theta0, double sigma1,
                                  double sigma2, double *score_out, void *workspace, int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_points > 0) || !obs_offsets || (!obs_points && n_obs > 0) || !centers || !score_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores: null pointer");
    const int bad = check_model(n_images, n_obs, n_points);
    if (bad) {
        static thread_local char msg[96];
        snprintf(msg, sizeof msg, "view_scores: %s", model_message(bad));
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    if (n_contrib < 0 || n_contrib >= kMaxItems)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores: the model has 2^31 or more co-visible observation pairs (n_contrib)");
    if (!std::isfinite(theta0) || !(sigma1 > 0.0) || !(sigma2 > 0.0) || !std::isfinite(sigma1) || !std::isfinite(sigma2))
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores: theta0 finite, sigma1 and sigma2 positive and finite");
    const int pos_bits = bits_for(n_obs + 1);
    const int key_bits = bits_for((long long)n_images * n_images) + pos_bits;
    Carver c{static_cast<char *>(workspace)};
    ScoreLayout l;
    if (!score_layout(c, n_obs, n_contrib, 31, key_bits, l) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "view_scores: workspace smaller than view_scores_workspace_bytes(n_images, n_obs, n_contrib)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    cudaMemsetAsync(score_out, 0, (size_t)n_images * n_images * sizeof(double), st);
    if (n_contrib == 0) return pmb200_internal_launch_status("view_scores");
    const int m = (int)n_obs, t = (int)n_contrib;
    EmitParams p;
    p.pt = l.pt_sorted; p.g = l.g_sorted; p.img = l.img_sorted; p.offs = l.offs; p.offsets = obs_offsets;
    p.xyz = xyz; p.centers = centers; p.n_images = n_images; p.m = m; p.pos_bits = pos_bits;
    p.theta0 = theta0; p.sigma1 = sigma1; p.sigma2 = sigma2; p.key = l.key_in; p.val = l.val_in;
    obs_emit_kernel<<<grid_blocks(m), kBlock, 0, st>>>(p);
    size_t bytes = l.cub2_bytes;
    if (cub::DeviceRadixSort::SortPairs(l.cub2, bytes, l.key_in, l.key_sorted, l.val_in, l.val_sorted, t, 0, key_bits, st) != cudaSuccess)
        return pmb200_internal_launch_status("view_scores (sort)");
    pair_sum_kernel<<<grid_blocks(t), kBlock, 0, st>>>(l.key_sorted, l.val_sorted, t, pos_bits, n_images, score_out);
    return pmb200_internal_launch_status("view_scores");
}

extern "C" int64_t pmb200_depth_ranges_workspace_bytes(int n_images, int64_t n_obs) {
    const int bad = check_model(n_images, n_obs, 0);
    if (bad) return pmb200_internal_fail(PMB200_EINVAL, bad == 1 ? "depth_ranges_workspace_bytes: 1 <= n_images < 65536"
                                                                 : "depth_ranges_workspace_bytes: 0 <= n_obs < 2^31");
    Carver c{nullptr};
    double *a, *b;
    void *temp;
    size_t tb;
    if (!range_layout(c, n_images, n_obs, a, b, temp, tb))
        return pmb200_internal_fail(PMB200_EINVAL, "depth_ranges_workspace_bytes: no CUDA device to size the CUB sort for");
    return (int64_t)c.used;
}

extern "C" int pmb200_depth_ranges(const double *xyz, int64_t n_points, const int *obs_offsets, const int *obs_points,
                                   const double *extrinsics, int n_images, int64_t n_obs, double *ranges_out, void *workspace,
                                   int64_t workspace_bytes, void *stream) {
    if ((!xyz && n_points > 0) || !obs_offsets || (!obs_points && n_obs > 0) || !extrinsics || !ranges_out || !workspace)
        return pmb200_internal_fail(PMB200_EINVAL, "depth_ranges: null pointer");
    const int bad = check_model(n_images, n_obs, n_points);
    if (bad) {
        static thread_local char msg[96];
        snprintf(msg, sizeof msg, "depth_ranges: %s", model_message(bad));
        return pmb200_internal_fail(PMB200_EINVAL, msg);
    }
    Carver c{static_cast<char *>(workspace)};
    double *z_in, *z_sorted;
    void *temp;
    size_t temp_bytes;
    if (!range_layout(c, n_images, n_obs, z_in, z_sorted, temp, temp_bytes) || workspace_bytes < (int64_t)c.used)
        return pmb200_internal_fail(PMB200_EINVAL, "depth_ranges: workspace smaller than depth_ranges_workspace_bytes(n_images, n_obs)");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int m = (int)n_obs;
    if (m > 0) {
        obs_depth_kernel<<<grid_blocks(m), kBlock, 0, st>>>(obs_points, obs_offsets, n_images, m, xyz, extrinsics, z_in);
        if (cub::DeviceSegmentedSort::SortKeys(temp, temp_bytes, (const double *)z_in, z_sorted, m, n_images, obs_offsets, obs_offsets + 1,
                                               st) != cudaSuccess)
            return pmb200_internal_launch_status("depth_ranges (sort)");
    }
    depth_pick_kernel<<<grid_blocks(n_images), kBlock, 0, st>>>(z_sorted, obs_offsets, n_images, ranges_out);
    return pmb200_internal_launch_status("depth_ranges");
}
