// pm_train.cu -- the per-step loss and metric work of training (reference models/net.py:321-342 patchmatchnet_loss,
// train.py:174-180 create_stage_images, utils.py:187-221 absolute_depth_error_metrics / threshold_metrics).
//
// The ground truth and mask of pyramid level l at pixel (y, x) are the full-resolution values at (y << l, x << l): what
// F.interpolate(scale_factor=0.5**l, mode="nearest") selects.  No pyramid is materialised.
//
// Reductions are deterministic and use no atomics:
//   - loss terms: a fixed decomposition into blocks of kThreads * kItems elements per job (one job per map, plus one mask
//     count per level); each thread accumulates its elements in float64 in index order, the block sums its threads by a
//     fixed shared-memory tree, and one final launch sums each job's block partials in index order;
//   - metrics: one block per (image, level), the same per-thread order and tree.
// Per-element terms are formed in float32 as torch forms them (no fused multiply-add), then widened.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/patchmatch_b200.h"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;                                  // elements per thread and block of the loss / backward launches
constexpr int kBlockElems = kThreads * kItems;
constexpr int kMetricThreads = 512;
constexpr int kLevels = 4;
constexpr int kMaxJobs = PMB200_DEPTH_LOSS_MAX_MAPS + kLevels;

struct Jobs {
    const float *map[kMaxJobs];  // NULL for a mask-count job
    float *grad[kMaxJobs];       // backward only
    int level[kMaxJobs];
    int first_block[kMaxJobs + 1];  // prefix sum of the jobs' block counts
    int n;
};

__host__ __device__ inline int64_t level_elems(int B, int H, int W, int l) { return (int64_t)B * (H >> l) * (W >> l); }

// full-resolution index of element i of a level-l map [B, H >> l, W >> l]
__device__ inline int64_t gt_index(int64_t i, int H, int W, int l) {
    const int wl = W >> l, hl = H >> l;
    const int x = (int)(i % wl);
    const int64_t r = i / wl;
    const int y = (int)(r % hl);
    const int64_t b = r / hl;
    return (b * H + ((int64_t)y << l)) * W + ((int64_t)x << l);
}

// torch's smooth_l1 with beta 1, in float32: z = |d - gt|; z < 1 ? 0.5 z z : z - 0.5
__device__ inline float smooth_l1(float d, float gt) {
    const float z = fabsf(__fsub_rn(d, gt));
    return z < 1.0f ? __fmul_rn(__fmul_rn(0.5f, z), z) : __fsub_rn(z, 0.5f);
}

template <int NT>
__device__ inline double block_sum(double v, double *sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
#pragma unroll
    for (int s = NT / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) sh[threadIdx.x] = sh[threadIdx.x] + sh[threadIdx.x + s];
        __syncthreads();
    }
    const double r = sh[0];
    __syncthreads();
    return r;
}

__device__ inline int find_job(const Jobs &jobs, int blk) {
    int j = 0;
    while (j + 1 < jobs.n && jobs.first_block[j + 1] <= blk) ++j;
    return j;
}

__global__ void __launch_bounds__(kThreads) loss_partials_kernel(Jobs jobs, const float *__restrict__ gt, const unsigned char *__restrict__ mask,
                                                                 int B, int H, int W, double *__restrict__ partials) {
    __shared__ double sh[kThreads];
    const int j = find_job(jobs, blockIdx.x);
    const int l = jobs.level[j];
    const int64_t n = level_elems(B, H, W, l);
    const int64_t base = (int64_t)(blockIdx.x - jobs.first_block[j]) * kBlockElems;
    const float *map = jobs.map[j];
    double acc = 0.0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        const int64_t i = base + k * kThreads + threadIdx.x;
        if (i >= n) break;
        const int64_t g = gt_index(i, H, W, l);
        if (!mask[g]) continue;
        acc += map ? (double)smooth_l1(map[i], gt[g]) : 1.0;
    }
    const double s = block_sum<kThreads>(acc, sh);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// one block per job; the jobs are the maps in order, then the mask counts of levels 0..3, so terms[j] is job j's sum
__global__ void __launch_bounds__(kThreads) loss_final_kernel(Jobs jobs, const double *__restrict__ partials, double *__restrict__ terms) {
    __shared__ double sh[kThreads];
    const int j = blockIdx.x;
    double acc = 0.0;
    for (int b = jobs.first_block[j] + threadIdx.x; b < jobs.first_block[j + 1]; b += kThreads) acc += partials[b];
    const double s = block_sum<kThreads>(acc, sh);
    if (threadIdx.x == 0) terms[j] = s;
}

__global__ void __launch_bounds__(kThreads) loss_backward_kernel(Jobs jobs, const float *__restrict__ gt, const unsigned char *__restrict__ mask,
                                                                 int B, int H, int W, const double *__restrict__ terms, int n_maps,
                                                                 const float *__restrict__ grad_loss, float scale) {
    const int j = find_job(jobs, blockIdx.x);
    const int l = jobs.level[j];
    const int64_t n = level_elems(B, H, W, l);
    const int64_t base = (int64_t)(blockIdx.x - jobs.first_block[j]) * kBlockElems;
    const float *map = jobs.map[j];
    float *out = jobs.grad[j];
    // d loss / d map = mask ? clamp(d - gt, -1, 1) * g * scale / count_l : 0  (smooth-L1 with beta 1, mean over the mask)
    const double coef = (double)__ldg(grad_loss) * (double)scale / terms[n_maps + l];
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
        const int64_t i = base + k * kThreads + threadIdx.x;
        if (i >= n) break;
        const int64_t g = gt_index(i, H, W, l);
        float v = 0.0f;
        if (mask[g]) {
            const float diff = fminf(fmaxf(__fsub_rn(map[i], gt[g]), -1.0f), 1.0f);
            v = (float)((double)diff * coef);
        }
        out[i] = v;
    }
}

// out row of image b: [abs_sum l0..3 | count l0..3 | count(|d - gt| > t_k) k < n_thr]
struct Thresholds {
    float t[PMB200_DEPTH_METRICS_MAX_THRESHOLDS];
    int n;
};

__global__ void __launch_bounds__(kMetricThreads) metrics_kernel(const float *m0, const float *m1, const float *m2, const float *m3,
                                                                 const float *__restrict__ gt, const unsigned char *__restrict__ mask,
                                                                 int H, int W, Thresholds thr, double *__restrict__ out) {
    __shared__ double sh[kMetricThreads];
    const int b = blockIdx.x, l = blockIdx.y;
    const float *map = l == 0 ? m0 : l == 1 ? m1 : l == 2 ? m2 : m3;
    const int hl = H >> l, wl = W >> l;
    const int64_t n = (int64_t)hl * wl;
    const float *mp = map + (int64_t)b * n;
    double abs_sum = 0.0, cnt = 0.0;
    int over[PMB200_DEPTH_METRICS_MAX_THRESHOLDS];
#pragma unroll
    for (int k = 0; k < PMB200_DEPTH_METRICS_MAX_THRESHOLDS; ++k) over[k] = 0;
    for (int64_t i = threadIdx.x; i < n; i += kMetricThreads) {
        const int x = (int)(i % wl), y = (int)(i / wl);
        const int64_t g = ((int64_t)b * H + ((int64_t)y << l)) * W + ((int64_t)x << l);
        if (!mask[g]) continue;
        const float e = fabsf(__fsub_rn(mp[i], gt[g]));
        abs_sum += (double)e;
        cnt += 1.0;
        if (l == 0) {
#pragma unroll
            for (int k = 0; k < PMB200_DEPTH_METRICS_MAX_THRESHOLDS; ++k) over[k] += (k < thr.n && e > thr.t[k]) ? 1 : 0;
        }
    }
    const int row = 2 * kLevels + thr.n;
    double *o = out + (int64_t)b * row;
    const double s = block_sum<kMetricThreads>(abs_sum, sh);
    const double c = block_sum<kMetricThreads>(cnt, sh);
    if (threadIdx.x == 0) { o[l] = s; o[kLevels + l] = c; }
    if (l == 0) {
#pragma unroll
        for (int k = 0; k < PMB200_DEPTH_METRICS_MAX_THRESHOLDS; ++k) {  // constant indices keep over[] in registers
            if (k >= thr.n) break;
            const double t = block_sum<kMetricThreads>((double)over[k], sh);
            if (threadIdx.x == 0) o[2 * kLevels + k] = t;
        }
    }
}

int build_jobs(Jobs &jobs, const float *const *maps_host, const int *levels_host, int n_maps, int B, int H, int W, bool counts) {
    if (n_maps < 1 || n_maps > PMB200_DEPTH_LOSS_MAX_MAPS) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: n_maps must be 1..16");
    if (B <= 0 || H <= 0 || W <= 0) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: B, H and W must be positive");
    if (!levels_host) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: null levels");
    jobs.n = n_maps + (counts ? kLevels : 0);
    jobs.first_block[0] = 0;
    for (int j = 0; j < jobs.n; ++j) {
        const bool is_map = j < n_maps;
        const int l = is_map ? levels_host[j] : j - n_maps;
        if (l < 0 || l >= kLevels) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: a level outside 0..3");
        if ((H >> l) <= 0 || (W >> l) <= 0) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: H and W must be at least 8");
        jobs.level[j] = l;
        jobs.map[j] = nullptr;
        jobs.grad[j] = nullptr;
        if (is_map && maps_host) {
            if (!maps_host[j]) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: null map pointer");
            jobs.map[j] = maps_host[j];
        }
        const int64_t blocks = (level_elems(B, H, W, l) + kBlockElems - 1) / kBlockElems;
        if (jobs.first_block[j] + blocks > (int64_t)INT32_MAX / 2) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: maps too large");
        jobs.first_block[j + 1] = jobs.first_block[j] + (int)blocks;
    }
    return 0;
}

}  // namespace

extern "C" int64_t pmb200_depth_loss_workspace_bytes(const int *levels_host, int n_maps, int B, int H, int W) {
    Jobs jobs;
    const int rc = build_jobs(jobs, nullptr, levels_host, n_maps, B, H, W, true);
    if (rc) return rc;
    return (int64_t)jobs.first_block[jobs.n] * (int64_t)sizeof(double);
}

extern "C" int pmb200_depth_loss(const float *const *maps_host, const int *levels_host, int n_maps, const float *depth_gt,
                                 const unsigned char *mask, int B, int H, int W, double *terms_out, void *workspace,
                                 int64_t workspace_bytes, void *stream) {
    if (!maps_host) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: null maps");
    Jobs jobs;
    int rc = build_jobs(jobs, maps_host, levels_host, n_maps, B, H, W, true);
    if (rc) return rc;
    if (!depth_gt || !mask || !terms_out || !workspace) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: null pointer");
    if (workspace_bytes < (int64_t)jobs.first_block[jobs.n] * (int64_t)sizeof(double))
        return pmb200_internal_fail(PMB200_EINVAL, "depth_loss: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    double *partials = (double *)workspace;
    loss_partials_kernel<<<jobs.first_block[jobs.n], kThreads, 0, st>>>(jobs, depth_gt, mask, B, H, W, partials);
    loss_final_kernel<<<jobs.n, kThreads, 0, st>>>(jobs, partials, terms_out);
    return pmb200_internal_launch_status("depth_loss");
}

extern "C" int pmb200_depth_loss_backward(const float *const *maps_host, const int *levels_host, int n_maps, const float *depth_gt,
                                          const unsigned char *mask, int B, int H, int W, const double *terms, const float *grad_loss,
                                          float scale, float *const *grads_host, void *stream) {
    if (!maps_host || !grads_host) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss_backward: null maps");
    Jobs jobs;
    int rc = build_jobs(jobs, maps_host, levels_host, n_maps, B, H, W, false);
    if (rc) return rc;
    if (!depth_gt || !mask || !terms || !grad_loss) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss_backward: null pointer");
    for (int j = 0; j < n_maps; ++j) {
        if (!grads_host[j]) return pmb200_internal_fail(PMB200_EINVAL, "depth_loss_backward: null gradient pointer");
        jobs.grad[j] = grads_host[j];
    }
    loss_backward_kernel<<<jobs.first_block[jobs.n], kThreads, 0, (cudaStream_t)stream>>>(jobs, depth_gt, mask, B, H, W, terms, n_maps,
                                                                                          grad_loss, scale);
    return pmb200_internal_launch_status("depth_loss_backward");
}

extern "C" int pmb200_depth_metrics(const float *const *maps_host, const float *depth_gt, const unsigned char *mask, int B, int H, int W,
                                    const float *thresholds_host, int n_thr, double *out, void *stream) {
    if (!maps_host || !depth_gt || !mask || !out) return pmb200_internal_fail(PMB200_EINVAL, "depth_metrics: null pointer");
    for (int l = 0; l < kLevels; ++l)
        if (!maps_host[l]) return pmb200_internal_fail(PMB200_EINVAL, "depth_metrics: null map pointer");
    if (B <= 0 || (H >> 3) <= 0 || (W >> 3) <= 0) return pmb200_internal_fail(PMB200_EINVAL, "depth_metrics: B must be positive, H and W at least 8");
    if (n_thr < 0 || n_thr > PMB200_DEPTH_METRICS_MAX_THRESHOLDS || (n_thr > 0 && !thresholds_host))
        return pmb200_internal_fail(PMB200_EINVAL, "depth_metrics: 0..8 thresholds");
    if ((int64_t)B > 65535) return pmb200_internal_fail(PMB200_EINVAL, "depth_metrics: B too large");
    Thresholds thr;
    thr.n = n_thr;
    for (int k = 0; k < PMB200_DEPTH_METRICS_MAX_THRESHOLDS; ++k) thr.t[k] = k < n_thr ? thresholds_host[k] : 0.0f;
    metrics_kernel<<<dim3(B, kLevels), kMetricThreads, 0, (cudaStream_t)stream>>>(maps_host[0], maps_host[1], maps_host[2], maps_host[3],
                                                                                  depth_gt, mask, H, W, thr, out);
    return pmb200_internal_launch_status("depth_metrics");
}
