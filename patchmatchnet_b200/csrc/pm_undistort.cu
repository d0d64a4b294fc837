// pm_undistort.cu -- undistortion of COLMAP cameras (beyond the reference; INTEGRATION.md "Undistortion (beyond the reference)",
// contract in include/patchmatch_b200.h).  The camera models and the per-pixel warp are pm_camera_math.cuh, shared with the
// host build of the CPU tests.
//
//   pmb200_undistort_extents: one block per camera; each thread maps a strided share of the 2H + 2W border points and keeps
//     its min / max per side, then the block reduces them.  Min and max are exact, so the result does not depend on the order.
//   pmb200_undistort_image: one thread per target pixel.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <cmath>

#include "../../include/patchmatch_b200.h"
#include "pm_camera_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

constexpr int kExtentBlock = 256;
constexpr int kWarpBlockX = 32, kWarpBlockY = 8;
constexpr int kMaxSide = 1 << 20;  // per image dimension

__global__ void __launch_bounds__(kExtentBlock) extents_kernel(const pmb200_camera *cameras, double *out) {
    __shared__ double red[8][kExtentBlock];
    const pmb200_camera cam = cameras[blockIdx.x];
    double acc[8];
    for (int s = 0; s < 4; ++s) {
        acc[2 * s] = INFINITY;       // min
        acc[2 * s + 1] = -INFINITY;  // max
    }
    const long long n = 2ll * cam.height + 2ll * cam.width;
    for (long long k = threadIdx.x; k < n; k += kExtentBlock) {
        int side;
        const double m = pmcam::border_point(cam.model, cam.params, cam.width, cam.height, k, side);
        acc[2 * side] = fmin(acc[2 * side], m);
        acc[2 * side + 1] = fmax(acc[2 * side + 1], m);
    }
    for (int j = 0; j < 8; ++j) red[j][threadIdx.x] = acc[j];
    __syncthreads();
    for (int o = kExtentBlock / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o)
            for (int j = 0; j < 8; ++j)
                red[j][threadIdx.x] = (j & 1) ? fmax(red[j][threadIdx.x], red[j][threadIdx.x + o])
                                              : fmin(red[j][threadIdx.x], red[j][threadIdx.x + o]);
        __syncthreads();
    }
    if (threadIdx.x < 8) out[8 * (size_t)blockIdx.x + threadIdx.x] = red[threadIdx.x][0];
}

struct WarpParams {
    pmb200_camera cam;
    double kp[4];  // fx', fy', cx', cy'
    int out_w, out_h;
};

__global__ void __launch_bounds__(kWarpBlockX * kWarpBlockY) warp_kernel(const unsigned char *__restrict__ src, const WarpParams p,
                                                                          unsigned char *__restrict__ dst) {
    const int x = blockIdx.x * kWarpBlockX + threadIdx.x, y = blockIdx.y * kWarpBlockY + threadIdx.y;
    if (x >= p.out_w || y >= p.out_h) return;
    unsigned char rgb[3];
    pmcam::undistort_pixel(p.cam.model, p.cam.params, p.cam.width, p.cam.height, src, p.kp, x, y, rgb);
    unsigned char *o = dst + ((int64_t)y * p.out_w + x) * 3;
    o[0] = rgb[0];
    o[1] = rgb[1];
    o[2] = rgb[2];
}

// nullptr when the camera is valid, else what is wrong with it
const char *camera_problem(const pmb200_camera &c) {
    if (c.model < 0 || c.model >= pmcam::kNumModels) return "model must be a COLMAP model id, 0..10";
    if (c.width < 1 || c.height < 1 || c.width > kMaxSide || c.height > kMaxSide) return "1 <= width, height <= 2^20";
    const int n = pmcam::num_params(c.model);
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(c.params[i])) return "every parameter must be finite";
    double fx, fy, cx, cy;
    pmcam::pinhole_part(c.model, c.params, fx, fy, cx, cy);
    if (fx == 0.0 || fy == 0.0) return "focal lengths must be non-zero";
    return nullptr;
}

int fail_camera(const char *what, int index, const char *problem) {
    static thread_local char msg[160];
    snprintf(msg, sizeof msg, "%s: camera %d: %s", what, index, problem);
    return pmb200_internal_fail(PMB200_EINVAL, msg);
}

}  // namespace

extern "C" int pmb200_undistort_extents(const pmb200_camera *cameras_host, int n_cameras, pmb200_camera *cameras_device,
                                        double *extents_out, void *stream) {
    if (!cameras_host || !cameras_device || !extents_out) return pmb200_internal_fail(PMB200_EINVAL, "undistort_extents: null pointer");
    if (n_cameras < 1 || n_cameras > 65535) return pmb200_internal_fail(PMB200_EINVAL, "undistort_extents: 1 <= n_cameras <= 65535");
    for (int i = 0; i < n_cameras; ++i)
        if (const char *why = camera_problem(cameras_host[i])) return fail_camera("undistort_extents", i, why);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (cudaMemcpyAsync(cameras_device, cameras_host, sizeof(pmb200_camera) * (size_t)n_cameras, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return pmb200_internal_launch_status("undistort_extents (camera upload)");
    extents_kernel<<<n_cameras, kExtentBlock, 0, st>>>(cameras_device, extents_out);
    return pmb200_internal_launch_status("undistort_extents");
}

extern "C" int pmb200_undistort_image(const unsigned char *src, const pmb200_camera *camera_host, const double *pinhole_host,
                                      int out_width, int out_height, unsigned char *dst, void *stream) {
    if (!src || !camera_host || !pinhole_host || !dst) return pmb200_internal_fail(PMB200_EINVAL, "undistort_image: null pointer");
    if (const char *why = camera_problem(*camera_host)) return fail_camera("undistort_image", 0, why);
    if (out_width < 1 || out_height < 1 || out_width > kMaxSide || out_height > kMaxSide)
        return pmb200_internal_fail(PMB200_EINVAL, "undistort_image: 1 <= out_width, out_height <= 2^20");
    for (int i = 0; i < 4; ++i)
        if (!std::isfinite(pinhole_host[i]) || (i < 2 && pinhole_host[i] == 0.0))
            return pmb200_internal_fail(PMB200_EINVAL, "undistort_image: the pinhole camera needs finite parameters and non-zero focal lengths");
    WarpParams p;
    p.cam = *camera_host;
    for (int i = 0; i < 4; ++i) p.kp[i] = pinhole_host[i];
    p.out_w = out_width;
    p.out_h = out_height;
    const dim3 block(kWarpBlockX, kWarpBlockY);
    const dim3 grid((out_width + kWarpBlockX - 1) / kWarpBlockX, (out_height + kWarpBlockY - 1) / kWarpBlockY);
    warp_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>(src, p, dst);
    return pmb200_internal_launch_status("undistort_image");
}
