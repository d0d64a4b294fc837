// pm_geo.cu -- geometric-consistency filtering of one reference depth map against V source depth maps in ONE launch
// (SURVEY.md 8f row f4; reference eval.py:86-190 `reproject_with_depth` / `check_geometric_consistency` and the
// per-view accumulation of `filter_depth`, eval.py:226-256).
//
// The reference runs this on one CPU thread in numpy + cv2.remap, one source view at a time, materialising ~20 H x W
// float64 temporaries per (reference, source) pair.  Here one thread owns one reference pixel and walks the source views:
// project with the pixel's depth, sample the source depth map, project back, threshold, accumulate -- the same warp /
// gather pattern as K-A with a depth map in place of the features.  No intermediate ever reaches memory: the launch
// reads (1 + V) depth maps + the confidence map and writes the three masks and the averaged depth.
//
// The per-pixel arithmetic (dtype by dtype the reference's) lives in pm_geo_math.cuh, shared with the host-side formula
// tests.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/patchmatch_b200.h"
#include "pm_geo_math.cuh"

extern "C" int pmb200_internal_fail(int code, const char *msg);
extern "C" int pmb200_internal_launch_status(const char *what);

namespace {

using pmgeo::kCamDoubles;

struct GeoParams {
    const float *ref_depth, *confidence, *src_depths;
    const double *cams;
    int V, H, W, Hs, Ws;
    double pixel_thres;
    float depth_thres, photo_thres;
    int mask_thres;
    int *mask_sum;
    unsigned char *photo_mask, *final_mask;
    double *depth_avg;
};

__global__ void __launch_bounds__(256) geometric_filter_kernel(const GeoParams p) {
    extern __shared__ double s_cam[];  // [V][60]
    for (int i = threadIdx.x; i < p.V * kCamDoubles; i += blockDim.x) s_cam[i] = p.cams[i];
    __syncthreads();
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= p.H * p.W) return;
    const int x = n % p.W, y = n / p.W;
    const pmgeo::PixelResult r = pmgeo::filter_pixel(s_cam, p.src_depths, p.V, p.Hs, p.Ws, x, y, __ldg(p.ref_depth + n),
                                                     __ldg(p.confidence + n), p.pixel_thres, p.depth_thres, p.photo_thres,
                                                     p.mask_thres);
    p.mask_sum[n] = r.count;
    p.photo_mask[n] = r.photo ? 1 : 0;
    p.final_mask[n] = r.final ? 1 : 0;
    p.depth_avg[n] = r.depth_avg;
}

// Source depth maps of different sizes (pmb200_geometric_filter_views): the extents travel in the parameter block and are
// staged in shared memory behind the cameras.
constexpr int kGeoMaxViews = 64;
struct GeoViews {
    pmgeo::SourceMap v[kGeoMaxViews];
};

__global__ void __launch_bounds__(256) geometric_filter_views_kernel(const GeoParams p, const GeoViews views) {
    extern __shared__ double s_cam[];  // [V][60], then V SourceMap
    pmgeo::SourceMap *s_views = reinterpret_cast<pmgeo::SourceMap *>(s_cam + p.V * kCamDoubles);
    for (int i = threadIdx.x; i < p.V * kCamDoubles; i += blockDim.x) s_cam[i] = p.cams[i];
    for (int i = threadIdx.x; i < p.V; i += blockDim.x) s_views[i] = views.v[i];
    __syncthreads();
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= p.H * p.W) return;
    const int x = n % p.W, y = n / p.W;
    const pmgeo::PixelResult r = pmgeo::filter_pixel(s_cam, p.src_depths, s_views, p.V, x, y, __ldg(p.ref_depth + n),
                                                     __ldg(p.confidence + n), p.pixel_thres, p.depth_thres, p.photo_thres,
                                                     p.mask_thres);
    p.mask_sum[n] = r.count;
    p.photo_mask[n] = r.photo ? 1 : 0;
    p.final_mask[n] = r.final ? 1 : 0;
    p.depth_avg[n] = r.depth_avg;
}

// ---- fusion half (reference eval.py:273-296): masked back-projection + colour gather + ORDER-PRESERVING compaction ----------
// Three small launches: per-block survivor counts, one-block exclusive scan of the counts, write.  A survivor's position is
// scan[block] + (survivors before it in the block), so the records come out in row-major pixel order exactly as the
// reference's boolean indexing produces them; each record is the 15-byte PLY vertex (float32 x, y, z, uint8 r, g, b).
constexpr int kFuseBlock = 256;

__global__ void __launch_bounds__(kFuseBlock) fuse_count_kernel(const unsigned char *mask, int n, int *counts) {
    const int i = blockIdx.x * kFuseBlock + threadIdx.x;
    const int c = __syncthreads_count(i < n && mask[i] != 0);
    if (threadIdx.x == 0) counts[blockIdx.x] = c;
}

__global__ void __launch_bounds__(1024) fuse_scan_kernel(int *counts, int nblocks, int *total) {  // in place: exclusive scan
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        const int i = base + threadIdx.x;
        const int v = i < nblocks ? counts[i] : 0;
        int x = v;
        for (int off = 1; off < 32; off <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, off);
            if ((threadIdx.x & 31) >= off) x += y;
        }
        if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int w = s_warp[threadIdx.x];
            for (int off = 1; off < 32; off <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, w, off);
                if (threadIdx.x >= off) w += y;
            }
            s_warp[threadIdx.x] = w;  // inclusive over warps
        }
        __syncthreads();
        const int before_warp = (threadIdx.x >> 5) ? s_warp[(threadIdx.x >> 5) - 1] : 0;
        const int carry = s_carry;
        if (i < nblocks) counts[i] = carry + before_warp + x - v;
        __syncthreads();
        if (threadIdx.x == 1023) s_carry = carry + before_warp + x;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_carry;
}

// kOriented: the 27-byte records of pmb200_fuse_points_oriented, with the pixel's normal from `normals` ([n,3], read only
// then).  The normal map is the last parameter, so the plain instantiation keeps its parameter block and its code.
template <bool kOriented>
__global__ void __launch_bounds__(kFuseBlock) fuse_write_kernel(const unsigned char *mask, const double *depth_avg, const float *rgb,
                                                                const double *cam, int W, int n, const int *offsets,
                                                                unsigned char *body, const float *normals) {
    __shared__ int s_warp[kFuseBlock / 32];
    __shared__ double s_cam[pmgeo::kFuseCamDoubles];
    if (threadIdx.x < pmgeo::kFuseCamDoubles) s_cam[threadIdx.x] = cam[threadIdx.x];
    const int i = blockIdx.x * kFuseBlock + threadIdx.x;
    const bool keep = i < n && mask[i] != 0;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; ++w) before += s_warp[w];
    if (!keep) return;
    const int rank = offsets[blockIdx.x] + before + __popc(m & ((1u << lane) - 1u));
    if constexpr (kOriented)
        pmgeo::fuse_point_oriented(s_cam, i % W, i / W, depth_avg[i], rgb + (size_t)i * 3, normals + (size_t)i * 3,
                                   body + (size_t)rank * pmgeo::kPlyOrientedVertexBytes);
    else
        pmgeo::fuse_point(s_cam, i % W, i / W, depth_avg[i], rgb + (size_t)i * 3, body + (size_t)rank * pmgeo::kPlyVertexBytes);
}

template <bool kOriented>
int fuse_points(const unsigned char *final_mask, const double *depth_avg, const float *ref_img_hwc, const float *normals_hwc,
                const double *cam25, int H, int W, unsigned char *ply_body_out, int *count_out, int *block_scratch, void *stream,
                const char *what) {
    const int n = H * W, nblocks = (n + kFuseBlock - 1) / kFuseBlock;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    fuse_count_kernel<<<nblocks, kFuseBlock, 0, st>>>(final_mask, n, block_scratch);
    fuse_scan_kernel<<<1, 1024, 0, st>>>(block_scratch, nblocks, count_out);
    fuse_write_kernel<kOriented><<<nblocks, kFuseBlock, 0, st>>>(final_mask, depth_avg, ref_img_hwc, cam25, W, n, block_scratch,
                                                                 ply_body_out, normals_hwc);
    return pmb200_internal_launch_status(what);
}

// ---- surface normals (pmb200_depth_normals): one thread per pixel over a 32 x 8 tile of the depth map staged in shared
// memory with a halo of r, the per-pixel arithmetic of pmgeo::normal_pixel.  No atomics: run-to-run bit-identical. ----------
constexpr int kNormTileX = 32, kNormTileY = 8;
constexpr int kNormPitchMax = kNormTileX + 2 * pmgeo::kNormalMaxRadius;

struct NormalParams {
    const float *depth;
    float *normals;
    int H, W, radius, min_inliers;
    double depth_thres;
    double kinv[9];
};

__global__ void __launch_bounds__(kNormTileX * kNormTileY, 3) depth_normals_kernel(const NormalParams p) {
    __shared__ float s_tile[kNormPitchMax * (kNormTileY + 2 * pmgeo::kNormalMaxRadius)];
    const int r = p.radius, pitch = kNormTileX + 2 * r, rows = kNormTileY + 2 * r;
    const int tx0 = blockIdx.x * kNormTileX - r, ty0 = blockIdx.y * kNormTileY - r;
    for (int i = threadIdx.x; i < pitch * rows; i += kNormTileX * kNormTileY) {
        const int gy = ty0 + i / pitch, gx = tx0 + i % pitch;
        s_tile[i] = (gx >= 0 && gx < p.W && gy >= 0 && gy < p.H) ? __ldg(p.depth + (size_t)gy * p.W + gx) : 0.0f;
    }
    __syncthreads();
    const int lx = threadIdx.x % kNormTileX, ly = threadIdx.x / kNormTileX;
    const int x = blockIdx.x * kNormTileX + lx, y = blockIdx.y * kNormTileY + ly;
    if (x >= p.W || y >= p.H) return;
    const int dx0 = -min(r, x), dx1 = min(r, p.W - 1 - x), dy0 = -min(r, y), dy1 = min(r, p.H - 1 - y);
    float nrm[3];
    pmgeo::normal_pixel(s_tile + (ly + r) * pitch + lx + r, pitch, x, y, dx0, dx1, dy0, dy1, p.kinv, p.depth_thres, p.min_inliers,
                        nrm);
    float *o = p.normals + ((size_t)y * p.W + x) * 3;
    o[0] = nrm[0];
    o[1] = nrm[1];
    o[2] = nrm[2];
}

}  // namespace

extern "C" int pmb200_fuse_points(const unsigned char *final_mask, const double *depth_avg, const float *ref_img_hwc,
                                  const double *cam25, int H, int W, unsigned char *ply_body_out, int *count_out,
                                  int *block_scratch, void *stream) {
    if (!final_mask || !depth_avg || !ref_img_hwc || !cam25 || !ply_body_out || !count_out || !block_scratch)
        return pmb200_internal_fail(PMB200_EINVAL, "fuse_points: null pointer");
    if (H < 1 || W < 1 || (long long)H * W >= (1ll << 31)) return pmb200_internal_fail(PMB200_EINVAL, "fuse_points: bad size");
    return fuse_points<false>(final_mask, depth_avg, ref_img_hwc, nullptr, cam25, H, W, ply_body_out, count_out, block_scratch,
                              stream, "fuse_points");
}

extern "C" int pmb200_fuse_points_oriented(const unsigned char *final_mask, const double *depth_avg, const float *ref_img_hwc,
                                           const float *normals_hwc, const double *cam25, int H, int W, unsigned char *ply_body_out,
                                           int *count_out, int *block_scratch, void *stream) {
    if (!final_mask || !depth_avg || !ref_img_hwc || !normals_hwc || !cam25 || !ply_body_out || !count_out || !block_scratch)
        return pmb200_internal_fail(PMB200_EINVAL, "fuse_points_oriented: null pointer");
    if (H < 1 || W < 1 || (long long)H * W >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "fuse_points_oriented: bad size");
    return fuse_points<true>(final_mask, depth_avg, ref_img_hwc, normals_hwc, cam25, H, W, ply_body_out, count_out, block_scratch,
                             stream, "fuse_points_oriented");
}

extern "C" int pmb200_depth_normals(const float *depth, const double *kinv_host, int H, int W, int radius, double depth_thres,
                                    int min_inliers, float *normals_out, void *stream) {
    if (!depth || !kinv_host || !normals_out) return pmb200_internal_fail(PMB200_EINVAL, "depth_normals: null pointer");
    if (H < 1 || W < 1 || (long long)H * W >= (1ll << 31) || (H + kNormTileY - 1) / kNormTileY > 65535)
        return pmb200_internal_fail(PMB200_EINVAL, "depth_normals: bad size");
    if (radius < 1 || radius > pmgeo::kNormalMaxRadius)
        return pmb200_internal_fail(PMB200_EINVAL, "depth_normals: radius must be in 1..7");
    if (!(depth_thres >= 0.0) || min_inliers < 1)
        return pmb200_internal_fail(PMB200_EINVAL, "depth_normals: depth_thres must be >= 0 and min_inliers >= 1");
    NormalParams p;
    p.depth = depth; p.normals = normals_out;
    p.H = H; p.W = W; p.radius = radius; p.min_inliers = min_inliers; p.depth_thres = depth_thres;
    for (int i = 0; i < 9; ++i) p.kinv[i] = kinv_host[i];
    const dim3 grid((W + kNormTileX - 1) / kNormTileX, (H + kNormTileY - 1) / kNormTileY);
    depth_normals_kernel<<<grid, kNormTileX * kNormTileY, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return pmb200_internal_launch_status("depth_normals");
}

extern "C" int pmb200_geometric_filter(const float *ref_depth, const float *confidence, const float *src_depths,
                                       const double *cams, int V, int H, int W, int Hs, int Ws, double geo_pixel_thres,
                                       float geo_depth_thres, float photo_thres, int geo_mask_thres, int *geo_mask_sum_out,
                                       unsigned char *photo_mask_out, unsigned char *final_mask_out, double *depth_avg_out,
                                       void *stream) {
    if (!ref_depth || !confidence || !src_depths || !cams || !geo_mask_sum_out || !photo_mask_out || !final_mask_out || !depth_avg_out)
        return pmb200_internal_fail(PMB200_EINVAL, "geometric_filter: null pointer");
    if (V < 1 || V > 64 || H < 1 || W < 1 || Hs < 1 || Ws < 1 || (long long)H * W >= (1ll << 31) || (long long)Hs * Ws >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "geometric_filter: bad size (1 <= V <= 64)");
    GeoParams p;
    p.ref_depth = ref_depth; p.confidence = confidence; p.src_depths = src_depths; p.cams = cams;
    p.V = V; p.H = H; p.W = W; p.Hs = Hs; p.Ws = Ws;
    p.pixel_thres = geo_pixel_thres; p.depth_thres = geo_depth_thres; p.photo_thres = photo_thres; p.mask_thres = geo_mask_thres;
    p.mask_sum = geo_mask_sum_out; p.photo_mask = photo_mask_out; p.final_mask = final_mask_out; p.depth_avg = depth_avg_out;
    const int threads = 256;
    const int blocks = (int)(((long long)H * W + threads - 1) / threads);
    geometric_filter_kernel<<<blocks, threads, (size_t)V * kCamDoubles * sizeof(double), reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return pmb200_internal_launch_status("geometric_filter");
}

extern "C" int pmb200_geometric_filter_views(const float *ref_depth, const float *confidence, const float *src_flat,
                                             const pmb200_view_extent *views_host, const double *cams, int V, int H, int W,
                                             double geo_pixel_thres, float geo_depth_thres, float photo_thres, int geo_mask_thres,
                                             int *geo_mask_sum_out, unsigned char *photo_mask_out, unsigned char *final_mask_out,
                                             double *depth_avg_out, void *stream) {
    if (!ref_depth || !confidence || !src_flat || !views_host || !cams || !geo_mask_sum_out || !photo_mask_out || !final_mask_out ||
        !depth_avg_out)
        return pmb200_internal_fail(PMB200_EINVAL, "geometric_filter_views: null pointer");
    if (V < 1 || V > kGeoMaxViews || H < 1 || W < 1 || (long long)H * W >= (1ll << 31))
        return pmb200_internal_fail(PMB200_EINVAL, "geometric_filter_views: bad size (1 <= V <= 64)");
    GeoViews views;
    for (int v = 0; v < V; ++v) {
        const pmb200_view_extent &e = views_host[v];
        if (e.height < 1 || e.width < 1 || (long long)e.height * e.width >= (1ll << 31) || e.offset < 0)
            return pmb200_internal_fail(PMB200_EINVAL, "geometric_filter_views: bad source extent");
        views.v[v].offset = e.offset;
        views.v[v].rows = e.height;
        views.v[v].cols = e.width;
    }
    GeoParams p;
    p.ref_depth = ref_depth; p.confidence = confidence; p.src_depths = src_flat; p.cams = cams;
    p.V = V; p.H = H; p.W = W; p.Hs = views.v[0].rows; p.Ws = views.v[0].cols;
    p.pixel_thres = geo_pixel_thres; p.depth_thres = geo_depth_thres; p.photo_thres = photo_thres; p.mask_thres = geo_mask_thres;
    p.mask_sum = geo_mask_sum_out; p.photo_mask = photo_mask_out; p.final_mask = final_mask_out; p.depth_avg = depth_avg_out;
    const int threads = 256;
    const int blocks = (int)(((long long)H * W + threads - 1) / threads);
    const size_t smem = (size_t)V * kCamDoubles * sizeof(double) + (size_t)V * sizeof(pmgeo::SourceMap);
    geometric_filter_views_kernel<<<blocks, threads, smem, reinterpret_cast<cudaStream_t>(stream)>>>(p, views);
    return pmb200_internal_launch_status("geometric_filter_views");
}
