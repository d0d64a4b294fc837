/*
 * patchmatch_b200.h -- C ABI of the H100-native (sm_90a) learned-PatchMatch hot path.
 *
 * This is the drop-in boundary: plain device pointers, sizes and a CUDA stream;
 * no torch types.  The reference (FangjinhuaWang/PatchmatchNet) has no native
 * layer at all -- its hot path is a chain of ATen calls inside
 * models/patchmatch.py / models/module.py -- so each entry point below names the
 * reference Python lines it replaces; INTEGRATION.md shows the ctypes binding a
 * maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - all tensors are fp32, dense, in the layout written beside them;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *     kernels are enqueued, never synchronised -- the calls are CUDA-graph capturable;
 *   - return value: 0 on success, negative PMB200_E* on a rejected argument,
 *     positive cudaError_t if the launch failed.  pmb200_last_error() returns a
 *     thread-local message for the last non-zero return.  Nothing aborts.
 *   - re-entrant: no global mutable state; safe to call from one host thread per
 *     GPU (the reference's nn.DataParallel threading model, train.py:282).
 *     The caller makes the right device current (cudaSetDevice / torch.cuda.device).
 */
#ifndef PATCHMATCH_B200_H_
#define PATCHMATCH_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PMB200_ABI_VERSION 1

#define PMB200_EINVAL (-1)       /* bad size / null pointer */
#define PMB200_EUNSUPPORTED (-2) /* combination the reference raises NotImplementedError for */
#define PMB200_EIO (-3)          /* map files: open / read / write failed (message carries strerror and the path) */
#define PMB200_EFORMAT (-4)      /* map files: not a PFM file / malformed header / payload does not match the header */

#define PMB200_MAX_VIEWS 16
#define PMB200_MAX_NEIGHBORS 32
#define PMB200_MAX_HYPOTHESES 256

int pmb200_abi_version(void);
const char *pmb200_last_error(void);

/* Measurement aid (tools/kbench.py, A/B tests): override a launch-configuration knob of the library for this process.
 * Keys: "ka_gen" (3 | 4: generation of the fused warp+correlation kernel), "ka3_dc", "ka3_dc_vw", "ka3_pipe", "ka3_minb"
 * (generation-3 rows per pass / gather pipeline / resident CTAs), "ka4_nw" (4 | 8 consumer warps = tile rows), "ka4_ctas"
 * (resident CTAs per SM the window ring is sized for), "ka4_cap" (texels per ring slot), "ka4_stages" (ring depth 2..4), "ka4_grid" (persistent CTAs),
 * "kb_tp", "kb_dy" (block shape of the adaptive-evaluation kernel), "stem_ppt" (output pixels per thread of the fused
 * conv0 -> conv1 kernel: 2 or 4); 0 = the built-in default.  "reset" restores every
 * default.  Results never depend on these knobs, only launch shapes do.  Returns 0, or PMB200_EINVAL for an unknown key.
 * The reference has no counterpart (its launch shapes are ATen's). */
int pmb200_set_tuning(const char *key, int value);

/* ------------------------------------------------------------------------------------
 * K-D5: channels-last convolution on Hopper's warpgroup tensor cores (wgmma / TMA), fp32-accurate (3xTF32 split).
 * Replaces, for the FLOP-bound layers in the fp32-accurate mode, the nn.Conv2d calls of reference models/net.py:9-70 (FeatureNet
 * conv2..10), models/patchmatch.py:288-311 (stage-2/3 offset convs), models/net.py:73-122 (Refinement).
 *   x_nhwc      [N,H,W,Cin] fp32, 16-byte aligned, Cin in {8,16,32,64}
 *   filter_tc5  pmb200_conv2d_tc5_filter_floats(Cin,Cout,KS) floats: [tap ky*KS+kx][Cin/32 blocks (1 if Cin <= 32)]
 *               [2 Npad rows: w_hi rows then w_lo rows, Npad = Cout rounded up to 16][min(Cin,32) channels]; every
 *               [2 Npad][row bytes] tile is ONE K-major wgmma operand (its first Npad rows double as the N = Npad operand)
 *               stored in the tensor core's shared-memory swizzle for that row size (16-byte chunk j of row r sits at chunk
 *               j ^ (r % 8) for 128-byte rows, j ^ ((r / 2) % 4) for 64-byte rows, j ^ ((r / 4) % 2) for 32-byte rows);
 *               w_hi = weight rounded to TF32, w_lo = (weight - w_hi) rounded to TF32; rows >= Cout of each half are zero
 *   y_nhwc      [N,Ho,Wo,y_channel_stride]; channels y_channel_offset .. +Cout are written
 * Ho = (H + 2 pad - dil (KS-1) - 1) / stride + 1.  bias may be NULL.  relu != 0 applies max(.,0).
 * pmb200_conv2d_tc5_supported: 1 when (Cin, Cout, KS, stride) is served (KS in {1,3,5}, stride in {1,2}, Cout <= 64). */
int pmb200_conv2d_tc5_supported(int Cin, int Cout, int KS, int stride);
int pmb200_conv2d_tc5_filter_floats(int Cin, int Cout, int KS);
int pmb200_conv2d_tc5(const float *x_nhwc, const float *filter_tc5, const float *bias, float *y_nhwc, int N, int H, int W, int Cin,
                      int Cout, int KS, int stride, int pad, int dil, int relu, int y_channel_stride, int y_channel_offset,
                      void *stream);
/* Stride-1 form of the same convolution (K-D5h): the input halo of an 8 x 8 output unit is fetched ONCE (one dense TMA box),
 * split once into channel-chunk planes [Cin/4][rows][cols][4 floats]; every filter tap is a shifted view of them (no-swizzle
 * K-major wgmma operand: 8 consecutive pixels of a plane are one core matrix).  Same arguments minus the stride.
 *   filter_tc5h  same float count as filter_tc5, layout [tap][Cin/4 chunks][w_hi rows Npad | w_lo rows Npad][4 floats] */
int pmb200_conv2d_tc5h(const float *x_nhwc, const float *filter_tc5h, const float *bias, float *y_nhwc, int N, int H, int W, int Cin,
                       int Cout, int KS, int pad, int dil, int relu, int y_channel_stride, int y_channel_offset, void *stream);
/* The shared-memory plan pmb200_conv2d_tc5h launches a layer of `units` 8 x 8 output units with, on a device of `sms` SMs whose
 * per-block opt-in limit is smem_optin bytes: plan[0] staging buffers (1 or 2), plan[1] filter stages, plan[2] 1 when the whole
 * filter stays resident, plan[3] dynamic shared-memory bytes, plan[4] CTAs per SM its shared memory allows (1 to 4), plan[5] plane sets
 * (2, or 1 when units <= sms).  Non-zero when the layer does not fit. */
int pmb200_conv2d_tc5h_plan(int Cin, int Cout, int KS, int dil, int units, int sms, int smem_optin, int *plan);
/* Debugging aid (not a reference interface): a device buffer of 256 int64 that following K-D5h launches stamp with clock64
 * for warpgroup 0 of CTA 0 ([role][unit 0..15][event 0..3]: producer, wgmmas done, split, epilogue done); NULL switches it off. */
int pmb200_debug_conv5h_trace(long long *device_buffer_256);

/* ------------------------------------------------------------------------------------
 * K-S: the two full-resolution layers of FeatureNet in one launch, exact fp32 (plain FFMA, weights in the constant bank):
 *     y = relu(conv1(relu(conv0(x))))   conv0 3 -> 8, conv1 8 -> 8, both 3x3 / pad 1, BatchNorm folded into weight and bias.
 * Replaces `self.conv1(self.conv0(x))` at reference models/net.py:44 (layers :18-19) in eval mode.
 *   x_nchw   device [N,3,H,W] contiguous (the caller's image planes are read in place: no layout conversion)
 *   y_nhwc   device [N,H,W,8], 16-byte aligned
 *   host_w0  HOST memory [8][3][3][3] (PyTorch layout), host_b0 [8]; host_w1 HOST memory [8][8][3][3], host_b1 [8]:
 *            copied into the kernel parameter block at launch (so a captured CUDA graph keeps the values it was captured with). */
int pmb200_conv_stem(const float *x_nchw, const float *host_w0, const float *host_b0, const float *host_w1, const float *host_b1,
                     float *y_nhwc, int N, int H, int W, void *stream);

/* ------------------------------------------------------------------------------------
 * K-R: Refinement (reference models/net.py:73-122) in two launches, exact fp32 (plain FFMA, weights in the constant bank).
 * pmb200_refine_low  (half resolution; :104-110):  d = (depth - depth_min) / (depth_max - depth_min);
 *                    low = relu(conv2(relu(conv1(d))))   conv1 1 -> 8, conv2 8 -> 8, 3x3 / pad 1, BatchNorm folded.
 * pmb200_refine_full (full resolution; :103, :112-120):  up = relu(bn(deconv(low))), c0 = relu(conv0(img)),
 *                    c3 = relu(conv3(cat(up, c0))), res = conv_res(c3), out = (nearest_up2x(d) + res) * span + depth_min.
 *   depth_half [N,1,h,w], depth_min / depth_max [N], low_nhwc [N,h,w,8] (16-byte aligned), img_nchw [N,3,2h,2w] contiguous,
 *   depth_out [N,1,2h,2w]: device.   Every host_* argument is HOST memory in PyTorch layout with BatchNorm folded:
 *   host_w1 [8][1][3][3], host_w2 [8][8][3][3], host_wd [8 in][8 out][3][3] (ConvTranspose2d), host_w0 [8][3][3][3],
 *   host_w3 [8][16][3][3], host_wr [1][8][3][3] (no bias), biases [8].  They travel in the kernel parameter block. */
int pmb200_refine_low(const float *depth_half, const float *depth_min, const float *depth_max, const float *host_w1, const float *host_b1,
                      const float *host_w2, const float *host_b2, float *low_nhwc, int N, int h, int w, void *stream);
int pmb200_refine_full(const float *low_nhwc, const float *img_nchw, const float *depth_half, const float *depth_min, const float *depth_max,
                       const float *host_wd, const float *host_bd, const float *host_w0, const float *host_b0, const float *host_w3,
                       const float *host_b3, const float *host_wr, float *depth_out, int N, int H, int W, void *stream);

/* ------------------------------------------------------------------------------------
 * Relative projections for every (source view, batch element):
 *     P = src_proj . inverse(ref_proj);  rt = [P[0,0..2], P[1,0..2], P[2,0..2], P[0..2,3]]
 * Replaces torch.matmul(src_proj, torch.inverse(ref_proj)) at models/module.py:148-150,
 * which the reference re-evaluates (with a host sync inside linalg.inv) once per source
 * view per PatchMatch iteration; here it runs once per stage with no host sync.
 * The 4x4 inverse is done in fp64 on the device and rounded to fp32.
 *   ref_proj        [B,4,4], row stride 4, batch stride `ref_batch_stride` floats
 *   src_projs_host  host array of V device pointers, each [B,4,4] with batch stride `src_batch_stride`
 *   rt_out          [V,B,12]
 */
int pmb200_relative_projection(const float *ref_proj, int64_t ref_batch_stride,
                               const float *const *src_projs_host, int64_t src_batch_stride,
                               int V, int B, float *rt_out, void *stream);

/* ------------------------------------------------------------------------------------
 * Pack n NCHW feature maps into one channels-last buffer [n,B,H,W,C] (one launch).
 * The fused kernels read features channels-last so that each bilinear tap is one
 * contiguous C-vector.  Not needed when the producer already emits channels-last.
 *   maps_host  host array of n device pointers, each [B,C,H,W] contiguous
 */
int pmb200_pack_nhwc(const float *const *maps_host, int n, int B, int C, int H, int W,
                     float *out_nhwc, void *stream);

/* ------------------------------------------------------------------------------------
 * Caller-side helper (feature pyramid top-down path, models/net.py:60-66): channels-last
 *     out = bilinear_upsample_x2(x) + y (+ bias[c])     x [N,h,w,C], y/out [N,2h,2w,C], C % 4 == 0
 * same sampling as F.interpolate(scale_factor=2, mode="bilinear", align_corners=False).
 * bias: NULL, or the [C] bias of the lateral 1x1 conv that produced y (so that conv can run bias-free).
 * Replaces ATen's channels-last bilinear kernel + separate bias/add passes (12 % + 4 % of the forward before).
 */
int pmb200_upsample2x_add_nhwc(const float *x_nhwc, const float *y_nhwc, const float *bias, float *out_nhwc,
                               int N, int h, int w, int C, void *stream);

/* ------------------------------------------------------------------------------------
 * Channels-last 2-D convolution for the small learned convs of the model (1..64 channels), tensor cores
 * (TF32 implicit GEMM), bias + ReLU fused:
 *     y[n,oy,ox,yco+co] = act(bias[co] + sum_{ky,kx,ci} x[n, oy*S-pad+ky*dil, ox*S-pad+kx*dil, ci] * w[co,ci,ky,kx])
 * Replaces, on the hot path, the offset convs propa_conv / eval_conv (models/patchmatch.py:288-311, called at
 * :486 and :498: nn.Conv2d 3x3, dilation = padding = propagation range) and, either side of it (SURVEY.md 8f rows
 * f1 / f3), ConvBnReLU (models/module.py:11-40, BatchNorm folded by the caller) and the plain convs of FeatureNet
 * (models/net.py:9-70) and Refinement (models/net.py:73-122, including its ConvTranspose2d: transposed2x = 1 runs the
 * equivalent stride-1 conv over the virtually zero-stuffed input, caller passes the flipped filter and pad = KS-1-pad_t).
 *   x            [N,H,W,Cin]      (16-byte aligned when Cin % 4 == 0)
 *   filter_frag  the filter in tensor-core fragment order for the chosen precision,
 *                pmb200_conv2d_filter_floats(Cin,Cout,KS,precision) floats, 16-byte aligned:
 *                [tap = ky*KS+kx][ks = 0..Cin'/8)[nt = 0..NT)[lane = 0..32)[2 or 4], lane = 4*g + t holding
 *                (b0, b1) = (w[nt*8+g][ks*8+2t][ky][kx], w[nt*8+g][ks*8+2t+1][ky][kx]) -- the MMA's k slots (t, t+4)
 *                are mapped to the adjacent channels (2t, 2t+1) -- zero where an index is outside the filter;
 *                Cin' = Cin rounded up to 8/16/32/64, NT = ceil(Cout/8) rounded up to 1,2,3,4 or 8.
 *                precision 1: the two values rounded to TF32 (nearest, ties away from zero);
 *                precision 3: four values (b0_hi, b1_hi, b0_lo, b1_lo), hi = tf32(w), lo = tf32(w - hi)
 *   bias         [Cout] or NULL
 *   add_up2x     NULL, or a coarser map [N,Ho/2,Wo/2,Cout] whose bilinear x2 upsample (F.interpolate scale_factor=2,
 *                align_corners=False) is added before the activation: the top-down step of the feature pyramid
 *                (models/net.py:60-66) fused into the lateral conv's epilogue (Ho, Wo, Cout even)
 *   y            [N,Ho,Wo,y_channel_stride], written at channels y_channel_offset .. +Cout (stride 0 = Cout: dense)
 *   precision    1: TF32 operands (the library's behaviour under torch.backends.cudnn.allow_tf32, torch's default:
 *                filter rounded by the host, activations truncated by the tensor core as for wgmma kind tf32);
 *                3: error-compensated 3xTF32, fp32-accurate
 *   rows_per_warp 0 = choose (tile = 16 columns x 4*rows_per_warp rows per 4-warp CTA); 1, 2 or 4 to force
 */
int pmb200_conv2d_filter_floats(int Cin, int Cout, int KS, int precision);
int pmb200_conv2d_nhwc(const float *x, const float *filter_frag, const float *bias, const float *add_up2x, float *y,
                       int N, int H, int W, int Cin, int Cout, int KS, int stride, int pad, int dil,
                       int relu, int precision, int transposed2x, int y_channel_stride, int y_channel_offset,
                       int rows_per_warp, void *stream);

/* One source view of a ragged pack (the *_views entry points): the view's first float is src_flat + offset, and batch item b
 * of it is [height, width(, C)] row-major starting at src_flat + offset + b * height * width (* C). */
typedef struct pmb200_view_extent {
    int64_t offset; /* floats from src_flat to (view v, batch 0); K-A: a multiple of 4 */
    int height;
    int width;
} pmb200_view_extent;

/* ------------------------------------------------------------------------------------
 * Geometric-consistency filtering of one reference depth map against V source depth maps, one launch
 * (SURVEY.md 8f row f4).  Replaces reproject_with_depth (eval.py:86-146), check_geometric_consistency (eval.py:149-190)
 * and the per-reference-view accumulation of filter_depth (eval.py:220, :226-256): numpy + cv2.remap on one CPU thread.
 *   ref_depth [H,W], confidence [H,W], src_depths [V,Hs,Ws]   float32
 *   cams [V,60] float64 (device): per source view, row-major, composed exactly as the reference composes them in float32
 *       and then widened:  inv(K_ref) (9) | (E_src . inv(E_ref))[:3,:4] (12) | K_src (9) | inv(K_src) (9) |
 *       (E_ref . inv(E_src))[:3,:4] (12) | K_ref (9)        (eval.py:116-139)
 *   geo_mask_sum_out [H,W] int32: source views consistent with the pixel (dist < geo_pixel_thres and relative depth
 *       difference < geo_depth_thres, eval.py:180-187); photo_mask_out / final_mask_out [H,W] uint8 (0/1):
 *       confidence > photo_thres, and that AND geo_mask_sum >= geo_mask_thres (eval.py:220, :254-255);
 *   depth_avg_out [H,W] float64: (sum of the consistent reprojected depths + ref_depth) / (geo_mask_sum + 1) (eval.py:252).
 * The source-depth sample reproduces cv2.remap(INTER_LINEAR, constant border 0): coordinates rounded to 1/32 pixel,
 * float32 weights, no fused multiply-add. */
int pmb200_geometric_filter(const float *ref_depth, const float *confidence, const float *src_depths,
                            const double *cams, int V, int H, int W, int Hs, int Ws, double geo_pixel_thres,
                            float geo_depth_thres, float photo_thres, int geo_mask_thres, int *geo_mask_sum_out,
                            unsigned char *photo_mask_out, unsigned char *final_mask_out, double *depth_avg_out,
                            void *stream);
/* pmb200_geometric_filter with source depth maps of different sizes (V <= 64): src_depths [V,Hs,Ws] replaced by src_flat and
 * one host extent per view; source view v's map is [height_v, width_v] at src_flat + offset_v, sampled at its own size
 * (eval.py:129 remaps each source on its own map).  PMB200_EINVAL when a view has a non-positive size, more than 2^31
 * pixels, or a negative offset. */
int pmb200_geometric_filter_views(const float *ref_depth, const float *confidence, const float *src_flat,
                                  const pmb200_view_extent *views_host, const double *cams, int V, int H, int W,
                                  double geo_pixel_thres, float geo_depth_thres, float photo_thres, int geo_mask_thres,
                                  int *geo_mask_sum_out, unsigned char *photo_mask_out, unsigned char *final_mask_out,
                                  double *depth_avg_out, void *stream);

/* Point-cloud half of the fusion for one reference view (reference eval.py:273-296): the pixels of final_mask, in row-major
 * order, back-projected with the averaged depth into the world frame, with their colours, written as the 15-byte vertex
 * records of the reference's fused.ply (binary little endian: float32 x, y, z, uint8 red, green, blue).
 *   final_mask  [H*W] bytes (0 / non-0), depth_avg [H*W] float64 (both as pmb200_geometric_filter writes them)
 *   ref_img_hwc [H*W*3] float32 in [0,1] (the reference's read_image output)
 *   cam25       25 doubles: inverse(ref_intrinsics) row-major (9) then inverse(ref_extrinsics) row-major (16), the float32
 *               inverses numpy computes, widened (ops.compose_fusion_camera)
 *   ply_body_out  capacity H*W*15 bytes; count_out: ONE int, the number of vertices written; block_scratch: ceil(H*W/256) ints
 * All pointers are device memory.  Three launches on `stream` (count, scan, write); no host synchronisation. */
int pmb200_fuse_points(const unsigned char *final_mask, const double *depth_avg, const float *ref_img_hwc, const double *cam25,
                       int H, int W, unsigned char *ply_body_out, int *count_out, int *block_scratch, void *stream);
/* pmb200_fuse_points with oriented records: the same launches and the same surviving pixels in the same order, each written
 * as a 27-byte vertex in the property order of COLMAP's fused.ply: float32 x, y, z, nx, ny, nz, uint8 red, green, blue.
 *   normals_hwc [H*W*3] float32 (device): the reference view's camera-frame normal map (pmb200_depth_normals).  The world
 *               normal is the rotation block of inverse(ref_extrinsics) (cam25[9..]) times it; a zero normal stays zero.
 *   ply_body_out  capacity H*W*27 bytes. */
int pmb200_fuse_points_oriented(const unsigned char *final_mask, const double *depth_avg, const float *ref_img_hwc,
                                const float *normals_hwc, const double *cam25, int H, int W, unsigned char *ply_body_out,
                                int *count_out, int *block_scratch, void *stream);

/* Per-pixel surface normals of one depth map (beyond the reference, which has none), one launch, no host synchronisation,
 * bit-identical from run to run.  Pixel p = (x, y) back-projects to P(p) = D(p) K^-1 (x, y, 1) (float64).  Its inliers are
 * the pixels q of the (2 radius + 1)^2 window around p, clipped at the image border, with a finite depth > 0 and
 * |D(q) - D(p)| <= depth_thres * D(p) (p included).  The normal is the unit eigenvector of the smallest eigenvalue of the
 * inliers' covariance about their centroid (float64, closed-form 3x3 solve), facing the camera (n . P(p) < 0), in the camera
 * frame.  It is (0, 0, 0) when D(p) is not finite and > 0, when there are fewer than min_inliers inliers, or when the middle
 * eigenvalue is <= 1e-6 times the largest (collinear or coincident points).
 *   depth [H*W] float32 (device); kinv_host: HOST, 9 doubles, K^-1 row-major at the map's size (the float32 inverse, widened)
 *   normals_out [H*W*3] float32 (device), the layout of COLMAP's normal maps
 * PMB200_EINVAL, nothing launched, for a null pointer, a bad size, radius outside 1..7, depth_thres < 0 or NaN, or
 * min_inliers < 1. */
int pmb200_depth_normals(const float *depth, const double *kinv_host, int H, int W, int radius, double depth_thres,
                         int min_inliers, float *normals_out, void *stream);

/* ------------------------------------------------------------------------------------
 * Meshes: TSDF integration of depth maps and marching cubes (beyond the reference, which has no mesher; INTEGRATION.md
 * "Meshes (beyond the reference)").  Definition:
 *
 * Grid.  The grid is anchored at the world origin.  Voxel (i, j, k) (int32) has its centre at ((i, j, k) + 0.5) * s, where s
 * is the voxel size.  Voxels come in blocks of 8^3.  Block key = the block's (bi, bj, bk) packed into 64 bits, 21 bits per
 * axis with an offset so that the keys sort in z, y, x order: (bk + 2^20) << 42 | (bj + 2^20) << 21 | (bi + 2^20).  Reject
 * (PMB200_EINVAL) any point whose voxel index does not fit: floor((p -+ tau) / s) must lie in [-2^23, 2^23) on every axis.
 *
 * Allocation.  The allocated blocks are the sorted unique keys of every block that meets the cube [p - tau, p + tau] of some
 * seed point p.  The truncation is tau = trunc * s, with trunc in [1, 4] voxels, so a point meets at most 8 blocks.  Memory
 * and work are proportional to the number of allocated blocks, whatever the cloud's extent: a far outlier adds its own few
 * blocks, never a dense box.
 *
 * Integration.  Each allocated voxel, with centre X in float64, runs through views v = 0..V-1 in order:
 *   Xc = R_v X + t_v, then u = K_v Xc / Xc.z; everything float64, the float32 camera values widened;
 *   skip the view if Xc.z <= 0;
 *   pixel (px, py) = floor(u + 0.5); skip the view if the pixel is outside that view's own W_v x H_v;
 *   d = depth_v[py, px] (float32); skip the view unless d is finite and > 0 (0 marks a pixel that is not an observation);
 *   sdf = d - Xc.z; skip the view if sdf < -tau;
 *   otherwise n += 1, F += min(1, sdf / tau), C += rgb_v[:, py, px].
 * After the last view: weight = n, tsdf = F / n (1 when n = 0), colour = clamp(round(255 * C / n)) as uint8 (round half to
 * even; 0 when n = 0).  There are no atomics: each voxel's sums are formed in one thread in view order, so reruns are
 * bit-identical.
 *
 * Extraction (marching cubes).  A voxel is valid when it is allocated and weight >= min_weight.  The cube whose minimum corner
 * is voxel a is meshed when all 8 of its corners are valid and its cube index (bit c set when corner c has tsdf < 0, corners
 * numbered 0 (0,0,0), 1 (1,0,0), 2 (1,1,0), 3 (0,1,0), 4..7 the same one voxel up in z) is not 0 or 255.  Vertices lie on cube
 * edges, and each edge belongs to its lower voxel, so a vertex shared by neighbouring cubes, including cubes in different
 * blocks, is written once.  Vertex position: X_a + t (X_b - X_a) with t = tsdf_a / (tsdf_a - tsdf_b); its colour is
 * interpolated the same way and rounded.  Triangles come from the 256-case table of csrc/pm_mesh_math.cuh, wound so that the
 * right-hand normal points from negative to positive tsdf, which is towards the cameras.  The output has no unreferenced
 * vertices: an edge gets a vertex only when one of its four cubes is meshed.  Output order:
 *   vertices by (block key, voxel index in the block with x fastest, edge axis x / y / z);
 *   faces by cube in the same order, then in table order.
 *
 * Calls (device pointers unless marked HOST; `stream` a cudaStream_t; *_workspace_bytes return bytes or a negative PMB200_E*):
 *   pmb200_tsdf_alloc: seed points [n,3] float32 -> the sorted unique block keys, uint64 [n_blocks], written at the START of
 *       the workspace, and n_blocks to *n_blocks_out (HOST).  Key generation, CUB radix sort and unique, then ONE host
 *       synchronisation of `stream` (the block count sizes the volume).  PMB200_EINVAL for a null pointer, n < 0 or
 *       n >= 2^28, s not finite and > 0, trunc outside 1..4, or a point whose voxel index does not fit.
 *   pmb200_tsdf_integrate: one launch, one CTA per block, every view.  views_host: HOST table of n_views >= 1 views; view v
 *       reads depth float32 [H_v,W_v] at depth_flat + depth_offset_v and image float32 [3,H_v,W_v] in [0,1] at
 *       image_flat + image_offset_v (signed element offsets, so the views may live in separate allocations of one device).
 *       The call copies the table into the workspace.  Outputs per voxel, index block * 512 + x + 8 y + 64 z: tsdf_out and
 *       weight_out float32, colour_out uint8 x4 (red, green, blue, 0): 12 bytes per voxel.  1 <= n_blocks < 2^22.
 *   pmb200_tsdf_mesh_count: per voxel its owned vertices and its cube's triangles, per block their totals, scanned;
 *       totals_out: TWO int64 (device), the vertex and face counts.  min_weight >= 1.
 *   pmb200_tsdf_mesh_write: with the same workspace, after the count call: vertices_out [nv,15] bytes, the records of the
 *       plain fused.ply (float32 x, y, z, uint8 red, green, blue); faces_out int32 [nf,3].  nv < 2^31.
 * Enqueue only, except the one synchronisation of pmb200_tsdf_alloc. */
typedef struct pmb200_tsdf_view {
    double K[9];            /* intrinsics, row-major */
    double Rt[12];          /* world -> camera [R | t], row-major 3x4 */
    int64_t depth_offset;   /* float32 elements from depth_flat */
    int64_t image_offset;   /* float32 elements from image_flat */
    int32_t height, width;
} pmb200_tsdf_view;

int64_t pmb200_tsdf_alloc_workspace_bytes(int64_t n_points);
int pmb200_tsdf_alloc(const float *points, int64_t n_points, double voxel_size, int trunc, int64_t *n_blocks_out,
                      void *workspace, int64_t workspace_bytes, void *stream);
int64_t pmb200_tsdf_integrate_workspace_bytes(int n_views);
int pmb200_tsdf_integrate(const uint64_t *block_keys, int64_t n_blocks, double voxel_size, int trunc,
                          const pmb200_tsdf_view *views_host, int n_views, const float *depth_flat, const float *image_flat,
                          float *tsdf_out, float *weight_out, unsigned char *colour_out, void *workspace,
                          int64_t workspace_bytes, void *stream);
int64_t pmb200_tsdf_mesh_workspace_bytes(int64_t n_blocks);
int pmb200_tsdf_mesh_count(const uint64_t *block_keys, int64_t n_blocks, const float *tsdf, const float *weight, int min_weight,
                           int64_t *totals_out, void *workspace, int64_t workspace_bytes, void *stream);
int pmb200_tsdf_mesh_write(const uint64_t *block_keys, int64_t n_blocks, double voxel_size, const float *tsdf,
                           const float *weight, const unsigned char *colour, int min_weight, unsigned char *vertices_out,
                           int *faces_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Rendering of point clouds and triangle meshes (beyond the reference, whose only viewer is an Open3D window; INTEGRATION.md
 * "Rendering (beyond the reference)").  This project's own definition, float32 throughout, every product, sum and
 * difference rounded on its own (no fused multiply-add); `/` and sqrt are IEEE.  Reruns give the same bits.
 *
 * Camera.  P_host (HOST, 12 floats) = K [R | t] composed in float64 and rounded to float32, row-major 3 x 4; centre_host
 * (HOST, 3 floats) = the camera centre -R^T t, rounded likewise.  A world point (x, y, z) maps to
 * u' = ((P00 x + P01 y) + P02 z) + P03, likewise v' (row 1) and z (row 2); u = u' / z, v = v' / z.  Pixel (x, y) is sampled
 * at (x, y), the convention of the cams files.  near_z > 0 (finite); anything with z <= near_z, or z, u or v not finite, is
 * skipped.
 * Z-buffer.  One uint64 per pixel, cleared to all ones; a fragment of primitive i at depth z writes
 * atomicMin((float_bits(z) << 32) | i): the nearest fragment wins, an exact depth tie goes to the lower index.
 * Points.  Point i covers the s x s square (s = point_size, odd, 1..15) centred on (rint(u), rint(v)) (round half to even),
 * clipped to the image; its depth is z.
 * Triangles.  A face is skipped when a vertex index is outside 0..n_vertices-1, when a vertex has z <= near_z, |u| or
 * |v| > 2^22 or a value that is not finite (no clipping), or when A = (u1 - u0)(v2 - v0) - (v1 - v0)(u2 - u0) is 0.  When
 * A < 0 vertices 1 and 2 swap and A = -A.  The box is ceil(min u) .. floor(max u) (and v), clipped to the image.  Edge i
 * (opposite vertex i) runs a -> b = 1 -> 2, 2 -> 0, 0 -> 1; its function at pixel p is
 * e = (b.u - a.u)(p.v - a.v) - (b.v - a.v)(p.u - a.u), evaluated from the edge's lower endpoint (smaller v, then smaller u)
 * and negated when that endpoint is b, so the two faces of a shared edge get the same magnitude.  p is covered when every
 * e_i > 0, or e_i == 0 on a top-left edge (b.v - a.v < 0, or == 0 and b.u - a.u > 0): faces sharing an edge cover each
 * pixel on it once.  b_i = e_i / A; z = 1 / ((b0 / z0 + b1 / z1) + b2 / z2), the fragment kept when 0 < z < inf.  No
 * back-face culling.  Perspective-correct weights w_i = (b_i / z_i) z.
 * Resolve.  A pixel no fragment reached gets the background (background_host, HOST, 3 bytes) and depth 0.  Otherwise the
 * depth is the winner's z and the colour c per channel is the point's colour, or ((w0 c0 + w1 c1) + w2 c2) over the face's
 * vertex colours; 160 where rgb is NULL.  With shade != 0 c is multiplied by f = 0.25 + 0.75 |n . d| / (|n| |d|), d = centre -
 * X: for a point X is the point and n its normal (normals NULL: f = 1); for a face X = ((w0 X0 + w1 X1) + w2 X2) and n is the
 * face normal (X1 - X0) x (X2 - X0) in the face's own vertex order, components (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0),
 * dot products ((x0 y0 + x1 y1) + x2 y2).  f = 1 when |n| |d| is not finite and > 0.  Channel = clamp(rint(c f), 0, 255).
 *
 * pmb200_render_points: xyz [n,3] float32, rgb [n,3] uint8 or NULL, normals [n,3] float32 or NULL, n < 2^32; out_rgb
 *   [H,W,3] uint8, out_depth [H,W] float32; workspace of pmb200_render_points_workspace_bytes(W, H) bytes (the z-buffer).
 *   A clear, one splat launch (a thread per point) and one resolve launch.
 * pmb200_render_mesh: vertices xyz [nv,3] float32, rgb [nv,3] uint8 or NULL; faces int32 [nf,3]; nv, nf < 2^31; workspace
 *   of pmb200_render_mesh_workspace_bytes(W, H, nv, nf) bytes.  The vertices are projected once; one thread per face
 *   rasterises faces whose clipped box is at most 16 x 16 pixels and appends larger ones to a list (atomic counter) that a
 *   second launch rasterises one face per CTA; then the resolve.
 * 1 <= W, H <= 16384.  PMB200_EINVAL, nothing launched, for a null pointer, a bad size or point size, a camera that is not
 * finite, or near_z not finite and > 0.  Enqueue only; no host synchronisation. */
int64_t pmb200_render_points_workspace_bytes(int width, int height);
int pmb200_render_points(const float *xyz, const unsigned char *rgb, const float *normals, int64_t n, const float *P_host,
                         const float *centre_host, int width, int height, int point_size, float near_z, int shade,
                         const unsigned char *background_host, unsigned char *out_rgb, float *out_depth, void *workspace,
                         int64_t workspace_bytes, void *stream);
int64_t pmb200_render_mesh_workspace_bytes(int width, int height, int64_t n_vertices, int64_t n_faces);
int pmb200_render_mesh(const float *xyz, const unsigned char *rgb, int64_t n_vertices, const int *faces, int64_t n_faces,
                       const float *P_host, const float *centre_host, int width, int height, float near_z, int shade,
                       const unsigned char *background_host, unsigned char *out_rgb, float *out_depth, void *workspace,
                       int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * DTU point-cloud evaluation (reference evaluations/dtu/*.m; INTEGRATION.md "DTU evaluation"), float64 throughout.
 * Both calls sort the cloud into a fine / coarse cell hash held in a caller-owned device workspace of
 * *_workspace_bytes(n) bytes (O(n), whatever the extent of the cloud; the size query returns bytes or a negative PMB200_E*).
 *
 * pmb200_thin_points (reducePts_haa.m): the points that survive thinning to a minimum distance `dst` when they are visited
 * in the order of `rank` (a permutation of 0 .. n-1, earlier = smaller).  A point survives iff no surviving point of
 * smaller rank lies within distance <= dst of it: the lexicographically-first maximal independent set, computed in parallel
 * rounds with a bound of 256 rounds.
 *   points [n,3] float64, rank [n] int32, keep_out [n] uint8 (1 = kept)
 *   undecided_out  ONE int (device): 0, or the number of points left undecided when the round bound was reached (their
 *                  keep_out is 0 and the result must not be used)
 * pmb200_nearest_distance (MaxDistCP.m): for each "from" point, min(exact distance to the nearest "to" point, max_dist) if it
 * lies in one of MaxDistCP's blocks of the box bb_host (BB_lo + k * max_dist <= x < BB_lo + k * max_dist + max_dist,
 * k = 0 .. floor((BB_hi - BB_lo) / max_dist) per axis), else max_dist.
 *   to_points [n_to,3], from_points [n_from,3], dist_out [n_from]: float64 device;  bb_host: HOST, 6 doubles (lo xyz, hi xyz)
 *   cell: edge of the fine search cells, max_dist / 256 <= cell (speed only: the result does not depend on it); the search
 *         visits at most 5^3 fine cells, then rings of 16^3-cell coarse cells out to max_dist (at most 35^3 coarse cells)
 * Sort + table launches, then the search; no host synchronisation.  Point and output pointers may be NULL for empty clouds. */
int64_t pmb200_thin_points_workspace_bytes(int64_t n);
int pmb200_thin_points(const double *points, const int *rank, int64_t n, double dst, unsigned char *keep_out, int *undecided_out,
                       void *workspace, int64_t workspace_bytes, void *stream);
int64_t pmb200_nearest_distance_workspace_bytes(int64_t n_to);
int pmb200_nearest_distance(const double *to_points, int64_t n_to, const double *from_points, int64_t n_from, const double *bb_host,
                            double max_dist, double cell, double *dist_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Tanks and Temples evaluation (beyond the reference; INTEGRATION.md "Tanks and Temples evaluation"), float64 throughout,
 * every product and sum rounded on its own (no fused multiply-add).  Points are [n,3] float64 device arrays, n < 2^31.
 * A 4 x 4 transform is HOST, row-major, finite, with last row exactly 0 0 0 1; a point p maps to
 * x' = ((m00 x + m01 y) + m02 z) + m03 per row.  No call synchronises the host.
 *
 * pmb200_crop_polygon (Open3D's SelectionPolygonVolume): writes points_out = T p and keep_out (uint8, 1 = kept).  With
 * w = orthogonal_axis (0 x, 1 y, 2 z) and in-plane axes (u, v) = (1, 2), (0, 2), (0, 1) for w = 0, 1, 2, a point is kept
 * when axis_min <= p_w <= axis_max and the number of crossings c < p_u is odd.  polygon_host: HOST [n_vertices,3] (only the
 * u and v columns are read), n_vertices <= 128.  Edge (i, j = i + 1 mod n_vertices) crosses when v_i < p_v <= v_j or
 * v_j < p_v <= v_i, at c = u_i + ((p_v - v_i) / (v_j - v_i)) * (u_j - u_i).
 *
 * pmb200_voxel_downsample (Open3D's VoxelDownSample): bounds_host HOST (min xyz, max xyz) over the cloud.  Origin
 * o = min - s/2; a point's voxel is floor((p - o) / s) per axis; PMB200_EINVAL when s * (2^31 - 1) < (max + s/2) - o on
 * some axis, or an index would exceed 2^31 - 1.  Output: one point per occupied voxel, the float64 sum of its points in
 * original order divided by their count, voxels in ascending (x, y, z) index order; points_out has room for n points and
 * count_out (ONE int64, device) receives the voxel count.  Reruns give the same bits.
 *
 * ICP correspondences: pmb200_icp_target sorts the target into the fine / coarse cell hash of the DTU calls (cell: speed
 * only) in a target workspace of pmb200_icp_target_workspace_bytes(n_target); that workspace is then read by any number of
 * pmb200_icp_query calls with the same n_target and cell.  pmb200_icp_query: for each source point p' = T p (the source is
 * never rewritten) the nearest target point with distance <= max_dist, ties to the smallest target index, written to
 * corr_out [n_source] (int32, -1 = none; corr_out may be NULL), and over the correspondences, with p = p' - origin and
 * q = target - origin (origin_host HOST, 3 doubles), the 18 sums moments_out (device): [0] count, [1] sum d^2,
 * [2..4] sum p, [5..7] sum q, [8..16] sum q_a p_b (row a, column b), [17] sum |p|^2.  The sums are per-CTA partials, then
 * one ordered sum: no atomics, so reruns give the same bits.  max_dist / 256 <= cell. */
int pmb200_crop_polygon(const double *points, int64_t n, const double *transform_host, int orthogonal_axis, double axis_min,
                        double axis_max, const double *polygon_host, int n_vertices, double *points_out, unsigned char *keep_out,
                        void *stream);
int64_t pmb200_voxel_downsample_workspace_bytes(int64_t n);
int pmb200_voxel_downsample(const double *points, int64_t n, const double *bounds_host, double voxel_size, double *points_out,
                            int64_t *count_out, void *workspace, int64_t workspace_bytes, void *stream);
int64_t pmb200_icp_target_workspace_bytes(int64_t n_target);
int pmb200_icp_target(const double *target, int64_t n_target, double cell, void *target_workspace, int64_t workspace_bytes,
                      void *stream);
int64_t pmb200_icp_query_workspace_bytes(int64_t n_source);
int pmb200_icp_query(const double *source, int64_t n_source, const double *transform_host, const double *origin_host,
                     double max_dist, const void *target_workspace, int64_t n_target, double cell, int *corr_out,
                     double *moments_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * ETH3D evaluation (beyond the reference; INTEGRATION.md "ETH3D evaluation (beyond the reference)"), float64 throughout,
 * every product, sum and difference rounded on its own (no fused multiply-add).  Points are [n,3] float64 device arrays,
 * n < 2^31, indexed with 64-bit offsets.  No call synchronises the host.
 *
 * Free beam.  A laser scan has an origin o and scene-frame points p (the scan's local points through its 4 x 4 matrix M, with
 * the rounding of pmb200_crop_polygon; o = (M03, M13, M23)).  With r0 = beam_start_radius >= 0 and T = tan_half_angle >= 0
 * (the tangent of the beam's divergence half-angle, computed once on the host), a = p - o, b = q - o, r = sqrt(a.a) and
 * t' = a.b, a query q lies in p's free beam iff
 *     0 < t'  and  t' < a.a  and  |a x b|^2 <= (r0 r + t' T)^2,
 * dot products evaluated as ((x0 y0 + x1 y1) + x2 y2), cross components as (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0).
 * A point with a = 0, or with a coordinate that is not finite, is never a beam, and a query with b = 0 or a non-finite b is
 * in no beam.  Coordinates relative to o must stay below 1e150 in magnitude, so that no product overflows.
 *
 * pmb200_beam_index: the angular index of one scan around origin_host (HOST, 3 doubles), written into a caller-owned
 *   workspace of pmb200_beam_index_workspace_bytes(n_scan) bytes (bytes or a negative PMB200_E*; the query needs a CUDA
 *   device to size the CUB sort).  Points are binned by the direction of a on an equirectangular grid of 2 R x R bins,
 *   R = min(1024, ceil(sqrt(n_scan / 64))), and sorted within a bin by range, farthest first.  Sort and three launches.
 * pmb200_beam_observed: for every query i with mask[i] != 0 (mask may be NULL: every query) and observed[i] == 0, sets
 *   observed[i] = 1 when q_i lies in the free beam of some point of the scan whose index the workspace holds (the same
 *   n_scan and origin as the pmb200_beam_index call); other entries are left as they are, so calling it once per scan ORs
 *   the scans together.  The index culls the points whose beams cannot hold q (by angle around b's direction and by range)
 *   with margins far above the rounding of the predicate, and evaluates the predicate exactly as above on every other point:
 *   the result is a brute-force evaluation's, bit for bit.  One launch.
 *
 * pmb200_voxel_score: the density-normalised score of one cloud at tolerance tau > 0.  Point i is good when dist[i] <= tau,
 *   bad when dist[i] > tau and (observed is NULL or observed[i] != 0), otherwise excluded.  Its voxel is floor(x / tau) per
 *   axis (anchored at the world origin); bounds_host (HOST, min xyz then max xyz) must enclose every point that is not
 *   excluded, and PMB200_EINVAL is returned, nothing launched, when floor(min / tau) or floor(max / tau) lies outside
 *   [-2^20, 2^20) on some axis.  The voxel keys are sorted in a caller-owned workspace of
 *   pmb200_voxel_score_workspace_bytes(n) bytes.  Outputs (device): counts_out [4] int64 = good, bad, excluded points and the
 *   number of voxels holding a good or bad point; fraction_sum_out [1] = the sum over those voxels of good / (good + bad).
 *   The sum is per-thread partials in voxel order, a fixed tree per block, then one ordered sum: no atomics, so reruns give
 *   the same bits. */
int64_t pmb200_beam_index_workspace_bytes(int64_t n_scan);
int pmb200_beam_index(const double *scan_points, int64_t n_scan, const double *origin_host, void *workspace, int64_t workspace_bytes,
                      void *stream);
int pmb200_beam_observed(const double *queries, int64_t n_queries, const unsigned char *mask, const void *index_workspace,
                         int64_t n_scan, const double *origin_host, double beam_start_radius, double tan_half_angle,
                         unsigned char *observed, void *stream);
int64_t pmb200_voxel_score_workspace_bytes(int64_t n);
int pmb200_voxel_score(const double *points, const double *dist, int64_t n, double tau, const unsigned char *observed,
                       const double *bounds_host, int64_t *counts_out, double *fraction_sum_out, void *workspace,
                       int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * COLMAP sparse model -> scene folder (reference colmap_input.py:318-373; INTEGRATION.md "COLMAP interop"), float64 throughout.
 * The model: points xyz [n_points,3]; observations in CSR form, obs_offsets [n_images+1] (int32, obs_offsets[0] = 0) and
 * obs_points [n_obs] (int32 dense point indices in each image's own 2D-point order, -1 entries removed); camera centres
 * [n_images,3] and extrinsics [n_images,4,4] row-major, composed on the host.  1 <= n_images < 65536, n_obs < 2^31.
 *
 * View scores: for i < j, score[i,j] = score[j,i] = sum over the entries x of obs_i, in obs_i's order, whose point is in obs_j of
 *     exp(-(theta - theta0)^2 / (2 sigma^2)),  theta = (180 / pi) acos(clamp(dot(c_i - x, c_j - x) / |c_i - x| / |c_j - x|)),
 *     sigma = sigma1 if theta <= theta0 else sigma2;  a point on c_i or c_j adds 0; the diagonal is 0.
 * Two calls over ONE caller-owned workspace:
 *   pmb200_view_scores_count   sorts the observations by point and counts the contributions T (pairs of an entry of obs_i and
 *                              a distinct image j > i that also observes its point); writes T to total_out (ONE int64, device).
 *                              Workspace: pmb200_view_scores_workspace_bytes(n_images, n_obs, 0).
 *   pmb200_view_scores         emits, sorts and sums the contributions into score_out [n_images,n_images] (zeroed by the
 *                              call); n_contrib = the T of the count call, whose results the workspace (now of at least
 *                              pmb200_view_scores_workspace_bytes(n_images, n_obs, T) bytes, the same first part) still holds.
 * T >= 2^31 is rejected.  Each pair is summed by one thread in obs_i order: deterministic, no floating-point atomics.
 * Depth ranges: per image, the z (row 2 of extrinsic . [x,y,z,1]) of every entry of obs_i, sorted; ranges_out [n_images,2] =
 *   (zs[int(n * 0.01)], zs[int(n * 0.99)]), NaN for an image without entries.
 * The size queries return bytes or a negative PMB200_E* (they need a CUDA device to size the CUB sorts).  Enqueues only. */
int64_t pmb200_view_scores_workspace_bytes(int n_images, int64_t n_obs, int64_t n_contrib);
int pmb200_view_scores_count(const int *obs_offsets, const int *obs_points, int n_images, int64_t n_obs, int64_t *total_out,
                             void *workspace, int64_t workspace_bytes, void *stream);
int pmb200_view_scores(const double *xyz, int64_t n_points, const int *obs_offsets, const int *obs_points, const double *centers,
                       int n_images, int64_t n_obs, int64_t n_contrib, double theta0, double sigma1, double sigma2, double *score_out,
                       void *workspace, int64_t workspace_bytes, void *stream);
int64_t pmb200_depth_ranges_workspace_bytes(int n_images, int64_t n_obs);
int pmb200_depth_ranges(const double *xyz, int64_t n_points, const int *obs_offsets, const int *obs_points, const double *extrinsics,
                        int n_images, int64_t n_obs, double *ranges_out, void *workspace, int64_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------
 * Undistortion of COLMAP cameras (beyond the reference; INTEGRATION.md "Undistortion (beyond the reference)"), float64
 * throughout, every operation rounded on its own (no fused multiply-add).  The camera models are COLMAP's 11, with its model
 * ids and parameter order (patchmatchnet_b200/csrc/pm_camera_math.cuh).  A camera is valid when its model is 0..10,
 * 1 <= width, height <= 2^20, its parameters are finite and its focal lengths non-zero; PMB200_EINVAL otherwise.
 *
 * pmb200_undistort_extents: for each camera c of cameras_host (HOST, n_cameras <= 65535), the border extents of COLMAP's
 *   UndistortCamera: with P the PINHOLE camera of the same fx, fy, cx, cy, each border pixel centre is mapped through
 *   P.WorldToImage(c.ImageToWorld(.)); extents_out [n_cameras,8] (device) = min and max of the mapped x over the left points
 *   (0.5, y + 0.5), min and max over the right points (W - 0.5, y + 0.5), then min and max of the mapped y over the top points
 *   (x + 0.5, 0.5) and the bottom points (x + 0.5, H - 0.5).  A point whose Newton iteration breaks down (NaN) is skipped.
 *   The call copies the cameras into cameras_device (device, room for n_cameras), then one launch, one block per camera.
 * pmb200_undistort_image: src uint8 [H,W,3] RGB (device; W, H = the camera's size), dst uint8 [out_height,out_width,3].
 *   pinhole_host: HOST (fx', fy', cx', cy') of the target PINHOLE camera.  Per target pixel (x, y):
 *     u = (x + 0.5 - cx') / fx', v = (y + 0.5 - cy') / fy';  (xs, ys) = c.WorldToImage(u, v) - 0.5;
 *     valid when xs, ys are finite, 0 <= xs <= W - 1 and 0 <= ys <= H - 1;
 *     x0 = floor(xs), dx = xs - x0, x1 = min(x0 + 1, W - 1), likewise y;
 *     channel = (1 - dy)((1 - dx) p00 + dx p01) + dy((1 - dx) p10 + dx p11) (p_ab = src[y_a, x_b]), rounded half away from
 *     zero and clamped to 0..255;  an invalid pixel is 0 in every channel.
 *   Offsets are int64.  One launch.
 * Enqueue only. */
typedef struct pmb200_camera {
    int32_t model;          /* COLMAP model id, 0..10 */
    int32_t width, height;
    int32_t reserved;       /* 0 */
    double params[12];      /* COLMAP's parameter order; entries past the model's count are ignored */
} pmb200_camera;

int pmb200_undistort_extents(const pmb200_camera *cameras_host, int n_cameras, pmb200_camera *cameras_device, double *extents_out,
                             void *stream);
int pmb200_undistort_image(const unsigned char *src, const pmb200_camera *camera_host, const double *pinhole_host, int out_width,
                           int out_height, unsigned char *dst, void *stream);

/* ------------------------------------------------------------------------------------
 * Training loss and metrics (reference models/net.py:321-342 patchmatchnet_loss, train.py:174-180 create_stage_images,
 * utils.py:187-221 absolute_depth_error_metrics / threshold_metrics; DESIGN.md K-L).
 *   depth_gt [B,H,W] float32 and mask [B,H,W] uint8 (0 / non-0) at full resolution.  The level-l ground truth and mask at
 *   (y, x) are the full-resolution values at (y << l, x << l) (F.interpolate(scale_factor=0.5**l, mode="nearest")).
 *   maps_host: HOST array of device pointers; map m is float32 [B, H >> l_m, W >> l_m] at level levels_host[m] in 0..3.
 *
 * pmb200_depth_loss: terms_out float64 [n_maps + 4]: for each map the sum over the level's masked pixels of smooth-L1(d - gt)
 *   (beta 1; each term formed in float32 as torch forms it, accumulated in float64), then the mask count of levels 0..3.
 *   Per-block partials go to the caller-owned workspace of pmb200_depth_loss_workspace_bytes(...) bytes (or a negative
 *   PMB200_E*), and one final launch sums them in index order: reruns are bit-identical.  1 <= n_maps <= 16.
 * pmb200_depth_loss_backward: grads_host[m] (device, the shape of map m) = mask ? clamp(d - gt, -1, 1) * g * scale / count_l : 0,
 *   with g = *grad_loss (device float32 scalar) and count_l from terms.  One launch over all maps.
 * pmb200_depth_metrics: maps_host[l] is the map of level l (4 pointers); out float64 [B, 8 + n_thr], per image:
 *   the sum of |d - gt| (difference in float32) over the masked pixels of levels 0..3, the mask counts of levels 0..3, then
 *   per threshold the number of masked level-0 pixels with float32 |d - gt| > thresholds_host[k].  n_thr <= 8.  One launch,
 *   one block per (image, level).
 * No atomics; enqueue only. */
#define PMB200_DEPTH_LOSS_MAX_MAPS 16
#define PMB200_DEPTH_METRICS_MAX_THRESHOLDS 8
int64_t pmb200_depth_loss_workspace_bytes(const int *levels_host, int n_maps, int B, int H, int W);
int pmb200_depth_loss(const float *const *maps_host, const int *levels_host, int n_maps, const float *depth_gt,
                      const unsigned char *mask, int B, int H, int W, double *terms_out, void *workspace,
                      int64_t workspace_bytes, void *stream);
int pmb200_depth_loss_backward(const float *const *maps_host, const int *levels_host, int n_maps, const float *depth_gt,
                               const unsigned char *mask, int B, int H, int W, const double *terms, const float *grad_loss,
                               float scale, float *const *grads_host, void *stream);
int pmb200_depth_metrics(const float *const *maps_host, const float *depth_gt, const unsigned char *mask, int B, int H, int W,
                         const float *thresholds_host, int n_thr, double *out, void *stream);

/* ------------------------------------------------------------------------------------
 * Depth / confidence map files either side of the path (SURVEY 8f row f5): PFM and COLMAP .bin, read straight into /
 * written straight from caller-owned host buffers (pinned, so the next step is one cudaMemcpyAsync).  Host code, no
 * stream.  Replaces reference datasets/data_io.py read_pfm :257-288, save_pfm :291-322, read_bin :165-191,
 * save_bin :194-223 -- identical bytes on disk, identical values in memory.  In-memory layout is [H,W,C] row-major, top
 * row first (what read_pfm / read_bin return); the PFM bottom-up row order and the planar [C][H][W] payload of .bin are
 * handled inside the I/O.  Messages of PMB200_EFORMAT are the reference's exception texts ("Not a PFM file.",
 * "Malformed PFM header.", numpy's "cannot reshape array of size N into shape (..)"). */
#define PMB200_MAP_PFM 1
#define PMB200_MAP_COLMAP_BIN 2

typedef struct {
    int format;             /* PMB200_MAP_* */
    int width, height, channels;
    int big_endian;         /* PFM: non-negative scale line (data_io.py:275-279); .bin: 0 */
    double scale;           /* PFM: |scale line| (data_io.py:277); .bin: 1 */
    int64_t data_offset;    /* first payload byte */
    int64_t payload_floats; /* whole float32 items after the header (np.fromfile) */
} pmb200_map_info;

/* Parse the header only (to size the destination buffer). */
int pmb200_map_probe(const char *path, int format, pmb200_map_info *info);
/* Read the whole map into out_host[H*W*C]; `info_out` may be NULL.  capacity_floats < H*W*C -> PMB200_EINVAL. */
int pmb200_map_read(const char *path, int format, float *out_host, int64_t capacity_floats, pmb200_map_info *info_out);
/* Write data_host[H,W,C] (C = 1 or 3).  PFM: the scale line is printf("%f", -scale) -- the reference negates the scale on a
 * little-endian host (data_io.py:315-318); .bin ignores `scale`. */
int pmb200_map_write(const char *path, int format, const float *data_host, int height, int width, int channels, double scale);

/* Caller-side helper (models/net.py:289-299): photometric confidence = probability mass of the four
 * hypotheses around the regressed hypothesis index, nearest-resized to [H_out, W_out].
 *   prob [B,D,h,w] (the last PatchMatch stage's probabilities)   confidence_out [B,H_out,W_out] */
int pmb200_photometric_confidence(const float *prob, float *confidence_out,
                                  int B, int D, int h, int w, int H_out, int W_out, void *stream);

/* ------------------------------------------------------------------------------------
 * K-A: fused homography warp + bilinear gather + group-wise correlation
 *      (+ view-weighted aggregation).
 * Replaces, per source view, differentiable_warping (models/module.py:130-181), the
 * broadcast multiply + mean at models/patchmatch.py:199-203 and -- when view_weights is
 * given -- the accumulation/normalisation at models/patchmatch.py:192-194,213-217.
 * The [B,C,D,H,W] warped tensor is never materialised.
 *   ref_nhwc      [B,H,W,C]
 *   src_nhwc      [V,B,Hs,Ws,C]
 *   rt            [V,B,12] from pmb200_relative_projection
 *   depth         [B,D,H,W]
 *   view_weights  [B,V,H,W] or NULL
 *   out           view_weights == NULL : per-view similarity [V,B,G,D,H,W]
 *                 view_weights != NULL : sum_v(sim_v * w_v) / (1e-5 + sum_v w_v)  [B,G,D,H,W]
 * Fast path for (C,G) in {(64,8),(32,8),(16,4)}; any other C % G == 0 runs a generic kernel.
 */
int pmb200_warp_corr(const float *ref_nhwc, const float *src_nhwc, const float *rt,
                     const float *depth, const float *view_weights, float *out,
                     int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D,
                     void *stream);

/* ------------------------------------------------------------------------------------
 * View-weighted aggregation of stored per-view similarities (first iteration on the
 * coarsest stage, where the weights come from PixelwiseNet run on those similarities):
 *     out = sum_v(sims[v] * w[:,v]) / (1e-5 + sum_v w[:,v])
 * Replaces models/patchmatch.py:192-194,213-217.
 *   sims [V,B,G,D,H,W]   view_weights [B,V,H,W]   out [B,G,D,H,W]
 */
int pmb200_aggregate_views(const float *sims, const float *view_weights, float *out,
                           int V, int B, int G, int D, int H, int W, void *stream);

/* ------------------------------------------------------------------------------------
 * K-A': reference-feature self-correlation at the learned evaluation neighbours.
 * Replaces PatchMatch.get_grid(evaluation) (models/patchmatch.py:361-426) and the
 * grid_sample + multiply + mean of FeatureWeightNet.forward (models/patchmatch.py:613-622).
 * Neighbour k samples at (x + dx_k + offsets[2k], y + dy_k + offsets[2k+1]) with the
 * reference's normalise(align_corners=True)/sample(align_corners=False) mismatch and
 * border padding reproduced.
 *   offsets  [B,2K,H,W] raw output of eval_conv;  K in {9,17};  dilation = propagation range
 *   out      [B,G,K,H,W]
 */
int pmb200_offset_corr(const float *ref_nhwc, const float *offsets, int offsets_channels_last, float *out,
                       int B, int C, int G, int H, int W, int K, int dilation, void *stream);
/* offsets_channels_last (here and below): 0 = planar [B,2K,H,W]; 1 = channels-last [B,H,W,2K], i.e. the memory a
 * conv2d on channels-last input produces -- consumed in place, no re-layout copy. */

/* ------------------------------------------------------------------------------------
 * Eval-mode fusion of the learned 1x1x1 heads (SURVEY.md 8f "f2").
 * A head is conv3d(G->16) + BN + ReLU, conv3d(16->8) + BN + ReLU, conv3d(8->1) + bias
 * (ConvBnReLU3D, models/module.py:43-72).  With BatchNorm in eval mode the BN folds into the
 * conv; the caller passes the folded weights (HOST pointer, copied into the kernel parameter
 * block, i.e. constant memory) and the kernels apply the head in their epilogue, so the
 * [B,G,D,H,W] similarity tensor (62-73 % of K-A's bytes) is never written.
 * Inference only: training-mode BatchNorm needs batch statistics and keeps the unfused path.
 */
typedef struct pmb200_mlp {
    float w0[16 * 8]; /* [16][G], rows padded to 8 inputs */
    float b0[16];
    float w1[8 * 16]; /* [8][16] */
    float b1[8];
    float w2[8];
    float b2;
} pmb200_mlp;

/* K-A + SimilarityNet head (models/patchmatch.py:547-549,570): weighted view average -> MLP.
 *   score_out [B,D,H,W];  view_weights [B,V,H,W] required.  (C,G) in {(64,8),(32,8),(16,4)}. */
int pmb200_warp_corr_score(const float *ref_nhwc, const float *src_nhwc, const float *rt,
                           const float *depth, const float *view_weights,
                           const pmb200_mlp *head_host, float *score_out, int score_stride,
                           int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D,
                           void *stream);
/* score_stride: element stride of score_out.  1 = dense [B,D,H,W]; 2 = write the .y lanes of an interleaved
 * (xnorm, score) buffer [B,D,H,W,2] whose .x lanes pmb200_init_propagate filled (xnorm_stride = 2), which
 * pmb200_adaptive_eval then gathers with ONE 8-byte load per tap (xnorm_score argument). */

/* K-A + PixelwiseNet (models/patchmatch.py:690-702): per view, max over hypotheses of
 * sigmoid(MLP(similarity)).  view_weights_out [B,V,H,W] (zeroed by the call, then atomic max).
 * sims_out: NULL, or [V,B,G,D,H,W] to also keep the per-view similarities so that the weighted
 * aggregation that follows (pmb200_aggregate_views_score) does not have to recompute them. */
int pmb200_warp_corr_view_weights(const float *ref_nhwc, const float *src_nhwc, const float *rt,
                                  const float *depth, const pmb200_mlp *head_host,
                                  float *view_weights_out, float *sims_out,
                                  int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D,
                                  void *stream);

/* ------------------------------------------------------------------------------------
 * K-A with a size per source view (views of different resolutions or orientations; the
 * reference's differentiable_warping samples each source at its own size).
 * A ragged source pack is one float buffer `src_flat` plus one extent per view:
 *   source view v, batch item b, is [height_v, width_v, C] channels-last starting at
 *   src_flat + offset_v + b * height_v * width_v * C.
 * offset_v counts floats and must be a multiple of 4 (16-byte aligned gathers); src_flat is
 * 32-byte aligned on the (C,G) fast paths.  views_host is a HOST array of V extents, copied into
 * the kernel parameter block (a captured CUDA graph keeps its own copy, like head_host).
 * Each view is exactly what the uniform entry point computes for a pack of that view's size:
 * the align_corners=True scale (width_v - 1) / (W - 1), (height_v - 1) / (H - 1), zero padding
 * at that view's borders and the behind-the-camera rule.  PMB200_EINVAL, output untouched,
 * when V is outside 1..PMB200_MAX_VIEWS, a view has a non-positive size or height*width >= 2^29,
 * an offset is negative or not a multiple of 4, or the pack reaches 2^31 float4 elements.
 * Always runs the third-generation kernel (the generic kernel for other (C,G)).
 */
/* pmb200_warp_corr with (Hs, Ws) replaced by per-view extents */
int pmb200_warp_corr_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                           const float *rt, const float *depth, const float *view_weights, float *out,
                           int V, int B, int C, int G, int H, int W, int D, void *stream);
/* pmb200_warp_corr_score with (Hs, Ws) replaced by per-view extents */
int pmb200_warp_corr_score_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                 const float *rt, const float *depth, const float *view_weights,
                                 const pmb200_mlp *head_host, float *score_out, int score_stride,
                                 int V, int B, int C, int G, int H, int W, int D, void *stream);
/* pmb200_warp_corr_view_weights with (Hs, Ws) replaced by per-view extents */
int pmb200_warp_corr_view_weights_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                        const float *rt, const float *depth, const pmb200_mlp *head_host,
                                        float *view_weights_out, float *sims_out,
                                        int V, int B, int C, int G, int H, int W, int D, void *stream);

/* View-weighted aggregation of stored per-view similarities + SimilarityNet head:
 *   score_out [B,D,H,W] = MLP( sum_v sims[v]*w[:,v] / (1e-5 + sum_v w[:,v]) ).  G in {4,8}. */
int pmb200_aggregate_views_score(const float *sims, const float *view_weights,
                                 const pmb200_mlp *head_host, float *score_out, int score_stride,
                                 int V, int B, int G, int D, int H, int W, void *stream);

/* K-A' + FeatureWeightNet head (models/patchmatch.py:597-601,624): sigmoid(MLP(correlation)).
 *   weight_out [B,K,H,W] */
int pmb200_offset_corr_weight(const float *ref_nhwc, const float *offsets, int offsets_channels_last,
                              const pmb200_mlp *head_host, float *weight_out,
                              int B, int C, int G, int H, int W, int K, int dilation, void *stream);

/* ------------------------------------------------------------------------------------
 * K-C: hypothesis initialisation + adaptive propagation + sort, one launch.
 * Replaces DepthInitialization.forward (models/patchmatch.py:53-94),
 * PatchMatch.get_grid(propagation) (:331-360,:396-426) and Propagation.forward (:115-124).
 *   mode 0  random init : `seed_map` is U[0,1) noise [B,48,H,W] (the caller draws it with
 *                          torch.rand so the generator stream matches the reference); Ns = 48
 *   mode 1  perturbation: `seed_map` is the current depth [B,1,H,W]; Ns samples at
 *                          inverse-depth steps (1/dmin - 1/dmax) * interval_scale, clamped
 *   mode 2  passthrough : Ns == 1, hypotheses = current depth
 *   offsets [B,2Kp,H,W] raw output of propa_conv, Kp in {0,4,8,16}; with Kp == 0 nothing is
 *           propagated and the samples keep initialisation order (no sort), as in the reference.
 *   out       [B,Ns+Kp,H,W]  (ascending along dim 1 when Kp > 0)
 *   xnorm_out [B,Ns+Kp,H,W] or NULL: (1/out - 1/dmax) / (1/dmin - 1/dmax), the normalised inverse
 *             depth that depth_weight gathers (models/patchmatch.py:655-657), for pmb200_adaptive_eval
 */
int pmb200_init_propagate(const float *seed_map, const float *offsets, int offsets_channels_last,
                          const float *depth_min, const float *depth_max, float *out, float *xnorm_out,
                          int xnorm_stride, int mode, int B, int H, int W, int Ns, int Kp, int dilation,
                          float interval_scale, void *stream);

/* ------------------------------------------------------------------------------------
 * K-B: adaptive evaluation tail, one launch.
 * Replaces depth_weight (models/patchmatch.py:650-669), the feature-weight product and
 * normalisation (:509-510), SimilarityNet's neighbour gather + weighted sum (:569-577),
 * softmax (:221) and depth regression (:226-237).
 *   score0          [B,D,H,W] per-hypothesis score from the 1x1x1 MLP
 *   depth_sample    [B,D,H,W]
 *   xnorm           [B,D,H,W] normalised inverse depth from pmb200_init_propagate, or NULL
 *                   (then it is recomputed from depth_sample at every tap: same result, slower)
 *   offsets         [B,2K,H,W] raw output of eval_conv
 *   feature_weight  [B,K,H,W]
 *   prob_out        [B,D,H,W]   depth_out [B,H,W]
 *   is_inverse      stage-1 last-iteration inverse-depth index regression (:227-234)
 */
int pmb200_adaptive_eval(const float *score0, const float *depth_sample, const float *xnorm,
                         const float *xnorm_score, /* NULL, or interleaved [B,D,H,W,2] replacing score0 + xnorm */
                         const float *offsets, int offsets_channels_last,
                         const float *feature_weight, const float *depth_min, const float *depth_max,
                         float *prob_out, float *depth_out,
                         int B, int D, int H, int W, int K, int dilation,
                         float interval_scale, int is_inverse, void *stream);
/* The block shape pmb200_adaptive_eval launches a [B,D,H,W] evaluation with K neighbours on a device of `sms` SMs:
 * plan[0] pixels per block (TP: 32, 16 when the map is too small to cover every SM twice, 8 when the shared-memory tile of
 * 32 or 16 pixels exceeds 48 KB), plan[1] hypothesis lanes (DY), plan[2] shared-memory bytes.  The kb_tp / kb_dy tuning
 * knobs, when both are set, replace (TP, DY) if TP * DY <= 256 and the tile fits 48 KB.  PMB200_EINVAL on a bad size. */
int pmb200_adaptive_eval_plan(int B, int D, int H, int W, int K, int sms, int *plan);

/* ====================================================================================
 * Backward entry points (training configuration).  Which gradients exist follows the
 * reference's graph (SURVEY.md 3.4): the warp grid is built under no_grad
 * (models/module.py:147), depth_weight and the incoming depth are detached
 * (models/patchmatch.py:74,85,503,506,669), FeatureWeightNet sees a detached reference
 * feature (:475).  All d_* outputs have the shape of the tensor they differentiate.
 * ==================================================================================== */

/* K-A backward: gradients w.r.t. the reference feature and the source features.
 *   grad_out  view_weights == NULL: [V,B,G,D,H,W] (per-view similarities)
 *             view_weights != NULL: [B,G,D,H,W]   (weighted average; the weights get no gradient here,
 *                                                  they arrive detached on every iteration that uses this mode)
 *   d_ref_nhwc [B,H,W,C]   d_src_nhwc [V,B,Hs,Ws,C] (zeroed by the call, then 128-bit vector atomics) */
int pmb200_warp_corr_backward(const float *ref_nhwc, const float *src_nhwc, const float *rt,
                              const float *depth, const float *view_weights, const float *grad_out,
                              float *d_ref_nhwc, float *d_src_nhwc,
                              int V, int B, int C, int G, int H, int W, int Hs, int Ws, int D,
                              void *stream);
/* pmb200_warp_corr_backward over a ragged source pack (the backward of pmb200_warp_corr_views): (Hs, Ws) replaced by one
 * HOST extent per view.  d_src_flat has the layout of src_flat (same offsets); the call zeroes it from src_flat's first
 * float to the end of the last view, padding between views included, then scatters into it.  Each view is exactly what
 * pmb200_warp_corr_backward computes for a pack of that view's size.  PMB200_EINVAL, nothing written, on the forward's
 * extent rules (V outside 1..PMB200_MAX_VIEWS, null extents, a non-positive size, height*width >= 2^29, an offset that
 * is negative or not a multiple of 4, a pack at or beyond 2^31 float4 elements); PMB200_EUNSUPPORTED for (C,G) other
 * than (64,8), (32,8), (16,4). */
int pmb200_warp_corr_views_backward(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views_host,
                                    const float *rt, const float *depth, const float *view_weights,
                                    const float *grad_out, float *d_ref_nhwc, float *d_src_flat,
                                    int V, int B, int C, int G, int H, int W, int D, void *stream);

/* aggregate_views backward: d_sims [V,B,G,D,H,W], d_view_weights [B,V,H,W]. */
int pmb200_aggregate_views_backward(const float *sims, const float *view_weights, const float *grad_out,
                                    float *d_sims, float *d_view_weights,
                                    int V, int B, int G, int D, int H, int W, void *stream);

/* K-A' backward: gradient of the self-correlation [B,G,K,H,W] w.r.t. the raw evaluation offsets [B,2K,H,W]. */
int pmb200_offset_corr_backward(const float *ref_nhwc, const float *offsets, const float *grad_out,
                                float *d_offsets, int B, int C, int G, int H, int W, int K, int dilation,
                                void *stream);

/* K-C backward: gradient of the sorted hypotheses [B,Ns+Kp,H,W] w.r.t. the raw propagation offsets [B,2Kp,H,W]. */
int pmb200_init_propagate_backward(const float *seed_map, const float *offsets,
                                   const float *depth_min, const float *depth_max,
                                   const float *grad_out, float *d_offsets,
                                   int mode, int B, int H, int W, int Ns, int Kp, int dilation,
                                   float interval_scale, void *stream);

/* K-B backward.  prob is the forward's probability output; grad_depth [B,H,W] and/or grad_prob [B,D,H,W]
 * (either may be NULL).  d_score0 [B,D,H,W] (zeroed by the call, atomics), d_depth_sample [B,D,H,W],
 * d_offsets [B,2K,H,W], d_feature_weight [B,K,H,W]. */
int pmb200_adaptive_eval_backward(const float *score0, const float *depth_sample, const float *xnorm,
                                  const float *offsets, const float *feature_weight,
                                  const float *depth_min, const float *depth_max, const float *prob,
                                  const float *grad_depth, const float *grad_prob,
                                  float *d_score0, float *d_depth_sample, float *d_offsets,
                                  float *d_feature_weight,
                                  int B, int D, int H, int W, int K, int dilation,
                                  float interval_scale, int is_inverse, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* PATCHMATCH_B200_H_ */
