// torch_binding.cpp -- TORCH_LIBRARY registration of the PatchMatch hot path: `torch.ops.pmb200.*`.
//
// A thin shim over the C ABI (include/patchmatch_b200.h, libpmb200.so).  It exists for the one thing a ctypes
// binding cannot do: be called from TorchScript.  The reference scripts its whole model for deployment
// (train.py:50-55 saves module_XXXXXX.pt, eval.py:38 loads it with torch.jit.load), so a drop-in PatchMatch must be
// scriptable; custom kernels are visible to TorchScript only as schema-registered operators.
//
// Conventions (SURVEY.md 8b): errors are raised with TORCH_CHECK (-> Python RuntimeError; NotImplementedError for
// the combinations the reference rejects with NotImplementedError), never status codes; every op runs under a
// CUDAGuard for its input's device on that device's CURRENT stream and keeps no global state, so DataParallel
// replicas on several threads are safe; nothing synchronises.  No arithmetic lives here.
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "../../include/patchmatch_b200.h"

namespace {

using at::Tensor;

void check(int rc, const char *what) {
    if (rc == 0) return;
    TORCH_CHECK_NOT_IMPLEMENTED(rc != PMB200_EUNSUPPORTED, "pmb200::", what, ": ", pmb200_last_error());
    TORCH_CHECK(false, "pmb200::", what, ": ", pmb200_last_error(), " (code ", rc, ")");
}

Tensor dev_f32(const Tensor &t, const char *name, int64_t ndim) {
    TORCH_CHECK(t.is_cuda(), name, ": the H100 path needs a CUDA tensor (got ", t.device(), "); there is no CPU fallback");
    TORCH_CHECK(t.scalar_type() == at::kFloat, name, ": expected float32, got ", t.scalar_type());
    TORCH_CHECK(t.dim() == ndim, name, ": expected ", ndim, " dims, got ", t.dim());
    return t.contiguous();
}

void *stream_of(const Tensor &t) { return c10::cuda::getCurrentCUDAStream(t.get_device()).stream(); }

// raw offset-conv output, consumed in place in planar NCHW or channels-last memory
Tensor offsets_arg(const Tensor &off, int64_t B, int64_t K, int64_t H, int64_t W, const char *name, int *channels_last) {
    TORCH_CHECK(off.is_cuda() && off.scalar_type() == at::kFloat, name, ": offsets must be a CUDA float32 tensor");
    TORCH_CHECK(off.dim() == 4 && off.size(0) == B && off.size(1) == 2 * K && off.size(2) == H && off.size(3) == W,
                name, ": offsets must be [B,2K,H,W]");
    if (off.is_contiguous()) { *channels_last = 0; return off; }
    if (off.is_contiguous(at::MemoryFormat::ChannelsLast)) { *channels_last = 1; return off; }
    *channels_last = 0;
    return off.contiguous();
}

// A scripted module keeps its packed / folded filters as CPU tensors (state-dict keys stay the reference's).  Uploading them
// on every forward is an implicit host sync from pageable memory and makes the scripted model impossible to capture in a CUDA
// graph, so device copies are cached per (source storage, version, device).  The cache holds the SOURCE tensor too: its address
// cannot be recycled for other contents while the entry lives.  Bounded: a scripted PatchmatchNet holds about 50 such tensors
// (filters and biases of FeatureNet, Refinement and the offset convs), so 512 entries serve several devices without eviction.
Tensor device_copy_cached(const Tensor &t, const c10::Device &dev) {
    if (t.device() == dev) return t.contiguous();
    struct Entry { Tensor src, copy; };
    static std::mutex mu;
    static auto *cache = new std::map<std::tuple<const void *, int64_t, int>, Entry>();  // never destroyed: outlives the CUDA context
    const auto key = std::make_tuple(static_cast<const void *>(t.data_ptr()), (int64_t)t._version(), (int)dev.index());
    std::lock_guard<std::mutex> lock(mu);
    auto it = cache->find(key);
    if (it != cache->end() && it->second.src.numel() == t.numel()) return it->second.copy;
    if (cache->size() >= 512) cache->clear();
    Entry e{t, t.to(dev)};  // memory format preserved: ATen's convolutions get the folded filter in the layout eager hands them
    (*cache)[key] = e;
    return e.copy;
}

// BatchNorm-folded G->16->8->1 head as the flat float image of `pmb200_mlp` (host memory)
struct Head {
    Tensor keep;
    const pmb200_mlp *ptr;
    explicit Head(const Tensor &h) {
        keep = h.to(at::kCPU, at::kFloat).contiguous();
        TORCH_CHECK(keep.numel() == (int64_t)(sizeof(pmb200_mlp) / sizeof(float)),
                    "head: expected ", sizeof(pmb200_mlp) / sizeof(float), " floats (the image of pmb200_mlp)");
        ptr = reinterpret_cast<const pmb200_mlp *>(keep.data_ptr<float>());
    }
};

struct WarpShape {
    int V, B, C, H, W, Hs, Ws, D;
};

WarpShape warp_shape(const Tensor &ref, const Tensor &src, const Tensor &rt, const Tensor &depth) {
    WarpShape s;
    s.B = (int)ref.size(0); s.H = (int)ref.size(1); s.W = (int)ref.size(2); s.C = (int)ref.size(3);
    s.V = (int)src.size(0); s.Hs = (int)src.size(2); s.Ws = (int)src.size(3); s.D = (int)depth.size(1);
    TORCH_CHECK(src.size(1) == s.B && src.size(4) == s.C && rt.size(0) == s.V && rt.size(1) == s.B && rt.size(2) == 12 &&
                    depth.size(0) == s.B && depth.size(2) == s.H && depth.size(3) == s.W,
                "warp_corr: inconsistent shapes");
    return s;
}

void check_xs(const Tensor &xs, int64_t B, int64_t D, int64_t H, int64_t W) {
    TORCH_CHECK(xs.is_cuda() && xs.scalar_type() == at::kFloat && xs.is_contiguous() && xs.dim() == 5 && xs.size(0) == B &&
                    xs.size(1) == D && xs.size(2) == H && xs.size(3) == W && xs.size(4) == 2,
                "xs must be a contiguous CUDA float32 [B,D,H,W,2] buffer");
}

// ---- reference module.py:148-150 --------------------------------------------------------------
Tensor relative_projection(const Tensor &ref_proj, at::TensorList src_projs) {
    TORCH_CHECK(ref_proj.is_cuda() && ref_proj.scalar_type() == at::kFloat && ref_proj.dim() == 3 && ref_proj.size(1) == 4 &&
                    ref_proj.size(2) == 4, "ref_proj: expected a CUDA float32 [B,4,4] tensor");
    const int64_t B = ref_proj.size(0), V = (int64_t)src_projs.size();
    TORCH_CHECK(V >= 1, "relative_projection: no source views");
    const Tensor ref = ref_proj.contiguous();
    std::vector<Tensor> mats;
    std::vector<const float *> ptrs;
    for (const Tensor &m : src_projs) {
        TORCH_CHECK(m.is_cuda() && m.scalar_type() == at::kFloat && m.dim() == 3 && m.size(0) == B && m.size(1) == 4 &&
                        m.size(2) == 4, "src_proj: expected a CUDA float32 [B,4,4] tensor");
        mats.push_back(m.contiguous());
        ptrs.push_back(mats.back().data_ptr<float>());
    }
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor out = at::empty({V, B, 12}, ref.options());
    check(pmb200_relative_projection(ref.data_ptr<float>(), 16, ptrs.data(), 16, (int)V, (int)B, out.data_ptr<float>(),
                                     stream_of(ref)),
          "relative_projection");
    return out;
}

// [n,B,H,W,C] channels-last pack; zero-copy when the maps already are back-to-back channels-last slices of one storage
Tensor pack_nhwc(at::TensorList maps) {
    TORCH_CHECK(!maps.empty(), "pack_nhwc: no maps");
    const Tensor &first = maps[0];
    TORCH_CHECK(first.is_cuda() && first.scalar_type() == at::kFloat && first.dim() == 4,
                "pack_nhwc: expected CUDA float32 [B,C,H,W] maps; there is no CPU fallback");
    const int64_t n = (int64_t)maps.size(), B = first.size(0), C = first.size(1), H = first.size(2), W = first.size(3);
    bool packed = (reinterpret_cast<uintptr_t>(first.data_ptr()) % 32) == 0;
    for (int64_t i = 0; i < n && packed; ++i) {
        const Tensor &m = maps[i];
        packed = m.sizes() == first.sizes() && m.stride(0) == H * W * C && m.stride(1) == 1 && m.stride(2) == W * C &&
                 m.stride(3) == C && m.storage().data() == first.storage().data() &&
                 m.storage_offset() == first.storage_offset() + i * first.numel();
    }
    if (packed) return first.as_strided({n, B, H, W, C}, {B * H * W * C, H * W * C, W * C, C, 1});
    std::vector<Tensor> keep;
    std::vector<const float *> ptrs;
    for (const Tensor &m : maps) {
        TORCH_CHECK(m.sizes() == first.sizes() && m.is_cuda() && m.scalar_type() == at::kFloat,
                    "pack_nhwc: maps must share one shape, dtype and device");
        keep.push_back(m.contiguous());
        ptrs.push_back(keep.back().data_ptr<float>());
    }
    c10::cuda::CUDAGuard guard(first.device());
    Tensor out = at::empty({n, B, H, W, C}, first.options().memory_format(at::MemoryFormat::Contiguous));
    check(pmb200_pack_nhwc(ptrs.data(), (int)n, (int)B, (int)C, (int)H, (int)W, out.data_ptr<float>(), stream_of(first)),
          "pack_nhwc");
    return out;
}

// ---- K-A: reference module.py:130-181 + patchmatch.py:192-217 -------------------------------------
Tensor warp_corr(const Tensor &ref_nhwc, const Tensor &src_nhwc, const Tensor &rt_, const Tensor &depth_,
                 const c10::optional<Tensor> &view_weights, int64_t G) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), src = dev_f32(src_nhwc, "src_nhwc", 5);
    const Tensor rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const WarpShape s = warp_shape(ref, src, rt, depth);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor vw, out;
    if (view_weights.has_value() && view_weights->numel() > 0) {
        vw = dev_f32(*view_weights, "view_weights", 4);
        TORCH_CHECK(vw.size(0) == s.B && vw.size(1) == s.V && vw.size(2) == s.H && vw.size(3) == s.W,
                    "warp_corr: view_weights must be [B,V,H,W]");
        out = at::empty({s.B, G, s.D, s.H, s.W}, ref.options());
    } else {
        out = at::empty({s.V, s.B, G, s.D, s.H, s.W}, ref.options());
    }
    check(pmb200_warp_corr(ref.data_ptr<float>(), src.data_ptr<float>(), rt.data_ptr<float>(), depth.data_ptr<float>(),
                           vw.defined() ? vw.data_ptr<float>() : nullptr, out.data_ptr<float>(), s.V, s.B, s.C, (int)G,
                           s.H, s.W, s.Hs, s.Ws, s.D, stream_of(ref)),
          "warp_corr");
    return out;
}

Tensor aggregate_views(const Tensor &sims_, const Tensor &view_weights) {
    const Tensor sims = dev_f32(sims_, "sims", 6), vw = dev_f32(view_weights, "view_weights", 4);
    const int64_t V = sims.size(0), B = sims.size(1), G = sims.size(2), D = sims.size(3), H = sims.size(4), W = sims.size(5);
    TORCH_CHECK(vw.size(0) == B && vw.size(1) == V && vw.size(2) == H && vw.size(3) == W,
                "aggregate_views: view_weights must be [B,V,H,W]");
    c10::cuda::CUDAGuard guard(sims.device());
    Tensor out = at::empty({B, G, D, H, W}, sims.options());
    check(pmb200_aggregate_views(sims.data_ptr<float>(), vw.data_ptr<float>(), out.data_ptr<float>(), (int)V, (int)B, (int)G,
                                 (int)D, (int)H, (int)W, stream_of(sims)),
          "aggregate_views");
    return out;
}

// K-A + PixelwiseNet (eval): -> (view weights [B,V,H,W], per-view similarities [V,B,G,D,H,W])
std::tuple<Tensor, Tensor> warp_corr_view_weights(const Tensor &ref_nhwc, const Tensor &src_nhwc, const Tensor &rt_,
                                                  const Tensor &depth_, const Tensor &head, int64_t G) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), src = dev_f32(src_nhwc, "src_nhwc", 5);
    const Tensor rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const WarpShape s = warp_shape(ref, src, rt, depth);
    const Head h(head);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor vw = at::empty({s.B, s.V, s.H, s.W}, ref.options());
    Tensor sims = at::empty({s.V, s.B, G, s.D, s.H, s.W}, ref.options());
    check(pmb200_warp_corr_view_weights(ref.data_ptr<float>(), src.data_ptr<float>(), rt.data_ptr<float>(),
                                        depth.data_ptr<float>(), h.ptr, vw.data_ptr<float>(), sims.data_ptr<float>(), s.V, s.B,
                                        s.C, (int)G, s.H, s.W, s.Hs, s.Ws, s.D, stream_of(ref)),
          "warp_corr_view_weights");
    return std::make_tuple(vw, sims);
}

// K-A + SimilarityNet (eval): raw score into the .y lanes of the interleaved (xnorm, score) buffer
void warp_corr_score_(const Tensor &ref_nhwc, const Tensor &src_nhwc, const Tensor &rt_, const Tensor &depth_,
                      const Tensor &view_weights, const Tensor &head, int64_t G, Tensor &xs) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), src = dev_f32(src_nhwc, "src_nhwc", 5);
    const Tensor rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const WarpShape s = warp_shape(ref, src, rt, depth);
    const Tensor vw = dev_f32(view_weights, "view_weights", 4);
    TORCH_CHECK(vw.size(0) == s.B && vw.size(1) == s.V && vw.size(2) == s.H && vw.size(3) == s.W,
                "warp_corr_score: view_weights must be [B,V,H,W]");
    check_xs(xs, s.B, s.D, s.H, s.W);
    const Head h(head);
    c10::cuda::CUDAGuard guard(ref.device());
    check(pmb200_warp_corr_score(ref.data_ptr<float>(), src.data_ptr<float>(), rt.data_ptr<float>(), depth.data_ptr<float>(),
                                 vw.data_ptr<float>(), h.ptr, xs.data_ptr<float>() + 1, 2, s.V, s.B, s.C, (int)G, s.H, s.W,
                                 s.Hs, s.Ws, s.D, stream_of(ref)),
          "warp_corr_score");
}

void aggregate_views_score_(const Tensor &sims_, const Tensor &view_weights, const Tensor &head, Tensor &xs) {
    const Tensor sims = dev_f32(sims_, "sims", 6), vw = dev_f32(view_weights, "view_weights", 4);
    const int64_t V = sims.size(0), B = sims.size(1), G = sims.size(2), D = sims.size(3), H = sims.size(4), W = sims.size(5);
    TORCH_CHECK(vw.size(0) == B && vw.size(1) == V && vw.size(2) == H && vw.size(3) == W,
                "aggregate_views_score: view_weights must be [B,V,H,W]");
    check_xs(xs, B, D, H, W);
    const Head h(head);
    c10::cuda::CUDAGuard guard(sims.device());
    check(pmb200_aggregate_views_score(sims.data_ptr<float>(), vw.data_ptr<float>(), h.ptr, xs.data_ptr<float>() + 1, 2, (int)V,
                                       (int)B, (int)G, (int)D, (int)H, (int)W, stream_of(sims)),
          "aggregate_views_score");
}

// ---- K-A': reference patchmatch.py:361-426, 613-624 -------------------------------------------------
Tensor offset_corr(const Tensor &ref_nhwc, const Tensor &offsets, int64_t G, int64_t K, int64_t dilation) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4);
    const int64_t B = ref.size(0), H = ref.size(1), W = ref.size(2), C = ref.size(3);
    int cl = 0;
    const Tensor off = offsets_arg(offsets, B, K, H, W, "offset_corr", &cl);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor out = at::empty({B, G, K, H, W}, ref.options());
    check(pmb200_offset_corr(ref.data_ptr<float>(), off.data_ptr<float>(), cl, out.data_ptr<float>(), (int)B, (int)C, (int)G,
                             (int)H, (int)W, (int)K, (int)dilation, stream_of(ref)),
          "offset_corr");
    return out;
}

Tensor offset_corr_weight(const Tensor &ref_nhwc, const Tensor &offsets, const Tensor &head, int64_t G, int64_t K,
                          int64_t dilation) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4);
    const int64_t B = ref.size(0), H = ref.size(1), W = ref.size(2), C = ref.size(3);
    int cl = 0;
    const Tensor off = offsets_arg(offsets, B, K, H, W, "offset_corr_weight", &cl);
    const Head h(head);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor out = at::empty({B, K, H, W}, ref.options());
    check(pmb200_offset_corr_weight(ref.data_ptr<float>(), off.data_ptr<float>(), cl, h.ptr, out.data_ptr<float>(), (int)B,
                                    (int)C, (int)G, (int)H, (int)W, (int)K, (int)dilation, stream_of(ref)),
          "offset_corr_weight");
    return out;
}

// ---- K-C: reference patchmatch.py:53-124 ------------------------------------------------------------
// -> (hypotheses [B,Ns+Kp,H,W] ascending when Kp > 0, interleaved buffer [B,Ns+Kp,H,W,2] with the normalised inverse
//     depth in its .x lanes; the .y lanes are for the score epilogues)
std::tuple<Tensor, Tensor> init_propagate(const Tensor &seed_map, const c10::optional<Tensor> &offsets,
                                          const Tensor &depth_min, const Tensor &depth_max, int64_t mode, int64_t Ns,
                                          int64_t Kp, int64_t dilation, double interval_scale) {
    const Tensor seed = dev_f32(seed_map, "seed_map", 4);
    const int64_t B = seed.size(0), S = seed.size(1), H = seed.size(2), W = seed.size(3);
    TORCH_CHECK(S == (mode == 0 ? 48 : 1), "init_propagate: seed_map has the wrong number of channels");
    const Tensor dmin = dev_f32(depth_min.reshape({-1}), "depth_min", 1), dmax = dev_f32(depth_max.reshape({-1}), "depth_max", 1);
    TORCH_CHECK(dmin.numel() == B && dmax.numel() == B, "init_propagate: depth_min/max must have B elements");
    Tensor off;
    int cl = 0;
    if (Kp > 0) {
        TORCH_CHECK(offsets.has_value(), "init_propagate: propagation offsets missing");
        off = offsets_arg(*offsets, B, Kp, H, W, "init_propagate", &cl);
    }
    c10::cuda::CUDAGuard guard(seed.device());
    Tensor out = at::empty({B, Ns + Kp, H, W}, seed.options());
    Tensor xs = at::empty({B, Ns + Kp, H, W, 2}, seed.options());
    check(pmb200_init_propagate(seed.data_ptr<float>(), off.defined() ? off.data_ptr<float>() : nullptr, cl,
                                dmin.data_ptr<float>(), dmax.data_ptr<float>(), out.data_ptr<float>(), xs.data_ptr<float>(), 2,
                                (int)mode, (int)B, (int)H, (int)W, (int)Ns, (int)Kp, (int)dilation, (float)interval_scale,
                                stream_of(seed)),
          "init_propagate");
    return std::make_tuple(out, xs);
}

// ---- K-B: reference patchmatch.py:502-510, 569-577, 219-237, 650-669 ----------------------------------
// xs = interleaved (normalised inverse depth, raw score) [B,D,H,W,2] -> (depth [B,H,W], probability [B,D,H,W])
std::tuple<Tensor, Tensor> adaptive_eval(const Tensor &xs, const Tensor &depth_sample, const Tensor &offsets,
                                         const Tensor &feature_weight, const Tensor &depth_min, const Tensor &depth_max,
                                         int64_t dilation, double interval_scale, bool is_inverse) {
    const Tensor ds = dev_f32(depth_sample, "depth_sample", 4), fw = dev_f32(feature_weight, "feature_weight", 4);
    const int64_t B = ds.size(0), D = ds.size(1), H = ds.size(2), W = ds.size(3), K = fw.size(1);
    check_xs(xs, B, D, H, W);
    TORCH_CHECK(fw.size(0) == B && fw.size(2) == H && fw.size(3) == W, "adaptive_eval: inconsistent shapes");
    int cl = 0;
    const Tensor off = offsets_arg(offsets, B, K, H, W, "adaptive_eval", &cl);
    const Tensor dmin = dev_f32(depth_min.reshape({-1}), "depth_min", 1), dmax = dev_f32(depth_max.reshape({-1}), "depth_max", 1);
    c10::cuda::CUDAGuard guard(ds.device());
    Tensor prob = at::empty({B, D, H, W}, ds.options()), depth = at::empty({B, H, W}, ds.options());
    check(pmb200_adaptive_eval(nullptr, ds.data_ptr<float>(), nullptr, xs.data_ptr<float>(), off.data_ptr<float>(), cl,
                               fw.data_ptr<float>(), dmin.data_ptr<float>(), dmax.data_ptr<float>(), prob.data_ptr<float>(),
                               depth.data_ptr<float>(), (int)B, (int)D, (int)H, (int)W, (int)K, (int)dilation,
                               (float)interval_scale, is_inverse ? 1 : 0, stream_of(ds)),
          "adaptive_eval");
    return std::make_tuple(depth, prob);
}

// same, from separate raw score / normalised inverse depth maps (the unfused configuration)
std::tuple<Tensor, Tensor> adaptive_eval_planar(const Tensor &score0, const Tensor &xnorm, const Tensor &depth_sample,
                                                const Tensor &offsets, const Tensor &feature_weight, const Tensor &depth_min,
                                                const Tensor &depth_max, int64_t dilation, double interval_scale,
                                                bool is_inverse) {
    const Tensor sc = dev_f32(score0, "score0", 4), xn = dev_f32(xnorm, "xnorm", 4);
    const Tensor ds = dev_f32(depth_sample, "depth_sample", 4), fw = dev_f32(feature_weight, "feature_weight", 4);
    const int64_t B = ds.size(0), D = ds.size(1), H = ds.size(2), W = ds.size(3), K = fw.size(1);
    TORCH_CHECK(sc.sizes() == ds.sizes() && xn.sizes() == ds.sizes() && fw.size(0) == B && fw.size(2) == H && fw.size(3) == W,
                "adaptive_eval: inconsistent shapes");
    int cl = 0;
    const Tensor off = offsets_arg(offsets, B, K, H, W, "adaptive_eval", &cl);
    const Tensor dmin = dev_f32(depth_min.reshape({-1}), "depth_min", 1), dmax = dev_f32(depth_max.reshape({-1}), "depth_max", 1);
    c10::cuda::CUDAGuard guard(ds.device());
    Tensor prob = at::empty({B, D, H, W}, ds.options()), depth = at::empty({B, H, W}, ds.options());
    check(pmb200_adaptive_eval(sc.data_ptr<float>(), ds.data_ptr<float>(), xn.data_ptr<float>(), nullptr, off.data_ptr<float>(),
                               cl, fw.data_ptr<float>(), dmin.data_ptr<float>(), dmax.data_ptr<float>(), prob.data_ptr<float>(),
                               depth.data_ptr<float>(), (int)B, (int)D, (int)H, (int)W, (int)K, (int)dilation,
                               (float)interval_scale, is_inverse ? 1 : 0, stream_of(ds)),
          "adaptive_eval");
    return std::make_tuple(depth, prob);
}

// reference net.py:289-299
Tensor photometric_confidence(const Tensor &prob, int64_t out_h, int64_t out_w) {
    const Tensor pr = dev_f32(prob, "prob", 4);
    c10::cuda::CUDAGuard guard(pr.device());
    Tensor out = at::empty({pr.size(0), out_h, out_w}, pr.options());
    check(pmb200_photometric_confidence(pr.data_ptr<float>(), out.data_ptr<float>(), (int)pr.size(0), (int)pr.size(1),
                                        (int)pr.size(2), (int)pr.size(3), (int)out_h, (int)out_w, stream_of(pr)),
          "photometric_confidence");
    return out;
}

// reference patchmatch.py:288-311 (propa_conv / eval_conv) -- the channels-last tensor-core conv of csrc/pm_conv.cu.
// x: logical [N,Cin,H,W] (made channels-last if it is not); filter_frag: the fragment-ordered filter
// (patchmatchnet_b200.ops.pack_conv_filter), moved to x's device when the scripted module holds it on the CPU;
// -> logical [N,cout,Ho,Wo] in channels-last memory, which the fused kernels consume in place.
Tensor conv2d_nhwc(const Tensor &x, const Tensor &filter_frag, const c10::optional<Tensor> &bias, int64_t cout, int64_t ks,
                   int64_t stride, int64_t pad, int64_t dil, bool relu, int64_t precision) {
    TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kFloat && x.dim() == 4,
                "conv2d_nhwc: x must be a 4-D CUDA float32 tensor; there is no CPU fallback");
    const Tensor xc = x.contiguous(at::MemoryFormat::ChannelsLast);
    const int64_t N = xc.size(0), cin = xc.size(1), H = xc.size(2), W = xc.size(3);
    const int want = pmb200_conv2d_filter_floats((int)cin, (int)cout, (int)ks, (int)precision);
    TORCH_CHECK(want > 0 && filter_frag.scalar_type() == at::kFloat && filter_frag.numel() == want,
                "conv2d_nhwc: filter must be ", want, " float32 values in fragment order for this precision (pack_conv_filter)");
    c10::cuda::CUDAGuard guard(xc.device());
    const Tensor frag = device_copy_cached(filter_frag, xc.device());
    Tensor b;
    const float *b_ptr = nullptr;
    if (bias.has_value() && bias->defined()) {
        b = bias->to(xc.device(), at::kFloat).contiguous();
        TORCH_CHECK(b.numel() == cout, "conv2d_nhwc: bias must have Cout elements");
        b_ptr = b.data_ptr<float>();
    }
    const int64_t Ho = (H + 2 * pad - dil * (ks - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (ks - 1) - 1) / stride + 1;
    TORCH_CHECK(Ho >= 1 && Wo >= 1, "conv2d_nhwc: empty output");
    Tensor out = at::empty({N, cout, Ho, Wo}, xc.options().memory_format(at::MemoryFormat::ChannelsLast));
    check(pmb200_conv2d_nhwc(xc.data_ptr<float>(), frag.data_ptr<float>(), b_ptr, nullptr, out.data_ptr<float>(), (int)N, (int)H, (int)W,
                             (int)cin, (int)cout, (int)ks, (int)stride, (int)pad, (int)dil, relu ? 1 : 0, (int)precision, 0, 0, 0,
                             0, stream_of(xc)),
          "conv2d_nhwc");
    return out;
}

// ---- the rest of the eval-mode network (reference models/net.py): what a scripted PatchmatchNet calls --------------------------

// optional [cout] bias on x's device (a scripted module may hold a folded bias on the CPU: cached like the filters)
const float *bias_arg(const c10::optional<Tensor> &bias, int64_t cout, const c10::Device &dev, Tensor &keep, const char *name) {
    if (!bias.has_value() || !bias->defined()) return nullptr;
    TORCH_CHECK(bias->scalar_type() == at::kFloat && bias->numel() == cout, name, ": bias must have Cout float32 elements");
    keep = device_copy_cached(*bias, dev);
    return keep.data_ptr<float>();
}

// `out`: channels-last CUDA float32 [N,C,Ho,Wo] with C >= out_channel_offset + cout
void check_conv_out(const Tensor &out, const Tensor &x, int64_t Ho, int64_t Wo, int64_t cout, int64_t offset, const char *name) {
    TORCH_CHECK(out.is_cuda() && out.scalar_type() == at::kFloat && out.dim() == 4 && out.device() == x.device() &&
                    out.size(0) == x.size(0) && out.size(2) == Ho && out.size(3) == Wo &&
                    out.is_contiguous(at::MemoryFormat::ChannelsLast),
                name, ": out must be a channels-last CUDA float32 [N,C,", Ho, ",", Wo, "] tensor on x's device");
    TORCH_CHECK(offset >= 0 && offset + cout <= out.size(1), name, ": channels ", offset, "..", offset + cout,
                " do not fit in out's ", out.size(1));
}

Tensor conv_x(const Tensor &x, const char *name) {
    TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kFloat && x.dim() == 4,
                name, ": x must be a 4-D CUDA float32 tensor; there is no CPU fallback");
    return x.contiguous(at::MemoryFormat::ChannelsLast);
}

// conv2d_nhwc with every argument of pmb200_conv2d_nhwc: the bilinear x2 upsample-add epilogue (FeatureNet's top-down path),
// the zero-stuffed transposed form (Refinement's ConvTranspose2d) and a channel window of a wider `out` (concat fusion)
void conv2d_nhwc_out(const Tensor &x, const Tensor &filter_frag, const c10::optional<Tensor> &bias, int64_t cout, int64_t ks,
                     int64_t stride, int64_t pad, int64_t dil, bool relu, int64_t precision, bool transposed2x,
                     const c10::optional<Tensor> &add_up2x, Tensor &out, int64_t out_channel_offset) {
    const Tensor xc = conv_x(x, "conv2d_nhwc_out");
    const int64_t N = xc.size(0), cin = xc.size(1), H = xc.size(2), W = xc.size(3);
    const int want = pmb200_conv2d_filter_floats((int)cin, (int)cout, (int)ks, (int)precision);
    TORCH_CHECK(want > 0 && filter_frag.scalar_type() == at::kFloat && filter_frag.numel() == want,
                "conv2d_nhwc_out: filter must be ", want, " float32 values in fragment order for this precision (pack_conv_filter)");
    const int64_t Hv = transposed2x ? 2 * H : H, Wv = transposed2x ? 2 * W : W;
    const int64_t Ho = (Hv + 2 * pad - dil * (ks - 1) - 1) / stride + 1, Wo = (Wv + 2 * pad - dil * (ks - 1) - 1) / stride + 1;
    TORCH_CHECK(Ho >= 1 && Wo >= 1, "conv2d_nhwc_out: empty output");
    check_conv_out(out, xc, Ho, Wo, cout, out_channel_offset, "conv2d_nhwc_out");
    const float *up_ptr = nullptr;
    if (add_up2x.has_value() && add_up2x->defined()) {
        const Tensor &u = *add_up2x;
        TORCH_CHECK(u.is_cuda() && u.scalar_type() == at::kFloat && u.dim() == 4 && u.is_contiguous(at::MemoryFormat::ChannelsLast),
                    "conv2d_nhwc_out: add_up2x must be a channels-last CUDA float32 tensor");
        TORCH_CHECK(u.size(0) == N && u.size(1) == cout && u.size(2) == Ho / 2 && u.size(3) == Wo / 2,
                    "conv2d_nhwc_out: add_up2x must be [N,cout,Ho/2,Wo/2]");
        up_ptr = u.data_ptr<float>();
    }
    c10::cuda::CUDAGuard guard(xc.device());
    const Tensor frag = device_copy_cached(filter_frag, xc.device());
    Tensor b;
    const float *b_ptr = bias_arg(bias, cout, xc.device(), b, "conv2d_nhwc_out");
    check(pmb200_conv2d_nhwc(xc.data_ptr<float>(), frag.data_ptr<float>(), b_ptr, up_ptr, out.data_ptr<float>(), (int)N, (int)H, (int)W,
                             (int)cin, (int)cout, (int)ks, (int)stride, (int)pad, (int)dil, relu ? 1 : 0, (int)precision,
                             transposed2x ? 1 : 0, (int)out.size(1), (int)out_channel_offset, 0, stream_of(xc)),
          "conv2d_nhwc_out");
}

// K-D5 / K-D5h (csrc/pm_conv5.cu): the wgmma convolution, tap form (any stride) or halo-tile form (halo = true, stride 1)
void conv2d_tc5_out(const Tensor &x, const Tensor &filter_tc5, const c10::optional<Tensor> &bias, int64_t cout, int64_t ks,
                    int64_t stride, int64_t pad, int64_t dil, bool relu, bool halo, Tensor &out, int64_t out_channel_offset) {
    TORCH_CHECK(!halo || stride == 1, "conv2d_tc5: the halo-tile form serves stride 1");
    const Tensor xc = conv_x(x, "conv2d_tc5");
    const int64_t N = xc.size(0), cin = xc.size(1), H = xc.size(2), W = xc.size(3);
    const int want = pmb200_conv2d_tc5_filter_floats((int)cin, (int)cout, (int)ks);
    TORCH_CHECK(want > 0 && filter_tc5.scalar_type() == at::kFloat && filter_tc5.numel() == want,
                "conv2d_tc5: filter must be ", want, " float32 values (pack_conv_filter_tc5 / pack_conv_filter_tc5h)");
    const int64_t Ho = (H + 2 * pad - dil * (ks - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (ks - 1) - 1) / stride + 1;
    TORCH_CHECK(Ho >= 1 && Wo >= 1, "conv2d_tc5: empty output");
    check_conv_out(out, xc, Ho, Wo, cout, out_channel_offset, "conv2d_tc5");
    c10::cuda::CUDAGuard guard(xc.device());
    const Tensor filt = device_copy_cached(filter_tc5, xc.device());
    Tensor b;
    const float *b_ptr = bias_arg(bias, cout, xc.device(), b, "conv2d_tc5");
    if (halo) {
        check(pmb200_conv2d_tc5h(xc.data_ptr<float>(), filt.data_ptr<float>(), b_ptr, out.data_ptr<float>(), (int)N, (int)H, (int)W,
                                 (int)cin, (int)cout, (int)ks, (int)pad, (int)dil, relu ? 1 : 0, (int)out.size(1),
                                 (int)out_channel_offset, stream_of(xc)),
              "conv2d_tc5h");
    } else {
        check(pmb200_conv2d_tc5(xc.data_ptr<float>(), filt.data_ptr<float>(), b_ptr, out.data_ptr<float>(), (int)N, (int)H, (int)W,
                                (int)cin, (int)cout, (int)ks, (int)stride, (int)pad, (int)dil, relu ? 1 : 0, (int)out.size(1),
                                (int)out_channel_offset, stream_of(xc)),
              "conv2d_tc5");
    }
}

Tensor conv2d_tc5(const Tensor &x, const Tensor &filter_tc5, const c10::optional<Tensor> &bias, int64_t cout, int64_t ks,
                  int64_t stride, int64_t pad, int64_t dil, bool relu, bool halo) {
    TORCH_CHECK(x.is_cuda() && x.dim() == 4, "conv2d_tc5: x must be a 4-D CUDA float32 tensor; there is no CPU fallback");
    const int64_t Ho = (x.size(2) + 2 * pad - dil * (ks - 1) - 1) / stride + 1, Wo = (x.size(3) + 2 * pad - dil * (ks - 1) - 1) / stride + 1;
    TORCH_CHECK(Ho >= 1 && Wo >= 1 && stride >= 1, "conv2d_tc5: empty output");
    Tensor out = at::empty({x.size(0), cout, Ho, Wo}, x.options().dtype(at::kFloat).memory_format(at::MemoryFormat::ChannelsLast));
    conv2d_tc5_out(x, filter_tc5, bias, cout, ks, stride, pad, dil, relu, halo, out, 0);
    return out;
}

// host weights of K-S / K-R: they travel in the kernel parameter block, so they must be contiguous float32 CPU tensors
const float *host_arg(const Tensor &t, std::initializer_list<int64_t> shape, const char *what, const char *name) {
    TORCH_CHECK(t.device().is_cpu() && t.scalar_type() == at::kFloat && t.is_contiguous() && t.sizes() == at::IntArrayRef(shape),
                what, ": ", name, " must be a contiguous float32 HOST tensor of shape ", at::IntArrayRef(shape));
    return t.data_ptr<float>();
}

Tensor per_image(const Tensor &t, int64_t N, const char *what, const char *name) {
    const Tensor r = dev_f32(t.reshape({-1}), name, 1);
    TORCH_CHECK(r.numel() == N, what, ": ", name, " must have one value per image");
    return r;
}

// K-S: relu(conv1(relu(conv0(x)))) of FeatureNet (reference models/net.py:18-19, :44) -> [N,8,H,W] channels-last
Tensor conv_stem(const Tensor &x_, const Tensor &w0, const Tensor &b0, const Tensor &w1, const Tensor &b1) {
    TORCH_CHECK(x_.is_cuda() && x_.scalar_type() == at::kFloat && x_.dim() == 4 && x_.size(1) == 3,
                "conv_stem: x must be a CUDA float32 [N,3,H,W] tensor; there is no CPU fallback");
    const Tensor x = x_.contiguous();
    const float *pw0 = host_arg(w0, {8, 3, 3, 3}, "conv_stem", "w0"), *pb0 = host_arg(b0, {8}, "conv_stem", "b0");
    const float *pw1 = host_arg(w1, {8, 8, 3, 3}, "conv_stem", "w1"), *pb1 = host_arg(b1, {8}, "conv_stem", "b1");
    c10::cuda::CUDAGuard guard(x.device());
    Tensor y = at::empty({x.size(0), 8, x.size(2), x.size(3)}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    check(pmb200_conv_stem(x.data_ptr<float>(), pw0, pb0, pw1, pb1, y.data_ptr<float>(), (int)x.size(0), (int)x.size(2),
                           (int)x.size(3), stream_of(x)),
          "conv_stem");
    return y;
}

// K-R, half resolution (reference models/net.py:104-110) -> [N,8,h,w] channels-last
Tensor refine_low(const Tensor &depth_half, const Tensor &depth_min, const Tensor &depth_max, const Tensor &w1, const Tensor &b1,
                  const Tensor &w2, const Tensor &b2) {
    const Tensor dh = dev_f32(depth_half, "depth_half", 4);
    TORCH_CHECK(dh.size(1) == 1, "refine_low: depth_half must be [N,1,h,w]");
    const int64_t N = dh.size(0), h = dh.size(2), w = dh.size(3);
    const Tensor lo = per_image(depth_min, N, "refine_low", "depth_min"), hi = per_image(depth_max, N, "refine_low", "depth_max");
    const float *pw1 = host_arg(w1, {8, 1, 3, 3}, "refine_low", "w1"), *pb1 = host_arg(b1, {8}, "refine_low", "b1");
    const float *pw2 = host_arg(w2, {8, 8, 3, 3}, "refine_low", "w2"), *pb2 = host_arg(b2, {8}, "refine_low", "b2");
    c10::cuda::CUDAGuard guard(dh.device());
    Tensor y = at::empty({N, 8, h, w}, dh.options().memory_format(at::MemoryFormat::ChannelsLast));
    check(pmb200_refine_low(dh.data_ptr<float>(), lo.data_ptr<float>(), hi.data_ptr<float>(), pw1, pb1, pw2, pb2, y.data_ptr<float>(),
                            (int)N, (int)h, (int)w, stream_of(dh)),
          "refine_low");
    return y;
}

// K-R, full resolution (reference models/net.py:103, :112-120) -> depth [N,1,2h,2w]
Tensor refine_full(const Tensor &low, const Tensor &img_, const Tensor &depth_half, const Tensor &depth_min, const Tensor &depth_max,
                   const Tensor &wd, const Tensor &bd, const Tensor &w0, const Tensor &b0, const Tensor &w3, const Tensor &b3,
                   const Tensor &wr) {
    TORCH_CHECK(low.is_cuda() && low.scalar_type() == at::kFloat && low.dim() == 4 && low.size(1) == 8 &&
                    low.is_contiguous(at::MemoryFormat::ChannelsLast),
                "refine_full: low must be a channels-last CUDA float32 [N,8,h,w] tensor; there is no CPU fallback");
    const int64_t N = low.size(0), h = low.size(2), w = low.size(3);
    const Tensor img = dev_f32(img_, "img", 4), dh = dev_f32(depth_half, "depth_half", 4);
    TORCH_CHECK(img.size(0) == N && img.size(1) == 3 && img.size(2) == 2 * h && img.size(3) == 2 * w,
                "refine_full: img must be [", N, ",3,", 2 * h, ",", 2 * w, "]");
    TORCH_CHECK(dh.size(0) == N && dh.size(1) == 1 && dh.size(2) == h && dh.size(3) == w,
                "refine_full: depth_half must be [", N, ",1,", h, ",", w, "]");
    const Tensor lo = per_image(depth_min, N, "refine_full", "depth_min"), hi = per_image(depth_max, N, "refine_full", "depth_max");
    const float *pwd = host_arg(wd, {8, 8, 3, 3}, "refine_full", "wd"), *pbd = host_arg(bd, {8}, "refine_full", "bd");
    const float *pw0 = host_arg(w0, {8, 3, 3, 3}, "refine_full", "w0"), *pb0 = host_arg(b0, {8}, "refine_full", "b0");
    const float *pw3 = host_arg(w3, {8, 16, 3, 3}, "refine_full", "w3"), *pb3 = host_arg(b3, {8}, "refine_full", "b3");
    const float *pwr = host_arg(wr, {1, 8, 3, 3}, "refine_full", "wr");
    c10::cuda::CUDAGuard guard(low.device());
    Tensor out = at::empty({N, 1, 2 * h, 2 * w}, low.options().memory_format(at::MemoryFormat::Contiguous));
    check(pmb200_refine_full(low.data_ptr<float>(), img.data_ptr<float>(), dh.data_ptr<float>(), lo.data_ptr<float>(), hi.data_ptr<float>(),
                             pwd, pbd, pw0, pb0, pw3, pb3, pwr, out.data_ptr<float>(), (int)N, (int)(2 * h), (int)(2 * w), stream_of(low)),
          "refine_full");
    return out;
}

// bilinear x2 upsample of x plus y (plus a per-channel bias), channels-last (FeatureNet's top-down step, models/net.py:60-66)
Tensor upsample2x_add(const Tensor &x_, const Tensor &y_, const c10::optional<Tensor> &bias) {
    TORCH_CHECK(x_.is_cuda() && y_.is_cuda() && x_.scalar_type() == at::kFloat && y_.scalar_type() == at::kFloat && x_.dim() == 4 &&
                    y_.dim() == 4, "upsample2x_add: x and y must be 4-D CUDA float32 tensors; there is no CPU fallback");
    const int64_t N = x_.size(0), C = x_.size(1), h = x_.size(2), w = x_.size(3);
    TORCH_CHECK(y_.size(0) == N && y_.size(1) == C && y_.size(2) == 2 * h && y_.size(3) == 2 * w, "upsample2x_add: y must be [N,C,2h,2w]");
    const Tensor x = x_.contiguous(at::MemoryFormat::ChannelsLast), y = y_.contiguous(at::MemoryFormat::ChannelsLast);
    c10::cuda::CUDAGuard guard(x.device());
    Tensor b;
    const float *b_ptr = bias_arg(bias, C, x.device(), b, "upsample2x_add");
    Tensor out = at::empty_like(y, y.options().memory_format(at::MemoryFormat::ChannelsLast));
    check(pmb200_upsample2x_add_nhwc(x.data_ptr<float>(), y.data_ptr<float>(), b_ptr, out.data_ptr<float>(), (int)N, (int)h, (int)w, (int)C,
                                     stream_of(x)),
          "upsample2x_add_nhwc");
    return out;
}

// ---- ragged source packs: views of different sizes (the *_views entry points of K-A) --------------------------------------------
constexpr int64_t kViewAlignFloats = 64;  // every view starts on a 256-byte boundary (ops.ViewPack.ALIGN_FLOATS)

// NCHW maps [B,C,H_v,W_v] sharing B and C -> (flat channels-last data, CPU int64 [V,3] extents (offset, height, width))
std::tuple<Tensor, Tensor> pack_nhwc_views(at::TensorList maps) {
    TORCH_CHECK(!maps.empty(), "pack_nhwc_views: no maps");
    const Tensor &first = maps[0];
    TORCH_CHECK(first.is_cuda() && first.scalar_type() == at::kFloat && first.dim() == 4,
                "pack_nhwc_views: expected CUDA float32 [B,C,H,W] maps; there is no CPU fallback");
    const int64_t V = (int64_t)maps.size(), B = first.size(0), C = first.size(1);
    Tensor extents = at::empty({V, 3}, at::TensorOptions().dtype(at::kLong));
    auto e = extents.accessor<int64_t, 2>();
    int64_t total = 0;
    std::vector<Tensor> keep;
    for (int64_t v = 0; v < V; ++v) {
        const Tensor &m = maps[v];
        TORCH_CHECK(m.is_cuda() && m.scalar_type() == at::kFloat && m.dim() == 4 && m.device() == first.device() && m.size(0) == B &&
                        m.size(1) == C, "pack_nhwc_views: maps must share batch size, channels, dtype and device");
        keep.push_back(m.contiguous());
        e[v][0] = total;
        e[v][1] = m.size(2);
        e[v][2] = m.size(3);
        total += (B * m.size(2) * m.size(3) * C + kViewAlignFloats - 1) / kViewAlignFloats * kViewAlignFloats;
    }
    c10::cuda::CUDAGuard guard(first.device());
    Tensor data = at::empty({total}, first.options().memory_format(at::MemoryFormat::Contiguous));
    for (int64_t v = 0; v < V; ++v) {
        const float *ptr = keep[v].data_ptr<float>();
        check(pmb200_pack_nhwc(&ptr, 1, (int)B, (int)C, (int)e[v][1], (int)e[v][2], data.data_ptr<float>() + e[v][0], stream_of(first)),
              "pack_nhwc_views");
    }
    return std::make_tuple(data, extents);
}

struct ViewsShape {
    int V, B, C, H, W, D;
    std::vector<pmb200_view_extent> ext;
};

ViewsShape views_shape(const Tensor &ref, const Tensor &src_flat, const Tensor &extents, const Tensor &rt, const Tensor &depth) {
    TORCH_CHECK(src_flat.is_cuda() && src_flat.scalar_type() == at::kFloat && src_flat.dim() == 1 && src_flat.is_contiguous(),
                "src_flat: expected the contiguous CUDA float32 data of a view pack (pack_nhwc_views)");
    TORCH_CHECK(extents.device().is_cpu() && extents.scalar_type() == at::kLong && extents.dim() == 2 && extents.size(1) == 3,
                "extents: expected a CPU int64 [V,3] tensor of (offset, height, width) (pack_nhwc_views)");
    ViewsShape s;
    s.B = (int)ref.size(0); s.H = (int)ref.size(1); s.W = (int)ref.size(2); s.C = (int)ref.size(3);
    s.V = (int)extents.size(0); s.D = (int)depth.size(1);
    TORCH_CHECK(rt.size(0) == s.V && rt.size(1) == s.B && rt.size(2) == 12 && depth.size(0) == s.B && depth.size(2) == s.H &&
                    depth.size(3) == s.W, "warp_corr: inconsistent shapes");
    const Tensor ex = extents.contiguous();
    const int64_t *p = ex.data_ptr<int64_t>();
    for (int v = 0; v < s.V; ++v) {
        const int64_t off = p[3 * v], h = p[3 * v + 1], w = p[3 * v + 2];
        TORCH_CHECK(off >= 0 && h > 0 && w > 0 && off + (int64_t)s.B * h * w * s.C <= src_flat.numel(),
                    "warp_corr: view ", v, " (offset ", off, ", ", h, "x", w, ") does not lie inside the pack's ", src_flat.numel(), " floats");
        s.ext.push_back(pmb200_view_extent{off, (int)h, (int)w});
    }
    return s;
}

Tensor warp_corr_views(const Tensor &ref_nhwc, const Tensor &src_flat, const Tensor &extents, const Tensor &rt_, const Tensor &depth_,
                       const c10::optional<Tensor> &view_weights, int64_t G) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const ViewsShape s = views_shape(ref, src_flat, extents, rt, depth);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor vw, out;
    if (view_weights.has_value() && view_weights->numel() > 0) {
        vw = dev_f32(*view_weights, "view_weights", 4);
        TORCH_CHECK(vw.size(0) == s.B && vw.size(1) == s.V && vw.size(2) == s.H && vw.size(3) == s.W,
                    "warp_corr: view_weights must be [B,V,H,W]");
        out = at::empty({s.B, G, s.D, s.H, s.W}, ref.options());
    } else {
        out = at::empty({s.V, s.B, G, s.D, s.H, s.W}, ref.options());
    }
    check(pmb200_warp_corr_views(ref.data_ptr<float>(), src_flat.data_ptr<float>(), s.ext.data(), rt.data_ptr<float>(),
                                 depth.data_ptr<float>(), vw.defined() ? vw.data_ptr<float>() : nullptr, out.data_ptr<float>(), s.V,
                                 s.B, s.C, (int)G, s.H, s.W, s.D, stream_of(ref)),
          "warp_corr_views");
    return out;
}

std::tuple<Tensor, Tensor> warp_corr_view_weights_views(const Tensor &ref_nhwc, const Tensor &src_flat, const Tensor &extents,
                                                        const Tensor &rt_, const Tensor &depth_, const Tensor &head, int64_t G) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const ViewsShape s = views_shape(ref, src_flat, extents, rt, depth);
    const Head h(head);
    c10::cuda::CUDAGuard guard(ref.device());
    Tensor vw = at::empty({s.B, s.V, s.H, s.W}, ref.options());
    Tensor sims = at::empty({s.V, s.B, G, s.D, s.H, s.W}, ref.options());
    check(pmb200_warp_corr_view_weights_views(ref.data_ptr<float>(), src_flat.data_ptr<float>(), s.ext.data(), rt.data_ptr<float>(),
                                              depth.data_ptr<float>(), h.ptr, vw.data_ptr<float>(), sims.data_ptr<float>(), s.V, s.B,
                                              s.C, (int)G, s.H, s.W, s.D, stream_of(ref)),
          "warp_corr_view_weights_views");
    return std::make_tuple(vw, sims);
}

void warp_corr_score_views_(const Tensor &ref_nhwc, const Tensor &src_flat, const Tensor &extents, const Tensor &rt_, const Tensor &depth_,
                            const Tensor &view_weights, const Tensor &head, int64_t G, Tensor &xs) {
    const Tensor ref = dev_f32(ref_nhwc, "ref_nhwc", 4), rt = dev_f32(rt_, "rt", 3), depth = dev_f32(depth_, "depth", 4);
    const ViewsShape s = views_shape(ref, src_flat, extents, rt, depth);
    const Tensor vw = dev_f32(view_weights, "view_weights", 4);
    TORCH_CHECK(vw.size(0) == s.B && vw.size(1) == s.V && vw.size(2) == s.H && vw.size(3) == s.W,
                "warp_corr_score: view_weights must be [B,V,H,W]");
    check_xs(xs, s.B, s.D, s.H, s.W);
    const Head h(head);
    c10::cuda::CUDAGuard guard(ref.device());
    check(pmb200_warp_corr_score_views(ref.data_ptr<float>(), src_flat.data_ptr<float>(), s.ext.data(), rt.data_ptr<float>(),
                                       depth.data_ptr<float>(), vw.data_ptr<float>(), h.ptr, xs.data_ptr<float>() + 1, 2, s.V, s.B,
                                       s.C, (int)G, s.H, s.W, s.D, stream_of(ref)),
          "warp_corr_score_views");
}

// the cached device copy of a host-held tensor: the folded filters a scripted network hands to ATen's convolutions
Tensor device_copy(const Tensor &t, const Tensor &like) {
    TORCH_CHECK(like.is_cuda(), "device_copy: `like` must be a CUDA tensor");
    c10::cuda::CUDAGuard guard(like.device());
    if (t.device() == like.device()) return t;
    return device_copy_cached(t, like.device());
}

int64_t abi_version() { return pmb200_abi_version(); }

}  // namespace

TORCH_LIBRARY(pmb200, m) {
    m.def("abi_version() -> int", &abi_version);
    m.def("relative_projection(Tensor ref_proj, Tensor[] src_projs) -> Tensor");
    m.def("pack_nhwc(Tensor[] maps) -> Tensor");
    m.def("warp_corr(Tensor ref_nhwc, Tensor src_nhwc, Tensor rt, Tensor depth, Tensor? view_weights, int G) -> Tensor");
    m.def("aggregate_views(Tensor sims, Tensor view_weights) -> Tensor");
    m.def("warp_corr_view_weights(Tensor ref_nhwc, Tensor src_nhwc, Tensor rt, Tensor depth, Tensor head, int G) -> (Tensor, Tensor)");
    m.def("warp_corr_score_(Tensor ref_nhwc, Tensor src_nhwc, Tensor rt, Tensor depth, Tensor view_weights, Tensor head, int G, Tensor(a!) xs) -> ()");
    m.def("aggregate_views_score_(Tensor sims, Tensor view_weights, Tensor head, Tensor(a!) xs) -> ()");
    m.def("offset_corr(Tensor ref_nhwc, Tensor offsets, int G, int K, int dilation) -> Tensor");
    m.def("offset_corr_weight(Tensor ref_nhwc, Tensor offsets, Tensor head, int G, int K, int dilation) -> Tensor");
    m.def("init_propagate(Tensor seed_map, Tensor? offsets, Tensor depth_min, Tensor depth_max, int mode, int Ns, int Kp, int dilation, float interval_scale) -> (Tensor, Tensor)");
    m.def("adaptive_eval(Tensor xs, Tensor depth_sample, Tensor offsets, Tensor feature_weight, Tensor depth_min, Tensor depth_max, int dilation, float interval_scale, bool is_inverse) -> (Tensor, Tensor)");
    m.def("adaptive_eval_planar(Tensor score0, Tensor xnorm, Tensor depth_sample, Tensor offsets, Tensor feature_weight, Tensor depth_min, Tensor depth_max, int dilation, float interval_scale, bool is_inverse) -> (Tensor, Tensor)");
    m.def("photometric_confidence(Tensor prob, int out_h, int out_w) -> Tensor");
    m.def("conv2d_nhwc(Tensor x, Tensor filter_frag, Tensor? bias, int cout, int ks, int stride, int pad, int dil, bool relu, int precision) -> Tensor");
    m.def("conv2d_nhwc_out(Tensor x, Tensor filter_frag, Tensor? bias, int cout, int ks, int stride, int pad, int dil, bool relu, int precision, bool transposed2x, Tensor? add_up2x, Tensor(a!) out, int out_channel_offset) -> ()");
    m.def("conv2d_tc5(Tensor x, Tensor filter_tc5, Tensor? bias, int cout, int ks, int stride, int pad, int dil, bool relu, bool halo) -> Tensor");
    m.def("conv2d_tc5_out(Tensor x, Tensor filter_tc5, Tensor? bias, int cout, int ks, int stride, int pad, int dil, bool relu, bool halo, Tensor(a!) out, int out_channel_offset) -> ()");
    m.def("conv_stem(Tensor x, Tensor w0, Tensor b0, Tensor w1, Tensor b1) -> Tensor");
    m.def("refine_low(Tensor depth_half, Tensor depth_min, Tensor depth_max, Tensor w1, Tensor b1, Tensor w2, Tensor b2) -> Tensor");
    m.def("refine_full(Tensor low, Tensor img, Tensor depth_half, Tensor depth_min, Tensor depth_max, Tensor wd, Tensor bd, Tensor w0, Tensor b0, Tensor w3, Tensor b3, Tensor wr) -> Tensor");
    m.def("upsample2x_add(Tensor x, Tensor y, Tensor? bias) -> Tensor");
    m.def("pack_nhwc_views(Tensor[] maps) -> (Tensor, Tensor)");
    m.def("warp_corr_views(Tensor ref_nhwc, Tensor src_flat, Tensor extents, Tensor rt, Tensor depth, Tensor? view_weights, int G) -> Tensor");
    m.def("warp_corr_view_weights_views(Tensor ref_nhwc, Tensor src_flat, Tensor extents, Tensor rt, Tensor depth, Tensor head, int G) -> (Tensor, Tensor)");
    m.def("warp_corr_score_views_(Tensor ref_nhwc, Tensor src_flat, Tensor extents, Tensor rt, Tensor depth, Tensor view_weights, Tensor head, int G, Tensor(a!) xs) -> ()");
    m.def("device_copy(Tensor t, Tensor like) -> Tensor");
}

// CUDA is the only backend: a CPU tensor reaches no kernel and the dispatcher raises, there is no fallback.
// relative_projection / pack_nhwc / pack_nhwc_views take tensor lists, which dispatch on their first element; the ops that take
// host weights (conv_stem, refine_*, device_copy) dispatch on their CUDA arguments.
TORCH_LIBRARY_IMPL(pmb200, CUDA, m) {
    m.impl("relative_projection", &relative_projection);
    m.impl("pack_nhwc", &pack_nhwc);
    m.impl("warp_corr", &warp_corr);
    m.impl("aggregate_views", &aggregate_views);
    m.impl("warp_corr_view_weights", &warp_corr_view_weights);
    m.impl("warp_corr_score_", &warp_corr_score_);
    m.impl("aggregate_views_score_", &aggregate_views_score_);
    m.impl("offset_corr", &offset_corr);
    m.impl("offset_corr_weight", &offset_corr_weight);
    m.impl("init_propagate", &init_propagate);
    m.impl("adaptive_eval", &adaptive_eval);
    m.impl("adaptive_eval_planar", &adaptive_eval_planar);
    m.impl("photometric_confidence", &photometric_confidence);
    m.impl("conv2d_nhwc", &conv2d_nhwc);
    m.impl("conv2d_nhwc_out", &conv2d_nhwc_out);
    m.impl("conv2d_tc5", &conv2d_tc5);
    m.impl("conv2d_tc5_out", &conv2d_tc5_out);
    m.impl("conv_stem", &conv_stem);
    m.impl("refine_low", &refine_low);
    m.impl("refine_full", &refine_full);
    m.impl("upsample2x_add", &upsample2x_add);
    m.impl("pack_nhwc_views", &pack_nhwc_views);
    m.impl("warp_corr_views", &warp_corr_views);
    m.impl("warp_corr_view_weights_views", &warp_corr_view_weights_views);
    m.impl("warp_corr_score_views_", &warp_corr_score_views_);
    m.impl("device_copy", &device_copy);
}
