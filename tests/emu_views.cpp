// emu_views.cpp -- the per-view (ragged source pack) instantiations of K-A compiled for the HOST on top of tests/warp_emu.h.
// TEST INFRASTRUCTURE: built by tests/test_multisize.py (g++, -DPM_EMU) into tests/_emu_views.so; never loaded by the product
// package.  The functions below do what the *_views entry points of pm_kernels.cu do (fill the parameter block and the view
// table, size the grid) and then run the kernel body under the emulator.
#define PM_EMU 1
#include "warp_emu.h"

#include "../patchmatchnet_b200/csrc/pm_kernels.cu"

namespace {

// what pmb200_warp_corr*_views put in the kernel's view table
ViewTable make_table(const pmb200_view_extent *views, int V, int H, int W) {
    ViewTable vt;
    for (int v = 0; v < V; ++v) {
        vt.base4[v] = (unsigned)(views[v].offset / 4);
        vt.hs[v] = views[v].height;
        vt.ws[v] = views[v].width;
        vt.sx[v] = (W > 1) ? (float)(views[v].width - 1) / (float)(W - 1) : 1.0f;
        vt.sy[v] = (H > 1) ? (float)(views[v].height - 1) / (float)(H - 1) : 1.0f;
    }
    return vt;
}

template <int C, int G, int EPI, int DC, int PIPE>
int run_wc3v(const WarpCorrParams &p, const ViewTable &vt, const MlpParams &m, float *sims_out) {
    if constexpr ((LaneMap<C, G>::PPW * DC) % 32 != 0) {
        return -2;
    } else {
        const int HW = p.H * p.W;
        constexpr int pix_per_block = kWarps2 * LaneMap<C, G>::PPW;
        dim3 grid((HW + pix_per_block - 1) / pix_per_block, (p.D + DC - 1) / DC, p.B);
        emu::launch(grid, dim3(kWarps2 * 32), 0, [&] { warp_corr3_views_kernel<C, G, EPI, DC, PIPE, 1>(p, vt, m, sims_out); });
        return 0;
    }
}

template <int C, int G, int EPI>
int run_wc3v_cfg(const WarpCorrParams &p, const ViewTable &vt, const MlpParams &m, float *sims_out, int dc, int pipe) {
#define EMU_TRY(DD, PP) \
    if (dc == DD && pipe == PP) return run_wc3v<C, G, EPI, DD, PP>(p, vt, m, sims_out);
    EMU_TRY(4, 0) EMU_TRY(4, 1) EMU_TRY(8, 0) EMU_TRY(8, 1) EMU_TRY(16, 0) EMU_TRY(16, 1)
#undef EMU_TRY
    return -2;
}

template <int C, int G>
int run_wc3v_epi(const WarpCorrParams &p, const ViewTable &vt, const MlpParams &m, float *sims_out, int epi, int dc, int pipe) {
    switch (epi) {
        case kEpiSims: return run_wc3v_cfg<C, G, kEpiSims>(p, vt, m, sims_out, dc, pipe);
        case kEpiAgg: return run_wc3v_cfg<C, G, kEpiAgg>(p, vt, m, sims_out, dc, pipe);
        case kEpiScore: return run_wc3v_cfg<C, G, kEpiScore>(p, vt, m, sims_out, dc, pipe);
        case kEpiViewW: return run_wc3v_cfg<C, G, kEpiViewW>(p, vt, m, sims_out, dc, pipe);
    }
    return -2;
}

WarpCorrParams make_params(const float *ref, const float *src, const ViewTable &vt, const float *rt, const float *depth, const float *vw,
                           float *out, int ostride, int V, int B, int H, int W, int D) {
    WarpCorrParams p;
    p.ref = ref; p.src = src; p.rt = rt; p.depth = depth; p.vw = vw; p.out = out;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = vt.hs[0]; p.Ws = vt.ws[0]; p.D = D;
    p.sx = vt.sx[0]; p.sy = vt.sy[0];
    p.ostride = ostride < 1 ? 1 : ostride;
    return p;
}

}  // namespace

extern "C" {

// Third-generation K-A over a ragged source pack.  epi: 0 per-view sims [V,B,G,D,H,W], 1 weighted average [B,G,D,H,W],
// 2 score [B,D,H,W]*ostride, 3 view weights [B,V,H,W] (out zero-filled; sims_out optional).  -2: combination not built.
int emu_warp_corr3_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views, const float *rt,
                         const float *depth, const float *vw, const pmb200_mlp *head, float *out, float *sims_out, int ostride, int V,
                         int B, int C, int G, int H, int W, int D, int epi, int dc, int pipe) {
    const ViewTable vt = make_table(views, V, H, W);
    const WarpCorrParams p = make_params(ref_nhwc, src_flat, vt, rt, depth, vw, out, ostride, V, B, H, W, D);
    MlpParams m{};
    if (head) m = to_device_layout(head);
    if (C == 64 && G == 8) return run_wc3v_epi<64, 8>(p, vt, m, sims_out, epi, dc, pipe);
    if (C == 32 && G == 8) return run_wc3v_epi<32, 8>(p, vt, m, sims_out, epi, dc, pipe);
    if (C == 16 && G == 4) return run_wc3v_epi<16, 4>(p, vt, m, sims_out, epi, dc, pipe);
    return -2;
}

// The generic kernel (any C % G == 0) over a ragged source pack; vw NULL: per-view sims, else the weighted average.
int emu_warp_corr_generic_views(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views, const float *rt,
                                const float *depth, const float *vw, float *out, int V, int B, int C, int G, int H, int W, int D) {
    const ViewTable vt = make_table(views, V, H, W);
    const WarpCorrParams p = make_params(ref_nhwc, src_flat, vt, rt, depth, vw, out, 1, V, B, H, W, D);
    const size_t total = (size_t)B * D * H * W;
    emu::launch(dim3((unsigned)((total + 127) / 128)), dim3(128), 0, [&] { warp_corr_generic_views_kernel(p, vt, C, G); });
    return 0;
}

}  // extern "C"
