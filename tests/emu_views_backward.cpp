// emu_views_backward.cpp -- the per-view (ragged source pack) instantiations of the K-A backward compiled for the HOST on top
// of tests/warp_emu.h.  TEST INFRASTRUCTURE: built by tests/test_multisize_train.py (g++, -DPM_EMU) into
// tests/_emu_views_backward.so; never loaded by the product package.  The function below does what
// pmb200_warp_corr_views_backward does (view table, parameter block, zero fill of the pack, grid) and then runs the kernel
// body under the emulator.
#define PM_EMU 1
#include "warp_emu.h"

#include "../patchmatchnet_b200/csrc/pm_backward.cu"

extern "C" {

int emu_warp_corr_views_backward(const float *ref_nhwc, const float *src_flat, const pmb200_view_extent *views, const float *rt,
                                 const float *depth, const float *vw, const float *grad_out, float *d_ref_nhwc, float *d_src_flat,
                                 int V, int B, int C, int G, int H, int W, int D) {
    BwdViewTable vt;
    long long end = 0;
    for (int v = 0; v < V; ++v) {
        vt.base[v] = views[v].offset;
        vt.hs[v] = views[v].height;
        vt.ws[v] = views[v].width;
        vt.sx[v] = (W > 1) ? (float)(views[v].width - 1) / (float)(W - 1) : 1.0f;
        vt.sy[v] = (H > 1) ? (float)(views[v].height - 1) / (float)(H - 1) : 1.0f;
        const long long e = views[v].offset + (long long)B * views[v].height * views[v].width * C;
        end = e > end ? e : end;
    }
    WarpCorrBwdParams p;
    p.ref = ref_nhwc; p.src = src_flat; p.rt = rt; p.depth = depth; p.vw = vw; p.gout = grad_out;
    p.dref = d_ref_nhwc; p.dsrc = d_src_flat;
    p.V = V; p.B = B; p.H = H; p.W = W; p.Hs = vt.hs[0]; p.Ws = vt.ws[0]; p.D = D;
    p.sx = vt.sx[0]; p.sy = vt.sy[0];
    memset(d_src_flat, 0, (size_t)end * sizeof(float));
    const int HW = H * W;
#define EMU_WBV(CC, GG)                                                                                  \
    do {                                                                                                 \
        const int pix_per_block = 4 * BwdMap<CC, GG>::PPW;                                               \
        emu::launch(dim3((HW + pix_per_block - 1) / pix_per_block, B), dim3(128), 0,                      \
                    [&] { warp_corr_backward_views_kernel<CC, GG>(p, vt); });                             \
        return 0;                                                                                        \
    } while (0)
    if (C == 64 && G == 8) EMU_WBV(64, 8);
    if (C == 32 && G == 8) EMU_WBV(32, 8);
    if (C == 16 && G == 4) EMU_WBV(16, 4);
#undef EMU_WBV
    return -2;
}

}  // extern "C"
