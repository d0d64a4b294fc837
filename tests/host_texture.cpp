// Host build of the texturer's per-face arithmetic (patchmatchnet_b200/csrc/pm_texture_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ -ffp-contract=off by a fixture of tests/test_texture.py into a temporary directory,
// so the CPU suite runs the kernels' own functions against oracle/texture_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_texture_math.cuh"

extern "C" {

// n faces x [n,9] (float32 corners) in one view -> q [n,9] (u, v, z per corner), candidate [n] (geometry only)
void ht_faces(const double *P, const double *C, double near_z, int W, int H, const float *x, int n, double *q, int *cand) {
    for (int i = 0; i < n; ++i)
        cand[i] = pmtex::candidate(P, C, near_z, W, H, x + 9 * i, x + 9 * i + 3, x + 9 * i + 6, q + 9 * i) ? 1 : 0;
}

void ht_scores(const int *data, const int *max_data, const int *same, int n, double *out) {
    for (int i = 0; i < n; ++i) out[i] = pmtex::score(data[i], max_data[i], same[i]);
}

// n corners: (u, v) [n,2], rectangle origin and placement [n,4] (x0, y0, ox, oy) -> uv [n,2]; and the cell uv of (ox, oy)
void ht_uvs(const double *uv_in, const int *frame, int n, int S, float *uv_out, float *cell_out) {
    for (int i = 0; i < n; ++i) {
        const int *f = frame + 4 * i;
        pmtex::corner_uv(uv_in[2 * i], uv_in[2 * i + 1], f[0], f[1], f[2], f[3], S, uv_out + 2 * i);
        pmtex::cell_uv(f[2], f[3], S, cell_out + 2 * i);
    }
}

}  // extern "C"
