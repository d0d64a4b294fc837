// Host build of the Poisson mesher's per-element formulas (patchmatchnet_b200/csrc/pm_poisson_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ by a fixture of tests/test_poisson.py into a temporary directory, so the CPU suite
// runs the kernels' own functions against oracle/poisson_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_poisson_math.cuh"

extern "C" {

int hp_keep(const float *p, const float *n, double *unit) { return pmpoisson::keep_point(p, n, unit) ? 1 : 0; }

double hp_quantile(const double *sorted, long long m, double q) {
    long long g = pmpoisson::quantile_index(q, m);
    if (g > m - 1) g = m - 1;
    return pmpoisson::quantile(q, m, sorted[g], sorted[g + 1 < m ? g + 1 : m - 1]);
}

int hp_place(const double *lo, const double *hi, int depth, double scale, double *h, long long *I0) {
    return pmpoisson::place_grid(lo, hi, depth, scale, *h, I0) ? 1 : 0;
}

double hp_grid_coord(float p, double h, long long I0) { return pmpoisson::grid_coord(p, h, I0); }
int hp_cell(double u, int N) { return pmpoisson::cell_of(u, N); }

// weights [8] and gradients [8,3] of the corners of a cell at fractions f[3]
void hp_corners(const double *f, double *w, double *g) {
    for (int k = 0; k < 8; ++k) {
        w[k] = pmpoisson::corner_weight(f, k);
        pmpoisson::corner_gradient(f, k, g + 3 * k);
    }
}

double hp_stencil(int dx, int dy, int dz) { return pmpoisson::stencil_weight(dx, dy, dz); }

}  // extern "C"
