// pm_poisson_math.cuh -- per-element formulas of the Poisson mesher (pm_poisson.cu; definition in include/patchmatch_b200.h
// and INTEGRATION.md "Poisson surface reconstruction (beyond the reference)"): the keep test, the box quantiles, grid
// placement, the trilinear hat weights and gradients, and the 27-point stencil.
//
// __host__ __device__ like pm_mesh_math.cuh: inlined into the kernels and into the host side of pm_poisson.cu, and compiled
// with g++ -ffp-contract=off by the CPU tests (tests/host_poisson.cpp), which check these functions against
// oracle/poisson_oracle.py.  Every float64 operation is written out so that no multiply-add is fused.
#pragma once

#include <math.h>
#include <stdint.h>

#include "pm_mesh_math.cuh"

namespace pmpoisson {

using pmmesh::add64;
using pmmesh::div64;
using pmmesh::mul64;
using pmmesh::sub64;

constexpr int kMinDepth = 5;
constexpr int kMaxDepth = 10;
constexpr long long kMaxPoints = 1ll << 28;
constexpr double kFixedScale = 4294967296.0;  // 2^32: the fixed-point unit of the rho and b sums

// A point is kept when xyz is finite and the normal is finite with a float64 length > 0; n_out is the normal divided by
// that length.
PMM_HD bool keep_point(const float *p, const float *n, double *n_out) {
    for (int a = 0; a < 3; ++a)
        if (!isfinite(p[a]) || !isfinite(n[a])) return false;
    const double x = n[0], y = n[1], z = n[2];
    const double len = sqrt(add64(add64(mul64(x, x), mul64(y, y)), mul64(z, z)));
    if (!(len > 0.0) || !isfinite(len)) return false;
    n_out[0] = div64(x, len);
    n_out[1] = div64(y, len);
    n_out[2] = div64(z, len);
    return true;
}

// The q quantile of m ascending values: pos = q (m - 1), g = floor(pos), t = pos - g, v[g] + t (v[g+1] - v[g]), with
// v[g+1] = v[g] at the end.  `at` reads element g and g + 1 of the sorted values.
PMM_HD double quantile(double q, long long m, double vg, double vg1) {
    const double pos = mul64(q, (double)(m - 1));
    const double t = sub64(pos, floor(pos));
    return add64(vg, mul64(t, sub64(vg1, vg)));
}
PMM_HD long long quantile_index(double q, long long m) { return (long long)floor(mul64(q, (double)(m - 1))); }

// Grid placement: E the largest extent of the box lo..hi, c its centre, h = scale E / N, I0 = floor(c / h) - N / 2.
// False when E is not positive and finite.
PMM_HD bool place_grid(const double *lo, const double *hi, int depth, double scale, double &h, long long *I0) {
    const int N = 1 << depth;
    double E = 0.0;
    for (int a = 0; a < 3; ++a) E = fmax(E, sub64(hi[a], lo[a]));
    if (!(E > 0.0) || !isfinite(E)) return false;
    h = div64(mul64(scale, E), (double)N);
    for (int a = 0; a < 3; ++a) {
        const double c = mul64(0.5, add64(lo[a], hi[a]));
        I0[a] = (long long)floor(div64(c, h)) - N / 2;
    }
    return true;
}

// Grid coordinate of a world coordinate: u = p / h - 0.5 - I0, so that node i sits at u = i.
PMM_HD double grid_coord(float p, double h, long long I0) { return sub64(sub64(div64((double)p, h), 0.5), (double)I0); }

// The cell of a grid coordinate inside the node box 0 <= u <= N: floor(u), with u = N in cell N - 1.
PMM_HD int cell_of(double u, int N) {
    const int c = (int)floor(u);
    return c > N - 1 ? N - 1 : (c < 0 ? 0 : c);
}

// Trilinear hat of the corner (c = 0: the cell's lower node, 1: its upper node) at fraction f along one axis, and its
// derivative along that axis.
PMM_HD double hat(double f, int c) { return c ? f : sub64(1.0, f); }
PMM_HD double hat_slope(int c) { return c ? 1.0 : -1.0; }

// Weight and gradient of corner k (bit a set: upper node along axis a) of the cell at fractions f[3].
PMM_HD double corner_weight(const double *f, int k) {
    return mul64(mul64(hat(f[0], k & 1), hat(f[1], (k >> 1) & 1)), hat(f[2], (k >> 2) & 1));
}
PMM_HD void corner_gradient(const double *f, int k, double *g) {
    const double wx = hat(f[0], k & 1), wy = hat(f[1], (k >> 1) & 1), wz = hat(f[2], (k >> 2) & 1);
    g[0] = mul64(mul64(hat_slope(k & 1), wy), wz);
    g[1] = mul64(mul64(wx, hat_slope((k >> 1) & 1)), wz);
    g[2] = mul64(mul64(wx, wy), hat_slope((k >> 2) & 1));
}

// A_ij = integral of grad phi_i . grad phi_j for the offset j - i: 8/3 at the centre, 0 at the 6 face neighbours, -1/6 at
// the 12 edge neighbours, -1/12 at the 8 corner neighbours, 0 beyond.
PMM_HD double stencil_weight(int dx, int dy, int dz) {
    if (dx < -1 || dx > 1 || dy < -1 || dy > 1 || dz < -1 || dz > 1) return 0.0;
    const int nz = (dx != 0) + (dy != 0) + (dz != 0);
    return nz == 0 ? 8.0 / 3.0 : nz == 1 ? 0.0 : nz == 2 ? -1.0 / 6.0 : -1.0 / 12.0;
}

}  // namespace pmpoisson
