// pm_sample_math.cuh -- per-face and per-sample arithmetic of the surface sampler (pm_sample.cu; definition in
// include/patchmatch_b200.h and INTEGRATION.md "Surface sampling of meshes (beyond the reference)"): the lattice size of a
// face, its sample count, the map from a sample's index to its lattice point (i, j), and the point and colour there.
//
// __host__ __device__ like pm_mesh_math.cuh, whose rounded float64 operations it uses: inlined into the kernels of
// pm_sample.cu and compiled with g++ by the CPU tests (tests/host_sample.cpp), which check these functions against
// oracle/sample_oracle.py bit for bit.  The host build is test infrastructure only.  Every float64 operation is written
// out in a fixed order, each rounded on its own (no fused multiply-add; the host build uses -ffp-contract=off).
#pragma once

#include "pm_mesh_math.cuh"

namespace pmsample {

using pmmesh::add64;
using pmmesh::div64;
using pmmesh::mul64;
using pmmesh::sub64;

constexpr long long kMaxLattice = 1ll << 31;  // n >= 2^31 is rejected (the caller is told to use a larger spacing)

#if defined(__CUDA_ARCH__)
PMM_HD double sqrt64(double a) { return __dsqrt_rn(a); }
#else
PMM_HD double sqrt64(double a) { return sqrt(a); }
#endif

PMM_HD bool finite3(const float *p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

// sqrt((dx dx + dy dy) + dz dz) of q - p, each operation rounded on its own
PMM_HD double edge_length(const double *p, const double *q) {
    const double dx = sub64(q[0], p[0]), dy = sub64(q[1], p[1]), dz = sub64(q[2], p[2]);
    return sqrt64(add64(add64(mul64(dx, dx), mul64(dy, dy)), mul64(dz, dz)));
}

// Lattice size n = max(1, ceil(L / s)), L the longest of |B - A|, |C - B|, |A - C|.  -> n, or 0 when a corner is not
// finite (the face emits nothing), or kMaxLattice when n >= 2^31 (including L / s = inf).
PMM_HD long long lattice_size(const float *a, const float *b, const float *c, double s) {
    if (!finite3(a) || !finite3(b) || !finite3(c)) return 0;
    const double A[3] = {(double)a[0], (double)a[1], (double)a[2]};
    const double B[3] = {(double)b[0], (double)b[1], (double)b[2]};
    const double C[3] = {(double)c[0], (double)c[1], (double)c[2]};
    const double lab = edge_length(A, B), lbc = edge_length(B, C), lca = edge_length(C, A);
    double L = lab;
    if (lbc > L) L = lbc;
    if (lca > L) L = lca;
    const double n = ceil(div64(L, s));
    if (!(n < (double)kMaxLattice)) return kMaxLattice;  // inf too (L and s are finite, s > 0: never NaN)
    return n < 1.0 ? 1 : (long long)n;
}

// Face samples of a lattice of size n: (n + 1)(n + 2) / 2 - 3, none for n <= 1.
PMM_HD long long face_samples(long long n) { return n <= 1 ? 0 : (n + 1) * (n + 2) / 2 - 3; }

// The inverse of face_samples on its range: the n >= 2 whose face_samples(n) is cnt > 0.  With m = n + 1,
// m (m + 1) / 2 = cnt + 3; m is guessed with a float64 square root and corrected with exact integer tests.
PMM_HD long long lattice_of_count(long long cnt) {
    const long long T = cnt + 3;
    long long m = (long long)((sqrt64(8.0 * (double)T + 1.0) - 1.0) * 0.5);
    if (m < 0) m = 0;
    while (m * (m + 1) / 2 > T) --m;
    while ((m + 1) * (m + 2) / 2 <= T) ++m;
    return m - 1;
}

// The k-th face sample (0 <= k < face_samples(n)) -> its lattice point (i, j).  Order: i from 0 to n, within each i, j from
// 0 to n - i, with (0, 0), (0, n) and (n, 0) left out.  The full lattice index p (row i starts at i (n + 1) - i (i - 1) / 2)
// is k + 1 in row 0 and k + 2 after it (skipping (0, 0) and (0, n)); (n, 0) is the last index and never reached.  Counted
// from the end, q = N - 1 - p lies in row i = n - t with t (t + 1) / 2 <= q < (t + 1)(t + 2) / 2: t is guessed with a
// float64 square root and corrected with exact integer tests, so the row inversion is exact.
PMM_HD void lattice_point(long long n, long long k, long long &i, long long &j) {
    const long long N = (n + 1) * (n + 2) / 2;
    const long long p = k < n - 1 ? k + 1 : k + 2;
    const long long q = N - 1 - p;
    long long t = (long long)((sqrt64(8.0 * (double)q + 1.0) - 1.0) * 0.5);  // 8 q + 1 would overflow int64 near n = 2^31
    if (t < 0) t = 0;
    while (t * (t + 1) / 2 > q) --t;
    while ((t + 1) * (t + 2) / 2 <= q) ++t;
    i = n - t;
    j = t - (q - t * (t + 1) / 2);
}

// The point of lattice (i, j) of size n on face A B C (float32 corners widened), a = (n - i - j) / n, b = i / n, c = j / n,
// P = (a A + b B) + c C per axis; colour round-half-even((a rA + b rB) + c rC) clamped to 0..255 (when ra is not NULL).
PMM_HD void lattice_sample(const float *a, const float *b, const float *c, const unsigned char *ra, const unsigned char *rb,
                           const unsigned char *rc, long long n, long long i, long long j, double *p, unsigned char *rgb) {
    const double dn = (double)n;
    const double wa = div64((double)(n - i - j), dn), wb = div64((double)i, dn), wc = div64((double)j, dn);
    for (int k = 0; k < 3; ++k)
        p[k] = add64(add64(mul64(wa, (double)a[k]), mul64(wb, (double)b[k])), mul64(wc, (double)c[k]));
    if (ra) {
        for (int k = 0; k < 3; ++k) {
            double v = rint(add64(add64(mul64(wa, (double)ra[k]), mul64(wb, (double)rb[k])), mul64(wc, (double)rc[k])));
            v = v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v);
            rgb[k] = (unsigned char)v;
        }
    }
}

}  // namespace pmsample
