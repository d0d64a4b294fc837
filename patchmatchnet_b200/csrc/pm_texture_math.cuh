// pm_texture_math.cuh -- the texturer's per-face arithmetic (definition in include/patchmatch_b200.h, "Mesh texturing"):
// float64 projection, the candidate test, the label score, the chart rectangle's corners and the texture coordinates.
// float64, each operation rounded on its own in the order written here (no fused multiply-add: the device code uses the
// __d*_rn intrinsics, the host build is compiled with -ffp-contract=off), so tests/host_texture.cpp and
// oracle/texture_oracle.py reproduce every bit.
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define PMTEX_HD __host__ __device__ inline
#else
#define PMTEX_HD inline
#endif

namespace pmtex {

constexpr int kRounds = 3;           // Jacobi rounds of the label smoothing
constexpr double kLambda = 0.5;      // weight of one edge neighbour with the same label
constexpr int kMargin = 2;           // texels around a chart's projected box
constexpr int kCell = 4;             // side of an untextured face's cell
constexpr int kMinPage = 4096;       // smallest page side
constexpr int kMaxPage = 16384;      // largest page side
constexpr double kGrey = 160.0;      // colour of an untextured face of a mesh without colours

#ifdef __CUDA_ARCH__
PMTEX_HD double add(double a, double b) { return __dadd_rn(a, b); }
PMTEX_HD double sub(double a, double b) { return __dsub_rn(a, b); }
PMTEX_HD double mul(double a, double b) { return __dmul_rn(a, b); }
PMTEX_HD double dvd(double a, double b) { return __ddiv_rn(a, b); }
#else
PMTEX_HD double add(double a, double b) { return a + b; }
PMTEX_HD double sub(double a, double b) { return a - b; }
PMTEX_HD double mul(double a, double b) { return a * b; }
PMTEX_HD double dvd(double a, double b) { return a / b; }
#endif

// ((r0 x + r1 y) + r2 z) + r3
PMTEX_HD double row(const double *r, double x, double y, double z) {
    return add(add(add(mul(r[0], x), mul(r[1], y)), mul(r[2], z)), r[3]);
}

// (u, v, z) of a world point under the float64 camera P (row-major 3 x 4); u = u' / z, v = v' / z
PMTEX_HD void project(const double *P, double x, double y, double z, double *q) {
    const double zz = row(P + 8, x, y, z);
    q[0] = dvd(row(P, x, y, z), zz);
    q[1] = dvd(row(P + 4, x, y, z), zz);
    q[2] = zz;
}

// a projected vertex lies in front of the near plane and inside the image: z > near, 0 <= u <= W - 1, 0 <= v <= H - 1
PMTEX_HD bool in_view(const double *q, double near_z, int W, int H) {
    return q[2] > near_z && q[2] < INFINITY && q[0] >= 0.0 && q[0] <= (double)(W - 1) && q[1] >= 0.0 && q[1] <= (double)(H - 1);
}

// n . (C - centroid) > 0, n = (X1 - X0) x (X2 - X0) (components (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)), centroid
// = ((X0 + X1) + X2) / 3, the dot product ((n0 d0 + n1 d1) + n2 d2)
PMTEX_HD bool front_facing(const double *X0, const double *X1, const double *X2, const double *C) {
    double a[3], b[3], d[3];
    for (int k = 0; k < 3; ++k) {
        a[k] = sub(X1[k], X0[k]);
        b[k] = sub(X2[k], X0[k]);
        d[k] = sub(C[k], dvd(add(add(X0[k], X1[k]), X2[k]), 3.0));
    }
    const double n0 = sub(mul(a[1], b[2]), mul(a[2], b[1]));
    const double n1 = sub(mul(a[2], b[0]), mul(a[0], b[2]));
    const double n2 = sub(mul(a[0], b[1]), mul(a[1], b[0]));
    return add(add(mul(n0, d[0]), mul(n1, d[1])), mul(n2, d[2])) > 0.0;
}

// the z-buffer counts make v a candidate: at least one winning pixel and at least 90 % of the covered pixels won
PMTEX_HD bool visible_enough(long long visible, long long covered) { return visible >= 1 && 10 * visible >= 9 * covered; }

// the candidate test of face X0 X1 X2 (float32 positions) in a view; q receives the three projections [3][3]
PMTEX_HD bool candidate(const double *P, const double *C, double near_z, int W, int H, const float *x0, const float *x1,
                        const float *x2, double *q) {
    const double X[3][3] = {{x0[0], x0[1], x0[2]}, {x1[0], x1[1], x1[2]}, {x2[0], x2[1], x2[2]}};
    bool ok = true;
    for (int k = 0; k < 3; ++k) {
        project(P, X[k][0], X[k][1], X[k][2], q + 3 * k);
        ok = ok && in_view(q + 3 * k, near_z, W, H);
    }
    return ok && front_facing(X[0], X[1], X[2], C);
}

// the smoothed label score of a candidate: D / max D + lambda * (edge neighbours carrying the candidate's view)
PMTEX_HD double score(int data, int max_data, int same_neighbours) {
    return add(dvd((double)data, (double)max_data), mul(kLambda, (double)same_neighbours));
}

// a chart's rectangle grows by floor(u) and ceil(u) of each corner (integers; the margin is added at the end)
PMTEX_HD int lo_pixel(double u) { return (int)floor(u); }
PMTEX_HD int hi_pixel(double u) { return (int)ceil(u); }

// texture coordinate of a corner at (u, v) of a chart whose rectangle starts at (x0, y0) and is placed at (ox, oy) on a
// page of side S: a = u - x0 + ox, b = v - y0 + oy; (float32((a + 0.5) / S), float32(1 - (b + 0.5) / S))
PMTEX_HD void corner_uv(double u, double v, int x0, int y0, int ox, int oy, int S, float *out) {
    const double a = add(sub(u, (double)x0), (double)ox), b = add(sub(v, (double)y0), (double)oy);
    out[0] = (float)dvd(add(a, 0.5), (double)S);
    out[1] = (float)sub(1.0, dvd(add(b, 0.5), (double)S));
}

// texture coordinate of an untextured face's corners: the centre of its cell at (ox, oy)
PMTEX_HD void cell_uv(int ox, int oy, int S, float *out) {
    out[0] = (float)dvd((double)(ox + kCell / 2), (double)S);
    out[1] = (float)sub(1.0, dvd((double)(oy + kCell / 2), (double)S));
}

// colour of an untextured face's cell: round-half-even(((c0 + c1 + c2) / 3)) per channel, grey without colours
PMTEX_HD unsigned char cell_colour(const unsigned char *c0, const unsigned char *c1, const unsigned char *c2, int k) {
    if (!c0) return (unsigned char)kGrey;
    return (unsigned char)rint(dvd(add(add((double)c0[k], (double)c1[k]), (double)c2[k]), 3.0));
}

}  // namespace pmtex
