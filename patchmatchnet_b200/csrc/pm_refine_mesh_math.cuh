// pm_refine_mesh_math.cuh -- the photometric mesh refinement's per-pixel and per-vertex arithmetic (definition in
// include/patchmatch_b200.h, "Mesh refinement"): grey levels, the pixel ray and its hit on the z-buffer's face, the bilinear
// sample and its derivative along the ray, the windowed ZNCC and its coefficients, fixed-point conversion and the vertex
// step.  float64 (float32 for the grey levels), each operation rounded on its own in the order written here (no fused
// multiply-add: the device code uses the __d*_rn / __f*_rn intrinsics, the host build is compiled with -ffp-contract=off),
// so tests/host_refine_mesh.cpp and oracle/refine_oracle.py reproduce every bit.
#pragma once

#include <math.h>
#include <stdint.h>

#include "pm_texture_math.cuh"

#ifdef __CUDACC__
#define PMRM_HD __host__ __device__ inline
#else
#define PMRM_HD inline
#endif

namespace pmrm {

using pmtex::add;
using pmtex::dvd;
using pmtex::mul;
using pmtex::sub;

constexpr int kRadius = 2;                  // the ZNCC window is (2 kRadius + 1)^2 pixels, clipped to the image
constexpr int kMinCount = 13;               // a window counts with at least this many valid pixels (more than half of 25)
constexpr double kMinVariance = 1e-4;       // and both grey variances above this (grey values in [0, 1])
constexpr double kDepthTolerance = 0.01;    // depth test in the source view: z <= (1 + 0.01) z-buffer depth
constexpr double kMinCosine = 0.3;          // both views see the face at less than acos(0.3) = 72.5 degrees of incidence
constexpr double kGradUnit = 1048576.0;     // 2^20: fixed-point unit of the gradient sums, per 1 / L
constexpr double kWeightUnit = 4294967296.0;  // 2^32: fixed-point unit of the weight sums, and of the footprint sums per L
constexpr double kEnergyUnit = 16777216.0;  // 2^24: fixed-point unit of the energy sum

#ifdef __CUDA_ARCH__
PMRM_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
PMRM_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
PMRM_HD double dsqrt(double a) { return __dsqrt_rn(a); }
PMRM_HD long long to_fixed(double a) { return __double2ll_rn(a); }
#else
PMRM_HD float fadd(float a, float b) { return a + b; }
PMRM_HD float fmul(float a, float b) { return a * b; }
PMRM_HD double dsqrt(double a) { return sqrt(a); }
PMRM_HD long long to_fixed(double a) { return (long long)nearbyint(a); }
#endif

// grey value of a pixel: ((0.299 r + 0.587 g) + 0.114 b), float32
PMRM_HD float grey(float r, float g, float b) {
    return fadd(fadd(fmul(0.299f, r), fmul(0.587f, g)), fmul(0.114f, b));
}

// one pixel of the next level: the 2 x 2 box mean ((a + b) + (c + d)) * 0.25, a b the upper row
PMRM_HD float box(float a, float b, float c, float d) { return fmul(fadd(fadd(a, b), fadd(c, d)), 0.25f); }

PMRM_HD double dot3(const double *a, const double *b) { return add(add(mul(a[0], b[0]), mul(a[1], b[1])), mul(a[2], b[2])); }

PMRM_HD void cross3(const double *a, const double *b, double *o) {
    o[0] = sub(mul(a[1], b[2]), mul(a[2], b[1]));
    o[1] = sub(mul(a[2], b[0]), mul(a[0], b[2]));
    o[2] = sub(mul(a[0], b[1]), mul(a[1], b[0]));
}

// camera centre C = -R^T t of Rt (row-major 3 x 4): C_c = -(((R0c t0 + R1c t1) + R2c t2))
PMRM_HD void centre(const double *Rt, double *C) {
    for (int c = 0; c < 3; ++c) C[c] = -add(add(mul(Rt[c], Rt[3]), mul(Rt[4 + c], Rt[7])), mul(Rt[8 + c], Rt[11]));
}

// the ray of pixel (x, y) with camera-z 1, r = R^T K^-1 (x, y, 1): y' = (y - cy) / fy, x' = ((x - cx) - s y') / fx,
// r_c = ((R0c x' + R1c y') + R2c)
PMRM_HD void ray(const double *K, const double *Rt, double x, double y, double *r) {
    const double yy = dvd(sub(y, K[5]), K[4]);
    const double xx = dvd(sub(sub(x, K[2]), mul(K[1], yy)), K[0]);
    for (int c = 0; c < 3; ++c) r[c] = add(add(mul(Rt[c], xx), mul(Rt[4 + c], yy)), Rt[8 + c]);
}

// face normal n = (X1 - X0) x (X2 - X0) of float32 corners, in float64
PMRM_HD void face_normal(const float *x0, const float *x1, const float *x2, double *n) {
    double a[3], b[3];
    for (int c = 0; c < 3; ++c) {
        a[c] = sub((double)x1[c], (double)x0[c]);
        b[c] = sub((double)x2[c], (double)x0[c]);
    }
    cross3(a, b, n);
}

struct Hit {
    double n[3];     // the face's normal
    double nr;       // n . r
    double t;        // X = C + t r
    double X[3];
    double beta[3];  // barycentrics of X, by the face's own corner order
};

// the hit of ray r from C on the plane of face x0 x1 x2: t = n . (X0 - C) / (n . r), X_c = C_c + t r_c, and
// beta_k = (n . ((X_{k+1} - X) x (X_{k+2} - X))) / (n . n); false when n . r is not < 0 (the ray does not meet the face's
// front) or t is not positive and finite
PMRM_HD bool hit(const double *C, const double *r, const float *x0, const float *x1, const float *x2, Hit &h) {
    face_normal(x0, x1, x2, h.n);
    h.nr = dot3(h.n, r);
    if (!(h.nr < 0.0)) return false;
    const double d[3] = {sub((double)x0[0], C[0]), sub((double)x0[1], C[1]), sub((double)x0[2], C[2])};
    h.t = dvd(dot3(h.n, d), h.nr);
    if (!(h.t > 0.0 && h.t < INFINITY)) return false;
    for (int c = 0; c < 3; ++c) h.X[c] = add(C[c], mul(h.t, r[c]));
    const float *xs[3] = {x0, x1, x2};
    const double nn = dot3(h.n, h.n);
    for (int k = 0; k < 3; ++k) {
        const float *p = xs[(k + 1) % 3], *q = xs[(k + 2) % 3];
        double a[3], b[3], e[3];
        for (int c = 0; c < 3; ++c) {
            a[c] = sub((double)p[c], h.X[c]);
            b[c] = sub((double)q[c], h.X[c]);
        }
        cross3(a, b, e);
        h.beta[k] = dvd(dot3(h.n, e), nn);
    }
    return true;
}

// the face faces C: n . (C - X0) > 0
PMRM_HD bool faces_point(const double *n, const float *x0, const double *C) {
    const double d[3] = {sub(C[0], (double)x0[0]), sub(C[1], (double)x0[1]), sub(C[2], (double)x0[2])};
    return dot3(n, d) > 0.0;
}

// neither view sees the face at grazing incidence: -(n . r) > c sqrt((n . n) (r . r)) for the reference ray r, and
// n . d > c sqrt((n . n) (d . d)) for d = C_j - X towards the source's centre, c = kMinCosine.  At grazing incidence the
// images alias the surface's texture and the photometric gradient points anywhere.
PMRM_HD bool oblique_ok(const Hit &h, const double *r, const double *Cj) {
    const double nn = dot3(h.n, h.n);
    const double d[3] = {sub(Cj[0], h.X[0]), sub(Cj[1], h.X[1]), sub(Cj[2], h.X[2])};
    return -h.nr > mul(kMinCosine, dsqrt(mul(nn, dot3(r, r)))) && dot3(h.n, d) > mul(kMinCosine, dsqrt(mul(nn, dot3(d, d))));
}

// X projects into a W x H source view: z > near and 0 <= u <= W - 1, 0 <= v <= H - 1 (q = (u, v, z), pmtex::project)
PMRM_HD bool lands(const double *q, double near_z, int W, int H) { return pmtex::in_view(q, near_z, W, H); }

// the depth test against the source z-buffer's depth zb (float32) at the rounded pixel: z <= (1 + tol) zb
PMRM_HD bool depth_ok(double z, float zb) { return z <= mul(add(1.0, kDepthTolerance), (double)zb); }

// bilinear sample of a W x H grey image at (u, v) inside [0, W - 1] x [0, H - 1] and its analytic derivatives: x0 = floor u,
// x1 = min(x0 + 1, W - 1), fx = u - x0 (likewise y); p q the upper row, s t the lower; top = p + fx (q - p),
// bot = s + fx (t - s), b = top + fy (bot - top); du = (q - p) + fy ((t - s) - (q - p)), dv = bot - top
PMRM_HD void bilinear(const float *img, int W, int H, double u, double v, double &b, double &du, double &dv) {
    const int x0 = (int)floor(u), y0 = (int)floor(v);
    const int x1 = x0 + 1 < W ? x0 + 1 : W - 1, y1 = y0 + 1 < H ? y0 + 1 : H - 1;
    const double fx = sub(u, (double)x0), fy = sub(v, (double)y0);
    const double p = img[(size_t)y0 * W + x0], q = img[(size_t)y0 * W + x1];
    const double s = img[(size_t)y1 * W + x0], t = img[(size_t)y1 * W + x1];
    const double dq = sub(q, p), dt = sub(t, s);
    const double top = add(p, mul(fx, dq)), bot = add(s, mul(fx, dt));
    b = add(top, mul(fy, sub(bot, top)));
    du = add(dq, mul(fy, sub(dt, dq)));
    dv = sub(bot, top);
}

// db/dt = du (du/dt) + dv (dv/dt) along ray r, at a point projecting to q = (u, v, z) under P:
// du/dt = ((P0 . r) - u (P2 . r)) / z, dv/dt = ((P1 . r) - v (P2 . r)) / z, Pk . r = ((Pk0 r0 + Pk1 r1) + Pk2 r2)
PMRM_HD double db_dt(const double *P, const double *q, const double *r, double du, double dv) {
    const double p0 = add(add(mul(P[0], r[0]), mul(P[1], r[1])), mul(P[2], r[2]));
    const double p1 = add(add(mul(P[4], r[0]), mul(P[5], r[1])), mul(P[6], r[2]));
    const double p2 = add(add(mul(P[8], r[0]), mul(P[9], r[1])), mul(P[10], r[2]));
    const double ut = dvd(sub(p0, mul(q[0], p2)), q[2]), vt = dvd(sub(p1, mul(q[1], p2)), q[2]);
    return add(mul(du, ut), mul(dv, vt));
}

// a window's sums (n valid pixels, Sa, Sb, Saa, Sbb, Sab) -> whether it counts, its energy 1 - ZNCC and the coefficients of
// dE/db_q = (c1 a_q + c2 b_q) + c0:  ma = Sa / n, mb = Sb / n, va = Saa / n - ma ma, vb = Sbb / n - mb mb,
// cov = Sab / n - ma mb, sigma = sqrt(va vb), Z = cov / sigma; c1 = -1 / (n sigma), c2 = Z / (n vb),
// c0 = ma / (n sigma) - (Z mb) / (n vb)
PMRM_HD bool window(int n, double Sa, double Sb, double Saa, double Sbb, double Sab, double &E, double *c) {
    if (n < kMinCount) return false;
    const double dn = (double)n;
    const double ma = dvd(Sa, dn), mb = dvd(Sb, dn);
    const double va = sub(dvd(Saa, dn), mul(ma, ma)), vb = sub(dvd(Sbb, dn), mul(mb, mb));
    if (!(va > kMinVariance) || !(vb > kMinVariance)) return false;
    const double cov = sub(dvd(Sab, dn), mul(ma, mb));
    const double sigma = dsqrt(mul(va, vb));
    const double Z = dvd(cov, sigma);
    const double ns = mul(dn, sigma), nv = mul(dn, vb);
    E = sub(1.0, Z);
    c[1] = -dvd(1.0, ns);
    c[2] = dvd(Z, nv);
    c[0] = sub(dvd(ma, ns), dvd(mul(Z, mb), nv));
    return true;
}

// dE/db_q from the summed coefficients of the counted windows that contain q
PMRM_HD double de_db(const double *c, double a, double b) { return add(add(mul(c[1], a), mul(c[2], b)), c[0]); }

// one pixel's contributions to corner k: gradient components ((g beta_k) / nr) n_c in units of 1 / L, the weight beta_k and
// the footprint beta_k t / f in units of L, each rounded to its fixed-point unit (half to even)
PMRM_HD void contributions(double g, const Hit &h, int k, double f, double L, long long *out) {
    const double s = dvd(mul(g, h.beta[k]), h.nr);
    for (int c = 0; c < 3; ++c) out[c] = to_fixed(mul(mul(mul(s, h.n[c]), L), kGradUnit));
    out[3] = to_fixed(mul(h.beta[k], kWeightUnit));
    out[4] = to_fixed(mul(dvd(dvd(mul(h.beta[k], h.t), f), L), kWeightUnit));
}

// the photometric step of a vertex from its sums (G [3], W, S fixed point), unit normal n, alpha and L:
// w = W / 2^32, s = ((S / 2^32) L) / w, g = (n . (G / 2^20 / L)) / w, d = -clamp((alpha s) s g, -s / 2, s / 2); 0 when W <= 0
PMRM_HD double step(const long long *G, long long Wf, long long Sf, const double *n, double alpha, double L) {
    if (Wf <= 0) return 0.0;
    const double w = dvd((double)Wf, kWeightUnit);
    const double s = dvd(mul(dvd((double)Sf, kWeightUnit), L), w);
    const double g3[3] = {dvd(dvd((double)G[0], kGradUnit), L), dvd(dvd((double)G[1], kGradUnit), L), dvd(dvd((double)G[2], kGradUnit), L)};
    const double g = dvd(dot3(n, g3), w);
    const double lim = mul(0.5, s);
    double d = mul(mul(mul(alpha, s), s), g);
    d = d > lim ? lim : (d < -lim ? -lim : d);
    return -d;
}

// the new coordinate: float32(((x + d n_c) - lambda U2_c))
PMRM_HD float moved(float x, double d, double n, double lambda, double u2) {
    return (float)sub(add((double)x, mul(d, n)), mul(lambda, u2));
}

}  // namespace pmrm
