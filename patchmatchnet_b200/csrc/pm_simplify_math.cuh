// pm_simplify_math.cuh -- per-edge arithmetic of the mesh simplifier (pm_simplify.cu; definition in include/patchmatch_b200.h
// and INTEGRATION.md "Mesh simplification (beyond the reference)"): quadrics, placement, cost, the flip test and the colour.
//
// __host__ __device__ like pm_mesh_math.cuh, whose rounded float64 operations it uses: inlined into the kernels of
// pm_simplify.cu and compiled with g++ by the CPU tests (tests/host_simplify.cpp), which check these functions against
// oracle/simplify_oracle.py bit for bit.  The host build is test infrastructure only.  Every float64 operation is written
// out in a fixed order, each rounded on its own (no fused multiply-add; the host build uses -ffp-contract=off).
#pragma once

#include <string.h>

#include "pm_mesh_math.cuh"

namespace pmsimp {

using pmmesh::add64;
using pmmesh::div64;
using pmmesh::mul64;
using pmmesh::sub64;

constexpr int kQ = 10;                  // unique entries of a symmetric 4x4 quadric: xx xy xz xd yy yz yd zz zd dd
constexpr double kBoundaryWeight = 1.0;  // W: a border edge's constraint plane weighs W |e|^2
constexpr double kDetRel = 1e-9;         // the 3x3 system is solved when |det| > kDetRel * s^3, s its largest diagonal entry
constexpr double kFarEdges = 1.0;        // ... and the solution lies within kFarEdges * |e| of the segment
constexpr double kFlatRel = 1e-9;        // the segment quadratic is flat when e^T A e <= kFlatRel * trace(A) * |e|^2
constexpr int kMaxValence = 32;          // a vertex with more incident faces is locked

#if defined(__CUDA_ARCH__)
PMM_HD double sqrt64(double a) { return __dsqrt_rn(a); }
#else
PMM_HD double sqrt64(double a) { return sqrt(a); }
#endif

PMM_HD double dot3(const double *a, const double *b) { return add64(add64(mul64(a[0], b[0]), mul64(a[1], b[1])), mul64(a[2], b[2])); }

// a x b, components (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0)
PMM_HD void cross3(const double *a, const double *b, double *o) {
    o[0] = sub64(mul64(a[1], b[2]), mul64(a[2], b[1]));
    o[1] = sub64(mul64(a[2], b[0]), mul64(a[0], b[2]));
    o[2] = sub64(mul64(a[0], b[1]), mul64(a[1], b[0]));
}

// (X1 - X0) x (X2 - X0)
PMM_HD void face_normal(const double *x0, const double *x1, const double *x2, double *n) {
    const double e1[3] = {sub64(x1[0], x0[0]), sub64(x1[1], x0[1]), sub64(x1[2], x0[2])};
    const double e2[3] = {sub64(x2[0], x0[0]), sub64(x2[1], x0[1]), sub64(x2[2], x0[2])};
    cross3(e1, e2, n);
}

// q += w (p p^T) for the plane p = (m / |m|, -(m / |m|) . X): each entry (p_i p_j) first, then times w; nothing when |m| = 0
PMM_HD void add_plane(const double *m, const double *x, double w, double *q) {
    const double len = sqrt64(dot3(m, m));
    if (!(len > 0.0)) return;
    const double u[3] = {div64(m[0], len), div64(m[1], len), div64(m[2], len)};
    const double p[4] = {u[0], u[1], u[2], -dot3(u, x)};
    int k = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j, ++k) q[k] = add64(q[k], mul64(w, mul64(p[i], p[j])));
}

// the area-weighted plane of face X0 X1 X2: A = |n| / 2
PMM_HD void add_face_quadric(const double *x0, const double *x1, const double *x2, double *q) {
    double n[3];
    face_normal(x0, x1, x2, n);
    add_plane(n, x0, mul64(sqrt64(dot3(n, n)), 0.5), q);
}

// the constraint plane of border edge (a, b), a < b, whose one face is X0 X1 X2: it contains the edge and is perpendicular to
// the face, m = (Xb - Xa) x n, weight W |Xb - Xa|^2, through Xa
PMM_HD void add_border_quadric(const double *xa, const double *xb, const double *x0, const double *x1, const double *x2, double *q) {
    double n[3], m[3];
    face_normal(x0, x1, x2, n);
    const double e[3] = {sub64(xb[0], xa[0]), sub64(xb[1], xa[1]), sub64(xb[2], xa[2])};
    cross3(e, n, m);
    add_plane(m, xa, mul64(kBoundaryWeight, dot3(e, e)), q);
}

// row i of the 4x4 quadric times (x, y, z, 1): ((Q_i0 x + Q_i1 y) + Q_i2 z) + Q_i3
PMM_HD double qrow(double a, double b, double c, double d, const double *v) {
    return add64(add64(add64(mul64(a, v[0]), mul64(b, v[1])), mul64(c, v[2])), d);
}

// v^T Q v with v = (x, y, z, 1): ((x r0 + y r1) + z r2) + r3, clamped at >= 0 (NaN -> 0)
PMM_HD double quadric_cost(const double *q, const double *v) {
    const double r0 = qrow(q[0], q[1], q[2], q[3], v), r1 = qrow(q[1], q[4], q[5], q[6], v), r2 = qrow(q[2], q[5], q[7], q[8], v),
                 r3 = qrow(q[3], q[6], q[8], q[9], v);
    const double c = add64(add64(add64(mul64(v[0], r0), mul64(v[1], r1)), mul64(v[2], r2)), r3);
    return c > 0.0 ? c : 0.0;
}

// clamp(((v - a) . e) / (e . e), 0, 1) with e = b - a; 0 when e . e = 0
PMM_HD double segment_param(const double *xa, const double *e, const double *v) {
    const double ee = dot3(e, e);
    if (!(ee > 0.0)) return 0.0;
    const double d[3] = {sub64(v[0], xa[0]), sub64(v[1], xa[1]), sub64(v[2], xa[2])};
    const double t = div64(dot3(d, e), ee);
    return t > 0.0 ? (t < 1.0 ? t : 1.0) : 0.0;
}

// The placement of edge (a, b) with q = Q_a + Q_b: the minimiser of q when the system passes the determinant test and lies
// within kFarEdges |e| of the segment, else the minimiser on the segment.  Returns 1 when the 3x3 solve was taken.
PMM_HD int placement(const double *q, const double *xa, const double *xb, double *v) {
    const double e[3] = {sub64(xb[0], xa[0]), sub64(xb[1], xa[1]), sub64(xb[2], xa[2])};
    const double ee = dot3(e, e);
    // cofactors of A = [[q0 q1 q2] [q1 q4 q5] [q2 q5 q7]]
    const double c00 = sub64(mul64(q[4], q[7]), mul64(q[5], q[5])), c01 = sub64(mul64(q[5], q[2]), mul64(q[1], q[7])),
                 c02 = sub64(mul64(q[1], q[5]), mul64(q[4], q[2])), c11 = sub64(mul64(q[0], q[7]), mul64(q[2], q[2])),
                 c12 = sub64(mul64(q[2], q[1]), mul64(q[0], q[5])), c22 = sub64(mul64(q[0], q[4]), mul64(q[1], q[1]));
    const double det = add64(add64(mul64(q[0], c00), mul64(q[1], c01)), mul64(q[2], c02));
    double s = fabs(q[0]);
    s = fabs(q[4]) > s ? fabs(q[4]) : s;
    s = fabs(q[7]) > s ? fabs(q[7]) : s;
    // g = A a + b, the gradient at a: the solve is taken relative to a, v = a - A^-1 g
    const double g[3] = {qrow(q[0], q[1], q[2], q[3], xa), qrow(q[1], q[4], q[5], q[6], xa), qrow(q[2], q[5], q[7], q[8], xa)};
    if (fabs(det) > mul64(kDetRel, mul64(mul64(s, s), s)) && ee > 0.0) {
        double w[3];
        w[0] = sub64(xa[0], div64(add64(add64(mul64(c00, g[0]), mul64(c01, g[1])), mul64(c02, g[2])), det));
        w[1] = sub64(xa[1], div64(add64(add64(mul64(c01, g[0]), mul64(c11, g[1])), mul64(c12, g[2])), det));
        w[2] = sub64(xa[2], div64(add64(add64(mul64(c02, g[0]), mul64(c12, g[1])), mul64(c22, g[2])), det));
        const double t = segment_param(xa, e, w);
        const double c[3] = {add64(xa[0], mul64(t, e[0])), add64(xa[1], mul64(t, e[1])), add64(xa[2], mul64(t, e[2]))};
        const double d[3] = {sub64(w[0], c[0]), sub64(w[1], c[1]), sub64(w[2], c[2])};
        if (dot3(d, d) <= mul64(mul64(kFarEdges, kFarEdges), ee)) {
            v[0] = w[0];
            v[1] = w[1];
            v[2] = w[2];
            return 1;
        }
    }
    // on the segment a + t e: f(t) = f(0) + 2 t e^T (A a + b) + t^2 e^T A e
    const double ae[3] = {add64(add64(mul64(q[0], e[0]), mul64(q[1], e[1])), mul64(q[2], e[2])),
                          add64(add64(mul64(q[1], e[0]), mul64(q[4], e[1])), mul64(q[5], e[2])),
                          add64(add64(mul64(q[2], e[0]), mul64(q[5], e[1])), mul64(q[7], e[2]))};
    const double eae = dot3(e, ae), eg = dot3(e, g);
    const double tr = add64(add64(q[0], q[4]), q[7]);
    double t = 0.5;
    if (eae > mul64(mul64(kFlatRel, tr), ee)) {
        t = -div64(eg, eae);
        t = t > 0.0 ? (t < 1.0 ? t : 1.0) : 0.0;  // NaN -> 0
    }
    v[0] = add64(xa[0], mul64(t, e[0]));
    v[1] = add64(xa[1], mul64(t, e[1]));
    v[2] = add64(xa[2], mul64(t, e[2]));
    return 0;
}

// colour at v: rint(ca + t (cb - ca)) per channel (round half to even), t the clamped segment parameter of v
PMM_HD void placement_colour(const double *xa, const double *xb, const double *v, const unsigned char *ca, const unsigned char *cb,
                             unsigned char *out) {
    const double e[3] = {sub64(xb[0], xa[0]), sub64(xb[1], xa[1]), sub64(xb[2], xa[2])};
    const double t = segment_param(xa, e, v);
    for (int c = 0; c < 3; ++c) out[c] = (unsigned char)rint(add64((double)ca[c], mul64(t, sub64((double)cb[c], (double)ca[c]))));
}

// A face X0 X1 X2 of the star, with vertex `slot` moved to v: false when it flips or becomes zero-area, i.e. when the old
// normal is non-zero and new . old <= 0.  Faces that were already zero-area pass.
PMM_HD bool face_keeps_orientation(const double *x0, const double *x1, const double *x2, int slot, const double *v) {
    double n0[3], n1[3];
    face_normal(x0, x1, x2, n0);
    if (n0[0] == 0.0 && n0[1] == 0.0 && n0[2] == 0.0) return true;
    double y0[3], y1[3], y2[3];
    for (int c = 0; c < 3; ++c) {
        y0[c] = slot == 0 ? v[c] : x0[c];
        y1[c] = slot == 1 ? v[c] : x1[c];
        y2[c] = slot == 2 ? v[c] : x2[c];
    }
    face_normal(y0, y1, y2, n1);
    return dot3(n1, n0) > 0.0;
}

// selection key: float32 bits of the cost (round to nearest) above the edge index; cost >= 0, so keys order like costs
PMM_HD unsigned long long edge_key(double cost, unsigned int edge) {
    const float c = (float)cost;
#if defined(__CUDA_ARCH__)
    const unsigned int bits = __float_as_uint(c);
#else
    unsigned int bits;
    memcpy(&bits, &c, 4);
#endif
    return ((unsigned long long)bits << 32) | edge;
}

}  // namespace pmsimp
