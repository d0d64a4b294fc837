// Host build of the mesh refinement's per-pixel and per-vertex arithmetic (patchmatchnet_b200/csrc/pm_refine_mesh_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ -ffp-contract=off by a fixture of tests/test_refine_mesh.py into a temporary
// directory, so the CPU suite runs the kernels' own functions against oracle/refine_oracle.py.  Never loaded by the package.
#include "../patchmatchnet_b200/csrc/pm_refine_mesh_math.cuh"

extern "C" {

void hr_grey(const float *rgb, int n, float *out) {
    for (int i = 0; i < n; ++i) out[i] = pmrm::grey(rgb[i], rgb[n + i], rgb[2 * n + i]);
}

void hr_box(const float *q, int n, float *out) {
    for (int i = 0; i < n; ++i) out[i] = pmrm::box(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
}

// n pixels (x, y) of one camera against n faces [n,9] -> ok [n], r [n,3], t, nr [n], X [n,3], beta [n,3]; C [3]; oblique [n]
// the incidence test towards a source centre Cj
void hr_hits(const double *K, const double *Rt, const double *xy, const float *tri, int n, const double *Cj, double *C, int *ok, double *r,
             double *t, double *nr, double *X, double *beta, int *oblique) {
    pmrm::centre(Rt, C);
    for (int i = 0; i < n; ++i) {
        pmrm::ray(K, Rt, xy[2 * i], xy[2 * i + 1], r + 3 * i);
        pmrm::Hit h;
        ok[i] = pmrm::hit(C, r + 3 * i, tri + 9 * i, tri + 9 * i + 3, tri + 9 * i + 6, h) ? 1 : 0;
        oblique[i] = ok[i] && pmrm::oblique_ok(h, r + 3 * i, Cj) ? 1 : 0;
        t[i] = h.t;
        nr[i] = h.nr;
        for (int c = 0; c < 3; ++c) { X[3 * i + c] = h.X[c]; beta[3 * i + c] = h.beta[c]; }
    }
}

// n samples (u, v) of a W x H image -> b, du, dv; and db/dt under P with (u, v, z) = q [n,3] and rays r [n,3]
void hr_samples(const float *img, int W, int H, const double *uv, const double *P, const double *q, const double *r, int n,
                double *out) {
    for (int i = 0; i < n; ++i) {
        double b, du, dv;
        pmrm::bilinear(img, W, H, uv[2 * i], uv[2 * i + 1], b, du, dv);
        out[4 * i] = b;
        out[4 * i + 1] = du;
        out[4 * i + 2] = dv;
        out[4 * i + 3] = pmrm::db_dt(P, q + 3 * i, r + 3 * i, du, dv);
    }
}

// n windows: counts [n], sums [n,5] -> ok [n], out [n,4] (E, c0, c1, c2)
void hr_windows(const int *cnt, const double *S, int n, int *ok, double *out) {
    for (int i = 0; i < n; ++i) {
        double E = 0.0, c[3] = {0.0, 0.0, 0.0};
        ok[i] = pmrm::window(cnt[i], S[5 * i], S[5 * i + 1], S[5 * i + 2], S[5 * i + 3], S[5 * i + 4], E, c) ? 1 : 0;
        out[4 * i] = E;
        out[4 * i + 1] = c[0];
        out[4 * i + 2] = c[1];
        out[4 * i + 3] = c[2];
    }
}

// n pixel contributions: g, n [3], nr, t, beta [3] -> [n,3 corners,5] fixed point
void hr_contributions(const double *g, const double *nrm, const double *nr, const double *t, const double *beta, int n, double f,
                      double L, long long *out) {
    for (int i = 0; i < n; ++i) {
        pmrm::Hit h;
        for (int c = 0; c < 3; ++c) { h.n[c] = nrm[3 * i + c]; h.beta[c] = beta[3 * i + c]; }
        h.nr = nr[i];
        h.t = t[i];
        for (int k = 0; k < 3; ++k) pmrm::contributions(g[i], h, k, f, L, out + 15 * i + 5 * k);
    }
}

// n vertices: sums [n,5], unit normals [n,3], positions [n,3], U2 [n,3] -> new positions [n,3]
void hr_steps(const long long *acc, const double *nrm, const float *x, const double *u2, int n, double alpha, double lambda, double L,
              float *out) {
    for (int i = 0; i < n; ++i) {
        const double d = pmrm::step(acc + 5 * i, acc[5 * i + 3], acc[5 * i + 4], nrm + 3 * i, alpha, L);
        for (int c = 0; c < 3; ++c) out[3 * i + c] = pmrm::moved(x[3 * i + c], d, nrm[3 * i + c], lambda, u2[3 * i + c]);
    }
}

}  // extern "C"
