// Host build of the surface sampler's per-face and per-sample arithmetic (patchmatchnet_b200/csrc/pm_sample_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ -ffp-contract=off by a fixture of tests/test_sample.py into a temporary directory,
// so the CPU suite runs the kernels' own functions against oracle/sample_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_sample_math.cuh"

extern "C" {

// nf faces, corners x [nf,9] -> lattice size n [nf] (0: not finite, 2^31: too large) and face sample count [nf]
void hs_sizes(const float *x, long long nf, double s, long long *n, long long *count) {
    for (long long f = 0; f < nf; ++f) {
        n[f] = pmsample::lattice_size(x + 9 * f, x + 9 * f + 3, x + 9 * f + 6, s);
        count[f] = n[f] >= pmsample::kMaxLattice ? 0 : pmsample::face_samples(n[f]);
    }
}

// m lattice points: the k-th sample of a lattice of size n on corners x [m,9] (colours c [m,9] or NULL) -> (i, j) [m,2],
// the size recovered from the count [m], the point p [m,3] and colour rgb [m,3]
void hs_points(const float *x, const unsigned char *c, const long long *n, const long long *k, long long m, long long *ij,
               long long *n_back, double *p, unsigned char *rgb) {
    for (long long t = 0; t < m; ++t) {
        long long i, j;
        pmsample::lattice_point(n[t], k[t], i, j);
        ij[2 * t] = i;
        ij[2 * t + 1] = j;
        n_back[t] = pmsample::lattice_of_count(pmsample::face_samples(n[t]));
        const unsigned char *ca = c ? c + 9 * t : nullptr;
        pmsample::lattice_sample(x + 9 * t, x + 9 * t + 3, x + 9 * t + 6, ca, c ? ca + 3 : nullptr, c ? ca + 6 : nullptr, n[t], i, j,
                                 p + 3 * t, rgb + 3 * t);
    }
}

}  // extern "C"
