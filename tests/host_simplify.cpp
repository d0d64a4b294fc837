// Host build of the simplifier's per-edge arithmetic (patchmatchnet_b200/csrc/pm_simplify_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ -ffp-contract=off by a fixture of tests/test_simplify.py into a temporary directory,
// so the CPU suite runs the kernels' own functions against oracle/simplify_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_simplify_math.cuh"

extern "C" {

// n edges: q [n,10], xa, xb [n,3], ca, cb [n,3] -> v [n,3], solved [n], colour [n,3], cost [n], key [n] (edge index i)
void hs_edges(const double *q, const double *xa, const double *xb, const unsigned char *ca, const unsigned char *cb, int n, double *v,
              int *solved, unsigned char *colour, double *cost, unsigned long long *key) {
    for (int i = 0; i < n; ++i) {
        solved[i] = pmsimp::placement(q + 10 * i, xa + 3 * i, xb + 3 * i, v + 3 * i);
        pmsimp::placement_colour(xa + 3 * i, xb + 3 * i, v + 3 * i, ca + 3 * i, cb + 3 * i, colour + 3 * i);
        cost[i] = pmsimp::quadric_cost(q + 10 * i, v + 3 * i);
        key[i] = pmsimp::edge_key(cost[i], (unsigned int)i);
    }
}

// n faces X0 X1 X2 [n,9]: the face quadric, the border quadric of edge (xa, xb) [n,6], and the flip test with `slot` -> v
void hs_faces(const double *x, const double *edge, const int *slot, const double *v, int n, double *qface, double *qborder, int *keeps) {
    for (int i = 0; i < n; ++i) {
        const double *p = x + 9 * i;
        for (int k = 0; k < 10; ++k) qface[10 * i + k] = qborder[10 * i + k] = 0.0;
        pmsimp::add_face_quadric(p, p + 3, p + 6, qface + 10 * i);
        pmsimp::add_border_quadric(edge + 6 * i, edge + 6 * i + 3, p, p + 3, p + 6, qborder + 10 * i);
        keeps[i] = pmsimp::face_keeps_orientation(p, p + 3, p + 6, slot[i], v + 3 * i) ? 1 : 0;
    }
}

}  // extern "C"
