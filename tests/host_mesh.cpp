// Host build of the TSDF mesher's per-voxel arithmetic (patchmatchnet_b200/csrc/pm_mesh_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ by a fixture of tests/test_mesh.py into a temporary directory, so the CPU suite runs
// the kernels' own functions against oracle/mesh_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_mesh_math.cuh"

extern "C" {

// the seed range of one coordinate; returns 0 when it is rejected
int hm_seed_range(float p, double s, double tau, int *lo, int *hi) { return pmmesh::seed_range(p, s, tau, *lo, *hi) ? 1 : 0; }

unsigned long long hm_block_key(long long bi, long long bj, long long bk) { return pmmesh::block_key(bi, bj, bk); }

// voxels given by their integer indices [n,3] through every view in order (the integration kernel's per-voxel loop, without
// the block culling, which never changes a result)
void hm_integrate(const int *idx, int n, double s, double tau, const double *K, const double *Rt, const int *hw, int V,
                  const float *depth_flat, const long long *depth_off, const float *image_flat, const long long *image_off,
                  float *tsdf, float *weight, unsigned char *rgb) {
    for (int i = 0; i < n; ++i) {
        const double X = pmmesh::voxel_centre(idx[3 * i], s), Y = pmmesh::voxel_centre(idx[3 * i + 1], s),
                     Z = pmmesh::voxel_centre(idx[3 * i + 2], s);
        pmmesh::VoxelSums a;
        pmmesh::sums_init(a);
        for (int v = 0; v < V; ++v) {
            const double *r = Rt + 12 * v;
            const double xc = pmmesh::rigid_row(r, X, Y, Z), yc = pmmesh::rigid_row(r + 4, X, Y, Z), zc = pmmesh::rigid_row(r + 8, X, Y, Z);
            int px, py;
            const int H = hw[2 * v], W = hw[2 * v + 1];
            if (!pmmesh::view_pixel(K + 9 * v, H, W, xc, yc, zc, px, py)) continue;
            const long long pix = (long long)py * W + px, plane = (long long)H * W;
            const float *img = image_flat + image_off[v] + pix;
            pmmesh::voxel_update(a, depth_flat[depth_off[v] + pix], zc, tau, img[0], img[plane], img[2 * plane]);
        }
        pmmesh::voxel_finish(a, tsdf[i], weight[i], rgb + 3 * i);
    }
}

int hm_cube_index(const float *corner_tsdf) { return pmmesh::cube_index(corner_tsdf); }

int hm_edge_offset(int e) { return pmmesh::edge_offset(e); }
int hm_edge_axis(int e) { return pmmesh::edge_axis(e); }
int hm_corner_offset(int c) { return pmmesh::corner_offset(c); }

void hm_edge_vertex(const double *xa, const double *xb, float ta, float tb, const unsigned char *ca, const unsigned char *cb,
                    float *pos, unsigned char *rgb) {
    pmmesh::edge_vertex(xa, xb, ta, tb, ca, cb, pos, rgb);
}

void hm_table(signed char *out) {
    for (int c = 0; c < 256; ++c)
        for (int k = 0; k < pmmesh::kTableWidth; ++k) out[c * pmmesh::kTableWidth + k] = pmmesh::kTriTable[c][k];
}

}  // extern "C"
