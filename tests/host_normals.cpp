// Host build of the normal estimation and oriented fusion arithmetic of patchmatchnet_b200/csrc/pm_geo_math.cuh.
// TEST INFRASTRUCTURE: compiled with g++ by a fixture of tests/test_normals.py into a temporary directory, so the CPU suite
// runs the kernels' own per-pixel functions against oracle/normals_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_geo_math.cuh"

extern "C" {

// every pixel of an [H,W] map through pmgeo::normal_pixel, the window clipped at the border as the kernel clips it
void hn_depth_normals(const float *depth, int H, int W, const double *kinv, int radius, double depth_thres, int min_inliers,
                      float *out) {
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const int dx0 = -(radius < x ? radius : x), dx1 = radius < W - 1 - x ? radius : W - 1 - x;
            const int dy0 = -(radius < y ? radius : y), dy1 = radius < H - 1 - y ? radius : H - 1 - y;
            pmgeo::normal_pixel(depth + (size_t)y * W + x, W, x, y, dx0, dx1, dy0, dy1, kinv, depth_thres, min_inliers,
                                out + ((size_t)y * W + x) * 3);
        }
}

// the oriented fusion's per-pixel function over the surviving pixels in row-major order; returns the count
int hn_fuse_points_oriented(const unsigned char *mask, const double *depth_avg, const float *rgb, const float *normals,
                            const double *cam25, int H, int W, unsigned char *body) {
    int n = 0;
    for (int i = 0; i < H * W; ++i)
        if (mask[i])
            pmgeo::fuse_point_oriented(cam25, i % W, i / W, depth_avg[i], rgb + (size_t)i * 3, normals + (size_t)i * 3,
                                       body + (size_t)(n++) * pmgeo::kPlyOrientedVertexBytes);
    return n;
}

}  // extern "C"
