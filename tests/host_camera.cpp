// Host build of the camera models and the undistortion warp (patchmatchnet_b200/csrc/pm_camera_math.cuh).
// TEST INFRASTRUCTURE: compiled with g++ -ffp-contract=off by a fixture of tests/test_undistort.py into a temporary directory,
// so the CPU suite runs the kernels' own functions against tests/undistort_oracle.py.  Never loaded by the product package.
#include "../patchmatchnet_b200/csrc/pm_camera_math.cuh"

extern "C" {

void hc_world_to_image(int model, const double *p, long long n, const double *u, const double *v, double *x, double *y) {
    for (long long i = 0; i < n; ++i) pmcam::world_to_image(model, p, u[i], v[i], x[i], y[i]);
}

void hc_image_to_world(int model, const double *p, long long n, const double *x, const double *y, double *u, double *v) {
    for (long long i = 0; i < n; ++i) pmcam::image_to_world(model, p, x[i], y[i], u[i], v[i]);
}

// every border point of a W x H camera: mapped coordinate and side
void hc_border_points(int model, const double *p, int W, int H, double *mapped, int *side) {
    const long long n = 2ll * H + 2ll * W;
    for (long long k = 0; k < n; ++k) mapped[k] = pmcam::border_point(model, p, W, H, k, side[k]);
}

// the warp of a whole image, pixel by pixel
void hc_undistort_image(int model, const double *p, int W, int H, const unsigned char *src, const double *kp, int out_w, int out_h,
                        unsigned char *dst) {
    for (int y = 0; y < out_h; ++y)
        for (int x = 0; x < out_w; ++x) pmcam::undistort_pixel(model, p, W, H, src, kp, x, y, dst + ((long long)y * out_w + x) * 3);
}

}  // extern "C"
