// pm_camera_math.cuh -- COLMAP's 11 camera models in float64, and the per-pixel warp of the undistortion (pm_undistort.cu;
// definition in include/patchmatch_b200.h and INTEGRATION.md "Undistortion (beyond the reference)").
//
// __host__ __device__ like pm_mesh_math.cuh: inlined into the kernels of pm_undistort.cu and compiled with g++ by the CPU tests
// (tests/host_camera.cpp), which check these functions against tests/undistort_oracle.py.  The host build is test
// infrastructure only.  Every float64 operation is written out (no fused multiply-add; the host build uses -ffp-contract=off)
// in the order the oracle evaluates it, so the host build and the oracle agree bit for bit and the GPU differs only where
// CUDA's atan / tan and libm's differ in the last bit.
//
// Model ids and parameter order are COLMAP's (colmap_input.CAMERA_MODELS / PARAM_TYPE).  "Normalised" coordinates (u, v) are
// camera-frame rays divided by z; distort() maps them to the distorted normalised coordinates, x = fx * xd + cx.
#pragma once

#include <float.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define PMC_HD __host__ __device__ __forceinline__
#else
#define PMC_HD inline
#endif

namespace pmcam {

enum Model {
    kSimplePinhole = 0, kPinhole = 1, kSimpleRadial = 2, kRadial = 3, kOpenCV = 4, kOpenCVFisheye = 5, kFullOpenCV = 6, kFOV = 7,
    kSimpleRadialFisheye = 8, kRadialFisheye = 9, kThinPrismFisheye = 10,
};
constexpr int kNumModels = 11;
constexpr int kMaxParams = 12;
constexpr int kNewtonIterations = 100;
constexpr double kNewtonStepNorm2 = 1e-20;  // stop once the step's squared norm is below this
constexpr double kNewtonRelStep = 1e-6;     // central differences of the Jacobian: step max(DBL_EPSILON, |1e-6 x|)
constexpr double kFovEpsilon = 1e-4;

#if defined(__CUDA_ARCH__)
PMC_HD double mul(double a, double b) { return __dmul_rn(a, b); }
PMC_HD double add(double a, double b) { return __dadd_rn(a, b); }
PMC_HD double sub(double a, double b) { return __dsub_rn(a, b); }
PMC_HD double dvd(double a, double b) { return __ddiv_rn(a, b); }
PMC_HD double root(double a) { return __dsqrt_rn(a); }
#else
PMC_HD double mul(double a, double b) { return a * b; }
PMC_HD double add(double a, double b) { return a + b; }
PMC_HD double sub(double a, double b) { return a - b; }
PMC_HD double dvd(double a, double b) { return a / b; }
PMC_HD double root(double a) { return sqrt(a); }
#endif

PMC_HD int num_params(int model) {
    switch (model) {
        case kSimplePinhole: return 3;
        case kPinhole: return 4;
        case kSimpleRadial: case kSimpleRadialFisheye: return 4;
        case kRadial: case kRadialFisheye: case kFOV: return 5;
        case kOpenCV: case kOpenCVFisheye: return 8;
        case kFullOpenCV: case kThinPrismFisheye: return 12;
        default: return -1;
    }
}

PMC_HD bool single_focal(int model) {
    return model == kSimplePinhole || model == kSimpleRadial || model == kRadial || model == kSimpleRadialFisheye ||
           model == kRadialFisheye;
}

// (fx, fy, cx, cy) of a model's pinhole part
PMC_HD void pinhole_part(int model, const double *p, double &fx, double &fy, double &cx, double &cy) {
    if (single_focal(model)) {
        fx = fy = p[0]; cx = p[1]; cy = p[2];
    } else {
        fx = p[0]; fy = p[1]; cx = p[2]; cy = p[3];
    }
}

// (u, v) scaled by theta_d / r for the fisheye models; (u, v) itself when r <= DBL_EPSILON
PMC_HD void fisheye(int model, const double *k, double u, double v, double r2, double &xd, double &yd) {
    const double r = root(r2);
    if (!(r > DBL_EPSILON)) {
        xd = u; yd = v;
        return;
    }
    const double th = atan(r), th2 = mul(th, th);
    double poly;
    if (model == kSimpleRadialFisheye) {
        poly = add(1.0, mul(k[0], th2));
    } else if (model == kRadialFisheye) {
        poly = add(add(1.0, mul(k[0], th2)), mul(k[1], mul(th2, th2)));
    } else {  // OPENCV_FISHEYE
        const double th4 = mul(th2, th2), th6 = mul(th4, th2), th8 = mul(th4, th4);
        poly = add(add(add(add(1.0, mul(k[0], th2)), mul(k[1], th4)), mul(k[2], th6)), mul(k[3], th8));
    }
    const double thd = mul(th, poly);
    xd = dvd(mul(u, thd), r);
    yd = dvd(mul(v, thd), r);
}

// distorted normalised coordinates (xd, yd) of the normalised point (u, v); x = fx * xd + cx
PMC_HD void distort(int model, const double *p, double u, double v, double &xd, double &yd) {
    const double u2 = mul(u, u), v2 = mul(v, v), r2 = add(u2, v2);
    switch (model) {
        case kSimpleRadial: {
            const double radial = mul(p[3], r2);
            xd = add(u, mul(u, radial)); yd = add(v, mul(v, radial));
            return;
        }
        case kRadial: {
            const double radial = add(mul(p[3], r2), mul(p[4], mul(r2, r2)));
            xd = add(u, mul(u, radial)); yd = add(v, mul(v, radial));
            return;
        }
        case kOpenCV: {
            const double k1 = p[4], k2 = p[5], p1 = p[6], p2 = p[7];
            const double uv = mul(u, v), radial = add(mul(k1, r2), mul(k2, mul(r2, r2)));
            const double du = add(add(mul(u, radial), mul(mul(2.0, p1), uv)), mul(p2, add(r2, mul(2.0, u2))));
            const double dv = add(add(mul(v, radial), mul(mul(2.0, p2), uv)), mul(p1, add(r2, mul(2.0, v2))));
            xd = add(u, du); yd = add(v, dv);
            return;
        }
        case kFullOpenCV: {
            const double k1 = p[4], k2 = p[5], p1 = p[6], p2 = p[7], k3 = p[8], k4 = p[9], k5 = p[10], k6 = p[11];
            const double r4 = mul(r2, r2), r6 = mul(r4, r2), uv = mul(u, v);
            const double radial = dvd(add(add(add(1.0, mul(k1, r2)), mul(k2, r4)), mul(k3, r6)),
                                      add(add(add(1.0, mul(k4, r2)), mul(k5, r4)), mul(k6, r6)));
            const double du = sub(add(add(mul(u, radial), mul(mul(2.0, p1), uv)), mul(p2, add(r2, mul(2.0, u2)))), u);
            const double dv = sub(add(add(mul(v, radial), mul(mul(2.0, p2), uv)), mul(p1, add(r2, mul(2.0, v2)))), v);
            xd = add(u, du); yd = add(v, dv);
            return;
        }
        case kOpenCVFisheye: case kSimpleRadialFisheye: case kRadialFisheye:
            fisheye(model, p + (model == kOpenCVFisheye ? 4 : 3), u, v, r2, xd, yd);
            return;
        case kFOV: {
            const double w = p[4], w2 = mul(w, w);
            double f;
            if (w2 < kFovEpsilon) {
                f = add(sub(dvd(mul(w2, r2), 3.0), dvd(w2, 12.0)), 1.0);
            } else if (r2 < kFovEpsilon) {
                const double t = tan(dvd(w, 2.0));
                f = dvd(mul(mul(-2.0, t), sub(mul(mul(mul(4.0, r2), t), t), 3.0)), mul(3.0, w));
            } else {
                const double r = root(r2);
                f = dvd(atan(mul(mul(r, 2.0), tan(dvd(w, 2.0)))), mul(r, w));
            }
            xd = mul(u, f); yd = mul(v, f);
            return;
        }
        case kThinPrismFisheye: {
            const double k1 = p[4], k2 = p[5], p1 = p[6], p2 = p[7], k3 = p[8], k4 = p[9], sx1 = p[10], sy1 = p[11];
            const double r = root(r2);
            double uu = u, vv = v;
            if (r > DBL_EPSILON) {
                const double th = atan(r);
                uu = dvd(mul(u, th), r);
                vv = dvd(mul(v, th), r);
            }
            const double uu2 = mul(uu, uu), vv2 = mul(vv, vv), rho2 = add(uu2, vv2);
            const double rho4 = mul(rho2, rho2), rho6 = mul(rho4, rho2), rho8 = mul(rho4, rho4), uv = mul(uu, vv);
            const double radial = add(add(add(mul(k1, rho2), mul(k2, rho4)), mul(k3, rho6)), mul(k4, rho8));
            xd = add(add(add(add(uu, mul(uu, radial)), mul(mul(2.0, p1), uv)), mul(p2, add(rho2, mul(2.0, uu2)))), mul(sx1, rho2));
            yd = add(add(add(add(vv, mul(vv, radial)), mul(mul(2.0, p2), uv)), mul(p1, add(rho2, mul(2.0, vv2)))), mul(sy1, rho2));
            return;
        }
        default:  // SIMPLE_PINHOLE, PINHOLE
            xd = u; yd = v;
            return;
    }
}

// pixel (x, y) of the normalised point (u, v)
PMC_HD void world_to_image(int model, const double *p, double u, double v, double &x, double &y) {
    double fx, fy, cx, cy, xd, yd;
    pinhole_part(model, p, fx, fy, cx, cy);
    distort(model, p, u, v, xd, yd);
    x = add(mul(fx, xd), cx);
    y = add(mul(fy, yd), cy);
}

// normalised point (u, v) of the pixel (x, y): the pinhole part inverted, then Newton's method on distort(u, v) = (xn, yn)
// from (xn, yn) (FOV: from its closed-form inverse), with a central-difference Jacobian.  NaN when the iteration breaks down.
PMC_HD void image_to_world(int model, const double *p, double x, double y, double &u, double &v) {
    double fx, fy, cx, cy;
    pinhole_part(model, p, fx, fy, cx, cy);
    const double xn = dvd(sub(x, cx), fx), yn = dvd(sub(y, cy), fy);
    u = xn; v = yn;
    if (model == kSimplePinhole || model == kPinhole) return;
    if (model == kFOV) {
        const double w = p[4];
        const double rd = root(add(mul(xn, xn), mul(yn, yn)));
        if (!(mul(w, w) < kFovEpsilon) && rd > DBL_EPSILON) {
            const double f = dvd(tan(mul(rd, w)), mul(mul(rd, 2.0), tan(dvd(w, 2.0))));
            u = mul(xn, f); v = mul(yn, f);
        }
    }
    for (int it = 0; it < kNewtonIterations; ++it) {
        const double s0 = fmax(DBL_EPSILON, fabs(mul(kNewtonRelStep, u))), s1 = fmax(DBL_EPSILON, fabs(mul(kNewtonRelStep, v)));
        double ex, ey, ax, ay, bx, by, cx_, cy_, dx_, dy_;
        distort(model, p, u, v, ex, ey);
        distort(model, p, sub(u, s0), v, ax, ay);
        distort(model, p, add(u, s0), v, bx, by);
        distort(model, p, u, sub(v, s1), cx_, cy_);
        distort(model, p, u, add(v, s1), dx_, dy_);
        const double j00 = dvd(sub(bx, ax), mul(2.0, s0)), j01 = dvd(sub(dx_, cx_), mul(2.0, s1));
        const double j10 = dvd(sub(by, ay), mul(2.0, s0)), j11 = dvd(sub(dy_, cy_), mul(2.0, s1));
        const double rx = sub(ex, xn), ry = sub(ey, yn);
        const double det = sub(mul(j00, j11), mul(j01, j10));
        const double sx = dvd(sub(mul(j11, rx), mul(j01, ry)), det), sy = dvd(sub(mul(j00, ry), mul(j10, rx)), det);
        u = sub(u, sx);
        v = sub(v, sy);
        const double n2 = add(mul(sx, sx), mul(sy, sy));
        if (n2 < kNewtonStepNorm2) return;
        if (!(n2 < INFINITY)) {  // NaN or infinite step: no solution from here
            u = v = NAN;
            return;
        }
    }
}

// The border point k of a W x H camera for the extents (k in [0, 2H + 2W)): the left (k < H) and right (H <= k < 2H) point of
// row y, then the top (2H <= k < 2H + W) and bottom point of column x, mapped through ImageToWorld and then the pinhole
// camera with the same fx, fy, cx, cy.  -> the mapped x for a row point, the mapped y for a column point; `side` is 0 left,
// 1 right, 2 top, 3 bottom.
PMC_HD double border_point(int model, const double *p, int W, int H, long long k, int &side) {
    double px, py;
    if (k < 2ll * H) {
        side = k < H ? 0 : 1;
        py = add((double)(k - (long long)side * H), 0.5);
        px = side == 0 ? 0.5 : sub((double)W, 0.5);
    } else {
        const long long c = k - 2ll * H;
        side = c < W ? 2 : 3;
        px = add((double)(c - (long long)(side - 2) * W), 0.5);
        py = side == 2 ? 0.5 : sub((double)H, 0.5);
    }
    double u, v, fx, fy, cx, cy;
    image_to_world(model, p, px, py, u, v);
    pinhole_part(model, p, fx, fy, cx, cy);
    return side < 2 ? add(mul(fx, u), cx) : add(mul(fy, v), cy);
}

// One target pixel (x, y) of the warp: its ray through the pinhole camera K' = (fx', fy', cx', cy'), through the distorted
// camera (model, p) of the W x H source image src (uint8 HWC RGB) to the source position (xs, ys) - 0.5, bilinear in float64
// (every operation rounded on its own), rounded half away from zero and clamped to 0..255.  0 in every channel when (xs, ys)
// is not finite or outside [0, W - 1] x [0, H - 1].
PMC_HD void undistort_pixel(int model, const double *p, int W, int H, const unsigned char *src, const double *kp, int x, int y,
                            unsigned char *out) {
    const double u = dvd(sub(add((double)x, 0.5), kp[2]), kp[0]);
    const double v = dvd(sub(add((double)y, 0.5), kp[3]), kp[1]);
    double xs, ys;
    world_to_image(model, p, u, v, xs, ys);
    xs = sub(xs, 0.5);
    ys = sub(ys, 0.5);
    if (!(xs >= 0.0 && xs <= (double)(W - 1) && ys >= 0.0 && ys <= (double)(H - 1))) {  // NaN fails too
        out[0] = out[1] = out[2] = 0;
        return;
    }
    const double fx0 = floor(xs), fy0 = floor(ys);
    const int x0 = (int)fx0, y0 = (int)fy0;
    const int x1 = x0 + 1 < W ? x0 + 1 : W - 1, y1 = y0 + 1 < H ? y0 + 1 : H - 1;
    const double dx = sub(xs, fx0), dy = sub(ys, fy0), ex = sub(1.0, dx), ey = sub(1.0, dy);
    const unsigned char *r0 = src + ((int64_t)y0 * W) * 3, *r1 = src + ((int64_t)y1 * W) * 3;
    for (int c = 0; c < 3; ++c) {
        const double a = add(mul(ex, (double)r0[3 * (int64_t)x0 + c]), mul(dx, (double)r0[3 * (int64_t)x1 + c]));
        const double b = add(mul(ex, (double)r1[3 * (int64_t)x0 + c]), mul(dx, (double)r1[3 * (int64_t)x1 + c]));
        const double val = round(add(mul(ey, a), mul(dy, b)));
        out[c] = (unsigned char)(val < 0.0 ? 0.0 : (val > 255.0 ? 255.0 : val));
    }
}

}  // namespace pmcam
