// cv::undistort's map and its uint8 remap on the device, shared by nb_item_images and nb_mask_views.  OpenCV's
// undistortion map walks each source row by repeated sums (initUndistortRectifyMap adds ir[0], ir[3], ir[6] once per
// column), so a pixel's map entry depends on every sum before it in its row: `row_sums` runs one of those sums for a
// whole row, and `undistort_point` / `fixed_point` turn a column's three sums into the 1/32 px source position.
// oracle/item_images.py restates every step in numpy and is pinned to cv2 by tests/test_item_images_cpu.py.  No
// expression here may be contracted: every product and sum is an explicit _rn intrinsic.
#pragma once
#include <climits>

#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kStripePixels = 4096;     // cv::undistort's map stripes: max(1, 4096 / W) rows

// cv::invert(DECOMP_LU) of the 3x3 camera matrix with Ar(1,2) = v0 - y0: the adjugate times 1 / det3
__device__ __forceinline__ void stripe_inverse(const double* K, int y0, double (&ir)[9]) {
    double m[9];
    for (int t = 0; t < 9; ++t) m[t] = K[t];
    m[5] = __dsub_rn(K[5], (double)y0);
    auto cof = [&](int a, int b, int c, int d) { return __dsub_rn(__dmul_rn(m[a], m[b]), __dmul_rn(m[c], m[d])); };
    const double det = __dadd_rn(__dsub_rn(__dmul_rn(m[0], cof(4, 8, 5, 7)), __dmul_rn(m[1], cof(3, 8, 5, 6))),
                                 __dmul_rn(m[2], cof(3, 7, 4, 6)));
    const double d = __ddiv_rn(1.0, det);
    ir[0] = __dmul_rn(cof(4, 8, 5, 7), d);
    ir[1] = __dmul_rn(cof(2, 7, 1, 8), d);
    ir[2] = __dmul_rn(cof(1, 5, 2, 4), d);
    ir[3] = __dmul_rn(cof(5, 6, 3, 8), d);
    ir[4] = __dmul_rn(cof(0, 8, 2, 6), d);
    ir[5] = __dmul_rn(cof(2, 3, 0, 5), d);
    ir[6] = __dmul_rn(cof(3, 7, 4, 6), d);
    ir[7] = __dmul_rn(cof(1, 6, 0, 7), d);
    ir[8] = __dmul_rn(cof(0, 4, 1, 3), d);
}

// The map's row-sum pass: component q (0: x, 1: y, 2: w) of source row sy of an H0 x W0 image under the camera `cam`
// (NB_ITEM_CAM_DOUBLES layout), written to out[0 .. W0)
__device__ __forceinline__ void row_sums(const double* cam, int sy, int q, int H0, int W0, double* out) {
    const int stripe = min(max(1, kStripePixels / W0), H0), y0 = sy / stripe * stripe;
    double ir[9];
    stripe_inverse(cam, y0, ir);
    const double step = q == 0 ? ir[0] : (q == 1 ? ir[3] : ir[6]);
    const double m = q == 0 ? ir[1] : (q == 1 ? ir[4] : ir[7]), c0 = q == 0 ? ir[2] : (q == 1 ? ir[5] : ir[8]);
    double s = __dadd_rn(__dmul_rn((double)(sy - y0), m), c0);
    for (int j = 0; j < W0; ++j) {
        out[j] = s;
        s = __dadd_rn(s, step);
    }
}

// saturate_cast<int>(c * 32) as SSE2's cvtsd2si rounds it (nearest-even; NaN or out of range -> INT_MIN), then the map's
// saturate_cast<short>(i >> 5) and the fraction i & 31
__device__ __forceinline__ void fixed_point(double c, int& whole, int& frac) {
    const double r = rint(__dmul_rn(c, 32.0));
    const int i = (r >= -2147483648.0 && r <= 2147483647.0) ? (int)r : INT_MIN;
    whole = min(max(i >> 5, -32768), 32767);
    frac = i & 31;
}

struct Camera {
    double fx, fy, u0, v0, k[8];   // k1 k2 p1 p2 k3 k4 k5 k6
};

// The distortion model of a camera in the NB_ITEM_CAM_DOUBLES layout, its first n_dist coefficients read
__device__ __forceinline__ Camera load_camera(const double* cam, int n_dist) {
    Camera c;
    c.fx = cam[0]; c.u0 = cam[2]; c.fy = cam[4]; c.v0 = cam[5];
    for (int t = 0; t < 8; ++t) c.k[t] = t < n_dist ? cam[9 + t] : 0.0;
    return c;
}

// initUndistortRectifyMap's source position of the map entry whose row sums are (X, Y, Wt)
__device__ __forceinline__ void undistort_point(const Camera& c, double X, double Y, double Wt, double& u, double& v) {
    const double w = __ddiv_rn(1.0, Wt), x = __dmul_rn(X, w), y = __dmul_rn(Y, w);
    const double x2 = __dmul_rn(x, x), y2 = __dmul_rn(y, y), r2 = __dadd_rn(x2, y2);
    const double xy2 = __dmul_rn(__dmul_rn(2.0, x), y);
    const double num = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c.k[4], r2), c.k[1]), r2), c.k[0]), r2));
    const double den = __dadd_rn(1.0, __dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c.k[7], r2), c.k[6]), r2), c.k[5]), r2));
    const double kr = __ddiv_rn(num, den);
    const double xd = __dadd_rn(__dadd_rn(__dmul_rn(x, kr), __dmul_rn(c.k[2], xy2)),
                                __dmul_rn(c.k[3], __dadd_rn(r2, __dmul_rn(2.0, x2))));
    const double yd = __dadd_rn(__dadd_rn(__dmul_rn(y, kr), __dmul_rn(c.k[2], __dadd_rn(r2, __dmul_rn(2.0, y2)))),
                                __dmul_rn(c.k[3], xy2));
    u = __dadd_rn(__dmul_rn(c.fx, xd), c.u0);
    v = __dadd_rn(__dmul_rn(c.fy, yd), c.v0);
}

// cv2.remap of a uint8 H0 x W0 image at the fixed-point source position (ix + fx / 32, iy + fy / 32): the bilinear
// weights * 32768 as integers, out-of-image neighbours 0, then (sum + 2^14) >> 15.  `binarise` reads each source pixel as
// (m != 0).
__device__ __forceinline__ int remap_u8(const unsigned char* src, int H0, int W0, int ix, int fx, int iy, int fy,
                                        bool binarise = false) {
    int sum = 0;
#pragma unroll
    for (int n = 0; n < 4; ++n) {
        const int yy = iy + (n >> 1), xx = ix + (n & 1);
        const bool in = yy >= 0 && yy < H0 && xx >= 0 && xx < W0;
        const int iw = ((n >> 1) ? fy : 32 - fy) * ((n & 1) ? fx : 32 - fx) * 32;
        int s = in ? (int)src[(size_t)yy * W0 + xx] : 0;
        if (binarise) s = s != 0;
        sum += s * iw;
    }
    return min((sum + (1 << 14)) >> 15, 255);
}

}  // namespace
}  // namespace nb
