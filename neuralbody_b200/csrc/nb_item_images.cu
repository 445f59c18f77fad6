// nb_item_images (include/neuralbody_b200.h): the training datasets' image steps after decoding, on the device.  One CTA
// per output row of one item.  OpenCV's undistortion map (nb_undistort.cuh) walks each source row by repeated sums, so a
// pixel's map entry depends on every sum before it in its row: 3k threads of the CTA run those sums for the row's k
// source rows into shared memory, then every thread takes output pixels, forms their k x k map entries from the sums
// (cv::undistort's distortion model and 1/32 px fixed point), remaps the float image bilinearly, sums the k x k cell as
// INTER_AREA's fast path does, remaps the mask at the cell's first pixel with the uint8 fixed-point weights, and applies
// the background and the class bits.  oracle/item_images.py restates every step in numpy and is pinned to cv2 by
// tests/test_item_images_cpu.py.  No expression here may be contracted: every product and sum is an explicit _rn
// intrinsic.
#include "nb_undistort.cuh"

namespace nb {
namespace {

constexpr int kItemThreads = 256;

__global__ void __launch_bounds__(kItemThreads) item_images_kernel(const __grid_constant__ nb_item_images_args a) {
    extern __shared__ double sums[];     // [k][3][W0]: the row sums x, y, w of the CTA's k source rows
    const int k = a.H0 / a.H, oy = blockIdx.x, b = blockIdx.y, W0 = a.W0, H0 = a.H0;
    const double* cam = a.cams + (size_t)b * NB_ITEM_CAM_DOUBLES;
    if (threadIdx.x < 3 * k)
        row_sums(cam, k * oy + threadIdx.x / 3, threadIdx.x % 3, H0, W0, sums + (size_t)threadIdx.x * W0);
    const Camera c = load_camera(cam, a.n_dist);
    __syncthreads();

    const unsigned char* img = a.img_u8 + (size_t)b * H0 * W0 * 3;
    const unsigned char* msk = a.msk_u8 + (size_t)b * H0 * W0;
    for (int ox = threadIdx.x; ox < a.W; ox += kItemThreads) {
        float acc[3] = {0.f, 0.f, 0.f};
        int mval = 0;
        for (int dy = 0; dy < k; ++dy) {
            for (int dx = 0; dx < k; ++dx) {
                const int sx = k * ox + dx;
                const double* rs = sums + (size_t)dy * 3 * W0;
                double u, v;
                undistort_point(c, rs[sx], rs[W0 + sx], rs[2 * W0 + sx], u, v);
                int ix, fx, iy, fy;
                fixed_point(u, ix, fx);
                fixed_point(v, iy, fy);
                const float ax = __fmul_rn((float)fx, 1.f / 32.f), ay = __fmul_rn((float)fy, 1.f / 32.f);
                const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
                const float w[4] = {__fmul_rn(by, bx), __fmul_rn(by, ax), __fmul_rn(ay, bx), __fmul_rn(ay, ax)};
                float px[3] = {0.f, 0.f, 0.f};
#pragma unroll
                for (int n = 0; n < 4; ++n) {
                    const int yy = iy + (n >> 1), xx = ix + (n & 1);
                    const bool in = yy >= 0 && yy < H0 && xx >= 0 && xx < W0;
                    const size_t p = in ? (size_t)yy * W0 + xx : 0;
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        const float s = in ? __fdiv_rn((float)img[p * 3 + ch], 255.f) : 0.f;
                        const float t = __fmul_rn(s, w[n]);
                        px[ch] = n == 0 ? t : __fadd_rn(px[ch], t);
                    }
                }
                for (int ch = 0; ch < 3; ++ch) acc[ch] = (dy == 0 && dx == 0) ? px[ch] : __fadd_rn(acc[ch], px[ch]);
                if (dy == 0 && dx == 0) mval = remap_u8(msk, H0, W0, ix, fx, iy, fy);
            }
        }
        if (k == 2)
            for (int ch = 0; ch < 3; ++ch) acc[ch] = __fmul_rn(acc[ch], 0.25f);
        const size_t o = ((size_t)b * a.H + oy) * a.W + ox;
        if (a.bkgd != NB_ITEM_BKGD_NONE && mval == 0)
            for (int ch = 0; ch < 3; ++ch) acc[ch] = a.bkgd == NB_ITEM_BKGD_WHITE ? 1.f : 0.f;
        for (int ch = 0; ch < 3; ++ch) a.img[o * 3 + ch] = acc[ch];
        a.msk[o] = (unsigned char)mval;
        if (a.class_rule != NB_ITEM_CLASS_NONE) {
            const int bm = a.bound[o], m = (unsigned char)(mval * bm);
            int bits = (m == 13 ? NB_TRAIN_CLASS_FACE : 0) | (bm == 1 ? NB_TRAIN_CLASS_BOUND : 0);
            if (a.class_rule == NB_ITEM_CLASS_H36M) {
                bits |= m == 1 ? NB_TRAIN_CLASS_BODY : 0;
                if (m == 100) bits &= ~NB_TRAIN_CLASS_BOUND;     // sample_ray_h36m takes the border out of the bound list
            } else {
                bits |= m != 0 ? NB_TRAIN_CLASS_BODY : 0;
            }
            a.class_map[o] = (unsigned char)bits;
        }
    }
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

int nb_item_images(const nb_item_images_args* a, void* stream) {
    static const char* who = "nb_item_images";
    if (!a || !a->img_u8 || !a->msk_u8 || !a->cams || !a->img || !a->msk) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->B < 1 || a->B > 65535 || a->H0 < 1 || a->W0 < 1 || a->W0 > NB_ITEM_MAX_W ||
        (long long)a->B * a->H0 * a->W0 >= (1LL << 31)) {
        set_error("%s: B in [1, 65535], H0 >= 1 and W0 in [1, %d] with B*H0*W0 < 2^31 (got %d x %d x %d)", who, NB_ITEM_MAX_W,
                  a->B, a->H0, a->W0);
        return NB_ERR_BAD_ARG;
    }
    if (!((a->H == a->H0 && a->W == a->W0) || (a->H >= 1 && a->W >= 1 && 2 * a->H == a->H0 && 2 * a->W == a->W0))) {
        set_error("%s: the output must be the source size or exactly half of it (got %d x %d from %d x %d)", who, a->H, a->W,
                  a->H0, a->W0);
        return NB_ERR_BAD_ARG;
    }
    if (a->n_dist != 4 && a->n_dist != 5 && a->n_dist != 8) {
        set_error("%s: n_dist must be 4, 5 or 8 (got %d)", who, a->n_dist);
        return NB_ERR_BAD_ARG;
    }
    if (a->bkgd < NB_ITEM_BKGD_NONE || a->bkgd > NB_ITEM_BKGD_WHITE) {
        set_error("%s: bkgd must be an NB_ITEM_BKGD_* value (got %d)", who, a->bkgd);
        return NB_ERR_BAD_ARG;
    }
    if (a->class_rule < NB_ITEM_CLASS_NONE || a->class_rule > NB_ITEM_CLASS_SNAPSHOT) {
        set_error("%s: class_rule must be an NB_ITEM_CLASS_* value (got %d)", who, a->class_rule);
        return NB_ERR_BAD_ARG;
    }
    const bool rule = a->class_rule != NB_ITEM_CLASS_NONE;
    if (rule != (a->bound != nullptr) || rule != (a->class_map != nullptr)) {
        set_error("%s: bound and class_map must both be set with a class rule and both be NULL without one", who);
        return NB_ERR_BAD_ARG;
    }
    const int k = a->H0 / a->H;
    const size_t smem = (size_t)3 * k * a->W0 * sizeof(double);
    static bool configured = false;
    cudaError_t e = cudaSuccess;
    if (!configured) {
        e = cudaFuncSetAttribute(item_images_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(3 * 2 * NB_ITEM_MAX_W * sizeof(double)));
        configured = e == cudaSuccess;
    }
    if (e == cudaSuccess) {
        item_images_kernel<<<dim3((unsigned)a->H, (unsigned)a->B), kItemThreads, smem, (cudaStream_t)stream>>>(*a);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
