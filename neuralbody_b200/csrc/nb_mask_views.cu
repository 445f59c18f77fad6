// nb_mask_views (include/neuralbody_b200.h): the demo and mesh datasets' mask views after decoding, on the device.  Pass 1
// is one CTA per undistorted row of one view: three threads run the row's map sums into shared memory (nb_undistort.cuh,
// as nb_item_images), then every thread takes pixels, forms their map entries and remaps the (optionally binarised)
// mask with the uint8 fixed-point weights.  Without a dilation pass 1 visits only the output pixels' sources (2y, 2x)
// and writes the output; with one it undistorts the whole view into the workspace and pass 2 takes each output pixel's
// 5 x 5 maximum there.  tools/mask_views_case.py restates the steps in numpy (on oracle/item_images.py's map) and is
// pinned to cv2 by tests/test_mask_views_cpu.py.
#include "nb_undistort.cuh"

namespace nb {
namespace {

constexpr int kMaskThreads = 256;
constexpr int kDilateThreads = 256;

// Row oy of view blockIdx.y's undistorted mask, sampled every k-th source row and column: out (nv, Ho, Wo)
__global__ void __launch_bounds__(kMaskThreads) mask_undistort_kernel(const __grid_constant__ nb_mask_views_args a,
                                                                      unsigned char* out, int Ho, int Wo, int k) {
    extern __shared__ double sums[];     // [3][W0]: the row sums x, y, w of the source row
    const int oy = blockIdx.x, b = blockIdx.y, W0 = a.W0, H0 = a.H0;
    const double* cam = a.cams + (size_t)b * NB_ITEM_CAM_DOUBLES;
    if (threadIdx.x < 3) row_sums(cam, k * oy, threadIdx.x, H0, W0, sums + (size_t)threadIdx.x * W0);
    const Camera c = load_camera(cam, a.n_dist);
    __syncthreads();

    const unsigned char* msk = a.msk_u8 + (size_t)b * H0 * W0;
    for (int ox = threadIdx.x; ox < Wo; ox += kMaskThreads) {
        const int sx = k * ox;
        double u, v;
        undistort_point(c, sums[sx], sums[W0 + sx], sums[2 * W0 + sx], u, v);
        int ix, fx, iy, fy;
        fixed_point(u, ix, fx);
        fixed_point(v, iy, fy);
        out[((size_t)b * Ho + oy) * Wo + ox] = (unsigned char)remap_u8(msk, H0, W0, ix, fx, iy, fy, a.binarise != 0);
    }
}

// cv2.dilate with a (2r+1) x (2r+1) window of ones, pixels outside the image not taking part, at source pixel (ky, kx)
__global__ void __launch_bounds__(kDilateThreads) mask_dilate_kernel(const __grid_constant__ nb_mask_views_args a,
                                                                     const unsigned char* und, int r, int k) {
    const long long i = (long long)blockIdx.x * kDilateThreads + threadIdx.x;
    if (i >= (long long)a.nv * a.H * a.W) return;
    const int x = (int)(i % a.W), y = (int)(i / a.W % a.H), b = (int)(i / ((long long)a.W * a.H));
    const int sy = k * y, sx = k * x;
    const unsigned char* src = und + (size_t)b * a.H0 * a.W0;
    const int y0 = max(sy - r, 0), y1 = min(sy + r, a.H0 - 1), x0 = max(sx - r, 0), x1 = min(sx + r, a.W0 - 1);
    int m = 0;
    for (int yy = y0; yy <= y1; ++yy)
        for (int xx = x0; xx <= x1; ++xx) m = max(m, (int)src[(size_t)yy * a.W0 + xx]);
    a.msks[i] = (unsigned char)m;
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_mask_views_workspace_bytes(int nv, int H0, int W0) {
    if (nv < 1 || nv > 65535 || H0 < 1 || W0 < 1 || (long long)nv * H0 * W0 >= (1LL << 31)) return 0;
    return (size_t)nv * H0 * W0;
}

int nb_mask_views(const nb_mask_views_args* a, void* stream) {
    static const char* who = "nb_mask_views";
    if (!a || !a->msk_u8 || !a->cams || !a->msks || (a->dilate && !a->workspace)) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->nv < 1 || a->nv > 65535 || a->H0 < 1 || a->W0 < 1 || a->W0 > NB_ITEM_MAX_W ||
        (long long)a->nv * a->H0 * a->W0 >= (1LL << 31)) {
        set_error("%s: nv in [1, 65535], H0 >= 1 and W0 in [1, %d] with nv*H0*W0 < 2^31 (got %d x %d x %d)", who,
                  NB_ITEM_MAX_W, a->nv, a->H0, a->W0);
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
    if (a->binarise != 0 && a->binarise != 1) {
        set_error("%s: binarise must be 0 or 1 (got %d)", who, a->binarise);
        return NB_ERR_BAD_ARG;
    }
    if (a->dilate != 0 && a->dilate != 5) {
        set_error("%s: dilate must be 0 or 5 (got %d)", who, a->dilate);
        return NB_ERR_BAD_ARG;
    }
    if (a->dilate && a->workspace_bytes < nb_mask_views_workspace_bytes(a->nv, a->H0, a->W0)) {
        set_error("%s: the workspace has %zu bytes, a dilation needs %zu", who, a->workspace_bytes,
                  nb_mask_views_workspace_bytes(a->nv, a->H0, a->W0));
        return NB_ERR_BAD_ARG;
    }
    const int k = a->H0 / a->H;
    static bool configured = false;
    cudaError_t e = cudaSuccess;
    if (!configured) {
        e = cudaFuncSetAttribute(mask_undistort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(3 * NB_ITEM_MAX_W * sizeof(double)));
        configured = e == cudaSuccess;
    }
    const size_t smem = (size_t)3 * a->W0 * sizeof(double);
    const cudaStream_t s = (cudaStream_t)stream;
    if (e == cudaSuccess) {
        if (a->dilate) {
            unsigned char* und = (unsigned char*)a->workspace;
            mask_undistort_kernel<<<dim3((unsigned)a->H0, (unsigned)a->nv), kMaskThreads, smem, s>>>(*a, und, a->H0, a->W0, 1);
            const long long n = (long long)a->nv * a->H * a->W;
            mask_dilate_kernel<<<(unsigned)((n + kDilateThreads - 1) / kDilateThreads), kDilateThreads, 0, s>>>(
                *a, und, a->dilate / 2, k);
        } else {
            mask_undistort_kernel<<<dim3((unsigned)a->H, (unsigned)a->nv), kMaskThreads, smem, s>>>(*a, a->msks, a->H, a->W, k);
        }
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
