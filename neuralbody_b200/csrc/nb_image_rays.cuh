// The demo datasets' render_utils.image_rays on the device (see nb_image_rays in include/neuralbody_b200.h): one thread per
// pixel.  image_ray<T> restates get_rays in the camera's scalar type with the roundings of upstream's np.dot calls over
// the pixels (numpy 2.3 / OpenBLAS 0.3.30; tools/demo_case.py spells them out and tests/golden/demo_*.npz pin them), then
// get_near_far in float32.  No expression here may be contracted: every product and sum is an explicit _rn intrinsic.
// The kernels are instantiated over the camera's scalar type: float in nb_image_rays.cu, double in nb_image_rays_f64.cu,
// one instance per object.  nb_gen_rays / nb_gen_rays_sharded (nb_capi.cu) do not use this file.
#pragma once

#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>

#include "nb_device.cuh"

namespace nb {
namespace {

constexpr int kRayThreads = 256;

// K_inv in K's scalar type TK, R / T / o in R's and T's TR: the training datasets' People-Snapshot camera is a float32 K with
// get_camera's float64 R and T (monocular_dataset.py:83-103), every other camera is one type
template <typename TK, typename TR = TK>
struct ImageCam {
    TK K_inv[9];
    TR R[9], T_[3], o[3];
    float bounds[6];
    int H, W;
};

// xy1 @ inv(K).T, component a, for the pixel (i, j) (np.arange's float32 coordinates)
__device__ __forceinline__ double pixel_camera(const double* Ki, double i, double j) {
    return __dadd_rn(__fma_rn(j, Ki[1], __dmul_rn(i, Ki[0])), Ki[2]);                          // ddot: an fma chain
}
__device__ __forceinline__ float pixel_camera(const float* Ki, float i, float j) {
    // sdot with unit strides: the float products summed in double, rounded once
    return __double2float_rn(__dadd_rn(__dadd_rn((double)__fmul_rn(i, Ki[0]), (double)__fmul_rn(j, Ki[1])), (double)Ki[2]));
}
// (pixel_camera - T) @ R, component a (R's column a, stride 3)
__device__ __forceinline__ double pixel_world(const double* p, const double* R, int a) {
    return __fma_rn(p[2], R[6 + a], __fma_rn(p[1], R[3 + a], __dmul_rn(p[0], R[a])));         // ddot: an fma chain
}
__device__ __forceinline__ float pixel_world(const float* p, const float* R, int a) {
    return __fadd_rn(__fmaf_rn(p[0], R[a], __fmul_rn(p[1], R[3 + a])), __fmul_rn(p[2], R[6 + a]));   // sdot, stride 3
}
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float to_f32(double v) { return __double2float_rn(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }

// get_rays (:8-21) at pixel (x, y), before any cast: xy1 @ inv(K).T in TK, then (pixel_camera - T) @ R - o in TR (a float
// pixel_camera is promoted exactly, as numpy promotes it against a float64 T)
template <typename TK, typename TR>
__device__ __forceinline__ void camera_ray_d(const ImageCam<TK, TR>& c, int x, int y, TR (&d)[3]) {
    const TK i = (TK)(float)x, j = (TK)(float)y;
    TR pc[3];
    for (int a = 0; a < 3; ++a) pc[a] = sub_rn((TR)pixel_camera(c.K_inv + 3 * a, i, j), c.T_[a]);
    for (int a = 0; a < 3; ++a) d[a] = sub_rn(pixel_world(pc, c.R, a), c.o[a]);
}

// np.minimum / np.maximum: a NaN operand propagates
__device__ __forceinline__ float np_min(float a, float b) { return (a != a || a < b) ? a : (b != b ? b : (b < a ? b : a)); }
__device__ __forceinline__ float np_max(float a, float b) { return (a != a || a > b) ? a : (b != b ? b : (b > a ? b : a)); }
__device__ __forceinline__ double np_min(double a, double b) { return (a != a || a < b) ? a : (b != b ? b : (b < a ? b : a)); }
__device__ __forceinline__ double np_max(double a, double b) { return (a != a || a > b) ? a : (b != b ? b : (b > a ? b : a)); }

// get_rays (:8-21), .astype(np.float32), get_near_far (:54-69) for pixel `pix`; -> mask_at_box
template <typename TK, typename TR>
__device__ __forceinline__ bool image_ray(const ImageCam<TK, TR>& c, int pix, float (&of)[3], float (&df)[3], float& near,
                                          float& far) {
    TR d[3];
    camera_ray_d(c, pix % c.W, pix / c.W, d);
    for (int a = 0; a < 3; ++a) {
        df[a] = to_f32(d[a]);
        of[a] = to_f32(c.o[a]);
    }
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(df[0], df[0]), __fmul_rn(df[1], df[1])), __fmul_rn(df[2], df[2])));
    float t1[3], t2[3];
    for (int a = 0; a < 3; ++a) {
        float v = __fdiv_rn(df[a], nrm);
        if (v < 1e-5f && v > -1e-10f) v = 1e-5f;
        if (v > -1e-5f && v < 1e-10f) v = -1e-5f;
        const float tmin = __fdiv_rn(__fsub_rn(c.bounds[a], of[a]), v), tmax = __fdiv_rn(__fsub_rn(c.bounds[3 + a], of[a]), v);
        t1[a] = np_min(tmin, tmax);
        t2[a] = np_max(tmin, tmax);
    }
    const float tn = np_max(np_max(t1[0], t1[1]), t1[2]), tf = np_min(np_min(t2[0], t2[1]), t2[2]);
    near = __fdiv_rn(tn, nrm);
    far = __fdiv_rn(tf, nrm);
    return tn < tf;
}

template <typename TK, typename TR>
__global__ void __launch_bounds__(kRayThreads) image_rays_mask_kernel(const __grid_constant__ ImageCam<TK, TR> c,
                                                                      unsigned char* __restrict__ mask) {
    const unsigned p = blockIdx.x * kRayThreads + threadIdx.x;     // H*W < 2^31: no unsigned wrap in the last block
    if (p >= (unsigned)(c.H * c.W)) return;
    float of[3], df[3], tn, tf;
    mask[p] = image_ray(c, (int)p, of, df, tn, tf) ? 1 : 0;
}

// the box-hit rays at their scanned offsets (the ray is recomputed: the same instructions give the same bits), and with an
// image its pixels' colours (the test split's rgb[mask_at_box])
template <typename TK, typename TR>
__global__ void __launch_bounds__(kRayThreads) image_rays_emit_kernel(const __grid_constant__ ImageCam<TK, TR> c,
                                                                      const unsigned char* __restrict__ mask,
                                                                      const int* __restrict__ offset, float* __restrict__ ray_o,
                                                                      float* __restrict__ ray_d, float* __restrict__ near,
                                                                      float* __restrict__ far, int* __restrict__ count,
                                                                      const float* __restrict__ image, float* __restrict__ rgb) {
    const unsigned p = blockIdx.x * kRayThreads + threadIdx.x;
    const unsigned n = (unsigned)(c.H * c.W);
    if (p >= n) return;
    const int m = mask[p], q = offset[p];
    if (p == n - 1) *count = q + m;
    if (!m) return;
    float of[3], df[3], tn, tf;
    image_ray(c, (int)p, of, df, tn, tf);
    for (int a = 0; a < 3; ++a) { ray_o[(size_t)q * 3 + a] = of[a]; ray_d[(size_t)q * 3 + a] = df[a]; }
    near[q] = tn;
    far[q] = tf;
    if (image)
        for (int a = 0; a < 3; ++a) rgb[(size_t)q * 3 + a] = image[(size_t)p * 3 + a];
}

// bit `shift` of a per-pixel byte map (mask_at_box: bit 0; the training sampler's class map: bits 0-2)
struct MaskBit {
    int shift;
    __host__ __device__ int operator()(unsigned char m) const { return (m >> shift) & 1; }
};

// the exclusive prefix count of bit `shift` over n bytes: the one scan both ray generators compact with
inline cudaError_t scan_mask_bit(void* scratch, size_t& scratch_bytes, const unsigned char* map, int shift, int* offset, int n,
                                 cudaStream_t s) {
    return cub::DeviceScan::ExclusiveSum(scratch, scratch_bytes, thrust::make_transform_iterator(map, MaskBit{shift}), offset,
                                         n, s);
}

// workspace: offsets (H*W) int32 | CUB scratch, 256-byte aligned each.  0 when the size query fails.
inline size_t image_rays_scan_bytes(int n) {
    size_t sb = 0;
    if (scan_mask_bit(nullptr, sb, nullptr, 0, nullptr, n, 0) != cudaSuccess) { cudaGetLastError(); return 0; }
    return sb;
}

inline int image_rays_pixels(int H, int W) {   // H*W, or -1 when it is not in [1, 2^31)
    if (H < 1 || W < 1 || (long long)H * W >= (1LL << 31)) return -1;
    return H * W;
}

template <typename TK, typename TR>
int image_rays_launch(const char* who, const nb_image_rays_args* a, const TR* K_inv, const TR* R, const TR* Tv, const TR* o,
                      void* stream) {
    if (!a || !K_inv || !R || !Tv || !o || !a->workspace || !a->ray_o || !a->ray_d || !a->near || !a->far ||
        !a->mask_at_box || !a->count) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (!a->image != !a->rgb) {
        set_error("%s: image and rgb must both be set or both be NULL", who);
        return NB_ERR_BAD_ARG;
    }
    const int n = image_rays_pixels(a->H, a->W);
    if (n < 0) {
        set_error("%s: H and W must be >= 1 with H*W < 2^31 (got %d x %d)", who, a->H, a->W);
        return NB_ERR_BAD_ARG;
    }
    const size_t need = nb_image_rays_workspace_bytes(a->H, a->W);
    if (need == 0 || a->workspace_bytes < need) {
        set_error("%s: workspace_bytes too small (%zu < %zu)", who, a->workspace_bytes, need);
        return NB_ERR_BAD_ARG;
    }
    ImageCam<TK, TR> c;
    for (int k = 0; k < 9; ++k) { c.K_inv[k] = (TK)K_inv[k]; c.R[k] = R[k]; }
    for (int k = 0; k < 3; ++k) { c.T_[k] = Tv[k]; c.o[k] = o[k]; }
    for (int k = 0; k < 6; ++k) c.bounds[k] = a->bounds[k];
    c.H = a->H; c.W = a->W;
    unsigned char* ws = (unsigned char*)a->workspace;
    int* offset = (int*)ws;
    const size_t scratch = align256((size_t)n * sizeof(int));
    size_t sb = need - scratch;
    const unsigned blocks = (unsigned)(((long long)n + kRayThreads - 1) / kRayThreads);   // 64-bit: n may be 2^31 - 1
    const cudaStream_t s = (cudaStream_t)stream;
    image_rays_mask_kernel<TK, TR><<<blocks, kRayThreads, 0, s>>>(c, a->mask_at_box);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess)
        e = scan_mask_bit(ws + scratch, sb, a->mask_at_box, 0, offset, n, s);
    if (e == cudaSuccess) {
        image_rays_emit_kernel<TK, TR><<<blocks, kRayThreads, 0, s>>>(c, a->mask_at_box, offset, a->ray_o, a->ray_d, a->near,
                                                                      a->far, a->count, a->image, a->rgb);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // namespace
}  // namespace nb
