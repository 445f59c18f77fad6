// nb_image_loss_fwd / nb_image_loss_bwd (include/neuralbody_b200.h): the image losses of upstream's training wrapper
// (lib/train/trainers/if_nerf_clight.py:24-32) without the boolean-mask index, whose nonzero waits for the host.
//   forward:  one launch.  Each CTA sums (pred - gt)^2 over its grid-stride share of the elements of the set rays in
//             float64 and counts them; thread 0 stores the CTA's partials, and the last CTA to arrive (an integer ticket)
//             adds the partials in CTA order and writes loss = (float)(sum / count) and count.  The grid depends on the
//             size only, so the loss is the same bits on every run; no floating-point atomics.
//   backward: one launch, element-wise: the chain autograd runs on the GPU for torch.mean((x[m] - y[m]) ** 2), i.e.
//             mean (g * (1 / N), torch's CUDA division by a scalar), pow (2 * d), the product, and for a mask the
//             index's scatter into zeros (0 + v); exact 0 on the rays outside the mask.
// tests/test_image_loss_cpu.py restates both in numpy / torch.
#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kLossThreads = 256;
constexpr int kLossMaxCtas = 2 * kGridSMs;      // a constant, not the device's SM count: the sum's order is the size's alone

struct LossWorkspace {
    double* sum;              // [kLossMaxCtas]
    long long* count;         // [kLossMaxCtas]
    unsigned int* ticket;     // CTAs done; the last one resets it to 0
};

inline size_t loss_layout(unsigned char* base, LossWorkspace* w) {
    const size_t s = align256(kLossMaxCtas * sizeof(double)), c = align256(kLossMaxCtas * sizeof(long long));
    if (w) {
        w->sum = (double*)base;
        w->count = (long long*)(base + s);
        w->ticket = (unsigned int*)(base + s + c);
    }
    return s + c + 256;
}

inline int loss_ctas(long long elems) {
    const long long b = (elems + kLossThreads - 1) / kLossThreads;
    return (int)(b < 1 ? 1 : (b > kLossMaxCtas ? kLossMaxCtas : b));
}

// fixed-order block sum of (s, c): shuffle tree per warp, then warp 0 over the warps' results; valid in thread 0
__device__ __forceinline__ void block_sum(double& s, long long& c) {
    __shared__ double ss[kLossThreads / 32];
    __shared__ long long sc[kLossThreads / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        c += __shfl_down_sync(0xffffffffu, c, o);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { ss[warp] = s; sc[warp] = c; }
    __syncthreads();
    if (warp == 0) {
        s = lane < kLossThreads / 32 ? ss[lane] : 0.0;
        c = lane < kLossThreads / 32 ? sc[lane] : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            s += __shfl_down_sync(0xffffffffu, s, o);
            c += __shfl_down_sync(0xffffffffu, c, o);
        }
    }
    __syncthreads();          // ss / sc are reused by the finishing CTA's second sum
}

__global__ void __launch_bounds__(kLossThreads) image_loss_fwd_kernel(const __grid_constant__ nb_image_loss_args a,
                                                                      const LossWorkspace w) {
    __shared__ bool last;
    const long long elems = 3LL * a.rays, stride = (long long)gridDim.x * kLossThreads;
    double s = 0.0;
    long long c = 0;
    for (long long e = (long long)blockIdx.x * kLossThreads + threadIdx.x; e < elems; e += stride) {
        if (a.mask && !a.mask[e / 3]) continue;
        const double d = (double)a.pred[e] - (double)a.gt[e];      // exact: two floats' difference fits a double
        s = fma(d, d, s);
        ++c;
    }
    block_sum(s, c);
    if (threadIdx.x == 0) {
        w.sum[blockIdx.x] = s;
        w.count[blockIdx.x] = c;
        __threadfence();
        last = atomicAdd(w.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    s = 0.0;
    c = 0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += kLossThreads) {
        s += __ldcg(w.sum + i);
        c += __ldcg(w.count + i);
    }
    block_sum(s, c);
    if (threadIdx.x == 0) {
        *a.loss = (float)(s / (double)c);            // no element: 0 / 0 = NaN, torch.mean of an empty tensor
        *a.count = c;
        *w.ticket = 0u;
    }
}

__global__ void __launch_bounds__(kLossThreads) image_loss_bwd_kernel(const __grid_constant__ nb_image_loss_args a,
                                                                      const float* __restrict__ d_loss,
                                                                      float* __restrict__ d_pred) {
    const long long elems = 3LL * a.rays;
    const long long e = (long long)blockIdx.x * kLossThreads + threadIdx.x;
    if (e >= elems) return;
    if (a.mask && !a.mask[e / 3]) {
        d_pred[e] = 0.0f;
        return;
    }
    // torch: mean's backward g / N on the GPU is g * (1.0f / (float)N); pow's is grad * (2.0 * d); rounded in that order
    const float inv = __fdiv_rn(1.0f, __ll2float_rn(*a.count));
    const float gm = __fmul_rn(*d_loss, inv);
    const float v = __fmul_rn(gm, __fmul_rn(2.0f, __fsub_rn(a.pred[e], a.gt[e])));
    d_pred[e] = a.mask ? __fadd_rn(0.0f, v) : v;       // the index's backward accumulates into zeros
}

int check_loss_args(const nb_image_loss_args* a, const char* who) {
    if (!a || (a->rays > 0 && (!a->pred || !a->gt)) || !a->count) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->rays < 0 || 3LL * a->rays >= (1LL << 31)) {
        set_error("%s: 0 <= 3 rays < 2^31 (got rays = %d)", who, a->rays);
        return NB_ERR_BAD_ARG;
    }
    return NB_OK;
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_image_loss_workspace_bytes(void) { return loss_layout(nullptr, nullptr); }

int nb_image_loss_fwd(const nb_image_loss_args* a, void* stream) {
    static const char* who = "nb_image_loss_fwd";
    int st = check_loss_args(a, who);
    if (st != NB_OK) return st;
    if (!a->loss || !a->workspace) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->workspace_bytes < nb_image_loss_workspace_bytes() || (uintptr_t)a->workspace % 256 != 0) {
        set_error("%s: workspace must be 256-byte aligned and hold %zu bytes (got %zu)", who, nb_image_loss_workspace_bytes(),
                  a->workspace_bytes);
        return NB_ERR_BAD_ARG;
    }
    LossWorkspace w;
    loss_layout((unsigned char*)a->workspace, &w);
    image_loss_fwd_kernel<<<loss_ctas(3LL * a->rays), kLossThreads, 0, (cudaStream_t)stream>>>(*a, w);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_image_loss_bwd(const nb_image_loss_args* a, const float* d_loss, float* d_pred, void* stream) {
    static const char* who = "nb_image_loss_bwd";
    int st = check_loss_args(a, who);
    if (st != NB_OK) return st;
    if (!d_loss || (a->rays > 0 && !d_pred)) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->rays == 0) return NB_OK;
    const long long elems = 3LL * a->rays;
    image_loss_bwd_kernel<<<(unsigned)((elems + kLossThreads - 1) / kLossThreads), kLossThreads, 0, (cudaStream_t)stream>>>(
        *a, d_loss, d_pred);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
