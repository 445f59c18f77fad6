// f-4: importance sampling between the coarse and the fine pass of a hierarchical render.
//
// Replaces, for one batch of rays, the reference's NeRF-baseline lines
//   z_vals_mid = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
//   z_samples  = sample_pdf(z_vals_mid, weights[..., 1:-1], N_importance, det=(perturb == 0.))   nerf_net_utils.py:55-90
//   z_vals, _  = torch.sort(torch.cat([z_vals, z_samples], -1), -1)                               volume_renderer.py:84-93
// One warp per ray: the coarse depths are re-derived exactly as the coarse render derived them (z_sample), the CDF is
// accumulated sequentially like torch.cumsum, the inverse CDF is a binary search (searchsorted side='right') and the
// S + N_importance depths are sorted with a bitonic network in shared memory.  The result feeds nb_render_args.z_vals.
#include "nb_device.cuh"

namespace nb {
namespace pdf {

constexpr int MAX_COARSE = 256, MAX_TOTAL = 512, WARPS = 4;

// SRC (nb_sample_pdf_src): each entry carries its origin (coarse index, -1 = importance sample) through the same swaps, so
// z_out is the same bit for bit and z_src says where every entry came from
template <bool SRC>
__global__ void __launch_bounds__(WARPS * 32) sample_pdf_kernel(const nb_importance_args A, int* __restrict__ z_src) {
    __shared__ float zc_s[WARPS][MAX_COARSE];
    __shared__ float cdf_s[WARPS][MAX_COARSE];
    __shared__ float buf_s[WARPS][MAX_TOTAL];
    __shared__ int src_s[SRC ? WARPS : 1][SRC ? MAX_TOTAL : 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long ray = (long long)blockIdx.x * WARPS + warp;
    if (ray >= A.n_rays_total) return;
    float* zc = zc_s[warp];
    float* cdf = cdf_s[warp];
    float* buf = buf_s[warp];
    const int S = A.n_samples, Ni = A.n_importance, M = S - 1;      // M bins (mid points), M - 1 weights
    const float near = __ldg(A.near + ray), far = __ldg(A.far + ray);
    for (int s = lane; s < S; s += 32) zc[s] = z_sample(near, far, A.t_vals, s, S, A.t_rand ? A.t_rand + ray * S : nullptr);
    // pdf = (w + 1e-5) / sum(w + 1e-5) over weights[1 : S-1]
    float part = 0.f;
    for (int i = lane; i < M - 1; i += 32) {
        const float w = __fadd_rn(__ldg(A.weights + ray * S + 1 + i), 1e-5f);
        cdf[i + 1] = w;
        part += w;
    }
    const float total = warp_sum(part);
    __syncwarp();
    if (lane == 0) {            // cdf = cat([0], cumsum(pdf)): sequential, like torch.cumsum on a contiguous row
        float acc = 0.f;
        cdf[0] = 0.f;
        for (int i = 1; i < M; ++i) { acc = __fadd_rn(acc, __fdiv_rn(cdf[i], total)); cdf[i] = acc; }
    }
    __syncwarp();
    auto bin = [&](int i) { return __fmul_rn(.5f, __fadd_rn(zc[i + 1], zc[i])); };
    for (int j = lane; j < Ni; j += 32) {
        const float u = A.u ? __ldg(A.u + ray * Ni + j) : linspace01(j, Ni);
        int lo = 0, hi = M;                         // first index whose cdf > u  (searchsorted side='right')
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
        const int below = max(0, lo - 1), above = min(M - 1, lo);
        const float c0 = cdf[below], c1 = cdf[above], b0 = bin(below), b1 = bin(above);
        float denom = __fsub_rn(c1, c0);
        if (denom < 1e-5f) denom = 1.f;
        const float t = __fdiv_rn(__fsub_rn(u, c0), denom);
        const float smp = __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
        buf[S + j] = smp;
        if (A.z_samples) A.z_samples[ray * Ni + j] = smp;
    }
    const int n = S + Ni;
    int P = 1;
    while (P < n) P <<= 1;
    for (int i = lane; i < S; i += 32) buf[i] = zc[i];
    for (int i = n + lane; i < P; i += 32) buf[i] = __int_as_float(0x7f800000);      // +inf padding sorts to the end
    int* src = SRC ? src_s[warp] : nullptr;
    if constexpr (SRC)
        for (int i = lane; i < P; i += 32) src[i] = i < S ? i : -1;
    __syncwarp();
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < P; i += 32) {
                const int x = i ^ j;
                if (x > i) {
                    const float a = buf[i], b = buf[x];
                    const bool asc = (i & k) == 0;
                    if ((a > b) == asc) {
                        buf[i] = b; buf[x] = a;
                        if constexpr (SRC) { const int t = src[i]; src[i] = src[x]; src[x] = t; }
                    }
                }
            }
            __syncwarp();
        }
    }
    for (int i = lane; i < n; i += 32) A.z_out[ray * n + i] = buf[i];
    if constexpr (SRC)
        for (int i = lane; i < n; i += 32) z_src[ray * n + i] = src[i];
}

}  // namespace pdf
}  // namespace nb

extern "C" int nb_sample_pdf(const nb_importance_args* a, void* stream) { return nb_sample_pdf_src(a, nullptr, stream); }

extern "C" int nb_sample_pdf_src(const nb_importance_args* a, int* z_src, void* stream) {
    using namespace nb;
    if (!a) { set_error("nb_sample_pdf: null args"); return NB_ERR_BAD_ARG; }
    if (a->n_rays_total < 0 || a->n_samples < 3 || a->n_importance < 1) {
        set_error("nb_sample_pdf: need n_rays_total >= 0, n_samples >= 3, n_importance >= 1");
        return NB_ERR_BAD_ARG;
    }
    if (a->n_samples > pdf::MAX_COARSE || a->n_samples + a->n_importance > pdf::MAX_TOTAL) {
        set_error("nb_sample_pdf: n_samples <= %d and n_samples + n_importance <= %d supported", pdf::MAX_COARSE, pdf::MAX_TOTAL);
        return NB_ERR_UNSUPPORTED;
    }
    if (!a->near || !a->far || !a->weights || !a->z_out) { set_error("nb_sample_pdf: a required device pointer is null"); return NB_ERR_BAD_ARG; }
    if (a->n_rays_total == 0) return NB_OK;
    const unsigned grid = (unsigned)((a->n_rays_total + pdf::WARPS - 1) / pdf::WARPS);
    if (z_src) pdf::sample_pdf_kernel<true><<<grid, pdf::WARPS * 32, 0, (cudaStream_t)stream>>>(*a, z_src);
    else pdf::sample_pdf_kernel<false><<<grid, pdf::WARPS * 32, 0, (cudaStream_t)stream>>>(*a, nullptr);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_sample_pdf launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}
