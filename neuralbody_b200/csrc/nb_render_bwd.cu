// Backward of the fused render (nb_render_bwd): gradients of rgb_map / depth_map / acc_map with respect to
// the four dense feature volumes, every decoder parameter and the latent table; nb_render_bwd_frame adds the frame
// transform R / Th, nb_render_bwd_rays also the rays ray_o / ray_d, nb_render_bwd_maps also the cotangents of disp_map
// and weights, nb_render_bwd_inputs also near / far, the sample depths and bounds.
//
// Upstream this is PyTorch autograd through raw2outputs (nerf_net_utils.py:6-51), the eight Conv1d layers
// and F.grid_sample (latent_xyzc.py:62-126), driven by Trainer.train (lib/train/trainers/trainer.py:46-53).
// Here the exact-fp32 forward kernel saves the per-point activations (kSaveDim floats/point), and the
// backward runs as a short sequence of fp32 kernels on the caller's stream:
//   1. composite_bwd_kernel   d(outputs) -> d(rgb logits, sigma) per sample              (thread per ray)
//   2. decoder_dgrad_kernel   back through the folded colour layer, fc_2, fc_1, fc_0 to the gathered
//                             features, then the trilinear scatter-add into the NCDHW volume grads
//   3. wgrad_kernel (x6), colsum_kernel, view_wgrad_kernel     weight / bias gradients (split over points)
//   4. unfold_* kernels       gradients of the folded Wc / bc back to feature_fc, latent_fc, view_fc, latent
//   5. ray / depth gradients only: pe_grad_kernel (the positional encodings' part per point), ray_grad_kernel (per ray)
// Training chunks are small (N_rand = 1024 rays), so this path is sized for correctness and simplicity:
// fp32 FFMA, no tensor cores; the forward hot path is untouched.
#include "nb_device.cuh"
#include "nb_train.h"

namespace nb {
namespace bwd {

struct BwdParams {
    RenderParams f;                 // the forward call's parameters (rays, transforms, packed weights)
    const float* save;              // (B,n,S,kSaveDim)
    const float* raw;               // (B,n,S,4)
    GradRequest req;                // the map cotangents and the input gradients (accumulated into)
    float* ws;                      // (B*n*S, kGradDim) scratch
    nb_decoder_weights w;           // raw decoder tensors
    float* d_vol[4];                // NCDHW fp32, caller-zeroed, accumulated into
    float* d_raw_out;               // composite backward writes d(rgb logits, sigma) of sample i at d_raw_out + i * d_raw_stride
    int d_raw_stride;
};

constexpr int kBwdMaxSamples = 256;     // coarse + importance samples of a fine pass (64 + 128) fit

// ------------------------------------------------------------------------------------------ 1. composite
// One WARP per ray.  The per-sample quantities (z, dist, exp, sigmoids: the expensive part) are computed by all lanes into
// shared memory; the two recurrences -- transmittance forwards, U_i = sum_{j>i} g_j alpha_j prod_{i<k<j} f_k backwards (no
// division => safe when 1 - alpha underflows) -- are run by lane 0 in the reference's order; the outputs are written by all
// lanes.  (The earlier thread-per-ray version kept 1024 threads busy on a 148-SM device: 0.16 ms per 192-sample pass.)
constexpr int CB_WARPS = 4;

struct RaySmem {                        // one warp's ray in the per-ray kernels
    float alpha[kBwdMaxSamples], f[kBwdMaxSamples], g[kBwdMaxSamples], T[kBwdMaxSamples], U[kBwdMaxSamples], z[kBwdMaxSamples + 1];
};

// d disp_map -> d depth_map, d acc_map through disp = 1 / max(1e-10, x), x = depth / acc (nerf_net_utils.py:44), by torch's
// own backward rules: reciprocal -d r^2; maximum hands x the whole of it where x > 1e-10 or x is NaN, half where x == 1e-10,
// nothing below; division d / acc to depth and -d (x / acc) to acc.  On a ray with acc == 0, x = 0 / 0 is NaN and so are
// both results, whatever d_disp is: upstream's autograd does the same.
__device__ __forceinline__ void disparity_bwd(float depth, float acc, float d_disp, float& dD, float& dA) {
    const float x = __fdiv_rn(depth, acc);
    const float r = disparity(depth, acc);
    const float dm = -(d_disp * (r * r));
    const float dx = (x > 1e-10f || x != x) ? dm : (x == 1e-10f ? dm * 0.5f : 0.f);
    dD += __fdiv_rn(dx, acc);
    dA += -dx * __fdiv_rn(x, acc);
}

// The part both per-ray kernels share, run by the whole warp of ray ri: z, alpha, f = 1 - alpha + 1e-10 and the per-sample
// cotangent g_i = dC . rgb_i + dD z_i + dA into sm, then lane 0's recurrences T (exclusive transmittance) and U; dC (the
// cotangent of rgb_map) is returned for the rgb logits.  The cotangents of disp_map and weights enter here and nowhere else:
//   weights:  g_i += d_weights_i -- exact, since w_i = alpha_i T_i is what the recurrences differentiate;
//   disp_map: folded into dD / dA (disparity_bwd) at the depth and acc of the forward's own composite_ray, recomputed here
//             so that max(1e-10, x) takes the forward's branch.  The white background does not enter disp.
// dD_out (if given) receives the depth cotangent after the disp fold: what d z_i takes through depth_map = sum w z.
__device__ __forceinline__ void ray_bwd_recurrences(const BwdParams& Q, size_t ri, float nrm, RaySmem& sm, float (&dC)[3], int lane,
                                                    float* dD_out = nullptr) {
    const RenderParams& P = Q.f;
    const int S = P.n_samples;
    const float near = P.near[ri], far = P.far[ri];
    const float* tr = P.t_rand ? P.t_rand + ri * S : nullptr;
    const float* zu = P.z_user ? P.z_user + ri * S : nullptr;
    const float4* raw = reinterpret_cast<const float4*>(Q.raw) + ri * S;
    const MapCotangents& d = Q.req.maps;
    dC[0] = dC[1] = dC[2] = 0.f;
    if (d.rgb) { dC[0] = d.rgb[ri * 3]; dC[1] = d.rgb[ri * 3 + 1]; dC[2] = d.rgb[ri * 3 + 2]; }
    float dD = d.depth ? d.depth[ri] : 0.f;
    float dA = d.acc ? d.acc[ri] : 0.f;
    if (P.white_bkgd) dA -= dC[0] + dC[1] + dC[2];            // rgb_map += 1 - acc_map
    for (int s = lane; s < S; s += 32) sm.z[s] = z_sample(near, far, P.t_vals, s, S, tr, zu);
    __syncwarp();
    if (d.disp) {
        const RayOut o = composite_ray(raw, sm.z, S, nrm, nullptr, lane);
        disparity_bwd(o.depth, o.acc, d.disp[ri], dD, dA);
    }
    if (dD_out) *dD_out = dD;
    const float* dW = d.weights ? d.weights + ri * S : nullptr;
    for (int s = lane; s < S; s += 32) {
        const float4 rw = raw[s];
        const float z = sm.z[s];
        const float dist = ((s + 1 < S) ? __fsub_rn(sm.z[s + 1], z) : 1e10f) * nrm;
        const float alpha = 1.f - expf(-fmaxf(rw.w, 0.f) * dist);
        const float c0 = 1.f / (1.f + expf(-rw.x)), c1 = 1.f / (1.f + expf(-rw.y)), c2 = 1.f / (1.f + expf(-rw.z));
        sm.alpha[s] = alpha;
        sm.f[s] = 1.f - alpha + 1e-10f;
        float g = dC[0] * c0 + dC[1] * c1 + dC[2] * c2 + dD * z + dA;
        if (dW) g += dW[s];
        sm.g[s] = g;
    }
    __syncwarp();
    if (lane == 0) {
        float T = 1.f;
        for (int s = 0; s < S; ++s) { sm.T[s] = T; T *= sm.f[s]; }       // exclusive transmittance
        float U = 0.f;
        for (int s = S - 1; s >= 0; --s) { sm.U[s] = U; U = sm.g[s] * sm.alpha[s] + sm.f[s] * U; }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(CB_WARPS * 32) composite_bwd_kernel(const BwdParams Q) {
    __shared__ RaySmem s_ray[CB_WARPS];
    const RenderParams& P = Q.f;
    const int S = P.n_samples;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t ri = (size_t)blockIdx.x * CB_WARPS + warp;
    if (ri >= (size_t)P.batch * P.n_rays) return;
    const float nrm = ray_norm(P.ray_d[ri * 3], P.ray_d[ri * 3 + 1], P.ray_d[ri * 3 + 2]);
    RaySmem& sm = s_ray[warp];
    float dC[3];
    ray_bwd_recurrences(Q, ri, nrm, sm, dC, lane);
    const float4* raw = reinterpret_cast<const float4*>(Q.raw) + ri * S;
    for (int s = lane; s < S; s += 32) {
        const float4 rw = raw[s];
        const float z = sm.z[s];
        const float dist = ((s + 1 < S) ? __fsub_rn(sm.z[s + 1], z) : 1e10f) * nrm;
        const float e = expf(-fmaxf(rw.w, 0.f) * dist);
        const float c0 = 1.f / (1.f + expf(-rw.x)), c1 = 1.f / (1.f + expf(-rw.y)), c2 = 1.f / (1.f + expf(-rw.z));
        const float Ti = sm.T[s];
        const float w = sm.alpha[s] * Ti;
        const float dalpha = sm.g[s] * Ti - Ti * sm.U[s];
        float4 o;
        o.x = w * dC[0] * c0 * (1.f - c0);
        o.y = w * dC[1] * c1 * (1.f - c1);
        o.z = w * dC[2] * c2 * (1.f - c2);
        o.w = (rw.w > 0.f) ? dalpha * dist * e : 0.f;
        *reinterpret_cast<float4*>(Q.d_raw_out + (ri * S + s) * Q.d_raw_stride) = o;
    }
}

// Ray gradients (nb_render_bwd_rays), one WARP per ray, after the per-sample records are complete: rec + i * rec_stride holds
// sample i's [d loss / d(world point) 3 | d loss / d(view direction) 3] (zero for a skipped sample).  With p_i = o + z_i d,
// u = d / |d| and dists_i = delta_i |d| (nerf_net_utils.py:28):
//   d o += sum_i g_i,   d d += sum_i z_i g_i + (du - u (u . du)) / |d| + u sum_i dL/d dists_i delta_i,
// where du = sum_i du_i and dL/d dists_i = dalpha_i relu(sigma_i) e_i; z, dist and the T / U recurrences are those of
// composite_bwd_kernel (ray_bwd_recurrences).
// DEPTH (nb_render_bwd_inputs): also d z_i = r_i . d + dD w_i + |d| (c_{i-1} - c_i), with r_i the record's d loss / d(world
// point), dD the depth cotangent after the disp fold and c_i = dL/d dists_i = dalpha_i relu(sigma_i) e_i (c_{S-1} = c_{-1} = 0:
// the last dist is 1e10 |d|, independent of z).  It is added to Q.req.depths.z and, with z_sample's coefficients, summed
// into .near / .far.  A skipped sample has r = 0, w = 0 and relu(sigma) = 0, so skipping stays exact.
template <bool DEPTH>
__global__ void __launch_bounds__(CB_WARPS * 32) ray_grad_kernel(const BwdParams Q, const float* __restrict__ rec, int rec_stride) {
    __shared__ RaySmem s_ray[CB_WARPS];
    const RenderParams& P = Q.f;
    const int S = P.n_samples;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t ri = (size_t)blockIdx.x * CB_WARPS + warp;
    if (ri >= (size_t)P.batch * P.n_rays) return;
    const float dx = P.ray_d[ri * 3], dy = P.ray_d[ri * 3 + 1], dz = P.ray_d[ri * 3 + 2];
    const float nrm = ray_norm(dx, dy, dz);
    RaySmem& sm = s_ray[warp];
    float dC[3];
    float dD = 0.f;
    ray_bwd_recurrences(Q, ri, nrm, sm, dC, lane, DEPTH ? &dD : nullptr);
    const float4* raw = reinterpret_cast<const float4*>(Q.raw) + ri * S;
    float go[3] = {0.f, 0.f, 0.f}, gd[3] = {0.f, 0.f, 0.f}, du[3] = {0.f, 0.f, 0.f}, dn = 0.f;
    for (int s = lane; s < S; s += 32) {
        const float z = sm.z[s];
        const float delta = (s + 1 < S) ? __fsub_rn(sm.z[s + 1], z) : 1e10f;
        const float sg = fmaxf(raw[s].w, 0.f);
        const float e = expf(-sg * (delta * nrm));
        const float Ti = sm.T[s];
        const float dalpha = sm.g[s] * Ti - Ti * sm.U[s];
        // kept for sg == 0 too: a skipped (empty) sample adds 0, except that the NaN dalpha of a ray with acc == 0 and a
        // disp_map cotangent makes d ray_d NaN, as upstream's dists * relu(sigma) does
        dn = fmaf(dalpha * sg * e, delta, dn);
        const float* r = rec + (ri * S + s) * rec_stride;
#pragma unroll
        for (int k = 0; k < 3; ++k) { go[k] += r[k]; gd[k] = fmaf(z, r[k], gd[k]); du[k] += r[3 + k]; }
        if constexpr (DEPTH) sm.f[s] = s + 1 < S ? dalpha * sg * e : 0.f;   // c_s (f is free after the recurrences)
    }
    if constexpr (DEPTH) {
        __syncwarp();
        const float* tr = P.t_rand ? P.t_rand + ri * S : nullptr;
        const DepthGrads& dzo = Q.req.depths;
        float dnear = 0.f, dfar = 0.f;
        for (int s = lane; s < S; s += 32) {
            const float* r = rec + (ri * S + s) * rec_stride;
            const float w = sm.alpha[s] * sm.T[s];
            const float dzs = fmaf(r[2], dz, fmaf(r[1], dy, r[0] * dx)) + dD * w + nrm * ((s > 0 ? sm.f[s - 1] : 0.f) - sm.f[s]);
            if (dzo.z) dzo.z[ri * S + s] += dzs;
            if (dzo.near || dzo.far) {
                float cn, cf;
                z_sample_coefs(P.t_vals, s, S, tr, cn, cf);
                dnear = fmaf(cn, dzs, dnear);
                dfar = fmaf(cf, dzs, dfar);
            }
        }
        dnear = warp_sum(dnear);
        dfar = warp_sum(dfar);
        if (lane == 0 && dzo.near) dzo.near[ri] += dnear;
        if (lane == 0 && dzo.far) dzo.far[ri] += dfar;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { go[k] = warp_sum(go[k]); gd[k] = warp_sum(gd[k]); du[k] = warp_sum(du[k]); }
    dn = warp_sum(dn);
    if (lane == 0) {
        if (Q.req.d_ray_o) {
#pragma unroll
            for (int k = 0; k < 3; ++k) Q.req.d_ray_o[ri * 3 + k] += go[k];
        }
        if (Q.req.d_ray_d) {
            const float u[3] = {__fdiv_rn(dx, nrm), __fdiv_rn(dy, nrm), __fdiv_rn(dz, nrm)};
            const float udu = fmaf(u[2], du[2], fmaf(u[1], du[1], u[0] * du[0]));
#pragma unroll
            for (int k = 0; k < 3; ++k) Q.req.d_ray_d[ri * 3 + k] += gd[k] + fmaf(-u[k], udu, du[k]) / nrm + u[k] * dn;
        }
    }
}

// fp32 path, ray gradients: per point, d(positional encodings) = view_fc[:, 256:346]^T d_wpre (the colour layer's input
// columns [PE(viewdir) 27 | PE(xyz) 63], latent_xyzc.py:104), back through both encodings -> rec + point * rec_stride =
// [d / d(world point) from PE(xyz) 3 | d / d(view direction) 3].  One warp per point; PE(xyz) is read from the activation
// record, PE(viewdir) recomputed as the forward computes it.
constexpr int PG_WARPS = 8;
__global__ void __launch_bounds__(PG_WARPS * 32) pe_grad_kernel(const BwdParams Q, float* __restrict__ rec, int rec_stride) {
    __shared__ float s_d[PG_WARPS][96], s_pe[PG_WARPS][kViewPE];
    const RenderParams& P = Q.f;
    const int S = P.n_samples;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t npts = (size_t)P.batch * P.n_rays * S;
    const float* vw = Q.w.view_w + kHidden;          // (128, 346) row-major: column 256 + j
    for (size_t g = (size_t)blockIdx.x * PG_WARPS + warp; g < npts; g += (size_t)gridDim.x * PG_WARPS) {
        const size_t ri = g / S;
        if (lane == 0) {
            const float dx = P.ray_d[ri * 3], dy = P.ray_d[ri * 3 + 1], dz = P.ray_d[ri * 3 + 2];
            const float nrm = ray_norm(dx, dy, dz);
            positional_embed<4>(__fdiv_rn(dx, nrm), __fdiv_rn(dy, nrm), __fdiv_rn(dz, nrm), [&](int j, float v) { s_pe[warp][j] = v; });
        }
        const float* dw = Q.ws + g * kGradDim + kGradW;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
        for (int n = 0; n < kColor; ++n) {
            const float d = dw[n];
            if (d == 0.f) continue;                      // relu: same address for the whole warp, so a uniform branch
            a0 = fmaf(d, vw[n * 346 + lane], a0);
            a1 = fmaf(d, vw[n * 346 + 32 + lane], a1);
            if (lane < kViewPE + kXyzPE - 64) a2 = fmaf(d, vw[n * 346 + 64 + lane], a2);
        }
        s_d[warp][lane] = a0; s_d[warp][32 + lane] = a1; s_d[warp][64 + lane] = a2;
        __syncwarp();
        if (lane < 6) {
            const int ax = lane % 3;
            const float v = lane < 3 ? positional_embed_bwd<10>(&s_d[warp][kViewPE], Q.save + g * kSaveDim + kSaveH2 + kHidden, ax)
                                     : positional_embed_bwd<4>(&s_d[warp][0], &s_pe[warp][0], ax);
            rec[g * rec_stride + lane] = v;
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------ 2. decoder dgrad
constexpr int TP = 64, NT = 256, LDX = 356, LDY = 324, KC = 8;

// out[p][n] = epi(p, n, sum_k in[p][k] * W[k][n]),  W row-major [K][N] in global memory
template <int K, int N, int LDI, int LDO, typename Epi>
__device__ __forceinline__ void gemm_tile(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ W,
                                          float* __restrict__ Ws, Epi&& epi) {
    static_assert(K % KC == 0 && N % 32 == 0, "shape");
    constexpr int TN = N / 32;
    const int tid = threadIdx.x, pg = tid & 7, ng = tid >> 3;
    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int t = 0; t < TN; ++t) acc[i][t] = 0.f;
    for (int k0 = 0; k0 < K; k0 += KC) {
        for (int i = tid; i < KC * N; i += NT) Ws[i] = __ldg(W + (size_t)k0 * N + i);
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
            float a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = in[(pg + 8 * i) * LDI + k0 + kk];
#pragma unroll
            for (int t = 0; t < TN; ++t) {
                const float wv = Ws[kk * N + ng + 32 * t];
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[i][t] = fmaf(a[i], wv, acc[i][t]);
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int t = 0; t < TN; ++t) out[(pg + 8 * i) * LDO + ng + 32 * t] = epi(pg + 8 * i, ng + 32 * t, acc[i][t]);
    __syncthreads();
}

// Also the input gradients of the request that depend on the sample position, each only when asked for: dR / dTh, d bounds
// [:, 0] = -sum d loss / d(canonical point) per frame, and the grid parts of the ray gradients (d ray_o += g, d ray_d += z g
// with g = d loss / d(world point)) and of d z (g . ray_d; through z_sample's coefficients into d near / d far).  The records
// of this path hold d_h1pre until the weight gradients have read them, so the ray and depth parts go straight into the
// outputs: d z has one writer per sample, the rest is summed per ray and frame in warp 0 (ray_sum_add, frame_sum_add).
__global__ void __launch_bounds__(NT, 1) decoder_dgrad_kernel(const BwdParams Q) {
    extern __shared__ __align__(16) float smem[];
    float* X = smem;                    // [64][356]
    float* Y = X + TP * LDX;            // [64][324]
    float* Ws = Y + TP * LDY;           // [KC][352]
    const RenderParams& P = Q.f;
    const int S = P.n_samples;
    const size_t npts = (size_t)P.batch * P.n_rays * S;
    const int tid = threadIdx.x;
    const float* wf = P.wf32;
    const GradRequest& q = Q.req;
    const bool frame_grads = q.sample_pos();
    FrameGradAcc acc;                   // warp 0: running per-frame sums of dR / dTh
    FrameGradAcc acc_bounds;            // warp 0: of d bounds[:, 0]
    for (size_t tile = blockIdx.x; tile * TP < npts; tile += gridDim.x) {
        const size_t p0 = tile * TP;
        auto gp = [&](int p) { return p0 + p; };
        auto in_range = [&](int p) { return p0 + p < npts; };
        // a. d_wpre[p][n] = (rgb_fc^T d_logits) * [w > 0]
        for (int i = tid; i < TP * kColor; i += NT) {
            const int p = i / kColor, n = i % kColor;
            float v = 0.f;
            if (in_range(p)) {
                const float* dr = Q.ws + gp(p) * kGradDim + kGradRaw;
                v = dr[0] * wf[oRgbW + n] + dr[1] * wf[oRgbW + kColor + n] + dr[2] * wf[oRgbW + 2 * kColor + n];
                if (!(Q.save[gp(p) * kSaveDim + kSaveW + n] > 0.f)) v = 0.f;
                Q.ws[gp(p) * kGradDim + kGradW + n] = v;
            }
            X[p * LDX + n] = v;
        }
        __syncthreads();
        // b. d_h2pre = (d_wpre Wc + alpha_fc^T d_sigma) * [h2 > 0]          Wc row-major [128][256] in the blob
        gemm_tile<kColor, kHidden, LDX, LDY>(X, Y, wf + oWc, Ws, [&](int p, int k, float v) {
            if (!in_range(p)) return 0.f;
            v += wf[oAlphaW + k] * Q.ws[gp(p) * kGradDim + kGradRaw + 3];
            if (!(Q.save[gp(p) * kSaveDim + kSaveH2 + k] > 0.f)) v = 0.f;
            Q.ws[gp(p) * kGradDim + kGradH2 + k] = v;
            return v;
        });
        // c. d_h1pre = (d_h2pre fc_2) * [h1 > 0]        fc_2.weight is [out=256][in=256] = the [K][N] this GEMM needs
        gemm_tile<kHidden, kHidden, LDY, LDX>(Y, X, Q.w.fc2_w, Ws, [&](int p, int k, float v) {
            if (!in_range(p) || !(Q.save[gp(p) * kSaveDim + kSaveH1 + k] > 0.f)) v = 0.f;
            if (in_range(p)) Q.ws[gp(p) * kGradDim + kGradH1 + k] = v;
            return v;
        });
        // d. d_h0pre = (d_h1pre fc_1) * [h0 > 0]
        gemm_tile<kHidden, kHidden, LDX, LDY>(X, Y, Q.w.fc1_w, Ws, [&](int p, int k, float v) {
            if (!in_range(p) || !(Q.save[gp(p) * kSaveDim + kSaveH0 + k] > 0.f)) v = 0.f;
            if (in_range(p)) Q.ws[gp(p) * kGradDim + kGradH0 + k] = v;
            return v;
        });
        // e. d_f = d_h0pre fc_0        ([256][352])
        gemm_tile<kHidden, kFeat, LDY, LDX>(Y, X, Q.w.fc0_w, Ws, [&](int, int, float v) { return v; });
        // f. backward of F.grid_sample (zeros padding): scatter-add into the NCDHW volume gradients and / or, for the frame
        // transform's gradients, d loss / d(canonical point) per (point, level) into Y (free after step e):
        // Y[p * 16 + 3 lvl + axis], the world point at + 12..14 and the frame (-1: none) at + 15
        if (Q.d_vol[0] || frame_grads) {
            for (int item = tid; item < TP * 4; item += NT) {   // (point, level): recompute the corner set-up
                const int p = item >> 2, lvl = item & 3;
                if (frame_grads && lvl == 0) Y[p * 16 + 15] = __int_as_float(-1);
                if (!in_range(p)) continue;
                const size_t g = gp(p);
                const size_t ri = g / S;
                const int s = (int)(g % S), b = (int)(ri / P.n_rays);
                // frame transform (threads of the same frame recompute it; cheap)
                FrameXf fx;
#pragma unroll
                for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
                const float z = z_sample(P.near[ri], P.far[ri], P.t_vals, s, S, P.t_rand ? P.t_rand + ri * S : nullptr, P.z_user ? P.z_user + ri * S : nullptr);
                const float wx = __fadd_rn(P.ray_o[ri * 3], __fmul_rn(P.ray_d[ri * 3], z));
                const float wy = __fadd_rn(P.ray_o[ri * 3 + 1], __fmul_rn(P.ray_d[ri * 3 + 1], z));
                const float wz = __fadd_rn(P.ray_o[ri * 3 + 2], __fmul_rn(P.ray_d[ri * 3 + 2], z));
                float gx, gy, gz;
                world_to_grid(fx, wx, wy, wz, gx, gy, gz);
                const int C = P.lvl_C[lvl], D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
                const int cbase = level_feature_base(lvl);
                Corners cn;
                corner_setup(unnormalize(gx, W), unnormalize(gy, H), unnormalize(gz, D), W, H, D, cn);
                if (Q.d_vol[0]) {
                    float* dv = Q.d_vol[lvl] + (size_t)b * C * D * H * W;
                    const size_t cs = (size_t)D * H * W;
                    for_each_corner(cn, W, H, D, [&](size_t vox, float wgt) {
                        for (int c = 0; c < C; ++c) {
                            const float dfv = X[p * LDX + cbase + c];
                            if (dfv != 0.f) atomicAdd(dv + (size_t)c * cs + vox, wgt * dfv);
                        }
                    });
                }
                if (frame_grads) {
                    float3 d = make_float3(0.f, 0.f, 0.f);
                    for (int q = cbase / 4; q < (cbase + C) / 4; ++q) {
                        const float4 df = *reinterpret_cast<const float4*>(X + p * LDX + 4 * q);
                        if (df.x == 0.f && df.y == 0.f && df.z == 0.f && df.w == 0.f) continue;
                        const float3 dq = gather_quad_dpos<float>(P, b, gx, gy, gz, q, df);
                        d.x += dq.x; d.y += dq.y; d.z += dq.z;
                    }
                    // d i / d g = (size - 1) / 2; the level-independent d g / d c is applied per point below
                    Y[p * 16 + 3 * lvl + 0] = d.x * (0.5f * (float)(W - 1));
                    Y[p * 16 + 3 * lvl + 1] = d.y * (0.5f * (float)(H - 1));
                    Y[p * 16 + 3 * lvl + 2] = d.z * (0.5f * (float)(D - 1));
                    if (lvl == 0) {
                        Y[p * 16 + 12] = wx; Y[p * 16 + 13] = wy; Y[p * 16 + 14] = wz;
                        Y[p * 16 + 15] = __int_as_float(b);
                    }
                }
            }
        }
        if (frame_grads) {   // warp 0: the tile's points -> dR / dTh terms, summed per frame
            __syncthreads();
            if (tid < 32) {
#pragma unroll 1
                for (int h = 0; h < TP / 32; ++h) {
                    const float* y = Y + (32 * h + tid) * 16;
                    const int b = __float_as_int(y[15]);
                    float t[12] = {};
                    float dcan[3] = {0.f, 0.f, 0.f};    // d loss / d(canonical point)
                    if (b >= 0) {
                        FrameXf fx;
#pragma unroll
                        for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
                        // levels summed in order; grid x / y / z pair with the dhw axes 2 / 1 / 0
                        dcan[0] = (((y[0] + y[3]) + y[6]) + y[9]) * grid_to_can_scale(fx, 2);
                        dcan[1] = (((y[1] + y[4]) + y[7]) + y[10]) * grid_to_can_scale(fx, 1);
                        dcan[2] = (((y[2] + y[5]) + y[8]) + y[11]) * grid_to_can_scale(fx, 0);
                        frame_grad_terms(fx, y[12], y[13], y[14], dcan[0], dcan[1], dcan[2], t);
                    }
                    if (q.d_R || q.d_Th) frame_sum_add(acc, b, t, tid, [&](FrameGradAcc& x) { frame_grad_flush(x, q.d_R, q.d_Th, tid); });
                    if (q.d_bounds) frame_sum_add(acc_bounds, b, dcan, tid, [&](FrameGradAcc& x) { bounds_grad_flush(x, q.d_bounds, tid); });
                    if (q.records()) {   // d loss / d(world point) through the grid: R dc = -(the dTh term)
                        const size_t g = gp(32 * h + tid);
                        const size_t ri = g / S;
                        const int s = (int)(g % S);
                        const unsigned int key = b < 0 ? ~0u : (unsigned int)ri;
                        const float gw[3] = {-t[9], -t[10], -t[11]};
                        if (q.d_ray_o || q.d_ray_d) {
                            const float z = b < 0 ? 0.f : z_sample(P.near[ri], P.far[ri], P.t_vals, s, S, P.t_rand ? P.t_rand + ri * S : nullptr,
                                                                   P.z_user ? P.z_user + ri * S : nullptr);
                            const float v[6] = {gw[0], gw[1], gw[2], z * gw[0], z * gw[1], z * gw[2]};
                            ray_sum_add(key, v, tid, [&](unsigned int r, int k, float sum) {
                                float* dst = k < 3 ? q.d_ray_o : q.d_ray_d;
                                if (dst) atomicAdd(dst + (size_t)r * 3 + k % 3, sum);
                            });
                        }
                        if (q.depths.any()) {   // the grid part of d z_i: one writer per sample, then per ray into d near / d far
                            const float v = b < 0 ? 0.f : fmaf(gw[2], P.ray_d[ri * 3 + 2], fmaf(gw[1], P.ray_d[ri * 3 + 1], gw[0] * P.ray_d[ri * 3]));
                            if (b >= 0 && q.depths.z) q.depths.z[g] += v;
                            if (q.depths.near || q.depths.far) {
                                float c[2] = {0.f, 0.f};
                                if (b >= 0) {
                                    z_sample_coefs(P.t_vals, s, S, P.t_rand ? P.t_rand + ri * S : nullptr, c[0], c[1]);
                                    c[0] *= v; c[1] *= v;
                                }
                                ray_sum_add(key, c, tid, [&](unsigned int r, int k, float sum) {
                                    float* dst = k ? q.depths.far : q.depths.near;
                                    if (dst) atomicAdd(dst + r, sum);
                                });
                            }
                        }
                    }
                }
            }
        }
        __syncthreads();
    }
    if (tid < 32) frame_grad_flush(acc, q.d_R, q.d_Th, tid);
    if (q.d_bounds && tid < 32) bounds_grad_flush(acc_bounds, q.d_bounds, tid);
}

// ------------------------------------------------------------------------------------------ 3. weight gradients
// dW[n * ldw + k] += sum_p A[p * lda + n] * Bm[p * ldb + k];  grid = (ceil(N/64), ceil(K/64), split over P)
__global__ void __launch_bounds__(256) wgrad_kernel(const float* __restrict__ A, int lda, const float* __restrict__ Bm, int ldb,
                                                    size_t npts, int N, int K, float* __restrict__ dW, int ldw) {
    __shared__ float As[16][65], Bs[16][65];
    const int n0 = blockIdx.x * 64, k0 = blockIdx.y * 64;
    const size_t per = (npts + gridDim.z - 1) / gridDim.z;
    const size_t pbeg = (size_t)blockIdx.z * per, pend = pbeg + per < npts ? pbeg + per : npts;
    const int tn = threadIdx.x >> 4, tk = threadIdx.x & 15;       // 16 x 16 threads, 4 x 4 outputs each
    float acc[4][4] = {};
    for (size_t p = pbeg; p < pend; p += 16) {
        for (int i = threadIdx.x; i < 16 * 64; i += 256) {
            const int pp = i >> 6, c = i & 63;
            const bool ok = p + pp < pend;
            As[pp][c] = (ok && n0 + c < N) ? A[(p + pp) * lda + n0 + c] : 0.f;
            Bs[pp][c] = (ok && k0 + c < K) ? Bm[(p + pp) * ldb + k0 + c] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int pp = 0; pp < 16; ++pp) {
            float a[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[pp][tn + 16 * i]; bv[i] = Bs[pp][tk + 16 * i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tn + 16 * i, k = k0 + tk + 16 * j;
            if (n < N && k < K && acc[i][j] != 0.f) atomicAdd(dW + (size_t)n * ldw + k, acc[i][j]);
        }
}

// out[seg * N + n] += sum_{p in segment seg} A[p * lda + n];  segments of seg_len consecutive points
__global__ void colsum_kernel(const float* __restrict__ A, int lda, size_t npts, size_t seg_len, int N, float* __restrict__ out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    const size_t per = (npts + gridDim.y - 1) / gridDim.y;
    const size_t pbeg = (size_t)blockIdx.y * per, pend = pbeg + per < npts ? pbeg + per : npts;
    size_t p = pbeg;
    while (p < pend) {
        const size_t seg = p / seg_len;
        const size_t send = (seg + 1) * seg_len < pend ? (seg + 1) * seg_len : pend;
        float acc = 0.f;
        for (; p < send; ++p) acc += A[p * lda + n];
        atomicAdd(out + seg * N + n, acc);
    }
}

// d view_fc[:, 256:283][n][j] += sum_rays (sum_s d_wpre[ray,s][n]) * PE4(viewdir(ray))[j];  block per ray, 128 threads
__global__ void view_wgrad_kernel(const BwdParams Q, float* __restrict__ d_view_w /* (128,346) */) {
    const RenderParams& P = Q.f;
    const size_t ri = blockIdx.x;
    const int n = threadIdx.x, S = P.n_samples;
    __shared__ float pe[kViewPE];
    if (n == 0) {
        const float dx = P.ray_d[ri * 3], dy = P.ray_d[ri * 3 + 1], dz = P.ray_d[ri * 3 + 2];
        const float nrm = ray_norm(dx, dy, dz);
        positional_embed<4>(__fdiv_rn(dx, nrm), __fdiv_rn(dy, nrm), __fdiv_rn(dz, nrm), [&](int j, float v) { pe[j] = v; });
    }
    __syncthreads();
    float acc = 0.f;
    for (int s = 0; s < S; ++s) acc += Q.ws[(ri * S + s) * kGradDim + kGradW + n];
    if (acc != 0.f)
        for (int j = 0; j < kViewPE; ++j) atomicAdd(d_view_w + n * 346 + 256 + j, acc * pe[j]);
}

// ------------------------------------------------------------------------------------------ 4. unfold Wc / bc
// Forward fold (nb_capi.cu): T = V L (V = view_fc[:, :256], L = latent_fc[:, :256]);  Wc = T F (F = feature_fc);
// u_b = Ll latent[idx_b] + b_l (Ll = latent_fc[:, 256:]);  bc_b = T b_f + V u_b + b_v.
// Inputs: dWcx (128,320) [cols 0..255 = dWc, 256..318 = d view_fc[:, 283:346]], dbc (B,128).
struct Unfold {
    nb_decoder_weights w;
    nb_decoder_weights g;            // gradient tensors (same shapes), accumulated into
    const float* dWcx;               // (128,320)
    const float* dbc;                // (B,128)
    float* T;                        // (128,256) scratch
    float* dT;                       // (128,256) scratch
    float* u;                        // (B,256) scratch
    float* du;                       // (B,256) scratch
};
#define NB_G(ptr) const_cast<float*>(ptr)

__global__ void unfold_stage1(const Unfold U) {     // T, u, d b_v, d view_fc[:, 283:346]
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = U.w.batch;
    if (idx < kColor * kHidden) {
        const int n = idx / kHidden, k = idx % kHidden;
        float acc = 0.f;
        for (int j = 0; j < kHidden; ++j) acc = fmaf(U.w.view_w[n * 346 + j], U.w.latent_w[j * 384 + k], acc);
        U.T[idx] = acc;
    } else if (idx < kColor * kHidden + B * kHidden) {
        const int r = idx - kColor * kHidden, b = r / kHidden, j = r % kHidden;
        const long long li = clamp_latent(U.w.latent_index[b], U.w.num_train_frame);
        float acc = U.w.latent_b[j];
        for (int i = 0; i < 128; ++i) acc = fmaf(U.w.latent_w[j * 384 + 256 + i], U.w.latent[li * 128 + i], acc);
        U.u[r] = acc;
    } else if (idx < kColor * kHidden + B * kHidden + kColor) {
        const int n = idx - kColor * kHidden - B * kHidden;
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc += U.dbc[b * kColor + n];
        NB_G(U.g.view_b)[n] += acc;
        for (int j = 0; j < kXyzPE; ++j) NB_G(U.g.view_w)[n * 346 + 283 + j] += U.dWcx[n * kColorK + kHidden + j];
    }
}
__global__ void unfold_stage2(const Unfold U) {     // dT, d feature_fc.W, d feature_fc.b, du
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = U.w.batch;
    if (idx < kColor * kHidden) {                    // dT[n][j] = sum_k dWc[n][k] F[j][k] + sum_b dbc[b][n] b_f[j]
        const int n = idx / kHidden, j = idx % kHidden;
        float acc = 0.f;
        for (int k = 0; k < kHidden; ++k) acc = fmaf(U.dWcx[n * kColorK + k], U.w.feature_w[j * kHidden + k], acc);
        for (int b = 0; b < B; ++b) acc = fmaf(U.dbc[b * kColor + n], U.w.feature_b[j], acc);
        U.dT[idx] = acc;
    } else if (idx < kColor * kHidden + kHidden * kHidden) {   // dF[j][k] = sum_n T[n][j] dWc[n][k]
        const int r = idx - kColor * kHidden, j = r / kHidden, k = r % kHidden;
        float acc = 0.f;
        for (int n = 0; n < kColor; ++n) acc = fmaf(U.T[n * kHidden + j], U.dWcx[n * kColorK + k], acc);
        NB_G(U.g.feature_w)[r] += acc;
    } else if (idx < kColor * kHidden + kHidden * kHidden + kHidden) {   // d b_f[j] = sum_b sum_n T[n][j] dbc[b][n]
        const int j = idx - kColor * kHidden - kHidden * kHidden;
        float acc = 0.f;
        for (int b = 0; b < B; ++b)
            for (int n = 0; n < kColor; ++n) acc = fmaf(U.T[n * kHidden + j], U.dbc[b * kColor + n], acc);
        NB_G(U.g.feature_b)[j] += acc;
    } else if (idx < kColor * kHidden + kHidden * kHidden + kHidden + B * kHidden) {   // du[b][j] = sum_n V[n][j] dbc[b][n]
        const int r = idx - kColor * kHidden - kHidden * kHidden - kHidden, b = r / kHidden, j = r % kHidden;
        float acc = 0.f;
        for (int n = 0; n < kColor; ++n) acc = fmaf(U.w.view_w[n * 346 + j], U.dbc[b * kColor + n], acc);
        U.du[r] = acc;
    }
}
__global__ void unfold_stage3(const Unfold U) {     // d view_fc[:, :256], d latent_fc, d latent, d b_l
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = U.w.batch;
    if (idx < kColor * kHidden) {                    // dV[n][j] = sum_k dT[n][k] L[j][k] + sum_b dbc[b][n] u[b][j]
        const int n = idx / kHidden, j = idx % kHidden;
        float acc = 0.f;
        for (int k = 0; k < kHidden; ++k) acc = fmaf(U.dT[n * kHidden + k], U.w.latent_w[j * 384 + k], acc);
        for (int b = 0; b < B; ++b) acc = fmaf(U.dbc[b * kColor + n], U.u[b * kHidden + j], acc);
        NB_G(U.g.view_w)[n * 346 + j] += acc;
    } else if (idx < kColor * kHidden + kHidden * 384) {
        const int r = idx - kColor * kHidden, j = r / 384, k = r % 384;
        float acc = 0.f;
        if (k < kHidden) {                           // dL[j][k] = sum_n V[n][j] dT[n][k]
            for (int n = 0; n < kColor; ++n) acc = fmaf(U.w.view_w[n * 346 + j], U.dT[n * kHidden + k], acc);
        } else {                                     // dLl[j][i] = sum_b du[b][j] latent[idx_b][i]
            for (int b = 0; b < B; ++b) {
                const long long li = clamp_latent(U.w.latent_index[b], U.w.num_train_frame);
                acc = fmaf(U.du[b * kHidden + j], U.w.latent[li * 128 + (k - kHidden)], acc);
            }
        }
        NB_G(U.g.latent_w)[r] += acc;
    } else if (idx < kColor * kHidden + kHidden * 384 + kHidden) {    // d b_l
        const int j = idx - kColor * kHidden - kHidden * 384;
        float acc = 0.f;
        for (int b = 0; b < B; ++b) acc += U.du[b * kHidden + j];
        NB_G(U.g.latent_b)[j] += acc;
    } else if (idx < kColor * kHidden + kHidden * 384 + kHidden + B * 128) {   // d latent[idx_b][i] += sum_j Ll[j][i] du[b][j]
        const int r = idx - kColor * kHidden - kHidden * 384 - kHidden, b = r / 128, i = r % 128;
        const long long li = clamp_latent(U.w.latent_index[b], U.w.num_train_frame);
        float acc = 0.f;
        for (int j = 0; j < kHidden; ++j) acc = fmaf(U.w.latent_w[j * 384 + 256 + i], U.du[b * kHidden + j], acc);
        atomicAdd(NB_G(U.g.latent) + li * 128 + i, acc);
    }
}

}  // namespace bwd

void launch_composite_bwd(const RenderParams& p, const float* raw, const GradRequest& req, float* d_raw_out, int d_raw_stride,
                          cudaStream_t stream) {
    bwd::BwdParams Q{};
    Q.f = p; Q.raw = raw; Q.req = req;
    Q.d_raw_out = d_raw_out; Q.d_raw_stride = d_raw_stride;
    const size_t nrays = (size_t)p.batch * p.n_rays;
    bwd::composite_bwd_kernel<<<(unsigned)((nrays + bwd::CB_WARPS - 1) / bwd::CB_WARPS), bwd::CB_WARPS * 32, 0, stream>>>(Q);
}

void launch_ray_grad(const RenderParams& p, const float* raw, const GradRequest& req, const float* rec, int rec_stride,
                     cudaStream_t stream) {
    bwd::BwdParams Q{};
    Q.f = p; Q.raw = raw; Q.req = req;
    const size_t nrays = (size_t)p.batch * p.n_rays;
    const unsigned grid = (unsigned)((nrays + bwd::CB_WARPS - 1) / bwd::CB_WARPS);
    if (req.depths.any()) bwd::ray_grad_kernel<true><<<grid, bwd::CB_WARPS * 32, 0, stream>>>(Q, rec, rec_stride);
    else bwd::ray_grad_kernel<false><<<grid, bwd::CB_WARPS * 32, 0, stream>>>(Q, rec, rec_stride);
}

int launch_unfold(const nb_decoder_weights& w, const nb_decoder_weights& g, const float* dWcx, const float* dbc, float* T, float* dT,
                  float* u, float* du, cudaStream_t stream) {
    bwd::Unfold U;
    U.w = w; U.g = g; U.dWcx = dWcx; U.dbc = dbc; U.T = T; U.dT = dT; U.u = u; U.du = du;
    const int B = w.batch;
    const int n1 = kColor * kHidden + B * kHidden + kColor;
    bwd::unfold_stage1<<<(n1 + 127) / 128, 128, 0, stream>>>(U);
    const int n2 = kColor * kHidden + kHidden * kHidden + kHidden + B * kHidden;
    bwd::unfold_stage2<<<(n2 + 127) / 128, 128, 0, stream>>>(U);
    const int n3 = kColor * kHidden + kHidden * 384 + kHidden + B * 128;
    bwd::unfold_stage3<<<(n3 + 127) / 128, 128, 0, stream>>>(U);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("unfold launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}
}  // namespace nb

using namespace nb;

extern "C" size_t nb_render_bwd_workspace_bytes(int batch, int n_rays, int n_samples) {
    const size_t npts = (size_t)batch * n_rays * n_samples;
    // per-point scratch + unfold scratch (dWcx, dbc, T, dT, u, du)
    return npts * kGradDim * 4 + ((size_t)kColor * kColorK + (size_t)batch * kColor + 2 * (size_t)kColor * kHidden +
                                  2 * (size_t)batch * kHidden) * 4 + 1024;
}
extern "C" size_t nb_render_save_bytes(int batch, int n_rays, int n_samples) {
    return (size_t)batch * n_rays * n_samples * kSaveDim * 4;
}

extern "C" size_t nb_render_save_bytes_for(const nb_render_args* f) {
    if (!f) return 0;
    if (f->precision == NB_PRECISION_TC_TF32X3) return train_save_bytes(f->batch, f->n_rays, f->n_samples);
    return nb_render_save_bytes(f->batch, f->n_rays, f->n_samples);
}
extern "C" size_t nb_render_bwd_workspace_bytes_for(const nb_render_args* f) {
    if (!f) return 0;
    if (f->precision != NB_PRECISION_TC_TF32X3) return nb_render_bwd_workspace_bytes(f->batch, f->n_rays, f->n_samples);
    RenderParams p;
    if (f->n_rays < 0 || f->n_samples <= 0 || fill_frame_params(f, "nb_render_bwd_workspace_bytes_for", &p) != NB_OK) return 0;
    return train_bwd_workspace_bytes(p, f->n_rays, f->n_samples);
}

extern "C" int nb_render_bwd(const nb_render_bwd_args* a, void* stream) { return nb_render_bwd_frame(a, nullptr, nullptr, stream); }

extern "C" int nb_render_bwd_frame(const nb_render_bwd_args* a, float* d_R, float* d_Th, void* stream) {
    return nb_render_bwd_rays(a, d_R, d_Th, nullptr, nullptr, stream);
}

extern "C" int nb_render_bwd_rays(const nb_render_bwd_args* a, float* d_R, float* d_Th, float* d_ray_o, float* d_ray_d, void* stream) {
    return nb_render_bwd_maps(a, nullptr, nullptr, d_R, d_Th, d_ray_o, d_ray_d, stream);
}

extern "C" int nb_render_bwd_maps(const nb_render_bwd_args* a, const float* d_disp_map, const float* d_weights, float* d_R,
                                  float* d_Th, float* d_ray_o, float* d_ray_d, void* stream) {
    nb_render_input_grads g{};
    g.d_R = d_R; g.d_Th = d_Th; g.d_ray_o = d_ray_o; g.d_ray_d = d_ray_d;
    return nb_render_bwd_inputs(a, d_disp_map, d_weights, &g, stream);
}

extern "C" int nb_render_bwd_inputs(const nb_render_bwd_args* a, const float* d_disp_map, const float* d_weights,
                                    const nb_render_input_grads* in, void* stream) {
    if (!a || !a->fwd || !a->save || !a->raw || !a->workspace || !a->weights || !a->grads) {
        set_error("nb_render_bwd: null argument");
        return NB_ERR_BAD_ARG;
    }
    const nb_render_input_grads none{};
    if (!in) in = &none;
    const GradRequest req{{a->d_rgb_map, a->d_depth_map, a->d_acc_map, d_disp_map, d_weights}, in->d_R, in->d_Th, in->d_ray_o,
                          in->d_ray_d, {in->d_near, in->d_far, in->d_z_vals}, in->d_bounds};
    const nb_render_args* f = a->fwd;
    if (f->z_vals && (in->d_near || in->d_far)) {
        set_error("nb_render_bwd: d_near / d_far need a forward that derived its depths from near / far (z_vals was given: "
                  "ask for d_z_vals)");
        return NB_ERR_BAD_ARG;
    }
    RenderParams p;
    int st = fill_frame_params(f, "nb_render_bwd", &p);
    if (st == NB_OK) st = fill_ray_params(f, "nb_render_bwd", &p);
    if (st != NB_OK) return st;
    if (f->n_samples > bwd::kBwdMaxSamples) { set_error("nb_render_bwd: n_samples <= %d supported (got %d)", bwd::kBwdMaxSamples, f->n_samples); return NB_ERR_UNSUPPORTED; }
    if (f->precision == NB_PRECISION_TC_TF32X3) {
        if (a->workspace_bytes < train_bwd_workspace_bytes(p, f->n_rays, f->n_samples)) { set_error("nb_render_bwd: workspace too small (see nb_render_bwd_workspace_bytes_for)"); return NB_ERR_BAD_ARG; }
        trn::TrainBwd t;
        t.save = a->save; t.raw = a->raw; t.req = req;
        t.weights = a->weights; t.grads = a->grads; t.workspace = (float*)a->workspace;
        for (int l = 0; l < 4; ++l) t.d_vol[l] = a->d_volumes[l];
        t.volume_dtype = f->volume_dtype;
        return launch_train_bwd(p, t, (cudaStream_t)stream);
    }
    if (f->precision != NB_PRECISION_FP32 || f->volume_dtype != NB_DTYPE_F32) {
        set_error("nb_render_bwd: the training path runs the exact kernel (NB_PRECISION_FP32 + fp32 volume)");
        return NB_ERR_UNSUPPORTED;
    }
    if (a->workspace_bytes < nb_render_bwd_workspace_bytes(f->batch, f->n_rays, f->n_samples)) {
        set_error("nb_render_bwd: workspace too small");
        return NB_ERR_BAD_ARG;
    }
    bwd::BwdParams Q{};
    Q.f = p;
    Q.save = a->save; Q.raw = a->raw; Q.req = req;
    Q.ws = (float*)a->workspace;
    Q.w = *a->weights;
    for (int l = 0; l < 4; ++l) Q.d_vol[l] = a->d_volumes[l];
    cudaStream_t s = (cudaStream_t)stream;
    const size_t nrays = (size_t)f->batch * f->n_rays, npts = nrays * f->n_samples;
    if (npts == 0) return NB_OK;
    const nb_decoder_weights& g = *a->grads;

    launch_composite_bwd(p, a->raw, req, Q.ws + kGradRaw, kGradDim, s);

    const size_t smem = ((size_t)bwd::TP * bwd::LDX + (size_t)bwd::TP * bwd::LDY + (size_t)bwd::KC * kFeat) * 4;
    const size_t ntiles = (npts + bwd::TP - 1) / bwd::TP;
    const unsigned dgrad_grid = (unsigned)(ntiles < kGridSMs ? ntiles : kGridSMs);
    cudaFuncSetAttribute(bwd::decoder_dgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    bwd::decoder_dgrad_kernel<<<dgrad_grid, bwd::NT, smem, s>>>(Q);

    // scratch after the per-point region
    float* extra = Q.ws + npts * kGradDim;
    float* dWcx = extra;                               extra += (size_t)kColor * kColorK;
    float* dbc = extra;                                extra += (size_t)f->batch * kColor;
    float* T = extra;                                  extra += (size_t)kColor * kHidden;
    float* dT = extra;                                 extra += (size_t)kColor * kHidden;
    float* u = extra;                                  extra += (size_t)f->batch * kHidden;
    float* du = extra;
    cudaMemsetAsync(dWcx, 0, ((size_t)kColor * kColorK + (size_t)f->batch * kColor) * 4, s);

    const int split = 64;
    auto wgrad = [&](int goff, int N, int soff, int K, float* dW, int ldw) {
        dim3 grid((N + 63) / 64, (K + 63) / 64, split);
        bwd::wgrad_kernel<<<grid, 256, 0, s>>>(Q.ws + goff, kGradDim, Q.save + soff, kSaveDim, npts, N, K, dW, ldw);
    };
    wgrad(kGradH0, kHidden, kSaveF, kFeat, NB_G(g.fc0_w), kFeat);
    wgrad(kGradH1, kHidden, kSaveH0, kHidden, NB_G(g.fc1_w), kHidden);
    wgrad(kGradH2, kHidden, kSaveH1, kHidden, NB_G(g.fc2_w), kHidden);
    wgrad(kGradW, kColor, kSaveH2, kColorK, dWcx, kColorK);
    wgrad(kGradRaw, 3, kSaveW, kColor, NB_G(g.rgb_w), kColor);
    wgrad(kGradRaw + 3, 1, kSaveH2, kHidden, NB_G(g.alpha_w), kHidden);
    auto colsum = [&](int goff, int N, float* out, size_t seg) {
        dim3 grid((N + 127) / 128, 32);
        bwd::colsum_kernel<<<grid, 128, 0, s>>>(Q.ws + goff, kGradDim, npts, seg, N, out);
    };
    colsum(kGradH0, kHidden, NB_G(g.fc0_b), npts);
    colsum(kGradH1, kHidden, NB_G(g.fc1_b), npts);
    colsum(kGradH2, kHidden, NB_G(g.fc2_b), npts);
    colsum(kGradRaw, 3, NB_G(g.rgb_b), npts);
    colsum(kGradRaw + 3, 1, NB_G(g.alpha_b), npts);
    colsum(kGradW, kColor, dbc, (size_t)f->n_rays * f->n_samples);           // per frame
    bwd::view_wgrad_kernel<<<(unsigned)nrays, kColor, 0, s>>>(Q, NB_G(g.view_w));

    st = launch_unfold(*a->weights, g, dWcx, dbc, T, dT, u, du, s);
    if (st != NB_OK) return st;
    if (req.records()) {   // the encodings' part per point into the d_h1pre columns (read by the weight / bias gradients above), then per ray
        float* rec = Q.ws + kGradH1;
        bwd::pe_grad_kernel<<<(unsigned)((npts + bwd::PG_WARPS - 1) / bwd::PG_WARPS < (size_t)kGridSMs * 16
                                             ? (npts + bwd::PG_WARPS - 1) / bwd::PG_WARPS : (size_t)kGridSMs * 16),
                              bwd::PG_WARPS * 32, 0, s>>>(Q, rec, kGradDim);
        launch_ray_grad(p, a->raw, req, rec, kGradDim, s);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_render_bwd: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

// ------------------------------------------------------------------------------------------------ diagnostics
// The per-ray stages around the decoder on caller-made raw records: composite_kernel (the maps and weights of a render) and
// composite_bwd_kernel / ray_grad_kernel (d raw, and the ray and depth gradients) exactly as the render calls launch them.
// tests/test_ray_stages_gpu.py compares them with a float64 raw2outputs.
static int debug_composite_params(const nb_render_args* a, const float* raw, const char* who, int max_samples, RenderParams* p) {
    if (!a || !raw) { set_error("%s: null args or raw", who); return NB_ERR_BAD_ARG; }
    if (a->batch <= 0) { set_error("%s: batch must be > 0", who); return NB_ERR_BAD_ARG; }
    *p = RenderParams{};
    p->batch = a->batch;
    const int st = fill_ray_params(a, who, p);
    if (st != NB_OK) return st;
    if (a->n_samples > max_samples) { set_error("%s: n_samples <= %d supported (got %d)", who, max_samples, a->n_samples); return NB_ERR_UNSUPPORTED; }
    p->stats = nullptr; p->trace = nullptr; p->save = nullptr;
    return NB_OK;
}

extern "C" int nb_debug_composite(const nb_render_args* a, const float* raw, void* stream) {
    RenderParams p;
    const int st = debug_composite_params(a, raw, "nb_debug_composite", kListMaxSamples, &p);
    if (st != NB_OK) return st;
    if (p.n_rays == 0) return NB_OK;
    for (int b = 0; b < p.batch; ++b) {
        p.frame = b;
        p.raw_ws = reinterpret_cast<float4*>(const_cast<float*>(raw)) + (size_t)b * p.n_rays * p.n_samples;
        launch_composite(p, (cudaStream_t)stream);
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_debug_composite: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

extern "C" int nb_debug_composite_bwd(const nb_render_args* a, const float* raw, const float* d_rgb_map, const float* d_depth_map,
                                      const float* d_acc_map, const float* d_disp_map, const float* d_weights, const float* rec,
                                      const nb_render_input_grads* in, float* d_raw, void* stream) {
    const char* who = "nb_debug_composite_bwd";
    RenderParams p;
    int st = debug_composite_params(a, raw, who, bwd::kBwdMaxSamples, &p);
    if (st != NB_OK) return st;
    if (!d_raw) { set_error("%s: d_raw is null", who); return NB_ERR_BAD_ARG; }
    const nb_render_input_grads none{};
    if (!in) in = &none;
    if (in->d_R || in->d_Th || in->d_bounds) { set_error("%s: d_R, d_Th and d_bounds need the decoder (nb_render_bwd_inputs)", who); return NB_ERR_BAD_ARG; }
    const GradRequest req{{d_rgb_map, d_depth_map, d_acc_map, d_disp_map, d_weights}, nullptr, nullptr, in->d_ray_o, in->d_ray_d,
                          {in->d_near, in->d_far, in->d_z_vals}, nullptr};
    if (req.records() && !rec) { set_error("%s: the ray and depth gradients need the per-sample record", who); return NB_ERR_BAD_ARG; }
    if (a->z_vals && (in->d_near || in->d_far)) { set_error("%s: d_near / d_far need depths derived from near / far (z_vals was given)", who); return NB_ERR_BAD_ARG; }
    if (p.n_rays == 0) return NB_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    launch_composite_bwd(p, raw, req, d_raw, 4, s);
    if (req.records()) launch_ray_grad(p, raw, req, rec, 8, s);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}
