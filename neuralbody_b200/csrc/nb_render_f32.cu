// Exact-fp32 fused render kernel (NB_PRECISION_FP32).
//
// One launch covers everything Renderer.render's chunk loop does upstream
// (lib/networks/renderer/if_clight_renderer.py:107-120): sampling, world->SMPL->grid,
// 4-level trilinear gather from the channels-last packed volume, the decoder MLP in
// fp32 FFMA, positional encodings, and the alpha composite.  No activation ever leaves
// shared memory.  This is the GPU-side oracle and the fallback for shapes the tensor-core
// kernel does not take; its roofline is the fp32 FFMA pipe, not the tensor cores.
//
// CTA = 256 threads, persistent over "groups" (one or more whole rays = <=64 sample
// points per tile).  Shared-memory plan (floats):
//   X [64][356]   gathered features (352) / fc_1 output / colour-layer output
//   Y [64][324]   fc_0, fc_2 outputs (cols 0..255) + PE(xyz) (cols 256..318) + 0 (col 319)
//   Ws[2][16][256] cp.async double buffer of the K-major weight stream
// Row strides 356 / 324 are == 4 (mod 32) so that the 8 interleaved point rows a
// thread owns (p = pg + 8 i) hit 8 distinct 16-byte bank groups.
#include "nb_device.cuh"

namespace nb {
namespace f32 {

constexpr int TP = 64;        // points per tile
constexpr int NT = 256;       // threads per CTA
constexpr int LDX = 356;
constexpr int LDY = 324;
constexpr int KC = 16;        // K rows per weight chunk

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// out[p][n] = act( sum_k Xs[p][k] * Wt[k][n] + bias[n] (+ vt[pray[p]][n]) )
// thread (pg = tid&7, ng = tid>>3) owns points pg + 8 i (i<8) and outputs ng*TN .. +TN.
template <int K, int N, int LDI, int LDO, bool RELU, bool RAYBIAS>
__device__ __forceinline__ void mlp_layer(const float* __restrict__ Xs, float* __restrict__ Ys,
                                          const float* __restrict__ Wt, const float* __restrict__ bias,
                                          float* __restrict__ Ws, const float* __restrict__ vt,
                                          const int* __restrict__ pray) {
    static_assert(K % KC == 0, "K must be a multiple of the chunk");
    constexpr int TN = N / 32;
    constexpr int NCHUNK = K / KC;
    constexpr int PIECES = KC * N / 4;    // float4 pieces per chunk
    const int tid = threadIdx.x;
    const int pg = tid & 7, ng = tid >> 3;
    const int n0 = ng * TN;

    float acc[8][TN];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int t = 0; t < TN; ++t) acc[i][t] = 0.f;

    auto load_chunk = [&](int c, int buf) {
        const float4* src = reinterpret_cast<const float4*>(Wt + (size_t)c * KC * N);
        float4* dst = reinterpret_cast<float4*>(Ws + buf * KC * 256);
#pragma unroll
        for (int i = tid; i < PIECES; i += NT) cp_async16(dst + i, src + i);
        cp_async_commit();
    };

    load_chunk(0, 0);
    for (int c = 0; c < NCHUNK; ++c) {
        if (c + 1 < NCHUNK) {
            load_chunk(c + 1, (c + 1) & 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* wb = Ws + (c & 1) * KC * 256;
#pragma unroll
        for (int kk = 0; kk < KC; kk += 4) {
            float4 a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i)
                a[i] = *reinterpret_cast<const float4*>(Xs + (pg + 8 * i) * LDI + c * KC + kk);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float w[TN];
#pragma unroll
                for (int t = 0; t < TN; t += 4) {
                    float4 wv = *reinterpret_cast<const float4*>(wb + (kk + j) * N + n0 + t);
                    w[t] = wv.x; w[t + 1] = wv.y; w[t + 2] = wv.z; w[t + 3] = wv.w;
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float av = (j == 0) ? a[i].x : (j == 1) ? a[i].y : (j == 2) ? a[i].z : a[i].w;
#pragma unroll
                    for (int t = 0; t < TN; ++t) acc[i][t] = fmaf(av, w[t], acc[i][t]);
                }
            }
        }
        __syncthreads();
    }

    float bv[TN];
#pragma unroll
    for (int t = 0; t < TN; ++t) bv[t] = __ldg(bias + n0 + t);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int p = pg + 8 * i;
        const float* vrow = RAYBIAS ? (vt + pray[p] * kColor + n0) : nullptr;
#pragma unroll
        for (int t = 0; t < TN; t += 4) {
            float4 o;
            float v0 = acc[i][t] + bv[t], v1 = acc[i][t + 1] + bv[t + 1];
            float v2 = acc[i][t + 2] + bv[t + 2], v3 = acc[i][t + 3] + bv[t + 3];
            if (RAYBIAS) { v0 += vrow[t]; v1 += vrow[t + 1]; v2 += vrow[t + 2]; v3 += vrow[t + 3]; }
            if (RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
            o.x = v0; o.y = v1; o.z = v2; o.w = v3;
            *reinterpret_cast<float4*>(Ys + p * LDO + n0 + t) = o;
        }
    }
    __syncthreads();
}

// Trilinear gather of one 64-point tile: work item = (point, channel quad); lanes run over the quads of one corner => contiguous
// 16-byte loads.  gcoord = [64][3] grid coords, X = [64][LDX].
template <typename VT>
__device__ __forceinline__ void gather_tile(const RenderParams& P, int b, const float* __restrict__ gcoord, float* __restrict__ X) {
    constexpr int QUADS = kFeat / 4;   // 88 per point
    for (int item = threadIdx.x; item < TP * QUADS; item += NT) {
        const int p = item / QUADS, q = item % QUADS;
        *reinterpret_cast<float4*>(X + p * LDX + q * 4) = gather_quad<VT>(P, b, gcoord[p * 3 + 0], gcoord[p * 3 + 1], gcoord[p * 3 + 2], q);
    }
}

// sigma = alpha_fc h2 of tile point tid / 4, h2 = its row of Y: four threads per point, each over every fourth channel
__device__ __forceinline__ float alpha_head(const float* __restrict__ Y, const float* __restrict__ wf, int tid) {
    const int p = tid >> 2, q = tid & 3;
    float acc = 0.f;
#pragma unroll 8
    for (int k = q; k < kHidden; k += 4) acc = fmaf(Y[p * LDY + k], __ldg(wf + oAlphaW + k), acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    return acc + __ldg(wf + oAlphaB);
}

struct RayInfo {
    float o[3], d[3], near, far, norm, vd[3];
};

// Work items of render_f32_kernel: groups of whole rays, 64 / S rays in one tile when S <= 64, else one ray of ceil(S / 64)
// tiles.  rays / tiles per group, groups per frame / in the launch.
struct Groups { int rays, tiles, per_frame, total; };

template <typename VT>
__global__ void __launch_bounds__(NT, 1) render_f32_kernel(const __grid_constant__ RenderParams P, const Groups grp) {
    extern __shared__ __align__(16) float smem[];
    float* X = smem;                           // [64][356]
    float* Y = X + TP * LDX;                   // [64][324]
    float* Ws = Y + TP * LDY;                  // [2][16][256]
    float* gcoord = Ws + 2 * KC * 256;         // [64][3] grid coords (x,y,z)
    int* pray = reinterpret_cast<int*>(gcoord + TP * 3);   // [64] local ray of each tile point (-1 = padding)
    int* prayc = pray + TP;                                // [64] same, padding clamped to ray 0
    int* pins = prayc + TP;                                // [64] f-1: sample projects into every mask view
    float* vt = reinterpret_cast<float*>(pins + TP);       // [G][128] per-ray view term
    const int G = grp.rays, S = P.n_samples;
    float* zbuf = vt + G * kColor;             // [G][S]
    float4* rawbuf = reinterpret_cast<float4*>(zbuf + ((G * S + 3) & ~3));  // [G][S]
    RayInfo* rays = reinterpret_cast<RayInfo*>(rawbuf + G * S);            // [G]
    __shared__ FrameXf xf;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float* wf = P.wf32;

    for (int g = blockIdx.x; g < grp.total; g += gridDim.x) {
        const int b = g / grp.per_frame;
        const int r0 = (g % grp.per_frame) * G;
        const int nr = min(G, P.n_rays - r0);

        // ---- per-frame transform + per-ray set-up
        load_frame_xf(P, b, xf, tid);
        if (tid < nr) {
            const size_t ri = (size_t)b * P.n_rays + r0 + tid;
            RayInfo& r = rays[tid];
#pragma unroll
            for (int j = 0; j < 3; ++j) { r.o[j] = __ldg(P.ray_o + ri * 3 + j); r.d[j] = __ldg(P.ray_d + ri * 3 + j); }
            r.near = __ldg(P.near + ri); r.far = __ldg(P.far + ri);
            r.norm = ray_norm(r.d[0], r.d[1], r.d[2]);
#pragma unroll
            for (int j = 0; j < 3; ++j) r.vd[j] = __fdiv_rn(r.d[j], r.norm);   // if_clight_renderer.py:68
        }
        __syncthreads();
        // view term vt[ray][n] = sum_j Wv^T[j][n] * PE4(viewdir)[j]   (per ray, not per sample)
        for (int idx = tid; idx < nr * kColor; idx += NT) {
            const int ry = idx / kColor, n = idx % kColor;
            float pe[kViewPE];
            positional_embed<4>(rays[ry].vd[0], rays[ry].vd[1], rays[ry].vd[2], [&](int j, float v) { pe[j] = v; });
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < kViewPE; ++j) acc = fmaf(pe[j], __ldg(wf + oWvt + j * kColor + n), acc);
            vt[idx] = acc;
        }

        for (int tile = 0; tile < grp.tiles; ++tile) {
            // ---- phase 1: geometry of the tile's points (one thread per point)
            if (tid < TP) {
                const int pgidx = tile * TP + tid;
                const int ry = pgidx / S, s = pgidx % S;
                const bool valid = ry < nr;
                pray[tid] = valid ? ry : -1;
                prayc[tid] = valid ? ry : 0;
                pins[tid] = 1;
                float* yrow = Y + tid * LDY + kHidden;
                if (valid) {
                    const RayInfo& r = rays[ry];
                    const size_t ri = (size_t)b * P.n_rays + r0 + ry;
                    const float z = z_sample(r.near, r.far, P.t_vals, s, S, P.t_rand ? P.t_rand + ri * S : nullptr, P.z_user ? P.z_user + ri * S : nullptr);
                    zbuf[ry * S + s] = z;
                    // pts = ray_o + ray_d * z   (if_clight_renderer.py:25)
                    const float wx = __fadd_rn(r.o[0], __fmul_rn(r.d[0], z));
                    const float wy = __fadd_rn(r.o[1], __fmul_rn(r.d[1], z));
                    const float wz = __fadd_rn(r.o[2], __fmul_rn(r.d[2], z));
                    float gx, gy, gz;
                    world_to_grid(xf, wx, wy, wz, gx, gy, gz);
                    if (P.mask_nv > 0) pins[tid] = inside_masks(P, xf, wx, wy, wz) ? 1 : 0;
                    gcoord[tid * 3 + 0] = gx; gcoord[tid * 3 + 1] = gy; gcoord[tid * 3 + 2] = gz;
                    positional_embed<10>(wx, wy, wz, [&](int j, float v) { yrow[j] = v; });   // PE of WORLD xyz (latent_xyzc.py:115)
                    yrow[kXyzPE] = 0.f;
                } else {
#pragma unroll 4
                    for (int j = 0; j < 64; ++j) yrow[j] = 0.f;
                    gcoord[tid * 3 + 0] = gcoord[tid * 3 + 1] = gcoord[tid * 3 + 2] = -4.f;   // outside => zero features
                }
            }
            __syncthreads();

            // ---- phase 2: trilinear gather (a7)
            gather_tile<VT>(P, b, gcoord, X);
            __syncthreads();

            // training forward: keep the per-point activations the backward pass needs (nb_render_bwd)
            // row p of the save buffer: [f 352 | h0 256 | h1 256 | h2 256 + PE 64 | w 128]
            auto save_rows = [&](const float* src, int ld, int width, int col0) {
                if (!P.save) return;
                for (int i = tid; i < TP * width; i += NT) {
                    const int p = i / width, c = i % width;
                    if (pray[p] >= 0) {
                        const size_t gp = ((size_t)b * P.n_rays + r0) * S + (size_t)tile * TP + p;
                        P.save[gp * kSaveDim + col0 + c] = src[p * ld + c];
                    }
                }
            };
            save_rows(X, LDX, kFeat, kSaveF);

            // ---- decoder (a8)
            mlp_layer<kFeat, kHidden, LDX, LDY, true, false>(X, Y, wf + oW0t, wf + oB0, Ws, nullptr, nullptr);
            save_rows(Y, LDY, kHidden, kSaveH0);
            mlp_layer<kHidden, kHidden, LDY, LDX, true, false>(Y, X, wf + oW1t, wf + oB1, Ws, nullptr, nullptr);
            save_rows(X, LDX, kHidden, kSaveH1);
            mlp_layer<kHidden, kHidden, LDX, LDY, true, false>(X, Y, wf + oW2t, wf + oB2, Ws, nullptr, nullptr);
            save_rows(Y, LDY, kColorK, kSaveH2);
            {
                const int p = tid >> 2;
                const float sigma = alpha_head(Y, wf, tid);
                if ((tid & 3) == 0 && pray[p] >= 0) reinterpret_cast<float*>(rawbuf + tile * TP + p)[3] = sigma;
            }
            // w = relu(Wc h2 + Wx PE(xyz) + bc + vt[ray]); padding rows borrow ray 0's view term (discarded)
            __syncthreads();
            mlp_layer<kColorK, kColor, LDY, LDX, true, true>(Y, X, wf + oWct, P.bc + b * kColor, Ws, vt, prayc);
            save_rows(X, LDX, kColor, kSaveW);
            {   // rgb = rgb_fc w: 4 threads per point, 3 outputs
                const int p = tid >> 2, q = tid & 3;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll 8
                for (int k = q; k < kColor; k += 4) {
                    const float xv = X[p * LDX + k];
                    a0 = fmaf(xv, __ldg(wf + oRgbW + k), a0);
                    a1 = fmaf(xv, __ldg(wf + oRgbW + kColor + k), a1);
                    a2 = fmaf(xv, __ldg(wf + oRgbW + 2 * kColor + k), a2);
                }
                a0 += __shfl_xor_sync(0xffffffffu, a0, 1); a0 += __shfl_xor_sync(0xffffffffu, a0, 2);
                a1 += __shfl_xor_sync(0xffffffffu, a1, 1); a1 += __shfl_xor_sync(0xffffffffu, a1, 2);
                a2 += __shfl_xor_sync(0xffffffffu, a2, 1); a2 += __shfl_xor_sync(0xffffffffu, a2, 2);
                if (q == 0 && pray[p] >= 0) {
                    float* rw = reinterpret_cast<float*>(rawbuf + tile * TP + p);
                    rw[0] = a0 + __ldg(wf + oRgbB + 0);
                    rw[1] = a1 + __ldg(wf + oRgbB + 1);
                    rw[2] = a2 + __ldg(wf + oRgbB + 2);
                }
            }
            __syncthreads();
            if (P.mask_nv > 0 && tid < TP && pray[tid] >= 0 && !pins[tid])      // if_clight_renderer_mmsk.py:54-59: raw = 0 outside
                rawbuf[tile * TP + tid] = make_float4(0.f, 0.f, 0.f, 0.f);
            __syncthreads();
        }

        // ---- composite (a10): one warp per ray
        for (int ry = warp; ry < nr; ry += NT / 32) {
            const size_t ri = (size_t)b * P.n_rays + r0 + ry;
            float* wout = P.weights ? P.weights + ri * S : nullptr;
            RayOut o = composite_ray(rawbuf + ry * S, zbuf + ry * S, S, rays[ry].norm, wout, lane);
            if (P.raw) {
                float4* rdst = reinterpret_cast<float4*>(P.raw) + ri * S;
                for (int s = lane; s < S; s += 32) rdst[s] = rawbuf[ry * S + s];
            }
            if (lane == 0) store_ray_outputs(P, ri, o);
        }
        __syncthreads();
    }
}

// f-3: density only, on arbitrary world points (Network.calculate_density, latent_xyzc.py:74-89; the mesh renderer's
// alpha decoder, if_mesh_renderer.py:36-39): gather -> fc_0 -> fc_1 -> fc_2 -> alpha_fc.  64 points per tile.
template <typename VT>
__global__ void __launch_bounds__(NT, 1) density_f32_kernel(const __grid_constant__ RenderParams P, const float* __restrict__ pts,
                                                            int n_points, float* __restrict__ sigma) {
    extern __shared__ __align__(16) float smem[];
    float* X = smem;
    float* Y = X + TP * LDX;
    float* Ws = Y + TP * LDY;
    float* gcoord = Ws + 2 * KC * 256;
    __shared__ FrameXf xf;
    const int tid = threadIdx.x;
    const float* wf = P.wf32;
    const int tiles_per_frame = (n_points + TP - 1) / TP;
    for (int t = blockIdx.x; t < tiles_per_frame * P.batch; t += gridDim.x) {
        const int b = t / tiles_per_frame, p0 = (t % tiles_per_frame) * TP;
        load_frame_xf(P, b, xf, tid);
        __syncthreads();
        if (tid < TP) {
            float gx = -4.f, gy = -4.f, gz = -4.f;
            if (p0 + tid < n_points) {
                const float* w = pts + ((size_t)b * n_points + p0 + tid) * 3;
                world_to_grid(xf, __ldg(w), __ldg(w + 1), __ldg(w + 2), gx, gy, gz);
            }
            gcoord[tid * 3 + 0] = gx; gcoord[tid * 3 + 1] = gy; gcoord[tid * 3 + 2] = gz;
        }
        __syncthreads();
        gather_tile<VT>(P, b, gcoord, X);
        __syncthreads();
        mlp_layer<kFeat, kHidden, LDX, LDY, true, false>(X, Y, wf + oW0t, wf + oB0, Ws, nullptr, nullptr);
        mlp_layer<kHidden, kHidden, LDY, LDX, true, false>(Y, X, wf + oW1t, wf + oB1, Ws, nullptr, nullptr);
        mlp_layer<kHidden, kHidden, LDX, LDY, true, false>(X, Y, wf + oW2t, wf + oB2, Ws, nullptr, nullptr);
        {
            const int p = tid >> 2;
            const float sg = alpha_head(Y, wf, tid);
            if ((tid & 3) == 0 && p0 + p < n_points) sigma[(size_t)b * n_points + p0 + p] = sg;
        }
        __syncthreads();
    }
}

size_t smem_bytes(int G, int S) {
    size_t fl = (size_t)TP * LDX + (size_t)TP * LDY + 2 * KC * 256 + TP * 3 + 3 * TP /*pray, prayc, pins*/ + (size_t)G * kColor +
                (size_t)((G * S + 3) & ~3);
    return fl * 4 + (size_t)G * S * 16 + (size_t)G * sizeof(RayInfo) + 16;
}

}  // namespace f32

// kernel<float> or kernel<__half> by the volume dtype: a persistent grid of min(work items, SMs) CTAs of NT threads with smem
// bytes of dynamic shared memory
template <typename Kernel, typename... Args>
static int launch_by_dtype(const char* name, Kernel k32, Kernel k16, int volume_dtype, int work, size_t smem, cudaStream_t stream,
                           Args... args) {
    if (work == 0) return NB_OK;
    const int sms = sm_count(), grid = work < sms ? work : sms;
    const Kernel kernel = volume_dtype == NB_DTYPE_F32 ? k32 : k16;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) {
        kernel<<<grid, f32::NT, smem, stream>>>(args...);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s launch failed: %s", name, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int launch_render_f32(const RenderParams& p, int volume_dtype, cudaStream_t stream) {
    const int S = p.n_samples;
    f32::Groups grp;
    if (S <= f32::TP) { grp.rays = f32::TP / S; grp.tiles = 1; }
    else { grp.rays = 1; grp.tiles = (S + f32::TP - 1) / f32::TP; }
    grp.per_frame = (p.n_rays + grp.rays - 1) / grp.rays;
    grp.total = grp.per_frame * p.batch;
    const size_t smem = f32::smem_bytes(grp.rays, S);
    if (smem > 227 * 1024) { set_error("n_samples=%d needs %zu B of shared memory (> 227 KB)", S, smem); return NB_ERR_UNSUPPORTED; }
    return launch_by_dtype("render_f32", f32::render_f32_kernel<float>, f32::render_f32_kernel<__half>, volume_dtype,
                           grp.total, smem, stream, p, grp);
}

int launch_density_f32(const RenderParams& p, int volume_dtype, const float* pts, int n_points, float* sigma, cudaStream_t stream) {
    const size_t smem = ((size_t)f32::TP * f32::LDX + (size_t)f32::TP * f32::LDY + 2 * f32::KC * 256 + f32::TP * 3) * 4;
    const int tiles = ((n_points + f32::TP - 1) / f32::TP) * p.batch;
    return launch_by_dtype("density_f32", f32::density_f32_kernel<float>, f32::density_f32_kernel<__half>, volume_dtype,
                           tiles, smem, stream, p, pts, n_points, sigma);
}

}  // namespace nb
