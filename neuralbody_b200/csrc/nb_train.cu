// Training path on the tensor cores (NB_PRECISION_TC_TF32X3): forward with an activation record + backward of the fused
// render over the COMPACT SAMPLE LIST, as chains of wgmma GEMMs.
//
// Upstream a training step is Trainer.train (lib/train/trainers/trainer.py:46-53) -> NetworkWrapper -> Renderer.render on a
// 1024-ray chunk (BASELINE config 3) and PyTorch autograd through raw2outputs (nerf_net_utils.py:6-51), the eight Conv1d
// layers and F.grid_sample (latent_xyzc.py:62-126).  Here:
//
//   forward   classify_compact_kernel (nb_render_tc_list.cu, ONE list for all frames): a sample whose trilinear cells are all
//             unoccupied has all-zero features, hence sigma = sigma_empty < 0: relu kills its density AND the gradient of
//             everything behind it, so neither pass evaluates it -- exact, as in the inference path.
//             gather_kernel      features (fp32, same accumulation order as the exact kernel) + both positional encodings
//             4 x gemm_tf32x3    fc_0, fc_1, fc_2, [folded colour layer | alpha_fc] -- activations live in HBM: a 1024-ray
//                                chunk lists ~1e5 samples, its whole record crosses HBM in ~0.2 ms
//             head_kernel        rgb_fc, raw records; then composite_kernel (shared with the inference path)
//   backward  composite_bwd_kernel (nb_render_bwd.cu) -> bwd_head_kernel -> 4 x gemm (dgrad, relu masks in the epilogue)
//             -> scatter_kernel (trilinear backward, 16-byte vector atomics into a channels-last gradient blob, then one
//             transposing add into the NCDHW gradients autograd expects) ; 4 x gemm (wgrad, split over the list, fp32
//             atomics) ; column sums for the biases ; the un-fold of the colour layer (nb_render_bwd.cu) ; only when a
//             gradient with respect to the sample position is asked for: frame_grad_kernel (dR / dTh, d bounds) and, for
//             the ray and depth gradients, gemm (the encodings' input gradient) before it (per-sample records) and
//             ray_grad_kernel (nb_render_bwd.cu) after it.
//
// gemm_tf32x3_kernel: C[128 x <=256 tile] = epilogue(A B^T), fp32 in HBM on both sides.  Operands are split on the way into
// shared memory into hi = x & 0xFFFFE000 (exactly representable in TF32) and lo = x - hi, and three wgmma tf32 passes
// (hi hi + lo hi + hi lo) accumulate in fp32 in registers (two warpgroups, 64 rows each, N = 256 per instruction): ~2^-21 relative error per product, i.e. fp32-grade, which the
// forward's 1e-3 parity gate on depth needs (one 11-bit rounding anywhere on the density path breaks it,
// tests/test_precision_model.py); TF32 rather than fp16 pairs because gradients underflow fp16's range.
#include "nb_device.cuh"
#include "nb_tc_ptx.cuh"
#include "nb_train.h"

namespace nb {
namespace trn {

// ================================================================================================ the GEMM
constexpr int GT = 256;                      // threads
#ifndef NB_TRN_KCH
#define NB_TRN_KCH 16
#endif
constexpr int KCH = NB_TRN_KCH;              // reduction elements per stage (KCH / 8 MMAs of K = 8 per pass)
constexpr int CTAS_PER_SM = 1;               // the 128 x 256 fp32 accumulator lives in registers: 128 per thread
// K-major no-swizzle operand planes: a core matrix is 8 rows x 16 B.  Row groups sit SBO = 144 B apart (not 128) and the
// 4-element K chunks LBO = rows/8 * 144 + 16 B apart: both strides are free descriptor fields, and these values make the
// transposing 4-byte stores of a row-contiguous operand and the 16-byte stores of a K-contiguous one bank-conflict-free.
#ifndef NB_TRN_SBO
#define NB_TRN_SBO 144
#endif
constexpr int SBO = NB_TRN_SBO;
#ifndef NB_TRN_LBO_PAD
#define NB_TRN_LBO_PAD 16
#endif
__host__ __device__ constexpr int lbo_bytes(int rows) { return rows / 8 * SBO + NB_TRN_LBO_PAD; }
constexpr int A_ROWS = 128, B_ROWS = 256;
constexpr int A_PLANE = (KCH / 4) * lbo_bytes(A_ROWS);    // 9280 at KCH = 16
constexpr int B_PLANE = (KCH / 4) * lbo_bytes(B_ROWS);    // 18496
constexpr int STAGE_BYTES = 2 * A_PLANE + 2 * B_PLANE;    // hi + lo of both operands: 55552
constexpr int GEMM_SMEM = 2 * STAGE_BYTES;                // 111104: two stages (one is stored while the other's MMAs run)
static_assert(CTAS_PER_SM * (GEMM_SMEM + 2048) <= 232448, "shared memory budget");
constexpr int KC_TPR = KCH / 4;                           // K-contiguous operand: threads per row
constexpr int KC_ROWS = GT / KC_TPR;                      //   rows per pass of the CTA
constexpr int RC_NKC = KCH / 4;                           // row-contiguous operand: 4-element K chunks per stage (one warp each)
constexpr int RC_WPK = (GT / 32) / RC_NKC;                //   warps sharing a K chunk (they split the 32-row blocks)
template <int R> struct TileRegs { static constexpr int N = R * KCH / 1024; };   // float4 per thread and R x KCH tile

// Operand element (row, k):  KC (K contiguous): p[row * ld + k];  RC (rows contiguous): p[k * ld + row].
// A 256-thread CTA moves one R x 32 tile per call, 16 bytes per load.
template <int R, bool KC>
__device__ __forceinline__ void load_tile(const float* __restrict__ p, long long ld, int row0, int rows_valid, int k0, int k_end,
                                          float4 (&v)[TileRegs<R>::N], int tid) {
    if (KC) {
        const int c = tid % KC_TPR, r = tid / KC_TPR;
        const int gk = k0 + 4 * c;
#pragma unroll
        for (int i = 0; i < TileRegs<R>::N; ++i) {
            const int grow = row0 + r + KC_ROWS * i;
            v[i] = (grow < rows_valid && gk < k_end) ? __ldg(reinterpret_cast<const float4*>(p + (long long)grow * ld + gk))
                                                      : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    } else {
        const int w = tid >> 5, lane = tid & 31, m4 = lane & 7, kk = lane >> 3;
        const int gk = k0 + 4 * (w % RC_NKC) + kk;
#pragma unroll
        for (int i = 0; i < TileRegs<R>::N; ++i) {
            const int grow = row0 + 32 * (w / RC_NKC + RC_WPK * i) + 4 * m4;
            v[i] = (grow < rows_valid && gk < k_end) ? __ldg(reinterpret_cast<const float4*>(p + (long long)gk * ld + grow))
                                                      : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    lo = x - hi;                                         // exact
}
template <int R, bool KC>
__device__ __forceinline__ void store_tile(unsigned char* __restrict__ hi_plane, unsigned char* __restrict__ lo_plane,
                                           const float4 (&v)[TileRegs<R>::N], int tid) {
    constexpr int LBO = lbo_bytes(R);
    if (KC) {
        const int c = tid % KC_TPR, r = tid / KC_TPR;
#pragma unroll
        for (int i = 0; i < TileRegs<R>::N; ++i) {
            const int row = r + KC_ROWS * i;
            const int off = c * LBO + (row >> 3) * SBO + (row & 7) * 16;
            float4 h, l;
            split_tf32(v[i].x, h.x, l.x); split_tf32(v[i].y, h.y, l.y); split_tf32(v[i].z, h.z, l.z); split_tf32(v[i].w, h.w, l.w);
            *reinterpret_cast<float4*>(hi_plane + off) = h;
            *reinterpret_cast<float4*>(lo_plane + off) = l;
        }
    } else {
        const int w = tid >> 5, lane = tid & 31, m4 = lane & 7, kk = lane >> 3;
#pragma unroll
        for (int i = 0; i < TileRegs<R>::N; ++i) {
            const float x[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int row = 32 * (w / RC_NKC + RC_WPK * i) + 4 * m4 + j;
                const int off = (w % RC_NKC) * LBO + (row >> 3) * SBO + (row & 7) * 16 + kk * 4;
                float h, l;
                split_tf32(x[j], h, l);
                *reinterpret_cast<float*>(hi_plane + off) = h;
                *reinterpret_cast<float*>(lo_plane + off) = l;
            }
        }
    }
}

template <bool A_KC, bool B_KC>
__global__ void __launch_bounds__(GT, CTAS_PER_SM) gemm_tf32x3_kernel(const __grid_constant__ GemmArgs G) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int M = G.dyn_m ? (int)__ldg(G.dyn_m) : G.M;
    const int Ktot = G.dyn_k ? (int)__ldg(G.dyn_k) : G.K;
    const int m0 = blockIdx.x * A_ROWS, n0 = blockIdx.y * B_ROWS;
    if (m0 >= M) return;
    int kbeg = 0, kend = Ktot;
    if (gridDim.z > 1) {                                 // split of the reduction (weight gradients): equal shares of the ACTUAL length
        const int per = (Ktot + KCH * (int)gridDim.z - 1) / (KCH * (int)gridDim.z) * KCH;
        kbeg = blockIdx.z * per;
        kend = min(Ktot, kbeg + per);
    }
    if (kbeg >= kend) return;
    const int nt = min(B_ROWS, G.N - n0);               // N is a multiple of 16; rows past nt are zero-filled in shared memory
    const int nchunks = (kend - kbeg + KCH - 1) / KCH;
    constexpr int LBO_A = lbo_bytes(A_ROWS), LBO_B = lbo_bytes(B_ROWS);
    const int wg = warp >> 2;                            // warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile

    // Two register sets: the loads of chunk c + 2 are issued when chunk c has been stored, so they have two MMA batches to
    // arrive; two shared-memory stages: the MMAs of chunk c run while chunk c + 1 is split and stored.
    float4 va0[TileRegs<A_ROWS>::N], vb0[TileRegs<B_ROWS>::N], va1[TileRegs<A_ROWS>::N], vb1[TileRegs<B_ROWS>::N];
    load_tile<A_ROWS, A_KC>(G.a, G.lda, m0, M, kbeg, kend, va0, tid);
    load_tile<B_ROWS, B_KC>(G.b, G.ldb, n0, G.N, kbeg, kend, vb0, tid);
    if (nchunks > 1) {
        load_tile<A_ROWS, A_KC>(G.a, G.lda, m0, M, kbeg + KCH, kend, va1, tid);
        load_tile<B_ROWS, B_KC>(G.b, G.ldb, n0, G.N, kbeg + KCH, kend, vb1, tid);
    }
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    auto chunk = [&](float4 (&va)[TileRegs<A_ROWS>::N], float4 (&vb)[TileRegs<B_ROWS>::N], int c) {
        const int s = c & 1;
        unsigned char* st = smem + s * STAGE_BYTES;
        if (c >= 2) {                                    // the MMAs of chunk c - 2 (both warpgroups) have read this stage
            tc::wgmma_wait<1>();
            tc::acc_fence(acc);
            __syncthreads();
        }
        store_tile<A_ROWS, A_KC>(st, st + A_PLANE, va, tid);
        store_tile<B_ROWS, B_KC>(st + 2 * A_PLANE, st + 2 * A_PLANE + B_PLANE, vb, tid);
        if (c + 2 < nchunks) {
            load_tile<A_ROWS, A_KC>(G.a, G.lda, m0, M, kbeg + (c + 2) * KCH, kend, va, tid);
            load_tile<B_ROWS, B_KC>(G.b, G.ldb, n0, G.N, kbeg + (c + 2) * KCH, kend, vb, tid);
        }
        tc::fence_proxy_async();
        __syncthreads();
        const uint32_t a_hi = tc::smem_u32(st) + 8 * wg * SBO, a_lo = a_hi + A_PLANE;
        const uint32_t b_hi = tc::smem_u32(st) + 2 * A_PLANE, b_lo = b_hi + B_PLANE;
        tc::wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {           // lo hi + hi lo + hi hi
            const uint32_t ab = pass == 0 ? a_lo : a_hi, bb = pass == 1 ? b_lo : b_hi;
#pragma unroll
            for (int j = 0; j < KCH / 8; ++j) {
                const uint64_t da = tc::make_smem_desc(ab + 2 * j * LBO_A, LBO_A, SBO);
                const uint64_t db = tc::make_smem_desc(bb + 2 * j * LBO_B, LBO_B, SBO);
                tc::wgmma_m64n256k8_tf32(acc, da, db, true);
            }
        }
        tc::wgmma_commit();
    };
    for (int c = 0; c < nchunks; c += 2) {
        chunk(va0, vb0, c);
        if (c + 1 < nchunks) chunk(va1, vb1, c + 1);
    }
    tc::wgmma_wait<0>();
    tc::acc_fence(acc);

    // ---- epilogue, straight from the accumulator registers: this thread holds rows r and r + 8, columns 8 j + 2 (lane % 4) + {0, 1}
    const int rbase = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = rbase + 8 * h;
        if (row >= M) continue;
        const float* bias = G.bias;
        if (bias && G.bias_frame_stride)
            bias += (size_t)((__float_as_uint(__ldg(&G.list[row].w)) & kListIdMask) / G.samples_per_frame) * G.bias_frame_stride;
#pragma unroll
        for (int j = 0; j < B_ROWS / 8; ++j) {
            const int cl = 8 * j + cq;
            if (cl >= nt) continue;
            const int col = n0 + cl;
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if (bias) {
                const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + col));
                v0 += bv.x; v1 += bv.y;
            }
            if (col < G.relu_cols) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }   // relu_cols is a multiple of 16
            if (G.mask) {
                const float2 mv = __ldg(reinterpret_cast<const float2*>(G.mask + (size_t)row * G.ldm + col));
                if (!(mv.x > 0.f)) v0 = 0.f;
                if (!(mv.y > 0.f)) v1 = 0.f;
            }
            float* dst = G.c + (size_t)row * G.ldc + col;
            if (G.atomic) {
                if (v0 != 0.f) atomicAdd(dst, v0);
                if (v1 != 0.f) atomicAdd(dst + 1, v1);
            } else {
                *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
            }
        }
    }
}

int launch_gemm(const GemmArgs& g, bool a_kc, bool b_kc, int max_m, int splits, cudaStream_t stream) {
    if (g.N % 16 || g.N <= 0 || (g.lda & 3) || (g.ldb & 3) || (!g.atomic && (g.ldc & 3))) {
        set_error("gemm_tf32x3: N must be a multiple of 16 and the leading dimensions multiples of 4");
        return NB_ERR_BAD_ARG;
    }
    if (max_m <= 0) return NB_OK;
    dim3 grid((max_m + A_ROWS - 1) / A_ROWS, (g.N + B_ROWS - 1) / B_ROWS, splits > 0 ? splits : 1);
    cudaError_t e;
#define NB_GEMM(AK, BK)                                                                                                  \
    do {                                                                                                                 \
        e = cudaFuncSetAttribute(gemm_tf32x3_kernel<AK, BK>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);    \
        if (e == cudaSuccess) { gemm_tf32x3_kernel<AK, BK><<<grid, GT, GEMM_SMEM, stream>>>(g); e = cudaGetLastError(); } \
    } while (0)
    if (a_kc && b_kc) NB_GEMM(true, true);
    else if (a_kc && !b_kc) NB_GEMM(true, false);
    else if (!a_kc && !b_kc) NB_GEMM(false, false);
    else NB_GEMM(false, true);
#undef NB_GEMM
    if (e != cudaSuccess) { set_error("gemm_tf32x3 launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

// ================================================================================================ record layout
SaveMap map_save(float* save, int batch, size_t pmax) {
    SaveMap m;
    float* p = save;
    m.count = reinterpret_cast<unsigned int*>(p);             p += 64;
    m.wcol = p;                                               p += (size_t)kWS * kH2X;
    m.bias3 = p;                                              p += ((size_t)batch * kWS + 63) / 64 * 64;
    m.list = reinterpret_cast<float4*>(p);                    p += pmax * 4;
    m.F = p;                                                  p += pmax * kFeat;
    m.H0 = p;                                                 p += pmax * kHidden;
    m.H1 = p;                                                 p += pmax * kHidden;
    m.H2X = p;                                                p += pmax * kH2X;
    m.WS = p;                                                 p += pmax * kWS;
    m.floats = (size_t)(p - save);
    return m;
}
size_t save_bytes(int batch, size_t pmax) { return map_save(nullptr, batch, pmax).floats * 4; }

// ================================================================================================ forward kernels
// Wcol (144 x 352): rows 0..127 = [Wc | Wx (PE xyz) | 0 | Wv (PE view) | 0 x 5], row 128 = [alpha_fc | 0], rows 129.. = 0;
// bias3 (B x 144) = [bc_b | alpha_b | 0].  All from the packed fp32 weight section (nb_layout.h).
__global__ void build_color_kernel(const float* __restrict__ wf, const float* __restrict__ bc, int batch, float* __restrict__ wcol,
                                   float* __restrict__ bias3) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < kWS * kH2X) {
        const int n = idx / kH2X, k = idx % kH2X;
        float v = 0.f;
        if (n < kColor) {
            if (k < kHidden) v = wf[oWc + (size_t)n * kHidden + k];
            else if (k < kHidden + kXyzPE) v = wf[oWct + (size_t)k * kColor + n];
            else if (k >= kViewCol && k < kViewCol + kViewPE) v = wf[oWvt + (size_t)(k - kViewCol) * kColor + n];
        } else if (n == kColor && k < kHidden) {
            v = wf[oAlphaW + k];
        }
        wcol[idx] = v;
    } else if (idx < kWS * kH2X + batch * kWS) {
        const int r = idx - kWS * kH2X, b = r / kWS, n = r % kWS;
        bias3[r] = n < kColor ? bc[b * kColor + n] : (n == kColor ? wf[oAlphaB] : 0.f);
    }
}

// One CTA per 32 list entries: grid coordinates + encodings by one thread per entry, then (entry, channel quad) work items --
// the 8 lanes of a quad row read one corner as 128 contiguous bytes.  Accumulation order = ATen's (and the exact kernel's).
constexpr int GP = 32;
template <typename VT>
__global__ void __launch_bounds__(256) gather_kernel(const __grid_constant__ RenderParams P, SaveMap sv) {
    __shared__ float gc[GP][3];
    __shared__ int fr[GP];
    const unsigned int count = *sv.count;
    const int S = P.n_samples;
    const unsigned int spf = (unsigned int)P.n_rays * S;
    for (unsigned int e0 = blockIdx.x * GP; e0 < count; e0 += gridDim.x * GP) {
        const int tid = threadIdx.x;
        if (tid < GP && e0 + tid < count) {
            const float4 en = sv.list[e0 + tid];
            const unsigned int id = __float_as_uint(en.w) & kListIdMask;
            const int b = id / spf;
            const size_t ri = id / S;
            FrameXf fx;
#pragma unroll
            for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
            float gx, gy, gz;
            world_to_grid(fx, en.x, en.y, en.z, gx, gy, gz);
            gc[tid][0] = gx; gc[tid][1] = gy; gc[tid][2] = gz;
            fr[tid] = b;
            float* xr = sv.H2X + (size_t)(e0 + tid) * kH2X;
            positional_embed<10>(en.x, en.y, en.z, [&](int j, float v) { xr[kXyzCol + j] = v; });      // latent_xyzc.py:115
            xr[kXyzCol + kXyzPE] = 0.f;
            const float dx = __ldg(P.ray_d + ri * 3), dy = __ldg(P.ray_d + ri * 3 + 1), dz = __ldg(P.ray_d + ri * 3 + 2);
            const float nrm = ray_norm(dx, dy, dz);
            positional_embed<4>(__fdiv_rn(dx, nrm), __fdiv_rn(dy, nrm), __fdiv_rn(dz, nrm), [&](int j, float v) { xr[kViewCol + j] = v; });
#pragma unroll
            for (int j = kViewCol + kViewPE; j < kH2X; ++j) xr[j] = 0.f;
        }
        __syncthreads();
        constexpr int QUADS = kFeat / 4;
        for (int item = tid; item < GP * QUADS; item += 256) {
            const int p = item / QUADS, qd = item % QUADS;
            if (e0 + p >= count) continue;
            *reinterpret_cast<float4*>(sv.F + (size_t)(e0 + p) * kFeat + qd * 4) = gather_quad<VT>(P, fr[p], gc[p][0], gc[p][1], gc[p][2], qd);
        }
        __syncthreads();
    }
}

// rgb = rgb_fc w + b (fp32, one warp per entry) and the raw record (rgb logits, sigma) of the entry's sample
__global__ void __launch_bounds__(256) head_kernel(const float* __restrict__ wf, SaveMap sv, float4* __restrict__ raw) {
    const unsigned int count = *sv.count;
    const int lane = threadIdx.x & 31;
    const unsigned int warps = gridDim.x * (blockDim.x >> 5);
    float rw[3][4];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) rw[c][j] = __ldg(wf + oRgbW + c * kColor + 4 * lane + j);
    for (unsigned int e = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); e < count; e += warps) {
        const float* ws = sv.WS + (size_t)e * kWS;
        const float4 w = *reinterpret_cast<const float4*>(ws + 4 * lane);
        float a0 = w.x * rw[0][0] + w.y * rw[0][1] + w.z * rw[0][2] + w.w * rw[0][3];
        float a1 = w.x * rw[1][0] + w.y * rw[1][1] + w.z * rw[1][2] + w.w * rw[1][3];
        float a2 = w.x * rw[2][0] + w.y * rw[2][1] + w.z * rw[2][2] + w.w * rw[2][3];
        a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
        if (lane == 0) {
            const unsigned int id = __float_as_uint(sv.list[e].w) & kListIdMask;
            raw[id] = make_float4(a0 + __ldg(wf + oRgbB), a1 + __ldg(wf + oRgbB + 1), a2 + __ldg(wf + oRgbB + 2), ws[kColor]);
        }
    }
}

// ================================================================================================ backward kernels
// d_raw (dense, per sample) -> the colour layer's output gradient G3 = [rgb_fc^T d_logits * [w > 0] | d_sigma | 0], and the
// gradients of rgb_fc (block-reduced, then atomics)
__global__ void __launch_bounds__(256) bwd_head_kernel(const float* __restrict__ wf, SaveMap sv, const float4* __restrict__ d_raw,
                                                       float* __restrict__ G3, float* __restrict__ g_rgb_w, float* __restrict__ g_rgb_b) {
    __shared__ float red[8][3 * kColor + 4];
    const unsigned int count = *sv.count;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int warps = gridDim.x * (blockDim.x >> 5);
    float rw[3][4], gw[3][4] = {}, gb[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) rw[c][j] = __ldg(wf + oRgbW + c * kColor + 4 * lane + j);
    for (unsigned int e = blockIdx.x * (blockDim.x >> 5) + warp; e < count; e += warps) {
        const unsigned int id = __float_as_uint(sv.list[e].w) & kListIdMask;
        const float4 d = __ldg(d_raw + id);
        const float4 w = *reinterpret_cast<const float4*>(sv.WS + (size_t)e * kWS + 4 * lane);
        const float wv[4] = {w.x, w.y, w.z, w.w};
        float o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            o[j] = wv[j] > 0.f ? d.x * rw[0][j] + d.y * rw[1][j] + d.z * rw[2][j] : 0.f;
            gw[0][j] = fmaf(d.x, wv[j], gw[0][j]); gw[1][j] = fmaf(d.y, wv[j], gw[1][j]); gw[2][j] = fmaf(d.z, wv[j], gw[2][j]);
        }
        float* g = G3 + (size_t)e * kWS;
        *reinterpret_cast<float4*>(g + 4 * lane) = make_float4(o[0], o[1], o[2], o[3]);
        if (lane < 4) *reinterpret_cast<float4*>(g + kColor + 4 * lane) = make_float4(lane == 0 ? d.w : 0.f, 0.f, 0.f, 0.f);
        gb[0] += d.x; gb[1] += d.y; gb[2] += d.z;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int j = 0; j < 4; ++j) red[warp][c * kColor + 4 * lane + j] = gw[c][j];
    if (lane == 0) { red[warp][3 * kColor] = gb[0]; red[warp][3 * kColor + 1] = gb[1]; red[warp][3 * kColor + 2] = gb[2]; }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 * kColor + 3; i += blockDim.x) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) s += red[w][i];
        if (s != 0.f) atomicAdd(i < 3 * kColor ? g_rgb_w + i : g_rgb_b + (i - 3 * kColor), s);
    }
}

// Trilinear backward (F.grid_sample, zeros padding): dF (count x 352) -> channels-last gradient blob, one 16-byte vector
// atomic per (entry, corner, channel quad)
__global__ void __launch_bounds__(256) scatter_kernel(const __grid_constant__ RenderParams P, SaveMap sv, const float* __restrict__ DF,
                                                      float* __restrict__ dblob, GradBlob gb) {
    __shared__ float gc[GP][3];
    __shared__ int fr[GP];
    const unsigned int count = *sv.count;
    const unsigned int spf = (unsigned int)P.n_rays * P.n_samples;
    for (unsigned int e0 = blockIdx.x * GP; e0 < count; e0 += gridDim.x * GP) {
        const int tid = threadIdx.x;
        if (tid < GP && e0 + tid < count) {
            const float4 en = sv.list[e0 + tid];
            const int b = (__float_as_uint(en.w) & kListIdMask) / spf;
            FrameXf fx;
#pragma unroll
            for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
            float gx, gy, gz;
            world_to_grid(fx, en.x, en.y, en.z, gx, gy, gz);
            gc[tid][0] = gx; gc[tid][1] = gy; gc[tid][2] = gz;
            fr[tid] = b;
        }
        __syncthreads();
        constexpr int QUADS = kFeat / 4;
        for (int item = tid; item < GP * QUADS; item += 256) {
            const int p = item / QUADS, qd = item % QUADS;
            if (e0 + p >= count) continue;
            int lvl, c0;
            feature_quad(qd, lvl, c0);
            const float4 g = *reinterpret_cast<const float4*>(DF + (size_t)(e0 + p) * kFeat + qd * 4);
            if (g.x == 0.f && g.y == 0.f && g.z == 0.f && g.w == 0.f) continue;
            const int C = P.lvl_C[lvl], D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
            Corners cn;
            corner_setup(unnormalize(gc[p][0], W), unnormalize(gc[p][1], H), unnormalize(gc[p][2], D), W, H, D, cn);
            float* dv = dblob + gb.off[lvl] + (size_t)fr[p] * gb.bstride[lvl];
            for_each_corner(cn, W, H, D, [&](size_t vox, float wgt) {
                atomicAdd(reinterpret_cast<float4*>(dv + vox * C + c0), make_float4(wgt * g.x, wgt * g.y, wgt * g.z, wgt * g.w));
            });
        }
        __syncthreads();
    }
}

// Frame-transform gradients (sp_input R, Th): the trilinear backward with respect to the sample position.  Same work items as
// scatter_kernel; each (entry, quad) adds sum_c dF_c d f_c / d i, scaled to d / d(canonical point), into its entry's shared
// slot; warp 0 then turns the 32 entries into dR / dTh terms and sums them per frame (one atomic per CTA, frame and element:
// the list is frame-major and each CTA walks it in order).  Reads the packed blob the forward gathered from.
// WIDE (ray, depth or bounds gradients asked for; dR / dTh may both be null then), each part only when its pointer is given:
//   rec: each entry's ray-gradient record rec + id * kRayRec = [d loss / d(world point) 3 | d loss / d(view direction) 3]:
//        the grid part R dc plus the two encodings' parts, from dPE (count x kPECols, the colour layer's input gradient in
//        columns kXyzCol..) and the sin / cos the forward saved in H2X;
//   d_bounds: d_bounds[b, 0, :] -= the per-frame sum of d loss / d(canonical point), the quantity whose image under R is the
//        dTh term, taken before R is applied.
// The frame-only variant takes 63 registers and runs 4 CTAs per SM; WIDE asks for at least 2, so that ptxas does not squeeze
// it into 64 registers and spill.
constexpr int kPECols = kH2X - kXyzCol;     // [PE(xyz) 63 | 0 | PE(view) 27 | 0 x 5]
constexpr int kRayRec = 8;
template <typename VT, bool WIDE>
__global__ void __launch_bounds__(256, WIDE ? 2 : 0) frame_grad_kernel(const __grid_constant__ RenderParams P, SaveMap sv, const float* __restrict__ DF,
                                                         float* __restrict__ dR, float* __restrict__ dTh, const float* __restrict__ dPE,
                                                         float* __restrict__ rec, float* __restrict__ d_bounds) {
    __shared__ float gc[GP][3], dc[GP][3];
    __shared__ int fr[GP];
    __shared__ float pe[WIDE ? 2 : 1][GP][3];   // WIDE: [PE(xyz) | PE(view)][entry][axis]
    const unsigned int count = *sv.count;
    const unsigned int spf = (unsigned int)P.n_rays * P.n_samples;
    const int tid = threadIdx.x;
    FrameGradAcc acc;
    FrameGradAcc acc_bounds;                    // WIDE: warp 0's running per-frame sums of d bounds[:, 0]
    for (unsigned int e0 = blockIdx.x * GP; e0 < count; e0 += gridDim.x * GP) {
        if (tid < GP) {
            fr[tid] = -1;
            dc[tid][0] = dc[tid][1] = dc[tid][2] = 0.f;
            if (e0 + tid < count) {
                const float4 en = sv.list[e0 + tid];
                const int b = (__float_as_uint(en.w) & kListIdMask) / spf;
                FrameXf fx;
#pragma unroll
                for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
                float gx, gy, gz;
                world_to_grid(fx, en.x, en.y, en.z, gx, gy, gz);
                gc[tid][0] = gx; gc[tid][1] = gy; gc[tid][2] = gz;
                fr[tid] = b;
            }
        }
        __syncthreads();
        constexpr int QUADS = kFeat / 4;
        for (int item = tid; item < GP * QUADS; item += 256) {
            const int p = item / QUADS, qd = item % QUADS;
            if (e0 + p >= count) continue;
            const float4 g = *reinterpret_cast<const float4*>(DF + (size_t)(e0 + p) * kFeat + qd * 4);
            if (g.x == 0.f && g.y == 0.f && g.z == 0.f && g.w == 0.f) continue;
            int lvl, c0;
            feature_quad(qd, lvl, c0);
            const float3 d = gather_quad_dpos<VT>(P, fr[p], gc[p][0], gc[p][1], gc[p][2], qd, g);
            // d i / d g = (size - 1) / 2 per level; the level-independent d g / d c is applied once per entry below
            atomicAdd(&dc[p][0], d.x * (0.5f * (float)(P.lvl_W[lvl] - 1)));
            atomicAdd(&dc[p][1], d.y * (0.5f * (float)(P.lvl_H[lvl] - 1)));
            atomicAdd(&dc[p][2], d.z * (0.5f * (float)(P.lvl_D[lvl] - 1)));
        }
        if (WIDE && rec && tid < 2 * GP * 3) {   // (encoding, entry, axis) items
            const int v = tid / (GP * 3), p = tid % (GP * 3) / 3, ax = tid % 3;
            float r = 0.f;
            if (e0 + p < count) {
                const float* d = dPE + (size_t)(e0 + p) * kPECols + (v ? kViewCol - kXyzCol : 0);
                const float* enc = sv.H2X + (size_t)(e0 + p) * kH2X + (v ? kViewCol : kXyzCol);
                r = v ? positional_embed_bwd<4>(d, enc, ax) : positional_embed_bwd<10>(d, enc, ax);
            }
            pe[v][p][ax] = r;
        }
        __syncthreads();
        if (tid < 32) {
            float t[12] = {};
            float dcan[3] = {0.f, 0.f, 0.f};    // WIDE: d loss / d(canonical point)
            const int b = fr[tid];
            if (b >= 0) {
                const float4 en = sv.list[e0 + tid];
                FrameXf fx;
#pragma unroll
                for (int j = 0; j < 9; ++j) load_frame_xf(P, b, fx, j);
                // grid x / y / z pair with the dhw axes 2 / 1 / 0
                frame_grad_terms(fx, en.x, en.y, en.z, dc[tid][0] * grid_to_can_scale(fx, 2), dc[tid][1] * grid_to_can_scale(fx, 1),
                                 dc[tid][2] * grid_to_can_scale(fx, 0), t);
                if constexpr (WIDE) {
                    dcan[0] = dc[tid][0] * grid_to_can_scale(fx, 2); dcan[1] = dc[tid][1] * grid_to_can_scale(fx, 1);
                    dcan[2] = dc[tid][2] * grid_to_can_scale(fx, 0);
                }
                if (WIDE && rec) {   // the grid part R dc is -(the dTh term)
                    float* r = rec + (size_t)(__float_as_uint(en.w) & kListIdMask) * kRayRec;
#pragma unroll
                    for (int k = 0; k < 3; ++k) { r[k] = pe[0][tid][k] - t[9 + k]; r[3 + k] = pe[1][tid][k]; }
                }
            }
            if (!WIDE || dR || dTh) frame_sum_add(acc, b, t, tid, [&](FrameGradAcc& x) { frame_grad_flush(x, dR, dTh, tid); });
            if (WIDE && d_bounds) frame_sum_add(acc_bounds, b, dcan, tid, [&](FrameGradAcc& x) { bounds_grad_flush(x, d_bounds, tid); });
        }
        __syncthreads();
    }
    if (tid < 32) frame_grad_flush(acc, dR, dTh, tid);
    if (WIDE && d_bounds && tid < 32) bounds_grad_flush(acc_bounds, d_bounds, tid);
}

// d_vol[b][c][v] += blob[b][v][c] for one level: 32 voxels x 32 channels through shared memory
__global__ void __launch_bounds__(256) unpack_grad_kernel(const float* __restrict__ blob, float* __restrict__ dvol, int C, size_t nvox, int batch) {
    __shared__ float t[32][33];
    const size_t v0 = (size_t)blockIdx.x * 32;
    const int c0 = blockIdx.y * 32, b = blockIdx.z;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int i = ty; i < 32; i += 8) {
        const size_t v = v0 + i;
        t[i][tx] = (v < nvox && c0 + tx < C) ? blob[((size_t)b * nvox + v) * C + c0 + tx] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const size_t v = v0 + tx;
        const float g = t[tx][i];
        if (v < nvox && c0 + i < C && g != 0.f) dvol[((size_t)b * C + c0 + i) * nvox + v] += g;
    }
}

// column sums of a (count x ld) gradient array, by frame when nframes > 1: out[frame * out_stride + col] += sum
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ A, int ld, int ncols, SaveMap sv, unsigned int spf, int rows_per_cta,
                                                     float* __restrict__ out, int out_stride, int by_frame) {
    const unsigned int count = *sv.count;
    const unsigned int r0 = blockIdx.x * rows_per_cta, r1 = min(count, r0 + rows_per_cta);
    const int col = threadIdx.x;
    if (col >= ncols || r0 >= r1) return;
    float acc = 0.f;
    int cur = by_frame ? (int)((__float_as_uint(sv.list[r0].w) & kListIdMask) / spf) : 0;
    for (unsigned int r = r0; r < r1; ++r) {
        if (by_frame) {
            const int f = (int)((__float_as_uint(sv.list[r].w) & kListIdMask) / spf);
            if (f != cur) { if (acc != 0.f) atomicAdd(out + (size_t)cur * out_stride + col, acc); acc = 0.f; cur = f; }
        }
        acc += A[(size_t)r * ld + col];
    }
    if (acc != 0.f) atomicAdd(out + (size_t)cur * out_stride + col, acc);
}

// dWcol (144 x 352) / dbias3 (B x 144) -> the inputs of the un-fold (dWcx 128 x 320, dbc B x 128) and the gradients that
// need no un-folding: view_fc[:, 256:283] (PE view), alpha_fc weight and bias
__global__ void finish_color_kernel(const float* __restrict__ dwcol, const float* __restrict__ dbias3, int batch, float* __restrict__ dWcx,
                                    float* __restrict__ dbc, float* __restrict__ g_view_w, float* __restrict__ g_alpha_w, float* __restrict__ g_alpha_b) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < kColor * kColorK) {
        const int n = idx / kColorK, k = idx % kColorK;
        dWcx[idx] = dwcol[(size_t)n * kH2X + k];
    } else if (idx < kColor * kColorK + kColor * kViewPE) {
        const int r = idx - kColor * kColorK, n = r / kViewPE, j = r % kViewPE;
        g_view_w[n * 346 + 256 + j] += dwcol[(size_t)n * kH2X + kViewCol + j];
    } else if (idx < kColor * kColorK + kColor * kViewPE + kHidden) {
        const int k = idx - kColor * kColorK - kColor * kViewPE;
        g_alpha_w[k] += dwcol[(size_t)kColor * kH2X + k];
    } else if (idx < kColor * kColorK + kColor * kViewPE + kHidden + batch * kColor) {
        const int r = idx - kColor * kColorK - kColor * kViewPE - kHidden, b = r / kColor, n = r % kColor;
        dbc[r] = dbias3[b * kWS + n];
    } else if (idx == kColor * kColorK + kColor * kViewPE + kHidden + batch * kColor) {
        float s = 0.f;
        for (int b = 0; b < batch; ++b) s += dbias3[b * kWS + kColor];
        g_alpha_b[0] += s;
    }
}

}  // namespace trn

// ================================================================================================ host side
using namespace trn;

static GradBlob grad_blob_map(const RenderParams& p) {
    GradBlob g;
    size_t off = 0;
    for (int l = 0; l < 4; ++l) {
        g.off[l] = off;
        g.bstride[l] = (size_t)p.lvl_D[l] * p.lvl_H[l] * p.lvl_W[l] * p.lvl_C[l];
        off += g.bstride[l] * p.batch;
    }
    g.floats = off;
    return g;
}

size_t train_save_bytes(int batch, int n_rays, int n_samples) { return save_bytes(batch, (size_t)batch * n_rays * n_samples); }

size_t train_bwd_workspace_bytes(const RenderParams& p, int n_rays, int n_samples) {
    const size_t pmax = (size_t)p.batch * n_rays * n_samples;
    const size_t per_point = 4 + kWS + 3 * kHidden + kFeat;
    const size_t fixed = (size_t)kWS * kH2X + (size_t)p.batch * kWS + 64 /* dwcol, dbias3 */ +
                         (size_t)kColor * kColorK + (size_t)p.batch * kColor + 2 * (size_t)kColor * kHidden + 2 * (size_t)p.batch * kHidden + 256;
    return (pmax * per_point + fixed + grad_blob_map(p).floats) * 4;
}

bool train_supported(const RenderParams& p) {
    return p.n_samples <= kListMaxSamples && (long long)p.batch * p.n_rays * p.n_samples <= (long long)kListIdMask;
}

int launch_train_fwd(const RenderParams& p_in, int volume_dtype, cudaStream_t stream) {
    RenderParams p = p_in;
    if (!train_supported(p)) { set_error("tc_tf32x3: n_samples <= %d and batch * n_rays * n_samples < 2^28", kListMaxSamples); return NB_ERR_UNSUPPORTED; }
    if (!p.save || !p.raw) { set_error("tc_tf32x3 (training precision) needs nb_render_args.save and .raw"); return NB_ERR_BAD_ARG; }
    if (p.n_rays == 0 || p.batch == 0) return NB_OK;
    const size_t pmax = (size_t)p.batch * p.n_rays * p.n_samples;
    SaveMap sv = map_save(p.save, p.batch, pmax);
    cudaError_t e = cudaMemsetAsync(sv.count, 0, 256, stream);
    if (e != cudaSuccess) { set_error("train fwd: memset failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    build_color_kernel<<<(kWS * kH2X + p.batch * kWS + 255) / 256, 256, 0, stream>>>(p.wf32, p.bc, p.batch, sv.wcol, sv.bias3);
    // 1. one list for all frames; skipped samples get their constant raw record
    p.train_list = 1;
    p.list_a = sv.list; p.list_b = sv.list; p.list_cap = pmax;
    p.list_count = sv.count;                 // class 3 -> count[3]; the kernels below read sv.count[3] through sv.count + 3
    p.stats = nullptr; p.frame_clock = nullptr;
    sv.count += 3;
    for (int b = 0; b < p.batch; ++b) {
        p.frame = b;
        p.raw_ws = reinterpret_cast<float4*>(p.raw) + (size_t)b * p.n_rays * p.n_samples;
        launch_classify(p, stream);
    }
    // 2. features + encodings, 3. the decoder as four GEMMs over the list
    const int grid_pts = (int)((pmax + GP - 1) / GP < kGridSMs * 8 ? (pmax + GP - 1) / GP : kGridSMs * 8);
    if (volume_dtype == NB_DTYPE_F32) gather_kernel<float><<<grid_pts, 256, 0, stream>>>(p, sv);
    else gather_kernel<__half><<<grid_pts, 256, 0, stream>>>(p, sv);
    const float* wf = p.wf32;
    GemmArgs g{};
    g.dyn_m = sv.count; g.M = 0; g.relu_cols = 1 << 30;
    int st;
    g.a = sv.F; g.lda = kFeat; g.b = wf + oW0t; g.ldb = kHidden; g.N = kHidden; g.K = kFeat; g.c = sv.H0; g.ldc = kHidden; g.bias = wf + oB0;
    if ((st = launch_gemm(g, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    g.a = sv.H0; g.lda = kHidden; g.b = wf + oW1t; g.K = kHidden; g.c = sv.H1; g.bias = wf + oB1;
    if ((st = launch_gemm(g, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    g.a = sv.H1; g.b = wf + oW2t; g.c = sv.H2X; g.ldc = kH2X; g.bias = wf + oB2;
    if ((st = launch_gemm(g, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    g.a = sv.H2X; g.lda = kH2X; g.b = sv.wcol; g.ldb = kH2X; g.N = kWS; g.K = kH2X; g.c = sv.WS; g.ldc = kWS;
    g.bias = sv.bias3; g.bias_frame_stride = kWS; g.list = sv.list; g.samples_per_frame = (unsigned int)p.n_rays * p.n_samples; g.relu_cols = kColor;
    if ((st = launch_gemm(g, true, true, (int)pmax, 1, stream)) != NB_OK) return st;
    // 4. rgb head + raw records, 5. raw2outputs
    head_kernel<<<kGridSMs * 4, 256, 0, stream>>>(wf, sv, reinterpret_cast<float4*>(p.raw));
    for (int b = 0; b < p.batch; ++b) {
        p.frame = b;
        p.raw_ws = reinterpret_cast<float4*>(p.raw) + (size_t)b * p.n_rays * p.n_samples;
        launch_composite(p, stream);
    }
    e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("train fwd launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int launch_train_bwd(const RenderParams& p, const TrainBwd& t, cudaStream_t stream) {
    const size_t pmax = (size_t)p.batch * p.n_rays * p.n_samples;
    if (pmax == 0) return NB_OK;
    SaveMap sv = map_save(const_cast<float*>(t.save), p.batch, pmax);
    sv.count += 3;
    const GradBlob gb = grad_blob_map(p);
    float* ws = t.workspace;
    float4* d_raw = reinterpret_cast<float4*>(ws);       ws += pmax * 4;
    float* G3 = ws;                                      ws += pmax * kWS;
    float* G2 = ws;                                      ws += pmax * kHidden;
    float* G1 = ws;                                      ws += pmax * kHidden;
    float* G0 = ws;                                      ws += pmax * kHidden;
    float* DF = ws;                                      ws += pmax * kFeat;
    float* dwcol = ws;                                   ws += (size_t)kWS * kH2X;
    float* dbias3 = ws;                                  ws += ((size_t)p.batch * kWS + 63) / 64 * 64;
    float* dWcx = ws;                                    ws += (size_t)kColor * kColorK;
    float* dbc = ws;                                     ws += (size_t)p.batch * kColor;
    float* T = ws;                                       ws += (size_t)kColor * kHidden;
    float* dT = ws;                                      ws += (size_t)kColor * kHidden;
    float* u = ws;                                       ws += (size_t)p.batch * kHidden;
    float* du = ws;                                      ws += (size_t)p.batch * kHidden;
    ws = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
    float* dblob = ws;
    const nb_decoder_weights& w = *t.weights;
    const nb_decoder_weights& g = *t.grads;
    auto G_ = [](const float* q) { return const_cast<float*>(q); };
    cudaMemsetAsync(dwcol, 0, ((size_t)kWS * kH2X + ((size_t)p.batch * kWS + 63) / 64 * 64) * 4, stream);

    // 1. d(outputs) -> d(raw) per sample (dense), 2. the colour layer's output gradient over the list
    const GradRequest& q = t.req;
    launch_composite_bwd(p, t.raw, q, reinterpret_cast<float*>(d_raw), 4, stream);
    bwd_head_kernel<<<kGridSMs * 2, 256, 0, stream>>>(p.wf32, sv, d_raw, G3, G_(g.rgb_w), G_(g.rgb_b));
    // 3. dgrad chain (relu masks = the saved activations)
    GemmArgs a{};
    a.dyn_m = sv.count; a.relu_cols = 0;
    int st;
    a.a = G3; a.lda = kWS; a.b = sv.wcol; a.ldb = kH2X; a.N = kHidden; a.K = kWS; a.c = G2; a.ldc = kHidden; a.mask = sv.H2X; a.ldm = kH2X;
    if ((st = launch_gemm(a, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    a.a = G2; a.lda = kHidden; a.b = w.fc2_w; a.ldb = kHidden; a.K = kHidden; a.c = G1; a.mask = sv.H1; a.ldm = kHidden;
    if ((st = launch_gemm(a, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    a.a = G1; a.b = w.fc1_w; a.c = G0; a.mask = sv.H0;
    if ((st = launch_gemm(a, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    if (t.d_vol[0] || q.sample_pos()) {
        a.a = G0; a.b = w.fc0_w; a.ldb = kFeat; a.N = kFeat; a.c = DF; a.ldc = kFeat; a.mask = nullptr;
        if ((st = launch_gemm(a, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
    }
    const int grid_pts = (int)((pmax + GP - 1) / GP < kGridSMs * 8 ? (pmax + GP - 1) / GP : kGridSMs * 8);
    if (t.d_vol[0]) {
        // 4. trilinear backward
        cudaMemsetAsync(dblob, 0, gb.floats * 4, stream);
        scatter_kernel<<<grid_pts, 256, 0, stream>>>(p, sv, DF, dblob, gb);
        for (int l = 0; l < 4; ++l) {
            const size_t nvox = (size_t)p.lvl_D[l] * p.lvl_H[l] * p.lvl_W[l];
            dim3 grid((unsigned)((nvox + 31) / 32), (p.lvl_C[l] + 31) / 32, p.batch);
            unpack_grad_kernel<<<grid, 256, 0, stream>>>(dblob + gb.off[l], t.d_vol[l], p.lvl_C[l], nvox, p.batch);
        }
    }
    // 5. weight gradients: dW[out][in] += G^T X, split over the list
    const int splits = 74;      // 2 x 2 tiles x 74 = two CTAs on every SM
    GemmArgs wg{};
    wg.dyn_k = sv.count; wg.atomic = 1; wg.relu_cols = 0;
    wg.a = G0; wg.lda = kHidden; wg.M = kHidden; wg.b = sv.F; wg.ldb = kFeat; wg.N = kFeat; wg.c = G_(g.fc0_w); wg.ldc = kFeat;
    if ((st = launch_gemm(wg, false, false, kHidden, splits, stream)) != NB_OK) return st;
    wg.a = G1; wg.b = sv.H0; wg.ldb = kHidden; wg.N = kHidden; wg.c = G_(g.fc1_w); wg.ldc = kHidden;
    if ((st = launch_gemm(wg, false, false, kHidden, splits, stream)) != NB_OK) return st;
    wg.a = G2; wg.b = sv.H1; wg.c = G_(g.fc2_w);
    if ((st = launch_gemm(wg, false, false, kHidden, splits, stream)) != NB_OK) return st;
    wg.a = G3; wg.lda = kWS; wg.M = kWS; wg.b = sv.H2X; wg.ldb = kH2X; wg.N = kH2X; wg.c = dwcol; wg.ldc = kH2X;
    if ((st = launch_gemm(wg, false, false, kWS, splits, stream)) != NB_OK) return st;
    // 6. bias gradients
    const unsigned int spf = (unsigned int)p.n_rays * p.n_samples;
    const int rows_per = 512, cs_grid = (int)((pmax + rows_per - 1) / rows_per);
    colsum_kernel<<<cs_grid, 256, 0, stream>>>(G0, kHidden, kHidden, sv, spf, rows_per, G_(g.fc0_b), 0, 0);
    colsum_kernel<<<cs_grid, 256, 0, stream>>>(G1, kHidden, kHidden, sv, spf, rows_per, G_(g.fc1_b), 0, 0);
    colsum_kernel<<<cs_grid, 256, 0, stream>>>(G2, kHidden, kHidden, sv, spf, rows_per, G_(g.fc2_b), 0, 0);
    colsum_kernel<<<cs_grid, 256, 0, stream>>>(G3, kWS, kWS, sv, spf, rows_per, dbias3, kWS, p.batch > 1);
    // 7. colour layer: split dWcol / dbias3, then the un-fold
    const int nfin = kColor * kColorK + kColor * kViewPE + kHidden + p.batch * kColor + 1;
    finish_color_kernel<<<(nfin + 255) / 256, 256, 0, stream>>>(dwcol, dbias3, p.batch, dWcx, dbc, G_(g.view_w), G_(g.alpha_w), G_(g.alpha_b));
    st = launch_unfold(w, g, dWcx, dbc, T, dT, u, du, stream);
    if (st != NB_OK) return st;
    if (q.sample_pos()) {
        // 8. the frame pass over DF, which steps 5-7 do not touch.  Ray and depth gradients first need the per-entry records
        // (skipped samples: 0) in G2 / G1, which steps 5 and 6 were the last to read: the encodings' input gradient
        // dPE = G3 Wcol[:, 256:352]^T, then the records by sample id, then per ray
        float* dPE = nullptr;
        float* rec = nullptr;
        if (q.records()) {
            dPE = G2; rec = G1;
            a.a = G3; a.lda = kWS; a.b = sv.wcol + kXyzCol; a.ldb = kH2X; a.N = kPECols; a.K = kWS; a.c = dPE; a.ldc = kPECols; a.mask = nullptr;
            if ((st = launch_gemm(a, true, false, (int)pmax, 1, stream)) != NB_OK) return st;
            cudaMemsetAsync(rec, 0, pmax * kRayRec * 4, stream);
        }
        const bool f32 = t.volume_dtype == NB_DTYPE_F32, wide = q.records() || q.d_bounds;
        auto* frame_pass = wide ? (f32 ? frame_grad_kernel<float, true> : frame_grad_kernel<__half, true>)
                                : (f32 ? frame_grad_kernel<float, false> : frame_grad_kernel<__half, false>);
        frame_pass<<<grid_pts, 256, 0, stream>>>(p, sv, DF, q.d_R, q.d_Th, dPE, rec, q.d_bounds);
        if (q.records()) launch_ray_grad(p, t.raw, q, rec, kRayRec, stream);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("train bwd launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // namespace nb

// ------------------------------------------------------------------------------------------------ diagnostics
// C = A B^T through gemm_tf32x3_kernel.  a: (M,K) [a_kc] or (K,M); b: (N,K) [b_kc] or (K,N); c: (M,N) fp32 (accumulated into
// when splits > 1: zero it first).  tests/test_train_gemm_gpu.py compares with an fp64 matmul.
extern "C" int nb_debug_gemm_tf32x3(const float* a, const float* b, float* c, int M, int N, int K, int a_kc, int b_kc, int splits,
                                    const float* bias, int relu, const float* mask, void* stream) {
    nb::trn::GemmArgs g{};
    g.a = a; g.lda = a_kc ? K : M; g.b = b; g.ldb = b_kc ? K : N; g.M = M; g.N = N; g.K = K; g.c = c; g.ldc = N;
    g.bias = bias; g.relu_cols = relu ? (1 << 30) : 0; g.mask = mask; g.ldm = N; g.atomic = splits > 1;
    return nb::trn::launch_gemm(g, a_kc != 0, b_kc != 0, M, splits, (cudaStream_t)stream);
}
