// extern "C" entry points of libneuralbody_b200.so (see include/neuralbody_b200.h) and the
// once-per-frame pack kernels (volume re-layout, decoder-weight fold + re-layout).
#include <stdarg.h>
#include <stdio.h>
#include "nb_device.cuh"
#include "nb_train.h"

namespace nb {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ------------------------------------------------------------------------------------------
// Volume pack: (B,C,D,H,W) fp32 -> [B][D][H][W][C] fp32/fp16 through a shared-memory
// transpose tile so that both the NCDHW reads (along W..DHW) and the channels-last writes
// (along C) are coalesced.  HBM-bound: reads 4 B and writes 4 or 2 B per element.
template <typename OT>
__device__ __forceinline__ OT cvt_out(float v);
template <>
__device__ __forceinline__ float cvt_out<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half cvt_out<__half>(float v) { return __float2half_rn(v); }

template <typename OT>
__global__ void __launch_bounds__(256) pack_volume_kernel(const float* __restrict__ src, OT* __restrict__ dst, int C,
                                                          size_t nvox /* D*H*W */, int batch,
                                                          unsigned* __restrict__ voxbits, size_t voxwords) {
    // tile: 32 voxels x 32 channels.  Also ORs "this voxel has a non-zero channel" into voxbits.
    __shared__ float tile[32][33];
    __shared__ unsigned tilemask;
    const size_t tiles_v = (nvox + 31) / 32;
    const int tiles_c = (C + 31) / 32;
    const size_t total = tiles_v * tiles_c * batch;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
    for (size_t t = blockIdx.x; t < total; t += gridDim.x) {
        const int b = (int)(t / (tiles_v * tiles_c));
        const size_t rem = t % (tiles_v * tiles_c);
        const int tc = (int)(rem / tiles_v);
        const size_t tv = rem % tiles_v;
        const float* s = src + (size_t)b * C * nvox;
        OT* d = dst + (size_t)b * C * nvox;
        if (threadIdx.x == 0) tilemask = 0u;
        bool nz = false;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int c = tc * 32 + ty + 8 * j;
            const size_t v = tv * 32 + tx;
            const float val = (c < C && v < nvox) ? __ldg(s + (size_t)c * nvox + v) : 0.f;
            nz |= (val != 0.f);
            tile[ty + 8 * j][tx] = val;
        }
        __syncthreads();
        if (nz) atomicOr(&tilemask, 1u << tx);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const size_t v = tv * 32 + ty + 8 * j;
            const int c = tc * 32 + tx;
            if (c < C && v < nvox) d[v * C + c] = cvt_out<OT>(tile[tx][ty + 8 * j]);
        }
        __syncthreads();
        if (threadIdx.x == 0 && tilemask) atomicOr(voxbits + (size_t)b * voxwords + tv, tilemask);
    }
}

// Cell occupancy: cell (cx,cy,cz), cx in [0,W] etc., is the trilinear cell whose low corner is voxel
// (cx-1, cy-1, cz-1); its bit is the OR of its (in-range) 8 corner voxels.  A sample whose cell bit is 0
// interpolates EXACT zeros at this level (SparseConvNet's .dense() is exactly 0 off the active set), so the
// gather can skip its 8 corner loads without changing a single bit of the result.
__global__ void cell_occupancy_kernel(const unsigned* __restrict__ voxbits, unsigned* __restrict__ cellbits, int D, int H,
                                      int W, size_t voxwords, size_t cellwords, int batch) {
    const size_t ncell = (size_t)(D + 1) * (H + 1) * (W + 1);
    const size_t padded = (ncell + 31) / 32 * 32;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < padded * batch; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / padded);
        const size_t c = i % padded;
        bool occ = false;
        if (c < ncell) {
            const int cx = (int)(c % (W + 1)), cy = (int)((c / (W + 1)) % (H + 1)), cz = (int)(c / ((size_t)(W + 1) * (H + 1)));
            const unsigned* vb = voxbits + (size_t)b * voxwords;
            for (int dz = -1; dz <= 0; ++dz)
                for (int dy = -1; dy <= 0; ++dy)
                    for (int dx = -1; dx <= 0; ++dx) {
                        const int x = cx + dx, y = cy + dy, z = cz + dz;
                        if (x >= 0 && x < W && y >= 0 && y < H && z >= 0 && z < D) {
                            const size_t v = ((size_t)z * H + y) * W + x;
                            occ |= (vb[v >> 5] >> (v & 31)) & 1u;
                        }
                    }
        }
        const unsigned word = __ballot_sync(0xffffffffu, occ);
        if ((threadIdx.x & 31) == 0) cellbits[(size_t)b * cellwords + (c >> 5)] = word;
    }
}

// ------------------------------------------------------------------------------------------
// Weight pack.  fold_T: T = view_fc[:, :256] * latent_fc[:, :256] (128x256, fp64) and
// u[b] = latent_fc[:, 256:] * latent[idx_b] + latent_fc.bias (256, fp64).
__global__ void fold_T_kernel(nb_decoder_weights w, double* __restrict__ T, double* __restrict__ u) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < kColor * kHidden) {
        const int n = idx / kHidden, k = idx % kHidden;
        double acc = 0.0;
        for (int j = 0; j < kHidden; ++j) acc += (double)w.view_w[n * 346 + j] * (double)w.latent_w[j * 384 + k];
        T[idx] = acc;
    } else if (idx < kColor * kHidden + w.batch * kHidden) {
        const int r = idx - kColor * kHidden;
        const int b = r / kHidden, j = r % kHidden;
        const long long li = clamp_latent(w.latent_index[b], w.num_train_frame);
        double acc = (double)w.latent_b[j];
        for (int i = 0; i < 128; ++i) acc += (double)w.latent_w[j * 384 + 256 + i] * (double)w.latent[li * 128 + i];
        u[r] = acc;
    }
}

// Wc = T * feature_fc.W (128x256); bc[b] = T feature_fc.b + view_fc[:, :256] u[b] + view_fc.b
__global__ void fold_Wc_kernel(nb_decoder_weights w, const double* __restrict__ T, const double* __restrict__ u,
                               float* __restrict__ f32, __half* __restrict__ f16, float* __restrict__ bc) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < kColor * kHidden) {
        const int n = idx / kHidden, k = idx % kHidden;
        double acc = 0.0;
        for (int j = 0; j < kHidden; ++j) acc += T[n * kHidden + j] * (double)w.feature_w[j * kHidden + k];
        const float v = (float)acc;
        f32[oWct + (size_t)k * kColor + n] = v;
        f32[oWc + (size_t)n * kHidden + k] = v;
    } else if (idx < kColor * kHidden + w.batch * kColor) {
        const int r = idx - kColor * kHidden;
        const int b = r / kColor, n = r % kColor;
        double acc = (double)w.view_b[n];
        for (int j = 0; j < kHidden; ++j)
            acc += T[n * kHidden + j] * (double)w.feature_b[j] + (double)w.view_w[n * 346 + j] * u[b * kHidden + j];
        bc[r] = (float)acc;
    }
}

// Everything that is a plain copy / transpose / fp16 re-layout.
__global__ void relayout_kernel(nb_decoder_weights w, float* __restrict__ f32, __half* __restrict__ f16) {
    const int stride = gridDim.x * blockDim.x;
    const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
    for (int i = t0; i < kHidden * kFeat; i += stride) {          // fc_0 (256,352)
        const int n = i / kFeat, k = i % kFeat;
        const float v = w.fc0_w[i];
        f32[oW0t + (size_t)k * kHidden + n] = v;
    }
    for (int i = t0; i < kHidden * kHidden; i += stride) {        // fc_1, fc_2 (256,256)
        const int n = i / kHidden, k = i % kHidden;
        const float v1 = w.fc1_w[i], v2 = w.fc2_w[i];
        f32[oW1t + (size_t)k * kHidden + n] = v1;
        f32[oW2t + (size_t)k * kHidden + n] = v2;
    }
    for (int i = t0; i < kHidden; i += stride) {
        f32[oB0 + i] = w.fc0_b[i]; f32[oB1 + i] = w.fc1_b[i]; f32[oB2 + i] = w.fc2_b[i];
        f32[oAlphaW + i] = w.alpha_w[i];
    }
    if (t0 == 0) { f32[oAlphaB] = w.alpha_b[0]; f32[oAlphaB + 1] = 0.f; f32[oAlphaB + 2] = 0.f; f32[oAlphaB + 3] = 0.f; }
    for (int i = t0; i < kColor * 64; i += stride) {              // Wx = view_fc[:, 283:346] (+ zero pad row 319)
        const int n = i / 64, j = i % 64;
        const float v = (j < kXyzPE) ? w.view_w[n * 346 + 283 + j] : 0.f;
        f32[oWct + (size_t)(kHidden + j) * kColor + n] = v;
    }
    for (int i = t0; i < kColor * 28; i += stride) {              // Wv = view_fc[:, 256:283]
        const int n = i / 28, j = i % 28;
        f32[oWvt + (size_t)j * kColor + n] = (j < kViewPE) ? w.view_w[n * 346 + 256 + j] : 0.f;
    }
    for (int i = t0; i < 3 * kColor; i += stride) f32[oRgbW + i] = w.rgb_w[i];
    if (t0 < 4) f32[oRgbB + t0] = (t0 < 3) ? w.rgb_b[t0] : 0.f;
}

// sigma of a sample whose gathered features are all zero: alpha_fc(relu(fc_2(relu(fc_1(relu(b_0)))))) (latent_xyzc.py:99-104)
__global__ void sigma_empty_kernel(nb_decoder_weights w, float* __restrict__ f32) {
    __shared__ float h0[kHidden], h1[kHidden], h2[kHidden];
    const int n = threadIdx.x;
    h0[n] = fmaxf(w.fc0_b[n], 0.f);
    __syncthreads();
    float a = w.fc1_b[n];
    for (int k = 0; k < kHidden; ++k) a = fmaf(w.fc1_w[n * kHidden + k], h0[k], a);
    h1[n] = fmaxf(a, 0.f);
    __syncthreads();
    a = w.fc2_b[n];
    for (int k = 0; k < kHidden; ++k) a = fmaf(w.fc2_w[n * kHidden + k], h1[k], a);
    h2[n] = fmaxf(a, 0.f);
    __syncthreads();
    if (n == 0) {
        float sgm = w.alpha_b[0];
        for (int k = 0; k < kHidden; ++k) sgm = fmaf(w.alpha_w[k], h2[k], sgm);
        f32[oSigmaEmpty] = sgm;
        f32[oSigmaEmpty + 1] = f32[oSigmaEmpty + 2] = f32[oSigmaEmpty + 3] = 0.f;
    }
}

// f-2: get_rays + get_near_far (if_nerf_data_utils.py:8-21, 54-69), one thread per pixel, fp64 like the numpy original.
__device__ __forceinline__ bool gen_ray(const nb_camera& cam, int pix, float (&of)[3], float (&df)[3], float& near, float& far) {
    const double i = (double)(float)(pix % cam.W), j = (double)(float)(pix / cam.W);   // np.arange(..., dtype=float32)
    // rays_o = -R^T T
    double o[3], pc[3], pw[3], d[3];
    for (int a = 0; a < 3; ++a) o[a] = -(cam.R[0 * 3 + a] * cam.T[0] + cam.R[1 * 3 + a] * cam.T[1] + cam.R[2 * 3 + a] * cam.T[2]);
    // pixel_camera = xy1 @ K_inv^T ; pixel_world = (pixel_camera - T) @ R
    for (int a = 0; a < 3; ++a) pc[a] = i * cam.K_inv[a * 3 + 0] + j * cam.K_inv[a * 3 + 1] + cam.K_inv[a * 3 + 2] - cam.T[a];
    for (int a = 0; a < 3; ++a) pw[a] = pc[0] * cam.R[0 * 3 + a] + pc[1] * cam.R[1 * 3 + a] + pc[2] * cam.R[2 * 3 + a];
    for (int a = 0; a < 3; ++a) d[a] = pw[a] - o[a];
    // the dataset casts to float32 BEFORE get_near_far (multi_view_demo_dataset.py / image_rays: ray_o.astype(np.float32))
    for (int a = 0; a < 3; ++a) { of[a] = (float)o[a]; df[a] = (float)d[a]; }
    const float nrm = ray_norm(df[0], df[1], df[2]);
    float tnear = -INFINITY, tfar = INFINITY;
    for (int a = 0; a < 3; ++a) {
        float v = __fdiv_rn(df[a], nrm);
        if (v < 1e-5f && v > -1e-10f) v = 1e-5f;
        if (v > -1e-5f && v < 1e-10f) v = -1e-5f;
        const float t0 = __fdiv_rn(__fsub_rn((float)cam.bounds[a], of[a]), v), t1 = __fdiv_rn(__fsub_rn((float)cam.bounds[3 + a], of[a]), v);
        tnear = fmaxf(tnear, fminf(t0, t1));
        tfar = fminf(tfar, fmaxf(t0, t1));
    }
    near = __fdiv_rn(tnear, nrm);
    far = __fdiv_rn(tfar, nrm);
    return tnear < tfar;
}

__global__ void gen_rays_kernel(nb_camera cam, float* __restrict__ ray_o, float* __restrict__ ray_d, float* __restrict__ near,
                                float* __restrict__ far, unsigned char* __restrict__ mask) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= cam.H * cam.W) return;
    float of[3], df[3], tn, tf;
    const bool hit = gen_ray(cam, idx, of, df, tn, tf);
    for (int a = 0; a < 3; ++a) { ray_o[idx * 3 + a] = of[a]; ray_d[idx * 3 + a] = df[a]; }
    near[idx] = tn;
    far[idx] = tf;
    mask[idx] = hit ? 1 : 0;
}

// one rank's interleaved shard, fixed shape: misses and pixels past the image become dead rays (near = far = 0)
__global__ void gen_rays_sharded_kernel(nb_camera cam, int rank, int world, int chunk, int n_local, float* __restrict__ ray_o,
                                        float* __restrict__ ray_d, float* __restrict__ near, float* __restrict__ far,
                                        unsigned char* __restrict__ mask) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_local) return;
    const long long pix = ((long long)(j / chunk) * world + rank) * chunk + j % chunk;
    float of[3] = {0.f, 0.f, 0.f}, df[3] = {0.f, 0.f, 1.f}, tn = 0.f, tf = 0.f;
    bool hit = false;
    if (pix < (long long)cam.H * cam.W) {
        hit = gen_ray(cam, (int)pix, of, df, tn, tf);
        if (!hit) tn = tf = 0.f;
    }
    for (int a = 0; a < 3; ++a) { ray_o[j * 3 + a] = of[a]; ray_d[j * 3 + a] = df[a]; }
    near[j] = tn;
    far[j] = tf;
    mask[j] = hit ? 1 : 0;
}

// fp16 split of an fp32 value: hi = fp16(x), lo = fp16(x - hi): hi + lo carries ~21 mantissa bits.
__device__ __forceinline__ __half f16_hi(float x) { return __float2half_rn(x); }
__device__ __forceinline__ __half f16_lo(float x) { return __float2half_rn(x - __half2float(__float2half_rn(x))); }

// The tensor-core kernel's weight stream (layout in nb_layout.h).  Runs after fold_Wc_kernel
// (reads the folded Wc from the fp32 section and the per-frame bias bc).
__global__ void stream_kernel(nb_decoder_weights w, const float* __restrict__ f32, const float* __restrict__ bc,
                              __half* __restrict__ seq, __half* __restrict__ frame_steps) {
    const int stride = gridDim.x * blockDim.x;
    const int t0 = blockIdx.x * blockDim.x + threadIdx.x;
    // L0 / L1 / L2: N = 256, stored per CTA half (pair layout, nb_layout.h): (hi, lo) planes grouped by 4 K-steps, then the bias step
    for (int layer = 0; layer < 3; ++layer) {
        const int K = layer == 0 ? kFeat : kHidden;
        const int nks = K / 16;
        const float* W = layer == 0 ? w.fc0_w : layer == 1 ? w.fc1_w : w.fc2_w;
        const float* Bv = layer == 0 ? w.fc0_b : layer == 1 ? w.fc1_b : w.fc2_b;
        __half* dst = seq + (layer == 0 ? sL0 : layer == 1 ? sL1 : sL2);
        for (int i = t0; i < (2 * nks + 1) * 256 * 16; i += stride) {
            const int sl = i / 4096, n = (i / 16) % 256, kk = i % 16;
            const int half = n >> 7, nl = n & 127;
            if (sl < 2 * nks) {
                const int ks = sl >> 1, lo = sl & 1;
                const int k = ks * 16 + kk;
                const float x = W[(size_t)n * K + (layer == 0 ? feat_tc_to_orig(k) : k)];
                dst[pair_step_offset(ks, lo, half, nks) + step_offset(nl, kk, 128)] = lo ? f16_lo(x) : f16_hi(x);
            } else {
                dst[pair_bias_offset(half, nks) + step_offset(nl, kk, 128)] =
                    kk == 0 ? f16_hi(Bv[n]) : kk == 1 ? f16_lo(Bv[n]) : __float2half_rn(0.f);
            }
        }
    }
    // L3: the folded colour layer, N = 128 as two 64-row halves.  common steps 0..20 -> seq, per-frame step 21 -> frame_steps[b][half]
    for (int i = t0; i < (kStepsL3 - 1 + w.batch) * kN3 * 16; i += stride) {
        int st = i / (kN3 * 16);
        const int n = (i / 16) % kN3, kk = i % 16;
        const int half = n / (kN3 / 2), nl = n % (kN3 / 2);
        int b = 0;
        __half* dst;
        if (st >= kStepsL3 - 1) { b = st - (kStepsL3 - 1); st = kStepsL3 - 1; dst = frame_steps + ((size_t)b * 2 + half) * kHalfTile3; }
        else dst = seq + sL3 + pair_l3_offset(st, half);
        float v = 0.f;
        bool lo = false;
        if (st < 16) {
            v = f32[oWct + (size_t)(st * 16 + kk) * kColor + n];
        } else {
            const int k2 = (st - 16) * 16 + kk;      // column of the per-point tile
            if (k2 < kXyzPE) v = w.view_w[n * 346 + 283 + k2];
            else if (k2 >= 64 && k2 < 64 + kViewPE) v = w.view_w[n * 346 + 256 + (k2 - 64)];
            else if (k2 == 92) v = bc[b * kColor + n];
            else if (k2 == 93) { v = bc[b * kColor + n]; lo = true; }
        }
        dst[step_offset(nl, kk, kN3 / 2)] = lo ? f16_lo(v) : f16_hi(v);
    }
}

}  // namespace nb

using namespace nb;

extern "C" {

int nb_abi_version(void) { return NB_ABI_VERSION; }
const char* nb_last_error(void) { return g_err; }
int nb_has_precision(int precision) {
    if (precision == NB_PRECISION_FP32) return 1;
    if (precision == NB_PRECISION_TC_FP16 || precision == NB_PRECISION_TC_FP16X3 || precision == NB_PRECISION_TC_TF32X3) return tc_available() ? 1 : 0;
    return 0;
}

static size_t dtype_size(int dtype) { return dtype == NB_DTYPE_F16 ? 2 : 4; }

size_t nb_packed_volume_level_offset(const int dims[NB_NUM_LEVELS][4], int batch, int dtype, int level) {
    size_t off = 0;
    for (int l = 0; l < level && l < NB_NUM_LEVELS; ++l)
        off += align256((size_t)batch * dims[l][0] * dims[l][1] * dims[l][2] * dims[l][3] * dtype_size(dtype));
    return off;
}

static size_t vox_words(const int d[4]) { return ((size_t)d[1] * d[2] * d[3] + 31) / 32; }
static size_t cell_words(const int d[4]) { return ((size_t)(d[1] + 1) * (d[2] + 1) * (d[3] + 1) + 31) / 32; }
// occupancy region after the four levels: per level [voxel bits (scratch)][cell bits], 256-B aligned each
static size_t occ_offset(const int dims[NB_NUM_LEVELS][4], int batch, int dtype, int level, int cell) {
    size_t off = nb_packed_volume_level_offset(dims, batch, dtype, NB_NUM_LEVELS);
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        if (l == level && !cell) return off;
        off += align256((size_t)batch * vox_words(dims[l]) * 4);
        if (l == level && cell) return off;
        off += align256((size_t)batch * cell_words(dims[l]) * 4);
    }
    return off;
}

size_t nb_packed_volume_bytes(const int dims[NB_NUM_LEVELS][4], int batch, int dtype) {
    return occ_offset(dims, batch, dtype, NB_NUM_LEVELS, 0);
}

int nb_pack_volume(const nb_volume_level levels[NB_NUM_LEVELS], int batch, int dtype, void* out_blob, size_t out_bytes,
                   void* stream) {
    if (!levels || !out_blob || batch <= 0) { set_error("nb_pack_volume: null argument or batch <= 0"); return NB_ERR_BAD_ARG; }
    if (dtype != NB_DTYPE_F32 && dtype != NB_DTYPE_F16) { set_error("nb_pack_volume: unknown dtype %d", dtype); return NB_ERR_BAD_ARG; }
    int dims[NB_NUM_LEVELS][4];
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        if (!levels[l].data || levels[l].C <= 0 || levels[l].C % 8 || levels[l].D <= 0 || levels[l].H <= 0 || levels[l].W <= 0) {
            set_error("nb_pack_volume: level %d has a null pointer or bad dims (C must be a multiple of 8)", l);
            return NB_ERR_BAD_ARG;
        }
        dims[l][0] = levels[l].C; dims[l][1] = levels[l].D; dims[l][2] = levels[l].H; dims[l][3] = levels[l].W;
    }
    if (out_bytes < nb_packed_volume_bytes(dims, batch, dtype)) { set_error("nb_pack_volume: out_bytes too small"); return NB_ERR_BAD_ARG; }
    cudaStream_t st = (cudaStream_t)stream;
    const size_t occ0 = occ_offset(dims, batch, dtype, 0, 0);
    cudaMemsetAsync((char*)out_blob + occ0, 0, nb_packed_volume_bytes(dims, batch, dtype) - occ0, st);
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        const size_t nvox = (size_t)levels[l].D * levels[l].H * levels[l].W;
        const size_t tiles = ((nvox + 31) / 32) * ((levels[l].C + 31) / 32) * batch;
        const int grid = (int)(tiles < kGridSMs * 16 ? tiles : kGridSMs * 16);
        char* dst = (char*)out_blob + nb_packed_volume_level_offset(dims, batch, dtype, l);
        unsigned* vb = (unsigned*)((char*)out_blob + occ_offset(dims, batch, dtype, l, 0));
        unsigned* cb = (unsigned*)((char*)out_blob + occ_offset(dims, batch, dtype, l, 1));
        if (dtype == NB_DTYPE_F16)
            pack_volume_kernel<__half><<<grid, 256, 0, st>>>(levels[l].data, (__half*)dst, levels[l].C, nvox, batch, vb, vox_words(dims[l]));
        else
            pack_volume_kernel<float><<<grid, 256, 0, st>>>(levels[l].data, (float*)dst, levels[l].C, nvox, batch, vb, vox_words(dims[l]));
        const size_t ncellp = cell_words(dims[l]) * 32 * batch;
        const int cgrid = (int)((ncellp + 255) / 256 < kGridSMs * 8 ? (ncellp + 255) / 256 : kGridSMs * 8);
        cell_occupancy_kernel<<<cgrid, 256, 0, st>>>(vb, cb, levels[l].D, levels[l].H, levels[l].W, vox_words(dims[l]),
                                                     cell_words(dims[l]), batch);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_pack_volume: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

size_t nb_packed_weights_bytes(int batch) { return packed_weights_bytes(batch < 1 ? 1 : batch); }

int nb_pack_weights(const nb_decoder_weights* w, void* out_blob, size_t out_bytes, void* stream) {
    if (!w || !out_blob) { set_error("nb_pack_weights: null argument"); return NB_ERR_BAD_ARG; }
    const void* ptrs[] = {w->fc0_w, w->fc0_b, w->fc1_w, w->fc1_b, w->fc2_w, w->fc2_b, w->alpha_w, w->alpha_b, w->feature_w,
                          w->feature_b, w->latent_w, w->latent_b, w->view_w, w->view_b, w->rgb_w, w->rgb_b, w->latent,
                          w->latent_index};
    for (size_t i = 0; i < sizeof(ptrs) / sizeof(ptrs[0]); ++i)
        if (!ptrs[i]) { set_error("nb_pack_weights: weight pointer #%zu is null", i); return NB_ERR_BAD_ARG; }
    if (w->batch <= 0 || w->num_train_frame <= 0) { set_error("nb_pack_weights: batch / num_train_frame must be > 0"); return NB_ERR_BAD_ARG; }
    if (out_bytes < packed_weights_bytes(w->batch)) { set_error("nb_pack_weights: out_bytes too small"); return NB_ERR_BAD_ARG; }
    cudaStream_t st = (cudaStream_t)stream;
    char* base = (char*)out_blob;
    float* f32 = (float*)base;
    __half* f16 = (__half*)(base + kF16ByteOffset);
    double* T = (double*)(base + kScratchByteOffset);
    float* bc = (float*)(base + kBcByteOffset);
    double* u = (double*)(base + u_byte_offset(w->batch));
    const int n1 = kColor * kHidden + w->batch * kHidden;
    fold_T_kernel<<<(n1 + 127) / 128, 128, 0, st>>>(*w, T, u);
    const int n2 = kColor * kHidden + w->batch * kColor;
    fold_Wc_kernel<<<(n2 + 127) / 128, 128, 0, st>>>(*w, T, u, f32, f16, bc);
    relayout_kernel<<<kGridSMs, 256, 0, st>>>(*w, f32, f16);
    sigma_empty_kernel<<<1, kHidden, 0, st>>>(*w, f32);
    stream_kernel<<<kGridSMs, 256, 0, st>>>(*w, f32, bc, f16, (__half*)(base + frame_step_byte_offset(w->batch)));
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_pack_weights: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_render_fwd_launches(int precision) { return precision == NB_PRECISION_FP32 ? 1 : precision == NB_PRECISION_TC_TF32X3 ? 9 : 3; }

size_t nb_render_fwd_workspace_bytes(int batch, int n_rays, int n_samples) {
    if (batch <= 0 || n_rays <= 0 || n_samples <= 0) return 0;
    return render_tc_list_workspace_bytes(batch, n_rays, n_samples);
}

}  // extern "C"

namespace nb {

int fill_frame_params(const nb_render_args* a, const char* who, RenderParams* out) {
    if (!a) { set_error("%s: null args", who); return NB_ERR_BAD_ARG; }
    if (a->batch <= 0) { set_error("%s: batch must be > 0", who); return NB_ERR_BAD_ARG; }
    if (!a->R || !a->Th || !a->bounds || !a->volume_blob || !a->weights_blob) {
        set_error("%s: a frame pointer (R, Th, bounds, volume_blob, weights_blob) is null", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->volume_dtype != NB_DTYPE_F32 && a->volume_dtype != NB_DTYPE_F16) { set_error("%s: bad volume_dtype", who); return NB_ERR_BAD_ARG; }
    static const int expectC[4] = {32, 64, 128, 128};
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        if (a->level_dims[l][0] != expectC[l]) {
            set_error("%s: level %d has %d channels, decoder expects %d (fc_0 is 352-wide)", who, l, a->level_dims[l][0], expectC[l]);
            return NB_ERR_UNSUPPORTED;
        }
        if (a->level_dims[l][1] <= 0 || a->level_dims[l][2] <= 0 || a->level_dims[l][3] <= 0) { set_error("%s: bad level dims", who); return NB_ERR_BAD_ARG; }
    }
    for (int i = 0; i < 3; ++i)
        if (!(a->voxel_size[i] > 0.f) || a->out_sh[i] <= 0) { set_error("%s: voxel_size/out_sh must be > 0", who); return NB_ERR_BAD_ARG; }

    RenderParams p{};
    p.batch = a->batch;
    p.R = a->R; p.Th = a->Th; p.bounds = a->bounds;
    for (int i = 0; i < 3; ++i) { p.voxel_size[i] = a->voxel_size[i]; p.out_sh[i] = (float)a->out_sh[i]; }
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        p.lvl_C[l] = a->level_dims[l][0]; p.lvl_D[l] = a->level_dims[l][1]; p.lvl_H[l] = a->level_dims[l][2]; p.lvl_W[l] = a->level_dims[l][3];
        p.lvl_off[l] = nb_packed_volume_level_offset(a->level_dims, a->batch, a->volume_dtype, l);
        p.lvl_bstride[l] = (size_t)p.lvl_C[l] * p.lvl_D[l] * p.lvl_H[l] * p.lvl_W[l];
        p.occ_off[l] = occ_offset(a->level_dims, a->batch, a->volume_dtype, l, 1);
        p.occ_bstride[l] = cell_words(a->level_dims[l]);
    }
    p.volume = a->volume_blob;
    const char* wb = (const char*)a->weights_blob;
    p.wf32 = (const float*)wb;
    p.wf16 = (const __half*)(wb + kF16ByteOffset);
    p.bc = (const float*)(wb + kBcByteOffset);
    p.wframe = (const __half*)(wb + frame_step_byte_offset(a->batch));
    *out = p;
    return NB_OK;
}

int fill_ray_params(const nb_render_args* a, const char* who, RenderParams* out) {
    if (a->n_rays < 0 || a->n_samples <= 0) { set_error("%s: bad n_rays/n_samples", who); return NB_ERR_BAD_ARG; }
    if (!a->ray_o || !a->ray_d || !a->near || !a->far || !a->rgb_map || !a->disp_map || !a->acc_map || !a->depth_map) {
        set_error("%s: a ray or output-map pointer (ray_o, ray_d, near, far, rgb_map, disp_map, acc_map, depth_map) is null", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->out_ray_stride < 0) { set_error("%s: out_ray_stride < 0", who); return NB_ERR_BAD_ARG; }
    if (a->mask_msks && (a->mask_R0 != nullptr) != (a->mask_Th0 != nullptr)) { set_error("%s: mask_R0 and mask_Th0 go together", who); return NB_ERR_BAD_ARG; }
    if (a->mask_msks && (a->batch != 1 || !a->mask_RT || !a->mask_Ks || a->mask_nv <= 0 || a->mask_H <= 0 || a->mask_W <= 0)) {
        set_error("%s: mask views need batch == 1 (as upstream), RT, Ks and positive nv/H/W", who);
        return NB_ERR_BAD_ARG;
    }

    RenderParams& p = *out;
    p.n_rays = a->n_rays; p.n_samples = a->n_samples;
    p.ray_o = a->ray_o; p.ray_d = a->ray_d; p.near = a->near; p.far = a->far; p.t_vals = a->t_vals; p.t_rand = a->t_rand; p.z_user = a->z_vals;
    p.rgb_stride = a->out_ray_stride ? a->out_ray_stride : 3;
    p.map_stride = a->out_ray_stride ? a->out_ray_stride : 1;
    p.white_bkgd = a->white_bkgd;
    p.skip_empty = a->skip_empty ? 1 : 0;
    p.rgb_map = a->rgb_map; p.disp_map = a->disp_map; p.acc_map = a->acc_map; p.weights = a->weights; p.depth_map = a->depth_map; p.raw = a->raw; p.trace = a->trace; p.save = a->save; p.stats = a->stats;
    p.mask_msks = a->mask_msks; p.mask_RT = a->mask_RT; p.mask_Ks = a->mask_Ks;
    p.mask_nv = a->mask_msks ? a->mask_nv : 0; p.mask_H = a->mask_H; p.mask_W = a->mask_W;
    p.mask_R0 = a->mask_msks ? a->mask_R0 : nullptr; p.mask_Th0 = a->mask_msks ? a->mask_Th0 : nullptr;
    return NB_OK;
}

}  // namespace nb

extern "C" {

int nb_gen_rays(const nb_camera* cam, float* ray_o, float* ray_d, float* near, float* far, unsigned char* mask_at_box, void* stream) {
    if (!cam || !ray_o || !ray_d || !near || !far || !mask_at_box || cam->H <= 0 || cam->W <= 0) {
        set_error("nb_gen_rays: null argument or empty image");
        return NB_ERR_BAD_ARG;
    }
    const int n = cam->H * cam->W;
    gen_rays_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*cam, ray_o, ray_d, near, far, mask_at_box);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_gen_rays: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_gen_rays_sharded(const nb_camera* cam, int rank, int world, int chunk, int n_local, float* ray_o, float* ray_d, float* near,
                        float* far, unsigned char* mask_at_box, void* stream) {
    if (!cam || !ray_o || !ray_d || !near || !far || !mask_at_box || cam->H <= 0 || cam->W <= 0 || world <= 0 || rank < 0 ||
        rank >= world || chunk <= 0 || n_local < 0) {
        set_error("nb_gen_rays_sharded: null argument, empty image or bad rank / world / chunk");
        return NB_ERR_BAD_ARG;
    }
    if (n_local == 0) return NB_OK;
    gen_rays_sharded_kernel<<<(n_local + 255) / 256, 256, 0, (cudaStream_t)stream>>>(*cam, rank, world, chunk, n_local, ray_o, ray_d,
                                                                                      near, far, mask_at_box);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("nb_gen_rays_sharded: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

int nb_decode_density(const nb_render_args* a, const float* points, int n_points, float* sigma, void* stream) {
    if (!a || !points || !sigma || n_points < 0) { set_error("nb_decode_density: null argument"); return NB_ERR_BAD_ARG; }
    RenderParams p;
    const int stp = fill_frame_params(a, "nb_decode_density", &p);
    if (stp != NB_OK) return stp;
    return launch_density_f32(p, a->volume_dtype, points, n_points, sigma, (cudaStream_t)stream);
}

size_t nb_decode_density_workspace_bytes(int batch, int n_points) {
    if (batch <= 0 || n_points <= 0) return 0;
    return density_tc_list_workspace_bytes(batch, n_points);
}

int nb_decode_density_list(const nb_render_args* a, const float* points, int n_points, float* sigma, void* stream) {
    if (!a || !points || !sigma || n_points < 0) { set_error("nb_decode_density_list: null argument or n_points < 0"); return NB_ERR_BAD_ARG; }
    if (a->precision != NB_PRECISION_TC_FP16X3 && a->precision != NB_PRECISION_TC_FP16) {
        set_error("nb_decode_density_list: precision %d; it runs NB_PRECISION_TC_FP16X3 or NB_PRECISION_TC_FP16 (exact fp32: "
                  "nb_decode_density)", a->precision);
        return NB_ERR_BAD_ARG;
    }
    RenderParams p;
    const int stp = fill_frame_params(a, "nb_decode_density_list", &p);
    if (stp != NB_OK) return stp;
    p.skip_empty = a->skip_empty ? 1 : 0; p.stats = a->stats; p.trace = a->trace;
    return launch_density_tc_list(p, a->volume_dtype, a->precision == NB_PRECISION_TC_FP16X3 ? 3 : 1, points, n_points, sigma,
                                  a->workspace, a->workspace_bytes, (cudaStream_t)stream);
}

int nb_render_fwd(const nb_render_args* a, void* stream) {
    if (a && a->n_rays == 0 && a->batch > 0 && a->n_samples > 0) return NB_OK;
    RenderParams p;
    int stp = fill_frame_params(a, "nb_render_fwd", &p);
    if (stp == NB_OK) stp = fill_ray_params(a, "nb_render_fwd", &p);
    if (stp != NB_OK) return stp;
    if (a->save && a->mask_msks) { set_error("nb_render_fwd: mask views are an inference feature (no activation record)"); return NB_ERR_UNSUPPORTED; }
    if (a->save && a->precision != NB_PRECISION_FP32 && a->precision != NB_PRECISION_TC_TF32X3) {
        set_error("nb_render_fwd: the activation record for nb_render_bwd is written by NB_PRECISION_FP32 and NB_PRECISION_TC_TF32X3 only");
        return NB_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == NB_PRECISION_TC_TF32X3) return launch_train_fwd(p, a->volume_dtype, st);
    if (a->precision == NB_PRECISION_FP32) return launch_render_f32(p, a->volume_dtype, st);
    if (a->precision == NB_PRECISION_TC_FP16 || a->precision == NB_PRECISION_TC_FP16X3) {
        const int passes = a->precision == NB_PRECISION_TC_FP16X3 ? 3 : 1;
        // one pipeline for every tensor-core call: classify (+ mask views) -> decoder over the frame's sample list -> composite;
        // skip_empty = 0 lists every sample (dense evaluation), bit-identical to the skipping run
        return launch_render_tc_list(p, a->volume_dtype, passes, a->workspace, a->workspace_bytes, st);
    }
    set_error("nb_render_fwd: unknown precision %d", a->precision);
    return NB_ERR_BAD_ARG;
}

}  // extern "C"
