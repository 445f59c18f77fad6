// nb_spconv_fwd / nb_spconv_bwd (include/neuralbody_b200.h): the reference's SparseConvNet encode (lib/networks/
// latent_xyzc.py:30-39,166-274, spconv 1.2.1 semantics as oracle/spconv_oracle.py restates them) as sparse convolutions
// over the active sites only, forward and backward, without a host wait.
//   active sets:  level 0 = the sites of the input points (the highest point index wins a shared site); level l+1 = the
//                 sites whose 3x3x3 stride-2 window (padding 1) holds an active level-l site.  Each level has a dense int32
//                 site -> row grid (-1 = inactive); rows are numbered in site order by a CUB scan, so the row order does
//                 not depend on scheduling.  Row buffers are sized from static bounds (level 0 <= n_points, level l+1 <=
//                 min(8 x level l, grid sites)); the counts stay on the device and every row kernel reads them there.
//   rulebooks:    per level, row -> the 27 neighbour rows (SubMConv3d); per strided conv, output row -> the 27 input rows
//                 and its transpose, input row -> the output row each offset feeds (for the data gradient).
//   convolution:  one gather-GEMM per 64-row tile, looping over the 27 offsets (offsets with no neighbour in the tile are
//                 skipped), fp32 FFMA; the same kernel with the transposed weights and the mirrored (SubM) or transposed
//                 (strided) rulebook is the data gradient.  The weight gradient is a gather-GEMM over rows per offset,
//                 reduced into dW with fp32 atomics.
//   BatchNorm:    the conv epilogue sums x and x^2 per channel in float64 (atomics); one 1-CTA kernel turns them into the
//                 batch statistics (train: biased variance to normalise, unbiased into running_var, num_batches_tracked
//                 += 1) or reads the running statistics (eval); then BN + ReLU is element-wise.
//   volumes:      each net_l is zeroed and its active rows scattered into (B, C, D, H, W).
// Everything the backward needs (grids, rulebooks, pre-BN and post-ReLU rows, statistics) stays in the workspace.
#include <cub/device/device_scan.cuh>
#include <thrust/iterator/transform_iterator.h>
#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kLayers = NB_SPCONV_LAYERS;
constexpr int kGrids = NB_NUM_LEVELS + 1;      // the input grid and the four strided levels
constexpr int kCode = NB_SPCONV_CODE_DIM;
constexpr int kThreads = 256;

struct LayerDef {
    int cin, cout, lin, stride;                // lin: grid level of the input rows; the output is at lin + (stride == 2)
};
// latent_xyzc.py:166-204: conv0 (2 SubM) down0 conv1 (2) down1 conv2 (3) down2 conv3 (3) down3 conv4 (3)
constexpr LayerDef kDefs[kLayers] = {
    {16, 16, 0, 1},   {16, 16, 0, 1},   {16, 32, 0, 2},   {32, 32, 1, 1},   {32, 32, 1, 1},   {32, 64, 1, 2},
    {64, 64, 2, 1},   {64, 64, 2, 1},   {64, 64, 2, 1},   {64, 128, 2, 2},  {128, 128, 3, 1}, {128, 128, 3, 1},
    {128, 128, 3, 1}, {128, 128, 3, 2}, {128, 128, 4, 1}, {128, 128, 4, 1}, {128, 128, 4, 1}};
constexpr int kOutLayer[NB_NUM_LEVELS] = {4, 8, 12, 16};      // net1..net4 are the outputs of these layers
inline int lout(int j) { return kDefs[j].lin + (kDefs[j].stride == 2); }

struct IsActive {
    __host__ __device__ int operator()(int v) const { return v >= 0 ? 1 : 0; }
};

struct Plan {
    int B;
    int dims[kGrids][3];
    long long sites[kGrids];                   // B * D * H * W
    long long cap[kGrids];                     // row bound
    size_t idx[kGrids], site[kGrids], nbr[kGrids], snbr[kGrids - 1], snbrT[kGrids - 1];
    size_t src0, counts, scan, cub, cub_bytes, feat0;
    size_t x[kLayers], y[kLayers], stats, coef;
    size_t dA, dB, dstat, bcoef;
    size_t total;
};

// Fills *p; returns 0 or a message for the caller's error.
const char* make_plan(int batch, int n_points, const int out_sh[3], Plan* p) {
    p->B = batch;
    for (int a = 0; a < 3; ++a) p->dims[0][a] = out_sh[a];
    for (int l = 1; l < kGrids; ++l)
        for (int a = 0; a < 3; ++a) p->dims[l][a] = (p->dims[l - 1][a] - 1) / 2 + 1;
    for (int l = 0; l < kGrids; ++l) {
        p->sites[l] = (long long)batch * p->dims[l][0] * p->dims[l][1] * p->dims[l][2];
        const long long bound = l == 0 ? (long long)n_points : 8 * p->cap[l - 1];
        p->cap[l] = bound < p->sites[l] ? bound : p->sites[l];
    }
    if (p->sites[0] >= (1LL << 31)) return "B * D * H * W of the input grid must be < 2^31";
    size_t off = 0;
    auto take = [&off](size_t bytes) { const size_t o = off; off += align256(bytes); return o; };
    for (int l = 0; l < kGrids; ++l) {
        p->idx[l] = take(p->sites[l] * 4);
        p->site[l] = take(p->cap[l] * 4);
        p->nbr[l] = take(p->cap[l] * 27 * 4);
    }
    for (int l = 0; l + 1 < kGrids; ++l) {
        p->snbr[l] = take(p->cap[l + 1] * 27 * 4);
        p->snbrT[l] = take(p->cap[l] * 27 * 4);
    }
    p->src0 = take(p->cap[0] * 4);
    p->counts = take(kGrids * 4);
    p->scan = take(p->sites[0] * 4);
    size_t cub_bytes = 0;
    for (int l = 0; l < kGrids; ++l) {
        size_t b = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, b, thrust::make_transform_iterator((int*)nullptr, IsActive()), (int*)nullptr,
                                      (int)p->sites[l]);
        if (b > cub_bytes) cub_bytes = b;
    }
    p->cub_bytes = cub_bytes;
    p->cub = take(cub_bytes);
    p->feat0 = take(p->cap[0] * kCode * 4);
    long long dmax = 0;
    for (int j = 0; j < kLayers; ++j) {
        const long long rows = p->cap[lout(j)];
        p->x[j] = take(rows * kDefs[j].cout * 4);
        p->y[j] = take(rows * kDefs[j].cout * 4);
        const long long a = rows * kDefs[j].cout, b = p->cap[kDefs[j].lin] * kDefs[j].cin;
        dmax = a > dmax ? a : dmax;
        dmax = b > dmax ? b : dmax;
    }
    p->stats = take((size_t)kLayers * 2 * 128 * sizeof(double));
    p->coef = take((size_t)kLayers * 2 * 128 * sizeof(float));
    p->dA = take(dmax * 4);
    p->dB = take(dmax * 4);
    p->dstat = take(2 * 128 * sizeof(double));
    p->bcoef = take(3 * 128 * sizeof(float));
    p->total = off;
    return nullptr;
}

__device__ __forceinline__ void decode(long long s, const int3 d, int& b, int& z, int& y, int& x) {
    x = (int)(s % d.z); s /= d.z;
    y = (int)(s % d.y); s /= d.y;
    z = (int)(s % d.x);
    b = (int)(s / d.x);
}
__device__ __forceinline__ int encode(int b, int z, int y, int x, const int3 d) { return ((b * d.x + z) * d.y + y) * d.z + x; }

// level 0: a site's value is the highest index of the points on it (the emulation's duplicate rule)
__global__ void mark_points_kernel(const int* __restrict__ coord, int n_points, int B, int3 d, int* __restrict__ idx) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= n_points) return;
    const int b = coord[4 * (size_t)i], z = coord[4 * (size_t)i + 1], y = coord[4 * (size_t)i + 2], x = coord[4 * (size_t)i + 3];
    if (b < 0 || b >= B || z < 0 || z >= d.x || y < 0 || y >= d.y || x < 0 || x >= d.z) return;
    atomicMax(idx + encode(b, z, y, x, d), i);
}

// level l+1: every output site whose window holds active row r (input c = 2 o - 1 + k, k in 0..2 per axis)
__global__ void mark_strided_kernel(const int* __restrict__ site, const int* __restrict__ count, int3 din, int3 dout,
                                    int* __restrict__ idx_out) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= *count) return;
    int b, c[3];
    decode(site[r], din, b, c[0], c[1], c[2]);
    const int ext[3] = {dout.x, dout.y, dout.z};
    int o[3][2], n[3];
    for (int a = 0; a < 3; ++a) {
        n[a] = 0;
        for (int k = 0; k < 3; ++k) {
            const int num = c[a] + 1 - k;
            if (num % 2 == 0 && num / 2 >= 0 && num / 2 < ext[a]) o[a][n[a]++] = num / 2;
        }
    }
    for (int i = 0; i < n[0]; ++i)
        for (int j = 0; j < n[1]; ++j)
            for (int k = 0; k < n[2]; ++k) idx_out[encode(b, o[0][i], o[1][j], o[2][k], dout)] = 0;
}

// site -> row (the scan's value), row -> site, and the row count; level 0 also keeps each row's point
__global__ void finalize_kernel(int* __restrict__ idx, const int* __restrict__ scan, int n_sites, int* __restrict__ site,
                                int* __restrict__ src0, int* __restrict__ count) {
    const int s = blockIdx.x * kThreads + threadIdx.x;
    if (s >= n_sites) return;
    const int v = idx[s];
    if (s == n_sites - 1) *count = scan[s] + (v >= 0);
    if (v < 0) return;
    const int r = scan[s];
    site[r] = s;
    if (src0) src0[r] = v;
    idx[s] = r;
}

__global__ void subm_rules_kernel(const int* __restrict__ site, const int* __restrict__ count, int3 d,
                                  const int* __restrict__ idx, int* __restrict__ nbr) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int r = (int)(e / 27), k = (int)(e % 27);
    if (r >= *count) return;
    int b, z, y, x;
    decode(site[r], d, b, z, y, x);
    z += k / 9 - 1; y += (k / 3) % 3 - 1; x += k % 3 - 1;
    nbr[e] = (z >= 0 && z < d.x && y >= 0 && y < d.y && x >= 0 && x < d.z) ? idx[encode(b, z, y, x, d)] : -1;
}

__global__ void strided_rules_kernel(const int* __restrict__ site_out, const int* __restrict__ count_out, int3 dout, int3 din,
                                     const int* __restrict__ idx_in, int* __restrict__ snbr, int* __restrict__ snbrT) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int o = (int)(e / 27), k = (int)(e % 27);
    if (o >= *count_out) return;
    int b, z, y, x;
    decode(site_out[o], dout, b, z, y, x);
    z = 2 * z - 1 + k / 9; y = 2 * y - 1 + (k / 3) % 3; x = 2 * x - 1 + k % 3;
    const int ri = (z >= 0 && z < din.x && y >= 0 && y < din.y && x >= 0 && x < din.z) ? idx_in[encode(b, z, y, x, din)] : -1;
    snbr[e] = ri;
    if (ri >= 0) snbrT[(size_t)ri * 27 + k] = o;
}

__global__ void gather_code_kernel(const float* __restrict__ code, int n_vert, const int* __restrict__ src0,
                                   const int* __restrict__ count, float* __restrict__ feat0) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int r = (int)(e / kCode), c = (int)(e % kCode);
    if (r >= *count) return;
    feat0[e] = code[(size_t)(src0[r] % n_vert) * kCode + c];
}

// out[r] = sum_k in[map[r][k']] @ B_k for the rows r < *count, k' = 26 - k when `mirror` (the transpose of a SubM rulebook),
// B_k = W[k] (K x N, W = [27][K][N]) or, TW, W[k]^T (W = [27][N][K]).  64-row tiles, 256 threads of 4 rows x N/16 columns.
// stats (N doubles of sum, then N of the sum of squares of the outputs) is accumulated into when non-null.
template <int K, int N, bool TW>
__global__ void __launch_bounds__(kThreads) gather_gemm_kernel(const float* __restrict__ in, const int* __restrict__ map,
                                                               int mirror, const float* __restrict__ W,
                                                               const int* __restrict__ count, float* __restrict__ out,
                                                               double* __restrict__ stats) {
    constexpr int TM = 64, KC = K < 32 ? K : 32, TN = N / 16;
    __shared__ float As[KC][TM + 1];
    __shared__ float Bs[KC][N + 1];
    __shared__ int src[TM];
    const int n = *count, r0 = blockIdx.x * TM;
    if (r0 >= n) return;
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    float acc[4][TN];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
    for (int k = 0; k < 27; ++k) {
        int s = -1;
        if (t < TM && r0 + t < n) s = map[(size_t)(r0 + t) * 27 + (mirror ? 26 - k : k)];
        if (t < TM) src[t] = s;
        if (!__syncthreads_or(s >= 0)) continue;
        float part[4][TN];             // this offset's products, summed apart and then added: shorter rounding chains
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) part[i][j] = 0.f;
        for (int kc = 0; kc < K; kc += KC) {
            for (int e = t; e < TM * KC; e += kThreads) {
                const int m = e / KC, c = e % KC, sm = src[m];
                As[c][m] = sm >= 0 ? __ldg(in + (size_t)sm * K + kc + c) : 0.f;
            }
            for (int e = t; e < KC * N; e += kThreads) {
                if (!TW) {
                    const int c = e / N, nn = e % N;
                    Bs[c][nn] = __ldg(W + ((size_t)k * K + kc + c) * N + nn);
                } else {
                    const int nn = e / KC, c = e % KC;
                    Bs[c][nn] = __ldg(W + ((size_t)k * N + nn) * K + kc + c);
                }
            }
            __syncthreads();
#pragma unroll 8
            for (int c = 0; c < KC; ++c) {
                float a[4], b[TN];
#pragma unroll
                for (int i = 0; i < 4; ++i) a[i] = As[c][ty * 4 + i];
#pragma unroll
                for (int j = 0; j < TN; ++j) b[j] = Bs[c][tx + 16 * j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < TN; ++j) part[i][j] = fmaf(a[i], b[j], part[i][j]);
            }
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < TN; ++j) acc[i][j] += part[i][j];
    }
    double s1[TN], s2[TN];
#pragma unroll
    for (int j = 0; j < TN; ++j) s1[j] = s2[j] = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty * 4 + i;
        if (r < n) {
#pragma unroll
            for (int j = 0; j < TN; ++j) {
                out[(size_t)r * N + tx + 16 * j] = acc[i][j];
                s1[j] += (double)acc[i][j];
                s2[j] += (double)acc[i][j] * (double)acc[i][j];
            }
        }
    }
    if (stats) {
        __shared__ double red[2][kThreads / 32][N];
        const int lane = t & 31, warp = t >> 5;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            s1[j] += __shfl_xor_sync(0xffffffffu, s1[j], 16);
            s2[j] += __shfl_xor_sync(0xffffffffu, s2[j], 16);
            if (lane < 16) {
                red[0][warp][tx + 16 * j] = s1[j];
                red[1][warp][tx + 16 * j] = s2[j];
            }
        }
        __syncthreads();
        for (int c = t; c < N; c += kThreads) {
            double a = 0.0, b = 0.0;
            for (int w = 0; w < kThreads / 32; ++w) { a += red[0][w][c]; b += red[1][w][c]; }
            atomicAdd(stats + c, a);
            atomicAdd(stats + N + c, b);
        }
    }
}

// dW[k] += sum over rows o < *count of in[map[o][k]]^T dx[o]: blockIdx.y = k, 256 rows per CTA in 32-row steps; each
// thread holds K/16 x N/16 entries and adds them into dW once.
template <int K, int N>
__global__ void __launch_bounds__(kThreads) wgrad_kernel(const float* __restrict__ in, const int* __restrict__ map,
                                                         const float* __restrict__ dx, const int* __restrict__ count,
                                                         float* __restrict__ dW) {
    constexpr int TR = 32, RC = 256, TI = K / 16, TJ = N / 16;
    __shared__ float As[TR][K + 1];
    __shared__ float Bs[TR][N + 1];
    __shared__ int src[TR];
    const int k = blockIdx.y, n = *count, r0 = blockIdx.x * RC;
    if (r0 >= n) return;
    const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
    const int r1 = r0 + RC < n ? r0 + RC : n;
    float acc[TI][TJ];
#pragma unroll
    for (int i = 0; i < TI; ++i)
#pragma unroll
        for (int j = 0; j < TJ; ++j) acc[i][j] = 0.f;
    for (int rt = r0; rt < r1; rt += TR) {
        int s = -1;
        if (t < TR && rt + t < r1) s = map[(size_t)(rt + t) * 27 + k];
        if (t < TR) src[t] = s;
        if (!__syncthreads_or(s >= 0)) continue;
        for (int e = t; e < TR * K; e += kThreads) {
            const int rr = e / K, c = e % K, sm = src[rr];
            As[rr][c] = sm >= 0 ? __ldg(in + (size_t)sm * K + c) : 0.f;
        }
        for (int e = t; e < TR * N; e += kThreads) {
            const int rr = e / N, c = e % N;
            Bs[rr][c] = src[rr] >= 0 ? __ldg(dx + (size_t)(rt + rr) * N + c) : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < TR; ++rr) {
            float a[TI], b[TJ];
#pragma unroll
            for (int i = 0; i < TI; ++i) a[i] = As[rr][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < TJ; ++j) b[j] = Bs[rr][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < TI; ++i)
#pragma unroll
                for (int j = 0; j < TJ; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TI; ++i)
#pragma unroll
        for (int j = 0; j < TJ; ++j) atomicAdd(dW + ((size_t)k * K + ty + 16 * i) * N + tx + 16 * j, acc[i][j]);
}

// BatchNorm statistics of one layer (one CTA of 128 threads): coef = (mean[C], 1 / sqrt(var + eps)[C])
__global__ void bn_stats_kernel(const double* __restrict__ sums, const int* __restrict__ count, int C, int training,
                                float momentum, float eps, float* __restrict__ rmean, float* __restrict__ rvar,
                                long long* __restrict__ nbt, float* __restrict__ coef) {
    const int c = threadIdx.x;
    if (c >= C) return;
    double mean, var;
    if (training) {
        const double n = *count > 1 ? (double)*count : 1.0;
        mean = sums[c] / n;
        var = sums[C + c] / n - mean * mean;
        var = var > 0.0 ? var : 0.0;
        const double unbiased = var * n / (n - 1.0 > 1.0 ? n - 1.0 : 1.0);
        rmean[c] = (1.f - momentum) * rmean[c] + momentum * (float)mean;
        rvar[c] = (1.f - momentum) * rvar[c] + momentum * (float)unbiased;
        if (c == 0) *nbt += 1;
    } else {
        mean = rmean[c];
        var = rvar[c];
    }
    coef[c] = (float)mean;
    coef[C + c] = (float)(1.0 / sqrt(var + (double)eps));
}

__global__ void bn_relu_kernel(const float* __restrict__ x, const float* __restrict__ coef, const float* __restrict__ gamma,
                               const float* __restrict__ beta, int C, const int* __restrict__ count, float* __restrict__ y) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= (size_t)*count * C) return;
    const int c = (int)(e % C);
    const float v = (x[e] - coef[c]) * coef[C + c];
    y[e] = fmaxf(v * gamma[c] + beta[c], 0.f);
}

__global__ void scatter_volume_kernel(const float* __restrict__ rows, const int* __restrict__ site, const int* __restrict__ count,
                                      int C, long long dhw, float* __restrict__ vol) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int r = (int)(e / C), c = (int)(e % C);
    if (r >= *count) return;
    const long long s = site[r], b = s / dhw;
    vol[(b * C + c) * dhw + s % dhw] = rows[e];
}

// rows[r] (+)= vol at row r's site
__global__ void gather_volume_kernel(const float* __restrict__ vol, const int* __restrict__ site, const int* __restrict__ count,
                                     int C, long long dhw, int accumulate, float* __restrict__ rows) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int r = (int)(e / C), c = (int)(e % C);
    if (r >= *count) return;
    const long long s = site[r], b = s / dhw;
    const float v = vol[(b * C + c) * dhw + s % dhw];
    rows[e] = accumulate ? rows[e] + v : v;
}

// sums = (sum dz, sum dz * xhat) per channel, dz = dy where the ReLU passed
__global__ void __launch_bounds__(kThreads) bn_bwd_reduce_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                                                 const float* __restrict__ x, const float* __restrict__ coef,
                                                                 int C, const int* __restrict__ count, double* __restrict__ sums) {
    __shared__ double red[2][kThreads];
    const int t = threadIdx.x, c = t % C, lane = t / C, lanes = kThreads / C, n = *count;
    const float mean = coef[c], istd = coef[C + c];
    double s1 = 0.0, s2 = 0.0;
    for (int r = blockIdx.x * lanes + lane; r < n; r += gridDim.x * lanes) {
        const size_t e = (size_t)r * C + c;
        const float dz = y[e] > 0.f ? dy[e] : 0.f;
        s1 += dz;
        s2 += (double)dz * (double)((x[e] - mean) * istd);
    }
    red[0][t] = s1;
    red[1][t] = s2;
    __syncthreads();
    if (lane == 0) {
        for (int l = 1; l < lanes; ++l) { s1 += red[0][l * C + c]; s2 += red[1][l * C + c]; }
        atomicAdd(sums + c, s1);
        atomicAdd(sums + C + c, s2);
    }
}

// d gamma, d beta, and dx = gamma istd (dz - k2 - xhat k3): k2 = mean(dz), k3 = mean(dz xhat) with batch statistics, 0 with
// the running ones
__global__ void bn_bwd_coef_kernel(const double* __restrict__ sums, const int* __restrict__ count, const float* __restrict__ gamma,
                                   const float* __restrict__ coef, int C, int training, float* __restrict__ dgamma,
                                   float* __restrict__ dbeta, float* __restrict__ bcoef) {
    const int c = threadIdx.x;
    if (c >= C) return;
    dgamma[c] = (float)sums[C + c];
    dbeta[c] = (float)sums[c];
    const double n = *count > 1 ? (double)*count : 1.0;
    bcoef[c] = gamma[c] * coef[C + c];
    bcoef[C + c] = training ? (float)(sums[c] / n) : 0.f;
    bcoef[2 * C + c] = training ? (float)(sums[C + c] / n) : 0.f;
}

__global__ void bn_bwd_apply_kernel(float* __restrict__ d, const float* __restrict__ y, const float* __restrict__ x,
                                    const float* __restrict__ coef, const float* __restrict__ bcoef, int C,
                                    const int* __restrict__ count) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    if (e >= (size_t)*count * C) return;
    const int c = (int)(e % C);
    const float dz = y[e] > 0.f ? d[e] : 0.f;
    const float xh = (x[e] - coef[c]) * coef[C + c];
    d[e] = bcoef[c] * (dz - bcoef[C + c] - xh * bcoef[2 * C + c]);
}

__global__ void code_grad_kernel(const float* __restrict__ dfeat0, const int* __restrict__ src0, const int* __restrict__ count,
                                 int n_vert, float* __restrict__ d_code) {
    const size_t e = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int r = (int)(e / kCode), c = (int)(e % kCode);
    if (r >= *count) return;
    atomicAdd(d_code + (size_t)(src0[r] % n_vert) * kCode + c, dfeat0[e]);
}

inline unsigned blocks(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }
inline int3 dims3(const Plan& p, int l) { return make_int3(p.dims[l][0], p.dims[l][1], p.dims[l][2]); }
inline long long dhw(const Plan& p, int l) { return (long long)p.dims[l][0] * p.dims[l][1] * p.dims[l][2]; }

// the layer's convolution (data gradient: transposed weights, rows of the input level)
void launch_conv(int j, bool bwd, const float* in, const int* map, int mirror, const float* W, const int* count, float* out,
                 double* stats, long long rows, cudaStream_t st) {
    const unsigned g = (unsigned)((rows + 63) / 64);
    const int ci = kDefs[j].cin, co = kDefs[j].cout;
#define NB_GG(KK, NN, TW) \
    if (K == KK && N == NN) { gather_gemm_kernel<KK, NN, TW><<<g, kThreads, 0, st>>>(in, map, mirror, W, count, out, stats); return; }
    if (!bwd) {
        const int K = ci, N = co;
        NB_GG(16, 16, false) NB_GG(16, 32, false) NB_GG(32, 32, false) NB_GG(32, 64, false) NB_GG(64, 64, false)
        NB_GG(64, 128, false) NB_GG(128, 128, false)
    } else {
        const int K = co, N = ci;
        NB_GG(16, 16, true) NB_GG(32, 16, true) NB_GG(32, 32, true) NB_GG(64, 32, true) NB_GG(64, 64, true)
        NB_GG(128, 64, true) NB_GG(128, 128, true)
    }
#undef NB_GG
}

void launch_wgrad(int j, const float* in, const int* map, const float* dx, const int* count, float* dW, long long rows,
                  cudaStream_t st) {
    const dim3 g((unsigned)((rows + 255) / 256), 27);
    const int K = kDefs[j].cin, N = kDefs[j].cout;
#define NB_WG(KK, NN) \
    if (K == KK && N == NN) { wgrad_kernel<KK, NN><<<g, kThreads, 0, st>>>(in, map, dx, count, dW); return; }
    NB_WG(16, 16) NB_WG(16, 32) NB_WG(32, 32) NB_WG(32, 64) NB_WG(64, 64) NB_WG(64, 128) NB_WG(128, 128)
#undef NB_WG
}

template <typename T>
T* at(const nb_spconv_args* a, size_t off) { return (T*)((char*)a->workspace + off); }

int check_args(const nb_spconv_args* a, const char* who, Plan* p) {
    if (!a) { set_error("%s: null args", who); return NB_ERR_BAD_ARG; }
    if (a->batch < 1 || a->n_points < 1 || a->n_vert < 1) {
        set_error("%s: batch, n_points and n_vert must be >= 1 (got %d, %d, %d)", who, a->batch, a->n_points, a->n_vert);
        return NB_ERR_BAD_ARG;
    }
    if (a->out_sh[0] < 1 || a->out_sh[1] < 1 || a->out_sh[2] < 1) { set_error("%s: out_sh must be >= 1", who); return NB_ERR_BAD_ARG; }
    if (a->training != 0 && a->training != 1) { set_error("%s: training must be 0 or 1", who); return NB_ERR_BAD_ARG; }
    if (!(a->eps > 0.f) || !(a->momentum >= 0.f && a->momentum <= 1.f)) {
        set_error("%s: eps must be > 0 and momentum in [0, 1]", who);
        return NB_ERR_BAD_ARG;
    }
    if (!a->coord || !a->code || !a->workspace) { set_error("%s: null coord, code or workspace", who); return NB_ERR_BAD_ARG; }
    for (int j = 0; j < kLayers; ++j)
        if (!a->weight[j] || !a->bn_weight[j] || !a->bn_bias[j] || !a->running_mean[j] || !a->running_var[j] ||
            (a->training && !a->num_batches_tracked[j])) {
            set_error("%s: layer %d has a null weight, bn_weight, bn_bias, running_mean, running_var or (training) "
                      "num_batches_tracked", who, j);
            return NB_ERR_BAD_ARG;
        }
    for (int l = 0; l < NB_NUM_LEVELS; ++l)
        if (!a->volumes[l]) { set_error("%s: volumes[%d] is null", who, l); return NB_ERR_BAD_ARG; }
    const char* msg = make_plan(a->batch, a->n_points, a->out_sh, p);
    if (msg) { set_error("%s: %s", who, msg); return NB_ERR_UNSUPPORTED; }
    if ((uintptr_t)a->workspace % 256 != 0 || a->workspace_bytes < p->total) {
        set_error("%s: workspace must be 256-byte aligned and hold %zu bytes (got %zu)", who, p->total, a->workspace_bytes);
        return NB_ERR_BAD_ARG;
    }
    return NB_OK;
}

int cuda_status(const char* who) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_spconv_workspace_bytes(int batch, int n_points, const int out_sh[3]) {
    if (batch < 1 || n_points < 1 || !out_sh || out_sh[0] < 1 || out_sh[1] < 1 || out_sh[2] < 1) return 0;
    Plan p;
    return make_plan(batch, n_points, out_sh, &p) ? 0 : p.total;
}

int nb_spconv_fwd(const nb_spconv_args* a, void* stream) {
    static const char* who = "nb_spconv_fwd";
    Plan p;
    const int stc = check_args(a, who, &p);
    if (stc != NB_OK) return stc;
    cudaStream_t st = (cudaStream_t)stream;
    int* counts = at<int>(a, p.counts);
    int* scan = at<int>(a, p.scan);
    // active sets and rulebooks
    for (int l = 0; l < kGrids; ++l) {
        int* idx = at<int>(a, p.idx[l]);
        cudaMemsetAsync(idx, 0xff, p.sites[l] * 4, st);
        if (l == 0)
            mark_points_kernel<<<blocks(a->n_points), kThreads, 0, st>>>(a->coord, a->n_points, a->batch, dims3(p, 0), idx);
        else
            mark_strided_kernel<<<blocks(p.cap[l - 1]), kThreads, 0, st>>>(at<int>(a, p.site[l - 1]), counts + l - 1,
                                                                            dims3(p, l - 1), dims3(p, l), idx);
        size_t cub_bytes = p.cub_bytes;
        cub::DeviceScan::ExclusiveSum(at<void>(a, p.cub), cub_bytes, thrust::make_transform_iterator(idx, IsActive()), scan,
                                      (int)p.sites[l], st);
        finalize_kernel<<<blocks(p.sites[l]), kThreads, 0, st>>>(idx, scan, (int)p.sites[l], at<int>(a, p.site[l]),
                                                                 l == 0 ? at<int>(a, p.src0) : nullptr, counts + l);
        subm_rules_kernel<<<blocks(p.cap[l] * 27), kThreads, 0, st>>>(at<int>(a, p.site[l]), counts + l, dims3(p, l), idx,
                                                                      at<int>(a, p.nbr[l]));
        if (l > 0) {
            cudaMemsetAsync(at<int>(a, p.snbrT[l - 1]), 0xff, p.cap[l - 1] * 27 * 4, st);
            strided_rules_kernel<<<blocks(p.cap[l] * 27), kThreads, 0, st>>>(at<int>(a, p.site[l]), counts + l, dims3(p, l),
                                                                             dims3(p, l - 1), at<int>(a, p.idx[l - 1]),
                                                                             at<int>(a, p.snbr[l - 1]), at<int>(a, p.snbrT[l - 1]));
        }
    }
    gather_code_kernel<<<blocks(p.cap[0] * kCode), kThreads, 0, st>>>(a->code, a->n_vert, at<int>(a, p.src0), counts,
                                                                       at<float>(a, p.feat0));
    // the 17 conv + BN + ReLU layers
    cudaMemsetAsync(at<double>(a, p.stats), 0, (size_t)kLayers * 2 * 128 * sizeof(double), st);
    for (int l = 0; l < NB_NUM_LEVELS; ++l) {
        const long long C = kDefs[kOutLayer[l]].cout;
        cudaMemsetAsync(a->volumes[l], 0, (size_t)p.B * C * dhw(p, l + 1) * 4, st);
    }
    const float* cur = at<float>(a, p.feat0);
    for (int j = 0; j < kLayers; ++j) {
        const LayerDef& d = kDefs[j];
        const int lo = lout(j), C = d.cout;
        const int* map = d.stride == 2 ? at<int>(a, p.snbr[d.lin]) : at<int>(a, p.nbr[d.lin]);
        float* x = at<float>(a, p.x[j]);
        float* y = at<float>(a, p.y[j]);
        double* stats = at<double>(a, p.stats) + (size_t)j * 256;
        float* coef = at<float>(a, p.coef) + (size_t)j * 256;
        launch_conv(j, false, cur, map, 0, a->weight[j], counts + lo, x, a->training ? stats : nullptr, p.cap[lo], st);
        bn_stats_kernel<<<1, 128, 0, st>>>(stats, counts + lo, C, a->training, a->momentum, a->eps, a->running_mean[j],
                                           a->running_var[j], a->num_batches_tracked[j], coef);
        bn_relu_kernel<<<blocks(p.cap[lo] * C), kThreads, 0, st>>>(x, coef, a->bn_weight[j], a->bn_bias[j], C, counts + lo, y);
        for (int l = 0; l < NB_NUM_LEVELS; ++l)
            if (kOutLayer[l] == j)
                scatter_volume_kernel<<<blocks(p.cap[lo] * C), kThreads, 0, st>>>(y, at<int>(a, p.site[lo]), counts + lo, C,
                                                                                  dhw(p, lo), a->volumes[l]);
        cur = y;
    }
    if (a->row_counts) cudaMemcpyAsync(a->row_counts, counts, kGrids * sizeof(int), cudaMemcpyDeviceToDevice, st);
    return cuda_status(who);
}

int nb_spconv_bwd(const nb_spconv_args* a, const nb_spconv_grads* g, void* stream) {
    static const char* who = "nb_spconv_bwd";
    Plan p;
    const int stc = check_args(a, who, &p);
    if (stc != NB_OK) return stc;
    if (!g || !g->d_code) { set_error("%s: null grads or d_code", who); return NB_ERR_BAD_ARG; }
    for (int j = 0; j < kLayers; ++j)
        if (!g->d_weight[j] || !g->d_bn_weight[j] || !g->d_bn_bias[j]) {
            set_error("%s: layer %d has a null d_weight, d_bn_weight or d_bn_bias", who, j);
            return NB_ERR_BAD_ARG;
        }
    cudaStream_t st = (cudaStream_t)stream;
    const int* counts = at<int>(a, p.counts);
    float* dY = at<float>(a, p.dA);
    float* dX = at<float>(a, p.dB);
    double* dstat = at<double>(a, p.dstat);
    float* bcoef = at<float>(a, p.bcoef);
    cudaMemsetAsync(g->d_code, 0, (size_t)a->n_vert * kCode * 4, st);
    for (int j = 0; j < kLayers; ++j)
        cudaMemsetAsync(g->d_weight[j], 0, (size_t)27 * kDefs[j].cin * kDefs[j].cout * 4, st);
    for (int j = kLayers - 1; j >= 0; --j) {
        const LayerDef& d = kDefs[j];
        const int lo = lout(j), C = d.cout;
        for (int l = 0; l < NB_NUM_LEVELS; ++l) {
            if (kOutLayer[l] != j) continue;
            const bool first = j == kLayers - 1;
            if (g->d_volumes[l])
                gather_volume_kernel<<<blocks(p.cap[lo] * C), kThreads, 0, st>>>(g->d_volumes[l], at<int>(a, p.site[lo]),
                                                                                 counts + lo, C, dhw(p, lo), first ? 0 : 1, dY);
            else if (first)
                cudaMemsetAsync(dY, 0, (size_t)p.cap[lo] * C * 4, st);
        }
        const float* x = at<float>(a, p.x[j]);
        const float* y = at<float>(a, p.y[j]);
        const float* coef = at<float>(a, p.coef) + (size_t)j * 256;
        cudaMemsetAsync(dstat, 0, 2 * 128 * sizeof(double), st);
        const long long rgrid = (p.cap[lo] * C + 8 * kThreads - 1) / (8 * kThreads);
        bn_bwd_reduce_kernel<<<(unsigned)(rgrid < 4 * kGridSMs ? rgrid : 4 * kGridSMs), kThreads, 0, st>>>(dY, y, x, coef, C,
                                                                                                          counts + lo, dstat);
        bn_bwd_coef_kernel<<<1, 128, 0, st>>>(dstat, counts + lo, a->bn_weight[j], coef, C, a->training, g->d_bn_weight[j],
                                              g->d_bn_bias[j], bcoef);
        bn_bwd_apply_kernel<<<blocks(p.cap[lo] * C), kThreads, 0, st>>>(dY, y, x, coef, bcoef, C, counts + lo);
        const float* in = j ? at<float>(a, p.y[j - 1]) : at<float>(a, p.feat0);
        const int* fmap = d.stride == 2 ? at<int>(a, p.snbr[d.lin]) : at<int>(a, p.nbr[d.lin]);
        launch_wgrad(j, in, fmap, dY, counts + lo, g->d_weight[j], p.cap[lo], st);
        const int* bmap = d.stride == 2 ? at<int>(a, p.snbrT[d.lin]) : at<int>(a, p.nbr[d.lin]);
        launch_conv(j, true, dY, bmap, d.stride == 1, a->weight[j], counts + d.lin, dX, nullptr, p.cap[d.lin], st);
        if (j == 0)
            code_grad_kernel<<<blocks(p.cap[0] * kCode), kThreads, 0, st>>>(dX, at<int>(a, p.src0), counts, a->n_vert, g->d_code);
        float* t = dY;
        dY = dX;
        dX = t;
    }
    return cuda_status(who);
}

}  // extern "C"
