// nb_eval_image (include/neuralbody_b200.h): the evaluator's per-view metrics on the device.  Nothing materialises the
// scattered images: a pixel's value is its ray's (at the mask's exclusive prefix count) when the mask is set, else the
// background.  Launches, in stream order:
//   1. box_partials:  per block, the min / max row and column of the set pixels it strides over;
//   2. a CUB scan:    the exclusive prefix count of the mask (the ray of each set pixel);
//   3. ray_partials:  per block, the two MSE sums (the fp32 ray terms and the float64 image terms) over the rays;
//   4. finish:        one CTA reduces both in a fixed order, checks the count and the box, writes mse and psnr;
//   5. ssim_tiles:    32 x 16 output pixels per CTA over the whole image (CTAs off the box return): the crops' uint8 bytes,
//                     and for the box's interior the separable 7 x 7 sums of x, y, xx, yy, xy per channel and the sum of S;
//   6. ssim_finish:   one CTA sums the tiles' S in a fixed order and writes the channel means and their mean.
// No expression here may be contracted: every product and sum is an explicit _rn intrinsic, so pred == gt gives S = 1
// exactly (2 ux uy and ux^2 + uy^2 round alike).  oracle/eval_metrics.py restates every output in numpy.
#include "nb_image_u8.cuh"
#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kEvalThreads = 256;
constexpr int kEvalMaxBlocks = 256;      // the partial-sum kernels' grid cap (grid-stride beyond it)
constexpr int kEvalItems = 4096;         // elements per block before the cap
constexpr int kTileX = 32, kTileY = 16;  // ssim_tiles: output pixels per CTA (32 x 8 threads, two rows each)
constexpr int kWin = 7, kPad = 3;
constexpr int kHaloX = kTileX + kWin - 1, kHaloY = kTileY + kWin - 1;

inline int partial_blocks(long long items) {
    return (int)max(1LL, min((long long)kEvalMaxBlocks, (items + kEvalItems - 1) / kEvalItems));
}

struct Workspace {
    int* offset;       // (H*W)
    void* scan;        // CUB scratch
    size_t scan_bytes;
    int4* box;         // (kEvalMaxBlocks) min x, min y, max x, max y
    double2* sums;     // (kEvalMaxBlocks) fp32-term sum, float64-term sum
    double* ssim;      // (tiles, 3)
};

inline int tiles(int H, int W) { return ((W + kTileX - 1) / kTileX) * ((H + kTileY - 1) / kTileY); }

// the layout of nb_eval_image_workspace_bytes; total 0 when the scan's size query fails
inline size_t layout(int H, int W, unsigned char* base, Workspace* w) {
    const size_t pixels = (size_t)H * W, sb = scan_bytes((int)pixels);
    if (sb == 0) return 0;
    size_t off = 0;
    auto take = [&](size_t bytes) { unsigned char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
    Workspace t;
    t.offset = (int*)take(pixels * sizeof(int));
    t.scan_bytes = sb;
    t.scan = take(sb);
    t.box = (int4*)take(kEvalMaxBlocks * sizeof(int4));
    t.sums = (double2*)take(kEvalMaxBlocks * sizeof(double2));
    t.ssim = (double*)take((size_t)tiles(H, W) * 3 * sizeof(double));
    if (w) *w = t;
    return off;
}

__device__ __forceinline__ int warp_min(int v) {
    for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_max(int v) {
    for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}
// a fixed tree: the same inputs in the same threads give the same bits
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}
// the block's sum in lane 0 of warp 0 (blockDim.x * blockDim.y == kEvalThreads); red holds kEvalThreads / 32 doubles
__device__ __forceinline__ double block_sum(double v, double* red) {
    const int t = threadIdx.y * blockDim.x + threadIdx.x;
    v = warp_sum(v);
    __syncthreads();
    if ((t & 31) == 0) red[t >> 5] = v;
    __syncthreads();
    v = 0.0;
    if (t < 32) {
        v = t < kEvalThreads / 32 ? red[t] : 0.0;
        v = warp_sum(v);
    }
    return v;
}

__global__ void __launch_bounds__(kEvalThreads) box_partials_kernel(const unsigned char* __restrict__ mask, int H, int W,
                                                                    int4* __restrict__ out) {
    __shared__ int4 red[kEvalThreads / 32];
    int x0 = INT_MAX, y0 = INT_MAX, x1 = -1, y1 = -1;
    const long long n = (long long)H * W, step = (long long)gridDim.x * kEvalThreads;
    for (long long p = (long long)blockIdx.x * kEvalThreads + threadIdx.x; p < n; p += step) {
        if (!mask[p]) continue;
        const int y = (int)(p / W), x = (int)(p - (long long)y * W);
        x0 = min(x0, x); x1 = max(x1, x);
        y0 = min(y0, y); y1 = max(y1, y);
    }
    x0 = warp_min(x0); y0 = warp_min(y0); x1 = warp_max(x1); y1 = warp_max(y1);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = make_int4(x0, y0, x1, y1);
    __syncthreads();
    if (threadIdx.x == 0) {
        int4 b = red[0];
        for (int i = 1; i < kEvalThreads / 32; ++i) {
            b.x = min(b.x, red[i].x); b.y = min(b.y, red[i].y); b.z = max(b.z, red[i].z); b.w = max(b.w, red[i].w);
        }
        out[blockIdx.x] = b;
    }
}

__global__ void __launch_bounds__(kEvalThreads) ray_partials_kernel(const float* __restrict__ pred, const float* __restrict__ gt,
                                                                    int values, double2* __restrict__ out) {
    __shared__ double red[kEvalThreads / 32];
    double s32 = 0.0, s64 = 0.0;
    for (int i = blockIdx.x * kEvalThreads + threadIdx.x; i < values; i += gridDim.x * kEvalThreads) {
        const float p = pred[i], g = gt[i];
        const float d = __fsub_rn(p, g);
        s32 = __dadd_rn(s32, (double)__fmul_rn(d, d));                    // numpy: (pred - gt) ** 2 in float32
        const double dd = __dsub_rn((double)p, (double)g);
        s64 = __dadd_rn(s64, __dmul_rn(dd, dd));                          // the float64 images' terms
    }
    s32 = block_sum(s32, red);
    s64 = block_sum(s64, red);
    if (threadIdx.x == 0) out[blockIdx.x] = make_double2(s32, s64);
}

__global__ void __launch_bounds__(kEvalThreads) finish_kernel(const __grid_constant__ nb_eval_image_args a, Workspace w,
                                                              int box_blocks, int sum_blocks) {
    __shared__ double red[kEvalThreads / 32];
    __shared__ int4 bred[kEvalThreads / 32];
    const int t = threadIdx.x;
    int x0 = INT_MAX, y0 = INT_MAX, x1 = -1, y1 = -1;
    double s32 = 0.0, s64 = 0.0;
    for (int i = t; i < box_blocks; i += kEvalThreads) {
        const int4 b = w.box[i];
        x0 = min(x0, b.x); y0 = min(y0, b.y); x1 = max(x1, b.z); y1 = max(y1, b.w);
    }
    for (int i = t; i < sum_blocks; i += kEvalThreads) {
        s32 = __dadd_rn(s32, w.sums[i].x);
        s64 = __dadd_rn(s64, w.sums[i].y);
    }
    x0 = warp_min(x0); y0 = warp_min(y0); x1 = warp_max(x1); y1 = warp_max(y1);
    if ((t & 31) == 0) bred[t >> 5] = make_int4(x0, y0, x1, y1);
    s32 = block_sum(s32, red);
    s64 = block_sum(s64, red);
    if (t != 0) return;
    for (int i = 1; i < kEvalThreads / 32; ++i) {
        x0 = min(x0, bred[i].x); y0 = min(y0, bred[i].y); x1 = max(x1, bred[i].z); y1 = max(y1, bred[i].w);
    }
    const long long pixels = (long long)a.H * a.W;
    const int count = w.offset[pixels - 1] + (a.mask_at_box[pixels - 1] != 0);
    nb_eval_image_result* r = a.result;
    int box[4] = {0, 0, 0, 0};
    if (a.eval_whole_img) {
        box[2] = a.W; box[3] = a.H;
    } else if (count > 0) {
        box[0] = x0; box[1] = y0; box[2] = x1 - x0 + 1; box[3] = y1 - y0 + 1;
    }
    int status = NB_EVAL_OK;
    if (count != a.n) status = NB_EVAL_COUNT;
    else if (box[2] < kWin || box[3] < kWin) status = NB_EVAL_SMALL;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    const double sum = a.eval_whole_img ? s64 : s32;
    const double mse = status == NB_EVAL_COUNT ? nan
                     : __ddiv_rn(sum, a.eval_whole_img ? (double)pixels * 3.0 : (double)a.n * 3.0);
    r->status = status;
    r->count = count;
    for (int k = 0; k < 4; ++k) r->box[k] = box[k];
    r->sq_sum = status == NB_EVAL_COUNT ? nan : sum;
    r->mse = mse;
    r->psnr = __dmul_rn(-10.0, log10(mse));
    r->ssim = nan;
    for (int c = 0; c < 3; ++c) r->ssim_channel[c] = nan;
}

__global__ void __launch_bounds__(kEvalThreads) ssim_tiles_kernel(const __grid_constant__ nb_eval_image_args a,
                                                                  const int* __restrict__ offset, double* __restrict__ part) {
    __shared__ float px[3][kHaloY][kHaloX], gx[3][kHaloY][kHaloX];   // the halo tile's pred / gt values per channel
    __shared__ double hs[5][kHaloY][kTileX];                         // horizontal 7-sums of x, y, xx, yy, xy
    __shared__ double red[kEvalThreads / 32];
    const int t = threadIdx.y * kTileX + threadIdx.x;
    const int tile = blockIdx.y * gridDim.x + blockIdx.x;
    const nb_eval_image_result* r = a.result;
    const int bx = r->box[0], by = r->box[1], bw = r->box[2], bh = r->box[3];
    const int tx0 = blockIdx.x * kTileX, ty0 = blockIdx.y * kTileY;
    // the box's interior (S positions whose window lies in the box) and this tile's part of it
    const int ix0 = max(bx + kPad, tx0), ix1 = min(bx + bw - kPad, tx0 + kTileX);
    const int iy0 = max(by + kPad, ty0), iy1 = min(by + bh - kPad, ty0 + kTileY);
    const bool ok = r->status == NB_EVAL_OK;
    const bool in_box = ok && tx0 < bx + bw && tx0 + kTileX > bx && ty0 < by + bh && ty0 + kTileY > by;
    const bool interior = in_box && ix0 < ix1 && iy0 < iy1;
    if (!interior) {
        if (t < 3) part[(size_t)tile * 3 + t] = 0.0;
        if (!in_box) return;
    }
    const float bk = a.white_bkgd ? 1.f : 0.f;
    const int W = a.W, H = a.H;
    // the crops' bytes of this tile's own pixels
    for (int i = t; i < kTileX * kTileY; i += kEvalThreads) {
        const int x = tx0 + i % kTileX, y = ty0 + i / kTileX;
        if (x < bx || x >= bx + bw || y < by || y >= by + bh) continue;
        const size_t p = (size_t)y * W + x;
        const size_t o = ((size_t)(y - by) * bw + (x - bx)) * 3;
        const bool m = a.mask_at_box[p] != 0;
        const size_t q = m ? (size_t)offset[p] * 3 : 0;
        for (int c = 0; c < 3; ++c) {
            a.crop_pred[o + 2 - c] = to_u8(m ? (double)a.rgb_pred[q + c] : (double)bk);
            a.crop_gt[o + 2 - c] = to_u8(m ? (double)a.rgb_gt[q + c] : (double)bk);
        }
    }
    if (!interior) return;
    for (int i = t; i < kHaloX * kHaloY; i += kEvalThreads) {
        const int hx = i % kHaloX, hy = i / kHaloX;
        // clamped: a halo pixel outside the image feeds no interior window
        const int x = min(max(tx0 - kPad + hx, 0), W - 1), y = min(max(ty0 - kPad + hy, 0), H - 1);
        const size_t p = (size_t)y * W + x;
        const bool m = a.mask_at_box[p] != 0;
        const size_t q = m ? (size_t)offset[p] * 3 : 0;
        for (int c = 0; c < 3; ++c) {
            px[c][hy][hx] = m ? a.rgb_pred[q + c] : bk;
            gx[c][hy][hx] = m ? a.rgb_gt[q + c] : bk;
        }
    }
    const double cov_norm = 49.0 / 48.0, C1 = 0.0004, C2 = 0.0036;   // (0.01 * 2)^2, (0.03 * 2)^2
    double acc[3] = {0.0, 0.0, 0.0};
    for (int c = 0; c < 3; ++c) {
        __syncthreads();
        for (int i = t; i < kHaloY * kTileX; i += kEvalThreads) {
            const int hx = i % kTileX, hy = i / kTileX;
            double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
            for (int k = 0; k < kWin; ++k) {
                const double x = px[c][hy][hx + k], y = gx[c][hy][hx + k];   // float32 values: the products are exact
                s[0] = __dadd_rn(s[0], x);
                s[1] = __dadd_rn(s[1], y);
                s[2] = __dadd_rn(s[2], __dmul_rn(x, x));
                s[3] = __dadd_rn(s[3], __dmul_rn(y, y));
                s[4] = __dadd_rn(s[4], __dmul_rn(x, y));
            }
            for (int q = 0; q < 5; ++q) hs[q][hy][hx] = s[q];
        }
        __syncthreads();
        const int x = tx0 + threadIdx.x;
        for (int row = threadIdx.y; row < kTileY; row += kEvalThreads / kTileX) {
            const int y = ty0 + row;
            if (x < ix0 || x >= ix1 || y < iy0 || y >= iy1) continue;
            double u[5];
            for (int q = 0; q < 5; ++q) {
                double s = 0.0;
                for (int k = 0; k < kWin; ++k) s = __dadd_rn(s, hs[q][row + k][threadIdx.x]);
                u[q] = __ddiv_rn(s, 49.0);
            }
            const double ux = u[0], uy = u[1];
            const double vx = __dmul_rn(cov_norm, __dsub_rn(u[2], __dmul_rn(ux, ux)));
            const double vy = __dmul_rn(cov_norm, __dsub_rn(u[3], __dmul_rn(uy, uy)));
            const double vxy = __dmul_rn(cov_norm, __dsub_rn(u[4], __dmul_rn(ux, uy)));
            const double A1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1), A2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
            const double B1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
            const double B2 = __dadd_rn(__dadd_rn(vx, vy), C2);
            acc[c] = __dadd_rn(acc[c], __ddiv_rn(__dmul_rn(A1, A2), __dmul_rn(B1, B2)));
        }
    }
    for (int c = 0; c < 3; ++c) {
        const double s = block_sum(acc[c], red);
        if (t == 0) part[(size_t)tile * 3 + c] = s;
    }
}

__global__ void __launch_bounds__(kEvalThreads) ssim_finish_kernel(nb_eval_image_result* __restrict__ r,
                                                                   const double* __restrict__ part, int n_tiles) {
    __shared__ double red[kEvalThreads / 32];
    double s[3] = {0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n_tiles; i += kEvalThreads)
        for (int c = 0; c < 3; ++c) s[c] = __dadd_rn(s[c], part[(size_t)i * 3 + c]);
    for (int c = 0; c < 3; ++c) s[c] = block_sum(s[c], red);
    if (threadIdx.x != 0 || r->status != NB_EVAL_OK) return;
    const double area = (double)(r->box[2] - 2 * kPad) * (double)(r->box[3] - 2 * kPad);
    for (int c = 0; c < 3; ++c) {
        s[c] = __ddiv_rn(s[c], area);
        r->ssim_channel[c] = s[c];
    }
    r->ssim = __ddiv_rn(__dadd_rn(__dadd_rn(s[0], s[1]), s[2]), 3.0);   // np.mean of three values
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_eval_image_workspace_bytes(int H, int W, int n) {
    if (H < 1 || W < 1 || (long long)H * W >= (1LL << 31) || n < 0 || 3LL * n >= (1LL << 31)) return 0;
    return layout(H, W, nullptr, nullptr);
}

int nb_eval_image(const nb_eval_image_args* a, void* stream) {
    static const char* who = "nb_eval_image";
    if (!a || !a->mask_at_box || !a->workspace || !a->result || !a->crop_pred || !a->crop_gt ||
        (a->n > 0 && (!a->rgb_pred || !a->rgb_gt))) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->H < 1 || a->W < 1 || (long long)a->H * a->W >= (1LL << 31) || a->n < 0 || 3LL * a->n >= (1LL << 31)) {
        set_error("%s: H, W >= 1 with H*W < 2^31 and 0 <= 3n < 2^31 (got %d x %d, n = %d)", who, a->H, a->W, a->n);
        return NB_ERR_BAD_ARG;
    }
    if ((a->white_bkgd != 0 && a->white_bkgd != 1) || (a->eval_whole_img != 0 && a->eval_whole_img != 1)) {
        set_error("%s: white_bkgd and eval_whole_img must be 0 or 1 (got %d, %d)", who, a->white_bkgd, a->eval_whole_img);
        return NB_ERR_BAD_ARG;
    }
    const size_t need = nb_eval_image_workspace_bytes(a->H, a->W, a->n);
    if (need == 0 || a->workspace_bytes < need) {
        set_error("%s: workspace_bytes too small (%zu < %zu)", who, a->workspace_bytes, need);
        return NB_ERR_BAD_ARG;
    }
    Workspace w;
    layout(a->H, a->W, (unsigned char*)a->workspace, &w);
    const cudaStream_t s = (cudaStream_t)stream;
    const int pixels = a->H * a->W, values = 3 * a->n;
    const int box_blocks = partial_blocks(pixels), sum_blocks = partial_blocks(values);
    const dim3 grid((unsigned)((a->W + kTileX - 1) / kTileX), (unsigned)((a->H + kTileY - 1) / kTileY));
    box_partials_kernel<<<box_blocks, kEvalThreads, 0, s>>>(a->mask_at_box, a->H, a->W, w.box);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = scan_mask(w.scan, w.scan_bytes, a->mask_at_box, w.offset, pixels, s);
    if (e == cudaSuccess) {
        ray_partials_kernel<<<sum_blocks, kEvalThreads, 0, s>>>(a->rgb_pred, a->rgb_gt, values, w.sums);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        finish_kernel<<<1, kEvalThreads, 0, s>>>(*a, w, box_blocks, sum_blocks);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ssim_tiles_kernel<<<grid, dim3(kTileX, kEvalThreads / kTileX), 0, s>>>(*a, w.offset, w.ssim);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) {
        ssim_finish_kernel<<<1, kEvalThreads, 0, s>>>(a->result, w.ssim, (int)(grid.x * grid.y));
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
