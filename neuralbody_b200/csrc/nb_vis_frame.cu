// nb_vis_frame (include/neuralbody_b200.h): the demo visualizers' uint8 BGR frame on the device.  Launches, in stream
// order:
//   1. a CUB scan:  the exclusive prefix count of the mask (the ray of each set pixel), as nb_eval_image's;
//   2. frame:       kVisPix pixels per thread, their 3 * kVisPix bytes packed into words in shared memory, then stored as
//                   consecutive words by consecutive threads; block 0 writes the status record.
// oracle/vis_frames.py restates the frame in numpy.
#include "nb_image_u8.cuh"
#include "nb_internal.h"

namespace nb {
namespace {

constexpr int kVisThreads = 256;
constexpr int kVisPix = 4;                                // pixels per thread: 12 bytes, three whole words
constexpr int kVisBlockPix = kVisThreads * kVisPix;
constexpr int kVisBlockWords = kVisBlockPix * 3 / 4;

struct VisWorkspace {
    int* offset;       // (H*W)
    void* scan;        // CUB scratch
    size_t scan_bytes;
};

// the layout of nb_vis_frame_workspace_bytes; total 0 when the scan's size query fails
inline size_t vis_layout(int H, int W, unsigned char* base, VisWorkspace* w) {
    const size_t pixels = (size_t)H * W, sb = scan_bytes((int)pixels);
    if (sb == 0) return 0;
    VisWorkspace t;
    t.offset = (int*)base;
    t.scan_bytes = sb;
    t.scan = base ? base + align256(pixels * sizeof(int)) : nullptr;
    if (w) *w = t;
    return align256(pixels * sizeof(int)) + align256(sb);
}

__global__ void __launch_bounds__(kVisThreads) vis_frame_kernel(const __grid_constant__ nb_vis_frame_args a,
                                                                 const int* __restrict__ offset) {
    __shared__ unsigned int words[kVisBlockWords];
    const long long pixels = (long long)a.H * a.W;
    const int count = offset[pixels - 1] + (a.mask_at_box[pixels - 1] != 0);
    const bool ok = count == a.n || a.n == 1;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.result->status = ok ? NB_VIS_OK : NB_VIS_COUNT;
        a.result->count = count;
    }
    if (!ok) return;
    const double bk = a.white_bkgd ? 1.0 : 0.0;
    const long long p0 = (long long)blockIdx.x * kVisBlockPix;
    const int t = threadIdx.x;
    unsigned int w[3] = {0u, 0u, 0u};
#pragma unroll
    for (int k = 0; k < kVisPix; ++k) {
        const long long p = p0 + t * kVisPix + k;
        if (p >= pixels) break;
        const bool m = a.mask_at_box[p] != 0;
        const size_t q = m ? (a.n == 1 ? 0 : (size_t)offset[p] * 3) : 0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const unsigned int b = to_u8(m ? (double)a.rgb_map[q + 2 - c] : bk);   // BGR
            const int pos = 3 * k + c;
            w[pos >> 2] |= b << (8 * (pos & 3));
        }
    }
    // stride 3 words per thread: no two lanes of a warp share a bank
    words[3 * t] = w[0];
    words[3 * t + 1] = w[1];
    words[3 * t + 2] = w[2];
    __syncthreads();
    const long long bytes = min((long long)kVisBlockPix, pixels - p0) * 3;
    unsigned char* out = a.frame + p0 * 3;                // p0 * 3 is a multiple of 4
    for (int i = t; i < kVisBlockWords; i += kVisThreads) {
        if (4LL * i + 4 <= bytes) {
            reinterpret_cast<unsigned int*>(out)[i] = words[i];
        } else {
            for (long long j = 4LL * i; j < bytes; ++j) out[j] = (unsigned char)(words[i] >> (8 * (j - 4LL * i)));
        }
    }
}

}  // namespace
}  // namespace nb

using namespace nb;

extern "C" {

size_t nb_vis_frame_workspace_bytes(int H, int W) {
    if (H < 1 || W < 1 || (long long)H * W >= (1LL << 31)) return 0;
    return vis_layout(H, W, nullptr, nullptr);
}

int nb_vis_frame(const nb_vis_frame_args* a, void* stream) {
    static const char* who = "nb_vis_frame";
    if (!a || !a->mask_at_box || !a->workspace || !a->result || !a->frame || (a->n > 0 && !a->rgb_map)) {
        set_error("%s: null argument", who);
        return NB_ERR_BAD_ARG;
    }
    if (a->H < 1 || a->W < 1 || (long long)a->H * a->W >= (1LL << 31) || a->n < 0 || 3LL * a->n >= (1LL << 31)) {
        set_error("%s: H, W >= 1 with H*W < 2^31 and 0 <= 3n < 2^31 (got %d x %d, n = %d)", who, a->H, a->W, a->n);
        return NB_ERR_BAD_ARG;
    }
    if (a->white_bkgd != 0 && a->white_bkgd != 1) {
        set_error("%s: white_bkgd must be 0 or 1 (got %d)", who, a->white_bkgd);
        return NB_ERR_BAD_ARG;
    }
    if ((uintptr_t)a->frame % 4 != 0) {
        set_error("%s: frame must be 4-byte aligned", who);
        return NB_ERR_BAD_ARG;
    }
    const size_t need = nb_vis_frame_workspace_bytes(a->H, a->W);
    if (need == 0 || a->workspace_bytes < need) {
        set_error("%s: workspace_bytes too small (%zu < %zu)", who, a->workspace_bytes, need);
        return NB_ERR_BAD_ARG;
    }
    VisWorkspace w;
    vis_layout(a->H, a->W, (unsigned char*)a->workspace, &w);
    const cudaStream_t s = (cudaStream_t)stream;
    const int pixels = a->H * a->W;
    cudaError_t e = scan_mask(w.scan, w.scan_bytes, a->mask_at_box, w.offset, pixels, s);
    if (e == cudaSuccess) {
        const unsigned blocks = (unsigned)((pixels + kVisBlockPix - 1) / kVisBlockPix);
        vis_frame_kernel<<<blocks, kVisThreads, 0, s>>>(*a, w.offset);
        e = cudaGetLastError();
    }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return NB_ERR_CUDA; }
    return NB_OK;
}

}  // extern "C"
