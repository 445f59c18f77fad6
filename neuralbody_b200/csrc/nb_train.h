// Training path on the tensor cores (nb_train.cu): declarations shared with nb_capi.cu / nb_render_bwd.cu.
#pragma once
#include "nb_internal.h"

namespace nb {

// the cotangents of the five output maps a backward call was given (device, dense; any may be null):
// rgb (B,n,3), depth / acc / disp (B,n), weights (B,n,S)
struct MapCotangents { const float *rgb, *depth, *acc, *disp, *weights; };

// the depth gradients a backward call was asked for (device, accumulated into; any may be null): d near / d far (B,n), only
// after a forward that derived z from them, and d z (B,n,S) per sample
struct DepthGrads {
    float *near, *far, *z;
    __host__ __device__ bool any() const { return near || far || z; }
};

// what one backward call was asked for: the map cotangents it was given and the input gradients it accumulates into
// (device; any pointer may be null)
struct GradRequest {
    MapCotangents maps;
    float *d_R, *d_Th;               // (B,3,3) / (B,3) frame transform
    float *d_ray_o, *d_ray_d;        // (B,n,3) rays
    DepthGrads depths;
    float* d_bounds;                 // (B,2,3): row 0
    // any per-frame gradient (the frame pass sums them per frame)
    __host__ __device__ bool frame() const { return d_R || d_Th || d_bounds; }
    // per-sample ray records: d z_i takes d loss / d(world point) along ray_d, so the depths need them too
    __host__ __device__ bool records() const { return d_ray_o || d_ray_d || depths.any(); }
    // any gradient with respect to the sample position
    __host__ __device__ bool sample_pos() const { return frame() || records(); }
};

namespace trn {

constexpr int kH2X = 352;                   // colour-layer input record: [h2 256 | PE(xyz) 63 | 0 | PE(viewdir) 27 | 0 x 5]
constexpr int kWS = 144;                    // colour-layer output record: [w 128 | sigma | 0 x 15]
constexpr int kXyzCol = 256, kViewCol = 320;

// C (M x N) = epilogue(A B^T): A is (M x K), B is (N x K), both fp32 in global memory
struct GemmArgs {
    const float* a; long long lda;
    const float* b; long long ldb;
    int M, N, K;
    const unsigned int* dyn_m;       // device: rows of A (the list length) instead of M, or null
    const unsigned int* dyn_k;       // device: reduction length instead of K (weight gradients), or null
    float* c; long long ldc;
    const float* bias;               // per column, added before the relu; null = none
    int bias_frame_stride;           // > 0: bias row = frame of the list entry (row) * this
    const float4* list; unsigned int samples_per_frame;
    int relu_cols;                   // relu on columns < relu_cols (multiple of 16)
    const float* mask; long long ldm;   // v = mask[row][col] > 0 ? v : 0 (relu backward), or null
    int atomic;                      // accumulate into c with atomicAdd (split reductions)
};
int launch_gemm(const GemmArgs& g, bool a_k_contiguous, bool b_k_contiguous, int max_m, int splits, cudaStream_t stream);

// the activation record of one forward call (nb_render_args.save)
struct SaveMap {
    unsigned int* count;             // list length (device)
    float* wcol;                     // (144, 352) colour layer + alpha_fc
    float* bias3;                    // (B, 144)
    float4* list;                    // (pmax) entries (world xyz, sample id | level bits)
    float *F, *H0, *H1, *H2X, *WS;   // (pmax, 352 / 256 / 256 / 352 / 144)
    size_t floats;
};
SaveMap map_save(float* save, int batch, size_t pmax);

struct GradBlob { size_t off[4], bstride[4], floats; };   // channels-last volume gradient, level offsets in floats

struct TrainBwd {
    const float* save; const float* raw;
    GradRequest req;
    const nb_decoder_weights* weights; const nb_decoder_weights* grads;
    float* d_vol[4];
    int volume_dtype;               // of the forward's volume blob (the frame-gradient pass reads it)
    float* workspace;
};

}  // namespace trn

size_t train_save_bytes(int batch, int n_rays, int n_samples);
size_t train_bwd_workspace_bytes(const RenderParams& p, int n_rays, int n_samples);   // p: the frame (batch, level dims)
bool train_supported(const RenderParams& p);
int launch_train_fwd(const RenderParams& p, int volume_dtype, cudaStream_t stream);
int launch_train_bwd(const RenderParams& p, const trn::TrainBwd& t, cudaStream_t stream);

// shared pieces living in other translation units
void launch_classify(const RenderParams& p, cudaStream_t stream);    // nb_render_tc_list.cu (p.frame, lists, raw_ws set by the caller)
void launch_composite(const RenderParams& p, cudaStream_t stream);   // nb_render_tc_list.cu
void launch_composite_bwd(const RenderParams& p, const float* raw, const GradRequest& req, float* d_raw_out, int d_raw_stride,
                          cudaStream_t stream);                                        // nb_render_bwd.cu
// per ray: the per-sample records rec + i * rec_stride = [d / d(world point) 3 | d / d(view direction) 3] plus the compositing
// term -> req.d_ray_o / d_ray_d; with any depth gradient asked for, also d z per sample (the records' world-point part along
// ray_d, the depth map and the dists) -> req.depths.z and, through z_sample, .near / .far                      nb_render_bwd.cu
void launch_ray_grad(const RenderParams& p, const float* raw, const GradRequest& req, const float* rec, int rec_stride,
                     cudaStream_t stream);
int launch_unfold(const nb_decoder_weights& w, const nb_decoder_weights& g, const float* dWcx, const float* dbc, float* T, float* dT,
                  float* u, float* du, cudaStream_t stream);                          // nb_render_bwd.cu

}  // namespace nb
