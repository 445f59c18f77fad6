// Internal declarations shared by the translation units of libneuralbody_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include "../../include/neuralbody_b200.h"
#include "nb_layout.h"

namespace nb {

void set_error(const char* fmt, ...);

// Grid-size unit of the persistent / grid-stride kernels: the SM count of the H100 SXM.  (Launches that must match the
// device's SM count exactly use sm_count() instead.)
constexpr int kGridSMs = 132;
inline int sm_count() {
    int dev = 0, sms = kGridSMs;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// Sample / point lists of the tensor-core pipelines: an entry's .w is its id | occupied-level bits << 28, so a list holds
// < 2^28 ids; a classification block and a composite warp take whole rays of at most kListMaxSamples samples.
constexpr uint32_t kListIdMask = 0x0FFFFFFFu;
constexpr int kListMaxSamples = 1024;

// Kernel-side view of one call (passed by value as a __grid_constant__): the caller's arguments as fill_frame_params and
// fill_ray_params translate them, then the per-launch state the list launchers set.
struct RenderParams {
    int batch, n_rays, n_samples;
    const float *ray_o, *ray_d, *near, *far, *t_vals, *t_rand;
    const float* z_user;       // (B,n,S) caller-supplied sample depths (nb_render_args.z_vals) or null
    const float *R, *Th, *bounds;
    float voxel_size[3];       // dhw
    float out_sh[3];           // dhw, as float (upstream: torch.tensor(out_sh).to(dhw))
    int   lvl_C[4], lvl_D[4], lvl_H[4], lvl_W[4];
    size_t lvl_off[4];         // byte offset of level l inside the volume blob
    size_t lvl_bstride[4];     // ELEMENT stride between frames of level l
    size_t occ_off[4];         // byte offset of level l's cell-occupancy bitmap inside the volume blob
    size_t occ_bstride[4];     // 32-bit words per frame of that bitmap
    const void* volume;
    const float* wf32;         // fp32 weight section
    const __half* wf16;        // fp16 weight stream (common steps)
    const __half* wframe;      // per-frame L3 step [B][144*16]
    const float* bc;           // [B][128]
    int white_bkgd;
    int skip_empty;            // tensor-core path: 1 = samples with all-zero features and sigma(empty) < 0 are not evaluated
    float *rgb_map, *disp_map, *acc_map, *weights, *depth_map, *raw;
    int rgb_stride, map_stride;   // floats between consecutive rays in rgb_map / in the three scalar maps (3 / 1 when dense)
    unsigned long long* trace;
    const unsigned char* mask_msks; const float* mask_RT; const float* mask_Ks;   // f-1 mask views (null = none)
    int mask_nv, mask_H, mask_W;
    const float *mask_R0, *mask_Th0;   // single-view _msk variant: SMPL -> snapshot-world transform, or null
    unsigned long long* stats; // u64[8] or null: [0] += tiles executed, [1] += listed samples, [2] += decoder-kernel ns,
                               // [3] += decoder launches, [4] += layer-0 K-steps executed (x 128 rows), [5] / [6] += coarse-level
                               // half tiles gathered from the staging / directly, [7] += fine-level half tiles gathered directly
    float* save;               // activation record for nb_render_bwd or null: (B,n,S,kSaveDim) for NB_PRECISION_FP32,
                               // trn::map_save's layout for NB_PRECISION_TC_TF32X3
    // list pipelines (nb_render_tc_list.cu, nb_train.cu), set by their launchers: one frame per launch
    int frame;                 // frame of this launch
    int train_list;            // training path (nb_train.cu): ONE list for all classes and frames (list_a upwards, list_count[3]),
                               // entry ids count samples across the whole batch; raw_ws stays the frame's
    // sample lists: entries (world xyz, frame sample id | level bits << 28), one list per sample CLASS (= finest occupied
    // level, nb_layout.h class_segments).  Two buffers of list_cap entries hold two classes each, growing towards each other:
    // class 3 from the start of A upwards, class 2 from the end of A downwards, class 1 / class 0 likewise in B.
    float4 *list_a, *list_b;
    size_t list_cap;
    unsigned int* list_count;  // [4] entries per class, appended by classify_compact_kernel
    unsigned long long* frame_clock;   // [0] max(~start), [1] max(end) of the decoder launch (%globaltimer ns)
    float4* raw_ws;            // (n, S) raw records of this frame: (rgb logits, sigma)
    // density queries (nb_decode_density_list): world points in, raw sigma out; the list entry ids are point ids
    const float* points;       // (n_points, 3) of this frame (the launch) / of frame 0 (the caller)
    float* sigma;              // (n_points) likewise
    int n_points;
};

// Check a call's fields and translate them into *p, or set an error that starts with `who` and return NB_ERR_*.  The frame
// (batch, R, Th, bounds, voxel_size, out_sh, level_dims, volume and weight blobs) is read by every entry point; the rays,
// samples, output maps and options by nb_render_fwd / nb_render_bwd only, which fill the frame first.
int fill_frame_params(const nb_render_args* a, const char* who, RenderParams* p);   // value-initialises *p
int fill_ray_params(const nb_render_args* a, const char* who, RenderParams* p);

int launch_render_f32(const RenderParams& p, int volume_dtype, cudaStream_t stream);
int launch_render_tc_list(const RenderParams& p, int volume_dtype, int passes, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t render_tc_list_workspace_bytes(int batch, int n_rays, int n_samples);
int launch_density_f32(const RenderParams& p, int volume_dtype, const float* pts, int n_points, float* sigma, cudaStream_t stream);
int launch_density_tc_list(const RenderParams& p, int volume_dtype, int passes, const float* pts, int n_points, float* sigma,
                           void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t density_tc_list_workspace_bytes(int batch, int n_points);
bool tc_available();

}  // namespace nb
