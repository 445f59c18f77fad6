/* neuralbody_b200 -- C ABI of the H100-native (sm_90a) volumetric-render hot path.
 *
 * The reference (zju3dv/neuralbody @ 3c516b9) is pure Python over PyTorch and has no FFI
 * of its own; its plugin boundary for this path is
 *     make_renderer(cfg, net).render(batch)       lib/networks/renderer/make_renderer.py:5-9
 *                                                 lib/networks/renderer/if_clight_renderer.py:94-122
 * This header is the C surface a binding for that boundary calls (the ctypes binding
 * shipped in neuralbody_b200/capi.py is the one a reference maintainer would add;
 * see INTEGRATION.md).  Conventions:
 *   - plain C types only; every pointer marked `device` is caller-owned CUDA memory that
 *     the library neither frees nor retains beyond the call;
 *   - all work is enqueued on the caller's stream (a cudaStream_t passed as void*); no
 *     hidden synchronisation, no allocation;
 *   - return value 0 = ok, <0 = error (see NB_ERR_*); nb_last_error() gives a thread-local
 *     message.  No exceptions cross the boundary.
 */
#ifndef NEURALBODY_B200_H
#define NEURALBODY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB_ABI_VERSION 6

#define NB_OK               0
#define NB_ERR_BAD_ARG     (-1)
#define NB_ERR_UNSUPPORTED (-2)
#define NB_ERR_CUDA        (-3)

/* element type of a packed feature volume */
#define NB_DTYPE_F32 0
#define NB_DTYPE_F16 1

/* arithmetic of the decoder MLP inside nb_render_fwd */
#define NB_PRECISION_FP32      0   /* exact: fp32 FFMA everywhere (GPU-side oracle, fallback)            */
#define NB_PRECISION_TC_FP16   1   /* wgmma tensor cores: fp16 operands, fp32 accumulate                 */
#define NB_PRECISION_TC_FP16X3 2   /* wgmma, density path as hi+lo fp16 pairs, 3 MMA passes: ~fp32-accurate */
#define NB_PRECISION_TC_TF32X3 3   /* training: sample list + wgmma tf32 GEMM chains, hi+lo TF32 pairs, 3 passes (fp32-grade);
                                      writes the activation record nb_render_bwd consumes; needs `save` and `raw` */

#define NB_NUM_LEVELS   4          /* SparseConvNet returns 4 dense volumes, latent_xyzc.py:179-204     */
#define NB_FEAT_DIM     352        /* 32+64+128+128 channels, latent_xyzc.py:20                         */
#define NB_XYZ_PE_DIM   63         /* embedder.py:53  (cfg.xyz_res = 10)                                */
#define NB_VIEW_PE_DIM  27         /* embedder.py:54  (cfg.view_res = 4)                                */

int         nb_abi_version(void);
const char* nb_last_error(void);
int         nb_has_precision(int precision);   /* 1 if nb_render_fwd implements NB_PRECISION_<precision> */

/* ------------------------------------------------------------------------------------------
 * Feature volumes.  Replaces the per-point F.grid_sample reads of NCDHW fp32 volumes in
 * Network.interpolate_features (lib/networks/latent_xyzc.py:62-72): the volumes returned by
 * net.encode_sparse_voxels (latent_xyzc.py:30-39) are re-laid-out ONCE per frame as
 * channels-last [B][D][H][W][C] so one trilinear corner is one contiguous vector.
 * Blob layout: level l starts at nb_packed_volume_level_offset(...), 256-byte aligned.
 */
typedef struct nb_volume_level {
    const float* data;   /* device, (B, C, D, H, W) fp32 contiguous, as `.dense()` returns it */
    int C, D, H, W;
} nb_volume_level;

size_t nb_packed_volume_bytes(const int dims[NB_NUM_LEVELS][4] /* C,D,H,W */, int batch, int dtype);
size_t nb_packed_volume_level_offset(const int dims[NB_NUM_LEVELS][4], int batch, int dtype, int level);
int    nb_pack_volume(const nb_volume_level levels[NB_NUM_LEVELS], int batch, int dtype,
                      void* out_blob /* device */, size_t out_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Decoder weights.  Replaces the eight nn.Conv1d(k=1) modules + nn.Embedding `latent` of
 * Network (lib/networks/latent_xyzc.py:13-28) as consumed by calculate_density_color (:91-126).
 * All pointers device fp32, Conv1d layout (out, in[, 1]).  The pack step performs the exact
 * fold  view_fc[:, :256] o latent_fc o (feature_fc (+) latent[latent_index])  (no activation
 * between those layers) in fp64, and emits fp32 K-major matrices for the exact kernel and fp16
 * canonical (K-major, no-swizzle) matrices of the wgmma shared-memory descriptor for the tensor-core kernel.
 */
typedef struct nb_decoder_weights {
    const float *fc0_w, *fc0_b;         /* (256,352) (256) */
    const float *fc1_w, *fc1_b;         /* (256,256) (256) */
    const float *fc2_w, *fc2_b;         /* (256,256) (256) */
    const float *alpha_w, *alpha_b;     /* (1,256)   (1)   */
    const float *feature_w, *feature_b; /* (256,256) (256) */
    const float *latent_w, *latent_b;   /* (256,384) (256) */
    const float *view_w, *view_b;       /* (128,346) (128) */
    const float *rgb_w, *rgb_b;         /* (3,128)   (3)   */
    const float *latent;                /* (num_train_frame,128) embedding table */
    const int64_t *latent_index;        /* device (batch) int64, sp_input['latent_index'] */
    int num_train_frame;
    int batch;
} nb_decoder_weights;

size_t nb_packed_weights_bytes(int batch);
int    nb_pack_weights(const nb_decoder_weights* w, void* out_blob /* device */, size_t out_bytes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Fused forward render.  One launch replaces the whole chunk loop of Renderer.render
 * (if_clight_renderer.py:107-120): get_sampling_points (:11-27) -> viewdir (:68) ->
 * Network.pts_to_can_pts / get_grid_coords / interpolate_features / calculate_density_color
 * (latent_xyzc.py:41-126, embedder.py:5-50) -> raw2outputs (nerf_net_utils.py:6-51).
 */
typedef struct nb_render_args {
    int batch;             /* B frames */
    int n_rays;            /* n rays per frame */
    int n_samples;         /* cfg.N_samples */
    const float* ray_o;    /* device (B,n,3) */
    const float* ray_d;    /* device (B,n,3), NOT normalised; near/far are parametric t */
    const float* near;     /* device (B,n) */
    const float* far;      /* device (B,n) */
    const float* t_vals;   /* device (S) = torch.linspace(0,1,S); NULL -> computed in-kernel */
    const float* t_rand;   /* device (B,n,S) uniform [0,1) jitter (cfg.perturb>0 and net.training), or NULL */
    const float* R;        /* device (B,3,3)  sp_input['R']  */
    const float* Th;       /* device (B,3)    sp_input['Th'] (either (B,1,3) or (B,3) upstream) */
    const float* bounds;   /* device (B,2,3)  sp_input['bounds'] (SMPL-frame box, xyz) */
    float voxel_size[3];   /* cfg.voxel_size, dhw order */
    int   out_sh[3];       /* sp_input['out_sh'], dhw order */
    int   level_dims[NB_NUM_LEVELS][4]; /* C,D,H,W of each packed level */
    const void* volume_blob;  /* device, from nb_pack_volume */
    int   volume_dtype;       /* NB_DTYPE_* of volume_blob */
    const void* weights_blob; /* device, from nb_pack_weights (same batch) */
    int   white_bkgd;      /* cfg.white_bkgd */
    int   precision;       /* NB_PRECISION_* */
    float* rgb_map;        /* device (B,n,3) */
    float* disp_map;       /* device (B,n)   */
    float* acc_map;        /* device (B,n)   */
    float* weights;        /* device (B,n,S) or NULL to skip */
    float* depth_map;      /* device (B,n)   */
    float* raw;            /* device (B,n,S,4) decoder output (rgb logits, sigma) or NULL; debugging / parity */
    int   out_ray_stride;  /* 0: rgb_map / disp_map / acc_map / depth_map are dense arrays ((B,n,3) and (B,n)).  > 0: floats
                              between consecutive rays in EACH of the four maps, so that they can be columns of one fused
                              (B,n,stride) record -- e.g. the 24-byte [rgb | disp | acc | depth] slab a ray-sharded render
                              all-gathers (stride 6, pointers slab+0, +3, +4, +5) */
    /* f-1, masked renderers (if_clight_renderer_mmsk.py:12-45; B = 1 only, as upstream): a sample is evaluated only if it
       projects into the foreground of every mask view; elsewhere raw = 0.  mask_msks NULL => no masking */
    const unsigned char* mask_msks;  /* device (nv, mask_H, mask_W) uint8 */
    const float* mask_RT;            /* device (nv,3,4) world->camera */
    const float* mask_Ks;            /* device (nv,3,3) */
    int   mask_nv, mask_H, mask_W;
    /* single-view variant (if_clight_renderer_msk.py:12-49, People-Snapshot demos): before projecting, a sample is taken from the
       world to the SMPL frame with this frame's (R, Th) and from there into the world of the snapshot frame the mask was
       shot in: q = ((p - Th) R) R0^T + Th0.  Both NULL => no such transform (the multi-view renderer) */
    const float* mask_R0;            /* device (3,3) batch['R0_snap'] or NULL */
    const float* mask_Th0;           /* device (3)   batch['Th0_snap'] or NULL */
    int   skip_empty;      /* tensor-core precisions: 1 = exact empty-sample skipping (samples whose trilinear cells are all
                              unoccupied have weight exactly 0 when sigma(empty) < 0; their MLP evaluation is skipped and `raw`,
                              if requested, holds (0, 0, 0, min(sigma_empty, 0)) for them instead of the decoder's rgb logits);
                              0 = every sample goes through the decoder (same maps bit for bit) */
    unsigned long long* stats; /* device u64[8] or NULL: [0] += 128-sample tiles executed, [1] += listed samples,
                                  [4] += layer-0 K-steps executed by those tiles (8 / 16 / 20 / 22 per tile, see below),
                                  [2] += ns spent in the decoder kernel (%globaltimer, first CTA start to last CTA end),
                                  [3] += decoder launches (tensor-core precisions), [5] / [6] += 64-row half tiles whose
                                  coarse-level (3 and 2) layer-0 features were gathered from the shared-memory staging /
                                  directly from global memory (more distinct voxels than the staging holds), [7] += 64-row
                                  half tiles whose fine-level (1 or 0) features were gathered directly, one per level */
    float* save;           /* device (B,n,S,1312) activation record for nb_render_bwd, or NULL (NB_PRECISION_FP32 only);
                              size from nb_render_save_bytes() */
    unsigned long long* trace; /* device, 4 x 4096 u64, or NULL: per-role (code<<48 | SM clock) timeline of CTA 0
                                  (tensor-core kernel only; diagnostics, see tools/trace_timeline.py) */
    void*  workspace;      /* device scratch of nb_render_fwd_workspace_bytes() bytes; REQUIRED by the tensor-core precisions (NULL
                              is fine for NB_PRECISION_FP32).  The samples of a frame that need the decoder (all of them with
                              skip_empty = 0) are compacted into four lists, one per finest occupied volume level, and the
                              decoder runs over full 128-sample tiles; a tile whose samples see no occupied cell in the finer
                              levels skips those levels' gather and layer-0 K-steps (exact: the features are zeros):
                              3 launches per frame (classify, decoder, composite) */
    size_t workspace_bytes;
    const float* z_vals;   /* device (B,n,S) or NULL.  When given, sample s of a ray sits at depth z_vals[b,r,s] (ascending) and
                              near / far / t_vals / t_rand are not read: the fine pass of hierarchical sampling (f-4; NeRF-style
                              volume_renderer.py:82-104 renders sorted(coarse z, importance z)).  Produced by nb_sample_pdf */
} nb_render_args;

int nb_render_fwd(const nb_render_args* args, void* stream);

/* Scratch bytes nb_render_fwd wants in nb_render_args.workspace for (batch, n_rays, n_samples): a 32-byte control block per
 * frame + two list buffers (each holds two of the four class lists, growing towards each other) + one frame's raw records
 * (16 B per sample each).  The buffer may be reused by
 * later calls on the same stream. */
size_t nb_render_fwd_workspace_bytes(int batch, int n_rays, int n_samples);

/* f-4: importance sampling between the coarse and the fine pass of a hierarchical (coarse + fine) render.  Neural Body's
 * own renderer has no fine pass; the spec is the reference's NeRF-baseline renderer: z_vals_mid, sample_pdf
 * (lib/networks/renderer/nerf_net_utils.py:55-90, det = (cfg.perturb == 0)) and the sort-merge of
 * lib/networks/renderer/volume_renderer.py:84-93.  The coarse depths are re-derived from (near, far, t_vals, t_rand)
 * exactly as nb_render_fwd derived them.  z_out then goes into nb_render_args.z_vals with n_samples = S + n_importance. */
typedef struct nb_importance_args {
    int n_rays_total;      /* B * n rays */
    int n_samples;         /* S of the coarse pass (3..256) */
    int n_importance;      /* cfg.N_importance (S + n_importance <= 512) */
    const float* near;     /* device (B*n) */
    const float* far;      /* device (B*n) */
    const float* t_vals;   /* device (S) or NULL, as in nb_render_args */
    const float* t_rand;   /* device (B*n,S) or NULL: the coarse pass's jitter */
    const float* weights;  /* device (B*n,S): the coarse pass's compositing weights */
    const float* u;        /* device (B*n,n_importance) uniforms [0,1) (the torch.rand of nerf_net_utils.py:70), or NULL for the
                              deterministic torch.linspace(0,1,n_importance) of the det branch */
    float* z_out;          /* device (B*n, S + n_importance): sorted(coarse z, importance z) */
    float* z_samples;      /* device (B*n, n_importance) or NULL: the importance samples alone (the reference's z_std input) */
} nb_importance_args;

int nb_sample_pdf(const nb_importance_args* args, void* stream);
/* nb_sample_pdf (the same launch, a bit-identical z_out) that also writes z_src: device (B*n, S + n_importance) int, for each
 * entry of z_out the coarse sample index it came from, or -1 for an importance sample.  It routes d z_out back to the coarse
 * depths (and so to near / far) when the fine pass is differentiated; on a tie either assignment holds the same z. */
int nb_sample_pdf_src(const nb_importance_args* args, int* z_src, void* stream);

/* f-3: density on arbitrary world points.  Replaces Network.calculate_density (lib/networks/latent_xyzc.py:74-89), the
 * alpha decoder of the mesh renderer (lib/networks/renderer/if_mesh_renderer.py:36-41).  Only the frame fields of `frame`
 * are read (batch, R, Th, bounds, voxel_size, out_sh, level_dims, volume_blob/dtype, weights_blob); exact fp32 arithmetic.
 * points: device (B, n_points, 3) world coordinates; sigma: device (B, n_points). */
int nb_decode_density(const nb_render_args* frame, const float* points, int n_points, float* sigma, void* stream);

/* The same density on the tensor cores (opt-in; nb_decode_density stays the exact reference).  Reads the frame fields of
 * nb_decode_density plus precision (NB_PRECISION_TC_FP16X3 or NB_PRECISION_TC_FP16; anything else is NB_ERR_BAD_ARG),
 * skip_empty, workspace / workspace_bytes (required, nb_decode_density_workspace_bytes), stats ([0]-[7] as for
 * nb_render_fwd, [1] = listed points) and trace.  sigma (B, n_points) is raw sigma, no relu.  With skip_empty = 1 a point
 * whose trilinear cells are unoccupied on all four levels (its features are all exactly 0, also outside the volume) gets
 * sigma_empty of the weight blob, whatever its sign; every other point goes through the decoder, and its sigma does not
 * depend on which points share its tile: it is the same bit for bit with skipping on or off and under any permutation of
 * the points.  n_points >= 2^28 returns NB_ERR_UNSUPPORTED before anything is enqueued; n_points = 0 is a no-op.  Per
 * frame: a classification launch and the decoder (plus a 1-thread launch that accounts stats[2] / [3] when stats is set),
 * after one memset of the control blocks per call. */
size_t nb_decode_density_workspace_bytes(int batch, int n_points);   /* control blocks + two list buffers of n_points entries */
int    nb_decode_density_list(const nb_render_args* frame, const float* points, int n_points, float* sigma, void* stream);

/* Marching cubes over a dense fp32 grid: the mesh step of the mesh renderer (lib/networks/renderer/if_mesh_renderer.py:42-48,
 * mcubes.marching_cubes(cube, cfg.mesh_th)).  A grid value is inside when it is > isovalue (equal counts as outside).
 * Vertices are the crossed grid edges p -> p + e_a, at p + t e_a with t = (iso - v(p)) / (v(p + e_a) - v(p)) in fp64, in
 * index coordinates; they follow grid-point order (x, y, z edge within a point).  Triangles follow the order of their
 * cells' min corners and the table order of csrc/nb_mc_table.h within a cell; (b - a) x (c - a) points towards decreasing
 * values.  The table separates the inside corners of every ambiguous face, so the mesh is closed wherever the surface
 * stays off the grid boundary.  Deterministic: no atomics decide any output position.
 * Usage: nb_mcubes_count, read counts on the host (one sync), allocate, nb_mcubes_emit with the same arguments and the
 * same workspace on the same stream (skip it when the mesh is empty).  Grids with 5 * cells >= 2^31 or 3 * points >= 2^31
 * (32-bit offsets) return NB_ERR_UNSUPPORTED before anything is enqueued; a grid with a dimension of 1 has no cell and an
 * empty mesh. */
typedef struct nb_mcubes_args {
    const float* grid;        /* device (nx, ny, nz) fp32, C order */
    int nx, ny, nz;
    double isovalue;          /* cfg.mesh_th */
    void* workspace;          /* device scratch of nb_mcubes_workspace_bytes(nx, ny, nz) bytes, kept from count to emit */
    size_t workspace_bytes;
    long long* counts;        /* device int64[2]: n_vertices, n_triangles (written by nb_mcubes_count) */
    double* vertices;         /* device (n_vertices, 3), index coordinates (nb_mcubes_emit) */
    long long* triangles;     /* device (n_triangles, 3) (nb_mcubes_emit) */
} nb_mcubes_args;
size_t nb_mcubes_workspace_bytes(int nx, int ny, int nz);   /* 0 for dims < 1 */
int    nb_mcubes_count(const nb_mcubes_args* a, void* stream);
int    nb_mcubes_emit(const nb_mcubes_args* a, void* stream);   /* after the caller read counts */

/* The mesh dataset's world grid and its mask-view test (lib/datasets/light_stage/multi_view_mesh_dataset.py:117-160,
 * prepare_inside_pts) on the device.  Grid point (i, j, k) is (x[i], y[j], z[k]); inside is written in the order of
 * meshgrid(x, y, z, indexing='ij').reshape(-1, 3), k fastest, and the grid itself is never materialised.  Per point, the
 * views are taken in order: the point is projected as base_utils.project does in fp32 (pts @ R^T + T, then @ K^T, then
 * xy / z), rounded half to even, converted as numpy's astype(int32) converts (NaN or outside int32 -> INT_MIN) and clipped to
 * [0, W-1] x [0, H-1]; the mask value there is read, and the point goes on to the next view only while that value is
 * exactly 1.  inside = the last value read (uint8, as upstream; callers treat it as a bool).  Validation (null pointers,
 * nv, H, W and grid dims >= 1, at most 2^31 points) happens before anything is enqueued; one launch. */
typedef struct nb_mesh_inside_args {
    const float* x;              /* device (nx) world x of the grid planes */
    const float* y;              /* device (ny) */
    const float* z;              /* device (nz) */
    int nx, ny, nz;
    const unsigned char* msks;   /* device (nv, H, W) uint8 mask views */
    const float* RT;             /* device (nv,3,4) world->camera, metres */
    const float* Ks;             /* device (nv,3,3) */
    int nv, H, W;
    unsigned char* inside;       /* device (nx, ny, nz) uint8, written */
} nb_mesh_inside_args;
int nb_mesh_inside(const nb_mesh_inside_args* a, void* stream);
/* The same test with a float64 camera (lib/datasets/light_stage/monocular_mesh_dataset.py:35-48, whose K, R and T are
 * float64, so numpy projects the float32 grid in float64): RT (nv,3,4) and Ks (nv,3,3) are device doubles passed here, and
 * a->RT / a->Ks must be NULL; everything else is read from `a` as nb_mesh_inside reads it.  Per point and view: the grid
 * point widened to double, pts @ R^T + T, then @ K^T, then xy / z, in double with the product and sum order of the fp32
 * chain; rounded half to even, converted as numpy's astype(int32) converts a float64 (NaN or outside int32 -> INT_MIN),
 * clipped.  The view loop and `inside` are nb_mesh_inside's.  Validated as nb_mesh_inside, before anything is enqueued. */
int nb_mesh_inside_f64(const nb_mesh_inside_args* a, const double* RT, const double* Ks, void* stream);

/* The demo datasets' per-view rays (render_utils.image_rays, lib/utils/render_utils.py:120-137, as called by
 * multi_view_demo_dataset.py:151, multi_view_perform_dataset.py:148 and monocular_demo_dataset.py:113) on the device, bit for
 * bit: get_rays (if_nerf_data_utils.py:8-21) in the camera's scalar type with the product and sum order numpy's BLAS uses
 * for upstream's two np.dot calls over the pixels, `.astype(np.float32)`, then get_near_far (:54-69) in float32 and the
 * `ray_o[mask_at_box]` compaction in row-major pixel order.  The per-view host operands are upstream's own: K_inv =
 * np.linalg.inv(K) and the camera centre o = -np.dot(R.T, T), both in the camera's dtype (their rounding belongs to the host
 * LAPACK / BLAS, so the caller computes them as upstream does); R (3,3) and T (3) row-major; all four are HOST memory, read
 * during the call.  The box is upstream's float32 can_bounds.
 * Writes mask_at_box (H*W) and the first n entries of ray_o / ray_d (n,3) and near / far (n), n = the number of pixels whose
 * ray enters the box, and n itself to `count` (device int32).  The caller reads count once (the one host synchronisation:
 * upstream's n varies per view).  Validation (null pointers, H, W >= 1, H*W < 2^31, workspace size) happens before anything is
 * enqueued; three launches (the box test, a CUB scan, the compacting write).
 * Shard mode (world >= 1): ONE RANK'S SHARD of a ray-sharded render (SURVEY 8e) in one launch, with a FIXED shape, so nothing
 * synchronises with the host.  Pixel chunk c (of `chunk` consecutive pixels) belongs to rank c % world; local ray j < n_local
 * is pixel ((j / chunk) * world + rank) * chunk + j % chunk, and its ray_o, ray_d, near, far and mask_at_box are the bits the
 * compacting call writes for that pixel.  A ray that misses the box (upstream drops it, image_rays :131-132) keeps ray_o /
 * ray_d with near = far = 0; a slot past the last pixel is o = 0, d = (0, 0, 1), near = far = 0.  Both are dead rays (every
 * sample sits at the camera centre, outside the volume, and is skipped) with mask_at_box = 0.  ray_o / ray_d (n_local,3),
 * near / far / mask_at_box (n_local); workspace and count are not read; image and rgb must be NULL.  rank in [0, world),
 * chunk >= 1 and n_local >= 0 are validated with the rest before anything is enqueued; n_local = 0 enqueues nothing. */
typedef struct nb_image_rays_args {
    int H, W;
    float bounds[6];             /* can_bounds (2,3): world box min, max */
    void* workspace;             /* device scratch of nb_image_rays_workspace_bytes(H, W) bytes */
    size_t workspace_bytes;
    float* ray_o;                /* device, room for H*W rays (n,3) */
    float* ray_d;                /* device, room for H*W rays (n,3), not normalised */
    float* near;                 /* device, room for H*W (n) */
    float* far;                  /* device, room for H*W (n) */
    unsigned char* mask_at_box;  /* device (H*W) 0 / 1 */
    int* count;                  /* device int32: n */
    const float* image;          /* device (H*W,3) or NULL: the view's image, whose box-hit pixels go to rgb (the training
                                    datasets' test split, if_nerf_data_utils.py:139-145) */
    float* rgb;                  /* device, room for H*W (n,3); set with image */
    int k_f32;                   /* nb_image_rays_f64 only, nonzero: K is float32 (K_inv's values are float32's and
                                    xy1 @ inv(K).T runs in float32, as for People-Snapshot's get_camera R and T) */
    int rank, world, chunk, n_local;  /* world = 0: the compacting call; world >= 1: shard mode (above) */
} nb_image_rays_args;
size_t nb_image_rays_workspace_bytes(int H, int W);   /* 0 for an invalid size */
/* float32 camera (monocular_demo_dataset.py:109-112: RT and K cast to float32) */
int nb_image_rays(const nb_image_rays_args* a, const float K_inv[9], const float R[9], const float T[3], const float o[3],
                  void* stream);
/* float64 camera (the multi-view demo / perform sets: gen_path's render_w2c and the annotation's K) */
int nb_image_rays_f64(const nb_image_rays_args* a, const double K_inv[9], const double R[9], const double T[3],
                      const double o[3], void* stream);

/* The training datasets' ray sampler (if_nerf_data_utils.sample_ray_h36m :153-219 for ZJU-MoCap's multi_view_dataset,
 * sample_ray :72-137 for People-Snapshot's monocular_dataset, split 'train') on the device.  Per batch item b the caller
 * hands the processed image and a class map built on the host from upstream's own masks; the call draws n_rays pixels in
 * upstream's rounds and writes, for each, the ray, near, far and colour upstream's item carries:
 *   - lists: the pixels of each class in row-major order (np.argwhere's), compacted by a CUB scan;
 *   - rounds (one CTA per item): m = n_rays - sampled, n_body = int(m * body_ratio), n_face = int(m * face_ratio) (in
 *     double, as Python), n_rand = m - n_body - n_face; candidates body, face (omitted when the face list is empty), bound,
 *     in that order; the ones whose ray enters the box are appended in that order, until n_rays are sampled;
 *   - a candidate's ray: get_rays (:8-21) at the pixel with the roundings of nb_image_rays, K_inv in K's dtype and R, T, o
 *     in float64; get_near_far (:54-69) in float64 on the float64 ray and the promoted float32 can_bounds; ray_o, ray_d,
 *     near and far rounded to float32 once; rgb gathered from the image.
 * Randomness: `draws` != NULL replays upstream's np.random.randint results (tests): item b's draws are
 * draws[draw_offset[b] .. draw_offset[b+1]), each round's body, face and bound draws in turn.  draws == NULL draws each
 * index from Philox4x32-10 keyed by `key` (counter: the item, the round and the candidate), mapped to [0, len) by the
 * 64-bit multiply-high.
 * status[b] (device int32): NB_TRAIN_RAYS_OK, or an error: upstream would loop forever (NB_TRAIN_RAYS_ROUNDS: no n_rays
 * after NB_TRAIN_RAYS_MAX_ROUNDS rounds), or would raise in randint (NB_TRAIN_RAYS_EMPTY: draws from an empty list), or
 * the replayed draws do not fit the lists (NB_TRAIN_RAYS_REPLAY).  The slots of an item whose status is not OK are
 * unspecified.  Validation (null pointers, sizes, ratios, kinds, workspace) happens before anything is enqueued; four
 * kinds of launch (three scans, the list scatter, the sampler); nothing synchronises with the host. */
#define NB_SCALAR_F32 0
#define NB_SCALAR_F64 1
#define NB_TRAIN_CAM_DOUBLES 30        /* per item: K_inv[9] | R[9] | T[3] | o[3] | can_bounds[6], row-major, as double */
#define NB_TRAIN_CLASS_BODY 1          /* class map bits */
#define NB_TRAIN_CLASS_FACE 2
#define NB_TRAIN_CLASS_BOUND 4
#define NB_TRAIN_RAYS_OK 0
#define NB_TRAIN_RAYS_ROUNDS 1
#define NB_TRAIN_RAYS_EMPTY 2
#define NB_TRAIN_RAYS_REPLAY 3
#define NB_TRAIN_RAYS_MAX_ROUNDS 64
typedef struct nb_train_rays_args {
    int B, H, W;
    int n_rays;                      /* N_rand, >= 1 */
    double body_ratio, face_ratio;   /* >= 0, body_ratio + face_ratio <= 1 */
    int k_kind;                      /* NB_SCALAR_*: K's dtype (People-Snapshot: float32; ZJU-MoCap: float64) */
    int rt_kind;                     /* R's and T's dtype: NB_SCALAR_F64 (both training datasets) */
    const unsigned char* class_map;  /* device (B,H,W): NB_TRAIN_CLASS_* bits */
    const float* image;              /* device (B,H,W,3) */
    const double* cams;              /* device (B, NB_TRAIN_CAM_DOUBLES): K_inv = np.linalg.inv(K) and o = -np.dot(R.T, T)
                                        as upstream computes them, each value exact in its kind */
    const long long* draws;          /* device, or NULL for Philox */
    const long long* draw_offset;    /* device (B+1), with draws */
    unsigned long long key[2];       /* Philox key, without draws */
    void* workspace;                 /* device scratch of nb_train_rays_workspace_bytes(B, H, W) bytes */
    size_t workspace_bytes;
    float* ray_o;                    /* device (B, n_rays, 3) */
    float* ray_d;                    /* device (B, n_rays, 3) */
    float* near;                     /* device (B, n_rays) */
    float* far;                      /* device (B, n_rays) */
    float* rgb;                      /* device (B, n_rays, 3) */
    int* coord;                      /* device (B, n_rays) row-major pixel index of each slot, or NULL */
    int* rounds;                     /* device (B) rounds run, or NULL */
    int* status;                     /* device (B) */
} nb_train_rays_args;
size_t nb_train_rays_workspace_bytes(int B, int H, int W);   /* 0 for an invalid size */
int nb_train_rays(const nb_train_rays_args* a, void* stream);

/* The training datasets' image steps after decoding (multi_view_dataset.py:121-145, monocular_dataset.py:74-103 upstream)
 * on the device, for B items of one size, bit for bit with OpenCV's:
 *   - cv2.undistort(img_u8 / 255 as float32, K, D) and cv2.undistort(msk_u8, K, D): the map of initUndistortRectifyMap in
 *     float64 (stripes of max(1, 4096 / W0) rows, each with its own inverse of the camera matrix; the per-column sums along
 *     each row), rounded to 1/32 px, then the bilinear remap with BORDER_CONSTANT 0 (float weights for the image, 15-bit
 *     fixed-point ones for the mask);
 *   - the resize to (H, W): a copy, or an exact 2x reduction (INTER_AREA's fast path for the image: the 2x2 cell summed
 *     row-major, times 0.25f; INTER_NEAREST for the mask: source pixel (2y, 2x));
 *   - the background: where the processed mask is 0, the image is 0 (NB_ITEM_BKGD_BLACK) or 1 (NB_ITEM_BKGD_WHITE);
 *   - optionally the sampler's class map (NB_TRAIN_CLASS_* bits) from the processed mask m and the bound mask bm,
 *     with mb = (uint8)(m * bm): NB_ITEM_CLASS_H36M (sample_ray_h36m): body mb == 1, face mb == 13, bound bm == 1 and
 *     mb != 100; NB_ITEM_CLASS_SNAPSHOT (sample_ray): body mb != 0, face mb == 13, bound bm == 1.
 * Validation (null pointers, sizes, the geometry, n_dist, the enums) happens before anything is enqueued; one launch; no
 * workspace; nothing synchronises with the host. */
#define NB_ITEM_CAM_DOUBLES 17         /* per item: K[9] row-major | k1 k2 p1 p2 k3 k4 k5 k6 (the first n_dist are read) */
#define NB_ITEM_MAX_W 4096
#define NB_ITEM_BKGD_NONE 0
#define NB_ITEM_BKGD_BLACK 1
#define NB_ITEM_BKGD_WHITE 2
#define NB_ITEM_CLASS_NONE 0
#define NB_ITEM_CLASS_H36M 1
#define NB_ITEM_CLASS_SNAPSHOT 2
typedef struct nb_item_images_args {
    int B, H0, W0;                   /* the decoded source size, W0 <= NB_ITEM_MAX_W */
    int H, W;                        /* the output size: (H0, W0), or exactly (H0 / 2, W0 / 2) */
    int n_dist;                      /* the distortion model's coefficient count: 4, 5 or 8 */
    int bkgd;                        /* NB_ITEM_BKGD_* */
    int class_rule;                  /* NB_ITEM_CLASS_* */
    const unsigned char* img_u8;     /* device (B,H0,W0,3) */
    const unsigned char* msk_u8;     /* device (B,H0,W0) */
    const double* cams;              /* device (B, NB_ITEM_CAM_DOUBLES): K and D at the source size, as float64 */
    const unsigned char* bound;      /* device (B,H,W) bound mask with a class rule, else NULL */
    float* img;                      /* device (B,H,W,3) */
    unsigned char* msk;              /* device (B,H,W) */
    unsigned char* class_map;        /* device (B,H,W) with a class rule, else NULL */
} nb_item_images_args;
int nb_item_images(const nb_item_images_args* a, void* stream);

/* The demo and mesh datasets' mask views after decoding (get_mask of multi_view_demo / multi_view_perform /
 * multi_view_mesh_dataset.py, the masks of monocular_demo / monocular_mesh_dataset.py upstream) on the device, for nv
 * views of one size, each with its own camera, bit for bit with OpenCV's host steps:
 *   - with `binarise`, the source is (m != 0) (upstream's (msk_cihp != 0).astype(np.uint8)), else the decoded values;
 *   - cv2.undistort(src, K, D) at the source size: nb_item_images' map and its 15-bit fixed-point uint8 remap;
 *   - with dilate = 5, cv2.dilate(., np.ones((5, 5))): the maximum over the 5 x 5 window, pixels outside the image not
 *     taking part (the default border);
 *   - the resize to (H, W): a copy, or an exact 2x reduction by INTER_NEAREST (source pixel (2y, 2x)).
 * Pass 1 undistorts every view at the source size into the workspace, pass 2 dilates and picks the output pixels.
 * Validation (null pointers, sizes, the geometry, n_dist, dilate, the workspace size) happens before anything is
 * enqueued; two launches; nothing synchronises with the host. */
typedef struct nb_mask_views_args {
    int nv, H0, W0;                  /* the decoded views' size, W0 <= NB_ITEM_MAX_W */
    int H, W;                        /* the output size: (H0, W0), or exactly (H0 / 2, W0 / 2) */
    int n_dist;                      /* the distortion model's coefficient count: 4, 5 or 8 */
    int binarise;                    /* 1: undistort (m != 0); 0: the decoded values */
    int dilate;                      /* 0 (none) or 5 (a 5 x 5 window) */
    const unsigned char* msk_u8;     /* device (nv,H0,W0) */
    const double* cams;              /* device (nv, NB_ITEM_CAM_DOUBLES): each view's K and D at the source size */
    void* workspace;                 /* device, nb_mask_views_workspace_bytes(nv, H0, W0) bytes */
    size_t workspace_bytes;
    unsigned char* msks;             /* device (nv,H,W) */
} nb_mask_views_args;
size_t nb_mask_views_workspace_bytes(int nv, int H0, int W0);   /* 0 for an invalid size */
int nb_mask_views(const nb_mask_views_args* a, void* stream);

/* The evaluator's per-view metrics (lib/evaluators/if_nerf.py upstream) on the device, from the rendered rays, the
 * test split's colours and mask_at_box:
 *   - scatter: ray k is the k-th set pixel of mask_at_box in row-major order (img[mask_at_box] = rgb); every other pixel
 *     is white_bkgd (0 or 1).  n must equal the mask's count, else status NB_EVAL_COUNT (upstream's numpy raises);
 *   - box: cv2.boundingRect of the mask (x, y, w, h; (0,0,0,0) for an empty mask), or the whole image with eval_whole_img;
 *   - mse: eval_whole_img 0: the mean over the n x 3 ray values of fp32(fp32(pred - gt)^2), the terms summed in float64;
 *     eval_whole_img 1: the mean over the float64 H x W x 3 images.  psnr = -10 log10(mse) in float64;
 *   - ssim: scikit-image 0.14.2's compare_ssim(X, Y, multichannel=True) over the box in float64: per channel the 7 x 7
 *     means of x, y, xx, yy, xy, cov_norm = 49/48, C1 = (0.01 * 2)^2, C2 = (0.03 * 2)^2 (a float image's data_range is 2),
 *     S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)), the channel value the mean of S over the box
 *     minus its 3-pixel border (those windows lie inside the box, so the filter's edge mode never enters), the result the
 *     mean of the three.  A box side under 7 is status NB_EVAL_SMALL (upstream's "win_size exceeds image extent");
 *   - crops: the box of each image as uint8 BGR, row-major, saturate_cast<uchar>(v * 255) with round-half-even (what
 *     cv2.imwrite makes of upstream's float64 img[..., [2,1,0]] * 255), at the start of crop_pred / crop_gt.
 * Fixed-order reductions and no floating-point atomics: the same inputs give the same bits.  `result` is written on the
 * device; the caller reads it (and the crops) back once.  Validation (null pointers, sizes, flags, workspace) happens
 * before anything is enqueued; six launches (the mask's box partials, a CUB scan, the ray sums, the first finish, the
 * SSIM tiles with the crops, the SSIM finish); nothing synchronises with the host. */
#define NB_EVAL_OK 0
#define NB_EVAL_COUNT 1                /* n != the number of set pixels of mask_at_box */
#define NB_EVAL_SMALL 2                /* a side of the box is under 7 pixels */
typedef struct nb_eval_image_result {
    int status;                        /* NB_EVAL_* */
    int count;                         /* set pixels of mask_at_box */
    int box[4];                        /* x, y, w, h of the region the SSIM and the crops cover */
    double sq_sum;                     /* the float64 sum of the MSE's terms */
    double mse, psnr, ssim;            /* NaN where the status says upstream raised before reaching them */
    double ssim_channel[3];
} nb_eval_image_result;
typedef struct nb_eval_image_args {
    int n;                             /* rays, 0 <= 3n < 2^31 */
    int H, W;                          /* the view, H*W < 2^31 */
    int white_bkgd;                    /* 0 / 1 */
    int eval_whole_img;                /* 0 / 1 */
    const float* rgb_pred;             /* device (n,3) */
    const float* rgb_gt;               /* device (n,3) */
    const unsigned char* mask_at_box;  /* device (H*W), nonzero = set */
    void* workspace;                   /* device scratch of nb_eval_image_workspace_bytes(H, W, n) bytes */
    size_t workspace_bytes;
    nb_eval_image_result* result;      /* device */
    unsigned char* crop_pred;          /* device, room for H*W*3 */
    unsigned char* crop_gt;            /* device, room for H*W*3 */
} nb_eval_image_args;
size_t nb_eval_image_workspace_bytes(int H, int W, int n);   /* 0 for an invalid size */
int nb_eval_image(const nb_eval_image_args* a, void* stream);

/* The demo visualizers' frame (lib/visualizers/if_nerf_demo.py and if_nerf_perform.py upstream) on the device: the uint8
 * BGR H x W x 3 array cv2.imwrite stores for upstream's float64 image img_pred[..., [2,1,0]] * 255, where
 * img_pred[mask_at_box] = rgb_map over a background of white_bkgd (0 or 1):
 *   - a set pixel takes the ray at the mask's exclusive prefix count (ray k is the k-th set pixel, row-major); with n = 1
 *     every set pixel takes ray 0 (numpy broadcasts a (1,3) value);
 *   - each value is saturate_cast<uchar>(v * 255): the float64 product rounded half to even, NaN or outside int32 to
 *     INT_MIN, then clamped to [0, 255].
 * A count other than n (and n != 1) is status NB_VIS_COUNT, upstream's numpy "shape mismatch"; the frame is then not
 * written.  Validation (null pointers, sizes, white_bkgd, a 4-byte aligned frame, workspace) happens before anything is
 * enqueued; two launches (a CUB scan of the mask, the frame with the status record); nothing synchronises with the host. */
#define NB_VIS_OK 0
#define NB_VIS_COUNT 1                 /* n != the number of set pixels of mask_at_box */
typedef struct nb_vis_frame_result {
    int status;                        /* NB_VIS_* */
    int count;                         /* set pixels of mask_at_box */
} nb_vis_frame_result;
typedef struct nb_vis_frame_args {
    int n;                             /* rays, 0 <= 3n < 2^31 */
    int H, W;                          /* the view, H*W < 2^31 */
    int white_bkgd;                    /* 0 / 1 */
    const float* rgb_map;              /* device (n,3) */
    const unsigned char* mask_at_box;  /* device (H*W), nonzero = set */
    void* workspace;                   /* device scratch of nb_vis_frame_workspace_bytes(H, W) bytes */
    size_t workspace_bytes;
    nb_vis_frame_result* result;       /* device */
    unsigned char* frame;              /* device (H,W,3) BGR, 4-byte aligned */
} nb_vis_frame_args;
size_t nb_vis_frame_workspace_bytes(int H, int W);   /* 0 for an invalid size */
int nb_vis_frame(const nb_vis_frame_args* a, void* stream);

/* The binary little-endian PLY body of a triangle mesh (nb_mcubes_emit's outputs), the bytes neuralbody_b200.mcubes.Mesh
 * .export writes after its header "... end_header\n":
 *   - nv vertex records of 24 bytes: the vertices array's own float64 bytes (x y z), in order;
 *   - nf face records of 13 bytes: uchar 3, then the face's three indices as little-endian int32.
 * `out` holds an nb_mesh_ply_result at its head and the body from NB_MESH_PLY_BODY_OFFSET on, so that one copy brings both
 * back.  A face index < 0 or >= max(nv, 1) (the bound Mesh.export checks) is status NB_MESH_PLY_FACE; the body then holds
 * that index's low 32 bits and must not be written out.  Nothing past NB_MESH_PLY_BODY_OFFSET + nb_mesh_ply_bytes(nv, nf)
 * is written.  Validation (null pointers, counts, nv < 2^31, alignment, out_bytes) happens before anything is enqueued; a
 * memset of the result record and one launch; nothing synchronises with the host. */
#define NB_MESH_PLY_OK 0
#define NB_MESH_PLY_FACE 1             /* a face index outside [0, max(nv, 1)) */
#define NB_MESH_PLY_BODY_OFFSET 16
typedef struct nb_mesh_ply_result {
    int status;                        /* NB_MESH_PLY_* */
    int reserved[3];
} nb_mesh_ply_result;
typedef struct nb_mesh_ply_args {
    long long nv;                      /* vertices, 0 <= nv < 2^31 */
    long long nf;                      /* faces, 0 <= nf <= 2^40 */
    const double* vertices;            /* device (nv,3), 8-byte aligned; may be NULL when nv = 0 */
    const long long* faces;            /* device (nf,3), 8-byte aligned; may be NULL when nf = 0 */
    unsigned char* out;                /* device, 16-byte aligned: nb_mesh_ply_result, then the body */
    size_t out_bytes;                  /* >= NB_MESH_PLY_BODY_OFFSET + nb_mesh_ply_bytes(nv, nf) */
} nb_mesh_ply_args;
size_t nb_mesh_ply_bytes(long long nv, long long nf);   /* 24 nv + 13 nf; 0 for invalid counts (and for an empty mesh) */
int nb_mesh_ply(const nb_mesh_ply_args* a, void* stream);

/* The image losses of upstream's training wrapper (lib/train/trainers/if_nerf_clight.py:24-32) on the device, without the
 * host wait of a boolean-mask index:
 *   img_loss  = mean over the set rays' elements of (rgb_map - rgb)^2   (mask = mask_at_box)
 *   img_loss0 = mean over all elements of (rgb0 - rgb)^2                (mask = NULL)
 * nb_image_loss_fwd writes the loss (float32; the sum in float64, then one rounding) and the number of elements averaged,
 * 3 x the set rays, in ONE launch: per-CTA partials over a grid that depends on `rays` only, finished in CTA order by the
 * last CTA (an integer ticket), so the loss is the same bits on every run; no floating-point atomics.  No element gives a
 * NaN loss, as torch.mean of an empty tensor.  nb_image_loss_bwd writes d_pred (rays,3), the cotangent autograd computes
 * on the GPU for upstream's expression, bit for bit: g * (1.0f / (float)count), times 2 * (pred - gt), in fp32 in that
 * order, on the set rays (plus 0, the index backward's scatter into zeros, when there is a mask) and exact 0 elsewhere; g is
 * the device scalar d_loss and count the forward's.  Validation happens before anything is enqueued; both enqueue one
 * launch on the caller's stream (none for rays = 0 in the backward); nothing allocates or synchronises.  The workspace is
 * zeroed once when allocated and the forward leaves it so; calls that share one must be ordered (one stream). */
typedef struct nb_image_loss_args {
    int rays;                          /* B*n rays of 3 channels, 0 <= 3 rays < 2^31 */
    const float* pred;                 /* device (rays,3): rgb_map or rgb0 */
    const float* gt;                   /* device (rays,3): batch['rgb'] */
    const unsigned char* mask;         /* device (rays), nonzero = set (bool or uint8); NULL = every ray */
    void* workspace;                   /* device, 256-byte aligned, nb_image_loss_workspace_bytes(); forward only */
    size_t workspace_bytes;
    float* loss;                       /* device scalar; written by the forward */
    long long* count;                  /* device scalar: elements averaged; written by the forward, read by the backward */
} nb_image_loss_args;
size_t nb_image_loss_workspace_bytes(void);
int nb_image_loss_fwd(const nb_image_loss_args* a, void* stream);
int nb_image_loss_bwd(const nb_image_loss_args* a, const float* d_loss, float* d_pred, void* stream);

/* The reference's SparseConvNet encode (lib/networks/latent_xyzc.py:30-39,166-274; spconv 1.2.1 semantics, restated in
 * oracle/spconv_oracle.py) as sparse convolutions over the active sites, forward and backward (opt-in from Python:
 * `sparse_encode: 'cuda'`).  17 layers in the reference's order (conv0 x2, down0, conv1 x2, down1, conv2 x3, down2, conv3
 * x3, down3, conv4 x3), each SubMConv3d(k=3) or SparseConv3d(k=3, s=2, p=1) without bias, then BatchNorm1d over the active
 * rows and ReLU; the outputs of layers 4, 8, 12 and 16 are net1..net4.
 *   - input: point i sits at coord[i] = (b, z, y, x) with feature code[i % n_vert]; several points on one site: the highest
 *     index wins; a point outside [0, batch) x out_sh is ignored.  Strided output extent floor((in - 1) / 2) + 1 per axis;
 *     a site is active iff its 3x3x3 window holds an active input.
 *   - BatchNorm: training = 1 normalises with the batch statistics (biased variance), then updates running_mean /
 *     running_var (unbiased) with `momentum` and adds 1 to num_batches_tracked; training = 0 uses the running statistics.
 *   - volumes[l]: (batch, C_l, D_l, H_l, W_l) fp32 with C = 32, 64, 128, 128 and the extents of strided levels 1..4; written
 *     whole, exact 0 off the active set.
 * fp32 FFMA arithmetic, float64 BatchNorm sums.  The row counts never leave the device: buffers are sized from bounds
 * (level 0 <= n_points, level l+1 <= min(8 x level l, B D_l H_l W_l)) in the workspace, whose size depends on
 * (batch, n_points, out_sh) only.  nb_spconv_bwd takes the same arguments and the workspace the forward call filled,
 * unchanged, and the cotangents of the four volumes; it WRITES every gradient (d_code, the conv weights, the BatchNorm
 * weights and biases); weight and BatchNorm sums use atomics, so the gradients are not bit-reproducible.  Validation (null
 * pointers, batch, n_points, n_vert, out_sh, training, eps, momentum, workspace) happens before anything is enqueued;
 * nothing allocates or synchronises with the host. */
#define NB_SPCONV_LAYERS 17
#define NB_SPCONV_CODE_DIM 16           /* the code embedding's width, c = nn.Embedding(6890, 16) */
typedef struct nb_spconv_args {
    int batch;                          /* B frames */
    int n_points;                       /* rows of coord (B * 6890 upstream) */
    int n_vert;                         /* rows of code (6890) */
    int out_sh[3];                      /* D, H, W of the input grid */
    const int* coord;                   /* device (n_points, 4) int32 (b, z, y, x) */
    const float* code;                  /* device (n_vert, 16) */
    const float* weight[NB_SPCONV_LAYERS];        /* device (3, 3, 3, Cin, Cout) each, spconv's layout */
    const float* bn_weight[NB_SPCONV_LAYERS];     /* device (Cout) */
    const float* bn_bias[NB_SPCONV_LAYERS];       /* device (Cout) */
    float* running_mean[NB_SPCONV_LAYERS];        /* device (Cout); updated when training */
    float* running_var[NB_SPCONV_LAYERS];         /* device (Cout); updated when training */
    long long* num_batches_tracked[NB_SPCONV_LAYERS];   /* device scalar; training only (may be NULL otherwise) */
    int training;                       /* 1: batch statistics, 0: running statistics */
    float momentum, eps;                /* BatchNorm1d(eps=1e-3, momentum=0.01) upstream */
    void* workspace;                    /* device, 256-byte aligned, nb_spconv_workspace_bytes() */
    size_t workspace_bytes;
    float* volumes[NB_NUM_LEVELS];      /* device, written */
    int* row_counts;                    /* device int32[5] or NULL: active sites of the input grid and of levels 1..4 */
} nb_spconv_args;
typedef struct nb_spconv_grads {
    const float* d_volumes[NB_NUM_LEVELS];        /* device, shaped as volumes; NULL = zero cotangent */
    float* d_code;                                /* device (n_vert, 16), written */
    float* d_weight[NB_SPCONV_LAYERS];            /* device, shaped as weight, written */
    float* d_bn_weight[NB_SPCONV_LAYERS];         /* device (Cout), written */
    float* d_bn_bias[NB_SPCONV_LAYERS];           /* device (Cout), written */
} nb_spconv_grads;
size_t nb_spconv_workspace_bytes(int batch, int n_points, const int out_sh[3]);   /* 0 for an invalid size */
int nb_spconv_fwd(const nb_spconv_args* a, void* stream);
int nb_spconv_bwd(const nb_spconv_args* a, const nb_spconv_grads* g, void* stream);

/* number of kernels nb_render_fwd enqueues per FRAME of a call: 1 for NB_PRECISION_FP32 (the single fused exact kernel),
 * 3 for the tensor-core inference precisions (classify, decoder, composite; plus one 32-byte memset per call), 9 for
 * NB_PRECISION_TC_TF32X3 (colour-matrix build, classify, gather, 4 GEMMs, rgb head, composite). */
int nb_render_fwd_launches(int precision);

/* ------------------------------------------------------------------------------------------
 * Backward of the fused render (training, BASELINE config 3).  Replaces PyTorch autograd through
 * raw2outputs (nerf_net_utils.py:6-51), Network.calculate_density_color (latent_xyzc.py:91-126) and
 * F.grid_sample (latent_xyzc.py:62-72) as driven by Trainer.train (lib/train/trainers/trainer.py:46-53).
 * Usage: run nb_render_fwd with NB_PRECISION_TC_TF32X3 (tensor cores, exact empty-sample skipping in both passes) or
 * NB_PRECISION_FP32 (the exact FFMA kernels; fp32 volume blob only), `raw` and `save` set; then call
 * nb_render_bwd with the same nb_render_args and the output gradients.  Gradients are ACCUMULATED into the
 * caller's (zeroed) buffers: `grads` mirrors nb_decoder_weights (same shapes; latent_index unused),
 * d_volumes[l] is the NCDHW fp32 gradient of level l (what autograd hands back to the SparseConvNet). */
typedef struct nb_render_bwd_args {
    const nb_render_args* fwd;          /* the forward call's arguments (unchanged) */
    const float* save;                  /* device, written by the forward call */
    const float* raw;                   /* device (B,n,S,4), written by the forward call */
    const float* d_rgb_map;             /* device (B,n,3) or NULL */
    const float* d_depth_map;           /* device (B,n)   or NULL */
    const float* d_acc_map;             /* device (B,n)   or NULL */
    const nb_decoder_weights* weights;  /* the raw decoder tensors the forward blob was packed from */
    const nb_decoder_weights* grads;    /* device gradient tensors, accumulated into */
    float* d_volumes[NB_NUM_LEVELS];    /* device (B,C,D,H,W) fp32 each, accumulated into; all NULL to skip */
    void* workspace;                    /* device scratch, nb_render_bwd_workspace_bytes() */
    size_t workspace_bytes;
} nb_render_bwd_args;

size_t nb_render_save_bytes(int batch, int n_rays, int n_samples);            /* NB_PRECISION_FP32 */
size_t nb_render_bwd_workspace_bytes(int batch, int n_rays, int n_samples);   /* NB_PRECISION_FP32 */
/* the same two sizes for the precision (and volume dimensions) of a forward call: NB_PRECISION_FP32 as above;
 * NB_PRECISION_TC_TF32X3: record = list + 1364 floats per sample of the batch (worst case: every sample listed), backward
 * scratch = 1268 floats per sample + a channels-last copy of the volume gradients */
size_t nb_render_save_bytes_for(const nb_render_args* fwd);
size_t nb_render_bwd_workspace_bytes_for(const nb_render_args* fwd);
int    nb_render_bwd(const nb_render_bwd_args* args, void* stream);
/* nb_render_bwd plus the gradients of the frame transform the forward call read (nb_render_args.R / .Th): what pose
 * refinement needs, i.e. upstream autograd through pts_to_can_pts -> get_grid_coords -> F.grid_sample's grid input
 * (latent_xyzc.py:41-72).  d_R: device (B,3,3) fp32, d_Th: device (B,3) fp32; both are ACCUMULATED into and either may
 * be NULL.  R and Th reach the outputs only through the grid coordinates (the positional encoding takes the world points),
 * so this is the trilinear backward with respect to the sample position, chained through the transform.  Both training
 * precisions; it reads the volume blob the forward gathered from.  nb_render_bwd(args, stream) is
 * nb_render_bwd_frame(args, NULL, NULL, stream) and enqueues no frame-gradient work.  No extra workspace. */
int    nb_render_bwd_frame(const nb_render_bwd_args* args, float* d_R, float* d_Th, void* stream);
/* nb_render_bwd_frame plus the gradients of the rays the forward call read (nb_render_args.ray_o / .ray_d): what camera
 * refinement needs, i.e. upstream autograd through pts = ray_o + ray_d * z (if_clight_renderer.py:25), the view direction
 * ray_d / |ray_d| (:68) and PE(world xyz) into view_fc (latent_xyzc.py:115), the canonical transform into grid_sample, and
 * dists * |ray_d| in raw2outputs (nerf_net_utils.py:28).  d_ray_o, d_ray_d: device (B,n,3) fp32; both are ACCUMULATED into
 * and either may be NULL.  The depths z are not differentiated here (nb_render_bwd_inputs does that); after a z_vals
 * (fine-pass) forward they are taken as given.  Both training precisions.  nb_render_bwd_frame(args, dR, dTh, stream) is
 * nb_render_bwd_rays(args, dR, dTh, NULL, NULL, stream) and enqueues no ray-gradient work.  No extra workspace. */
int    nb_render_bwd_rays(const nb_render_bwd_args* args, float* d_R, float* d_Th, float* d_ray_o, float* d_ray_d, void* stream);
/* nb_render_bwd_rays plus the cotangents of the two remaining output maps, so that a loss on any output of the render
 * differentiates as upstream's autograd does (raw2outputs, nerf_net_utils.py:37-45).  d_disp_map: device (B,n) fp32,
 * d_weights: device (B,n,S) fp32, both dense; either may be NULL.  They enter the per-ray compositing backward only:
 *   weights:  w_i = alpha_i T_i, differentiated exactly like the other maps;
 *   disp_map: 1 / max(1e-10, depth / acc) with torch's backward rules (reciprocal; maximum: all of the gradient to
 *             depth / acc where it is > 1e-10 or NaN, half where it equals 1e-10, none below; division).  depth and acc are
 *             recomputed as the forward composited them, before the white background; the output maps are not read.
 * NaN semantics are upstream's: on a ray with acc_map == 0, disp_map is NaN (0 / 0), and with a non-NULL d_disp_map its
 * gradient is NaN whatever the cotangent (0 * NaN = NaN).  relu(sigma) masks it out of every sample's sigma, so the
 * decoder, volume, R / Th and ray_o gradients stay finite; d_ray_d, which takes dists * relu(sigma) with relu(sigma) = 0,
 * is NaN on exactly those rays.  Both training precisions; S <= 256 as for every backward.
 * nb_render_bwd_rays(args, dR, dTh, do, dd, stream) is nb_render_bwd_maps(args, NULL, NULL, dR, dTh, do, dd, stream).
 * No extra workspace and no extra launch. */
int    nb_render_bwd_maps(const nb_render_bwd_args* args, const float* d_disp_map, const float* d_weights, float* d_R,
                          float* d_Th, float* d_ray_o, float* d_ray_d, void* stream);
/* nb_render_bwd_maps plus the gradients of the remaining float inputs upstream's autograd reaches: the depths and the box.
 * Every pointer is a device fp32 buffer ACCUMULATED into, and any may be NULL (a NULL struct = all NULL).
 *   d_R, d_Th, d_ray_o, d_ray_d: as for nb_render_bwd_maps.
 *   d_near, d_far (B,n): through z = near (1 - t) + far t and the stratified jitter (if_clight_renderer.py:11-23).  Only for
 *     a forward that derived its depths from near / far: with nb_render_args.z_vals set they return NB_ERR_BAD_ARG before
 *     anything is enqueued.
 *   d_z_vals (B,n,S): d loss / d z_i per sample, after either kind of forward:
 *     d z_i = g_i . ray_d + dD w_i + |ray_d| (c_{i-1} - c_i),  c_i = dalpha_i relu(sigma_i) exp(-relu(sigma_i) dist_i),
 *     c_{S-1} = c_{-1} = 0 (the last dist is 1e10 |ray_d|), where g_i is d loss / d(world point i) (grid and PE(xyz) parts)
 *     and dD the depth_map cotangent after the disp_map fold.  d_near / d_far are the sums of d z_i times z_i's coefficients.
 *   d_bounds (B,2,3): row 0 -= the per-frame sum of d loss / d(canonical point) (get_grid_coords, latent_xyzc.py:49-60
 *     subtracts bounds[:, 0]); row 1 is not touched.
 * NaN semantics follow nb_render_bwd_maps: on a ray with acc_map == 0 and a d_disp_map cotangent, d_near, d_far and that
 * ray's d_z_vals are NaN; d_bounds stays finite.  Both training precisions; S <= 256.  With the four new pointers NULL this is
 * nb_render_bwd_maps and enqueues the same kernels.  No extra workspace. */
typedef struct nb_render_input_grads {
    float* d_R;  float* d_Th;          /* as nb_render_bwd_rays */
    float* d_ray_o; float* d_ray_d;    /* as nb_render_bwd_rays */
    float* d_near; float* d_far;       /* (B,n); only for a forward that derived z from near/far (z_vals == NULL) */
    float* d_z_vals;                   /* (B,n,S): dL/dz_i per sample, either kind of forward */
    float* d_bounds;                   /* (B,2,3): row 0 accumulated, row 1 untouched */
} nb_render_input_grads;
int    nb_render_bwd_inputs(const nb_render_bwd_args* args, const float* d_disp_map, const float* d_weights,
                            const nb_render_input_grads* grads, void* stream);

/* ------------------------------------------------------------------------------------------
 * Diagnostics.
 */
/* The training path's GEMM in isolation (csrc/nb_train.cu): c (M,N) = epilogue(a b^T), fp32 in and out, 3 x TF32 passes.
 * a: (M,K) if a_k_contiguous else (K,M); b: (N,K) if b_k_contiguous else (K,N); N % 16 == 0, leading dimensions % 4 == 0.
 * splits > 1 splits the reduction over CTAs and ACCUMULATES into c (zero it first).  bias (N) / mask (M,N) may be NULL. */
int nb_debug_gemm_tf32x3(const float* a, const float* b, float* c, int M, int N, int K, int a_k_contiguous, int b_k_contiguous,
                         int splits, const float* bias, int relu, const float* mask, void* stream);
/* The render's compositing (raw2outputs) in isolation, on caller-made raw records instead of the decoder's.  The ray fields
 * of `a` are read and validated as nb_render_fwd reads them (batch, n_rays, n_samples <= 1024, ray_o, ray_d, near, far, t_vals,
 * t_rand, z_vals, white_bkgd, the four maps, weights, out_ray_stride); no frame field is read.  raw: device (B,n,S,4) (rgb
 * logits, sigma).  Writes the maps and weights a render writes from those records, with the same kernel, one launch per frame. */
int nb_debug_composite(const nb_render_args* a, const float* raw, void* stream);
/* Its backward as the training backward runs it: d_raw (B,n,S,4) = d loss / d(rgb logits, sigma) from the five map
 * cotangents (device, dense, any NULL; see nb_render_bwd_maps).  With `rec` (device (B,n,S,8): per sample d loss / d(world
 * point) 3 | d loss / d(view direction) 3 | 2 unused, standing in for the decoder's part) it also ACCUMULATES d_ray_o, d_ray_d,
 * d_near, d_far and d_z_vals of `grads` (as nb_render_bwd_inputs; d_R, d_Th, d_bounds must be NULL).  n_samples <= 256.  Sizes and
 * pointers are validated before anything is enqueued. */
int nb_debug_composite_bwd(const nb_render_args* a, const float* raw, const float* d_rgb_map, const float* d_depth_map,
                           const float* d_acc_map, const float* d_disp_map, const float* d_weights, const float* rec,
                           const nb_render_input_grads* grads, float* d_raw, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NEURALBODY_B200_H */
