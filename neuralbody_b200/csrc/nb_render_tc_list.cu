// The tensor-core render path: three launches over a frame's COMPACT SAMPLE LIST (nb_render_args.workspace).
//
//   1. classify_compact_kernel   every sample of the frame is classified with the four cell-occupancy bitmaps; occupied
//                                samples are appended to the list of their CLASS = finest occupied level (one atomicAdd per
//                                class and 1024-sample block), the others get their constant raw record
//                                (0, 0, 0, min(sigma_empty, 0)) at once.  With skip_empty = 0 every sample is listed.
//                                Layer 0 consumes the features coarse level first, so a class-c tile runs only the leading
//                                2 / 4 / 5 / 6 of its six 64-channel K segments (gather AND MMAs): exact, the skipped
//                                segments are all zeros.
//   2. render_tc_list_kernel     the decoder MLP (latent_xyzc.py:91-126) over the list, 128 entries per tile, on the Hopper
//                                tensor cores (wgmma, see below).
//   3. composite_kernel          raw2outputs (nerf_net_utils.py:6-51), one warp per ray.
//
// Precision: the density path (layers 0-2) runs in the 3-pass mode as A_hi W_hi + A_lo W_hi + A_hi W_lo with fp16 (hi, lo)
// pairs of both operands and fp32 accumulation (~fp32-accurate), or as A_hi W_hi only in the 1-pass mode.  h2 is converted to
// its hi halves only (rounded to nearest): the colour layer is a 1-pass layer, and sigma = alpha_fc . relu(acc) and the 3-wide
// rgb head are fp32 dot products on the accumulator registers.
//
// Results do not depend on the (non-deterministic) order of the blocks in the list: a tile row is evaluated
// independently of its neighbours.  The list and the raw (rgb logits, sigma) records cross HBM once each way.
//
// Density queries (nb_decode_density_list, the mesh renderer) run the same pipeline on world points instead of ray
// samples: classify_points_kernel lists the points (a point whose cells are unoccupied on every level gets sigma_empty at
// once with skip_empty = 1), and density_tc_list_kernel, the decoder with layer 3 and the rgb head left out, writes raw
// sigma (layers 0-2 and alpha_fc) for the listed ones.  There is no composite.
#include "nb_tc_common.cuh"
#include <type_traits>

namespace nb {
namespace tcl {

using tcr::Quad;

constexpr int TP = 128;                                            // list rows per tile
constexpr int NUM_SEGS = 6;

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ------------------------------------------------------------------------------------------------ 1. classify + compact
constexpr int CLS_THREADS = 256;

// bit l = the level-l trilinear cell at grid coordinates (gx, gy, gz) holds a non-zero voxel of frame b.  A cell with no
// corner inside the volume (outside the box, where grid_sample pads with zeros) holds none.
__device__ __forceinline__ uint32_t occupied_levels(const RenderParams& P, int b, float gx, float gy, float gz) {
    const uint32_t* occ_base = reinterpret_cast<const uint32_t*>(P.volume);
    uint32_t lm = 0;
#pragma unroll
    for (int lvl = 0; lvl < 4; ++lvl) {
        const int D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
        Corners cn;
        corner_setup(unnormalize(gx, W), unnormalize(gy, H), unnormalize(gz, D), W, H, D, cn);
        if (cn.x0 != -2 && cn.x0 < W && cn.y0 < H && cn.z0 < D) {
            const uint32_t* cellbits = occ_base + P.occ_off[lvl] / 4 + (size_t)b * P.occ_bstride[lvl];
            const uint32_t cell = ((uint32_t)(cn.z0 + 1) * (H + 1) + (cn.y0 + 1)) * (W + 1) + (cn.x0 + 1);
            lm |= ((__ldg(cellbits + (cell >> 5)) >> (cell & 31)) & 1u) << lvl;
        }
    }
    return lm;
}

// Appends a CLS_THREADS block's entries to the lists of their class.  Thread tid holds N entries e[k] of class cls[k] (0..3,
// -1 = not listed); entry k of thread tid is entry k * CLS_THREADS + tid of the block, and each class keeps that order.
// The classes are counted with ballots and reserved with one atomicAdd per class and block, so a block's entries of a class
// stay contiguous.  Classes 3 / 1 grow upwards from the start of list_a / list_b, classes 2 / 0 downwards from their end.
template <int N>
__device__ __forceinline__ void append_to_lists(const RenderParams& P, const float4 (&e)[N], const int (&cls)[N]) {
    constexpr int WARPS = CLS_THREADS / 32;
    __shared__ int wcnt[4][N * WARPS];
    __shared__ unsigned int sbase[4];
    __shared__ int stotal[4];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t bal = __ballot_sync(0xffffffffu, cls[k] == c);
            if (lane == 0) wcnt[c][k * WARPS + warp] = __popc(bal);
        }
    __syncthreads();
    if (tid < 4) {
        int total = 0;
        for (int w = 0; w < N * WARPS; ++w) total += wcnt[tid][w];
        stotal[tid] = total;
        sbase[tid] = total ? atomicAdd(P.list_count + tid, (unsigned int)total) : 0u;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) {
        const int slot = k * WARPS + warp, c = cls[k];
        const uint32_t same = __match_any_sync(0xffffffffu, c);
        if (c >= 0) {
            int local = __popc(same & ((1u << lane) - 1));
            for (int w = 0; w < slot; ++w) local += wcnt[c][w];
            float4* buf = c >= 2 ? P.list_a : P.list_b;
            const size_t at = (c & 1) ? (size_t)sbase[c] + local : P.list_cap - (size_t)sbase[c] - stotal[c] + local;
            buf[at] = e[k];
        }
    }
}

// One CTA per block of rays_per_block = kListMaxSamples / S rays, CLS_PER_THREAD samples per thread, SAMPLE-major inside
// the block so that consecutive list entries are the same depth sample of neighbouring rays (they share their corner lines).
// 256-thread CTAs: eight of them are resident per SM, which hides the one atomicAdd round trip each block waits for.
constexpr int CLS_PER_THREAD = kListMaxSamples / CLS_THREADS;
__global__ void __launch_bounds__(CLS_THREADS) classify_compact_kernel(const __grid_constant__ RenderParams P, int rays_per_block) {
    __shared__ FrameXf xf;
    const int tid = threadIdx.x;
    const int S = P.n_samples, b = P.frame;
    const int r0 = blockIdx.x * rays_per_block;
    const int nr = min(rays_per_block, P.n_rays - r0);
    load_frame_xf(P, b, xf, tid);
    __syncthreads();
    // robustly negative sigma on all-zero features => such a sample has compositing weight exactly 0 and is not evaluated
    const bool can_skip = P.skip_empty && __ldg(P.wf32 + oSigmaEmpty) < -1e-3f;
    const uint32_t id0 = P.train_list ? (uint32_t)b * (uint32_t)P.n_rays * (uint32_t)S : 0u;   // training lists span the batch

    float4 gm[CLS_PER_THREAD];
    int cls[CLS_PER_THREAD];                          // 0..3 = finest occupied level (list class), -1 = not listed
    bool live[CLS_PER_THREAD];
#pragma unroll
    for (int k = 0; k < CLS_PER_THREAD; ++k) {
        const int j = k * CLS_THREADS + tid;
        const int ry = j % rays_per_block, s = j / rays_per_block;
        live[k] = ry < nr && s < S;
        cls[k] = -1;
        gm[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (live[k]) {
            const size_t ri = (size_t)b * P.n_rays + r0 + ry;
            const float ox = __ldg(P.ray_o + ri * 3), oy = __ldg(P.ray_o + ri * 3 + 1), oz = __ldg(P.ray_o + ri * 3 + 2);
            const float dx = __ldg(P.ray_d + ri * 3), dy = __ldg(P.ray_d + ri * 3 + 1), dz = __ldg(P.ray_d + ri * 3 + 2);
            const float z = z_sample(__ldg(P.near + ri), __ldg(P.far + ri), P.t_vals, s, S, P.t_rand ? P.t_rand + ri * S : nullptr, P.z_user ? P.z_user + ri * S : nullptr);
            gm[k].x = __fadd_rn(ox, __fmul_rn(dx, z));
            gm[k].y = __fadd_rn(oy, __fmul_rn(dy, z));
            gm[k].z = __fadd_rn(oz, __fmul_rn(dz, z));
            float gx, gy, gz;
            world_to_grid(xf, gm[k].x, gm[k].y, gm[k].z, gx, gy, gz);
            const bool inside = P.mask_nv == 0 || inside_masks(P, xf, gm[k].x, gm[k].y, gm[k].z);   // f-1 mask views
            const uint32_t lm = inside ? occupied_levels(P, b, gx, gy, gz) : 0u;
            if (inside && (lm != 0u || !can_skip)) cls[k] = (lm && !P.train_list) ? __ffs((int)lm) - 1 : 3;
            gm[k].w = __uint_as_float(((uint32_t)((r0 + ry) * S + s) + id0) | (lm << 28));
        }
    }
    append_to_lists(P, gm, cls);
    const float4 empty = make_float4(0.f, 0.f, 0.f, fminf(__ldg(P.wf32 + oSigmaEmpty), 0.f));   // skipped sample: weight exactly 0
#pragma unroll
    for (int k = 0; k < CLS_PER_THREAD; ++k)
        if (cls[k] < 0 && live[k]) P.raw_ws[(__float_as_uint(gm[k].w) & kListIdMask) - id0] = empty;
}

// ------------------------------------------------------------------------------------------------ 1'. classify points
// Density queries: one thread per world point of frame P.frame.  A point whose cells are unoccupied on all four levels has
// all-zero features, so its raw sigma is sigma_empty whatever the sign: with skip_empty it is written at once.  Every other
// point (all of them with skip_empty = 0) is appended to the list of its class as classify_compact_kernel does, in point
// order inside the block (neighbouring grid points share their corner voxels).  Entry: (world xyz, point id | level bits << 28).
__global__ void __launch_bounds__(CLS_THREADS) classify_points_kernel(const __grid_constant__ RenderParams P) {
    __shared__ FrameXf xf;
    const int tid = threadIdx.x;
    const int b = P.frame, n = P.n_points;
    const int i = blockIdx.x * CLS_THREADS + tid;
    load_frame_xf(P, b, xf, tid);
    __syncthreads();
    float4 e[1] = {make_float4(0.f, 0.f, 0.f, 0.f)};
    int cls[1] = {-1};                                // 0..3 = finest occupied level (list class), -1 = not listed
    if (i < n) {
        const float* q = P.points + (size_t)i * 3;
        e[0].x = __ldg(q); e[0].y = __ldg(q + 1); e[0].z = __ldg(q + 2);
        float gx, gy, gz;
        world_to_grid(xf, e[0].x, e[0].y, e[0].z, gx, gy, gz);
        const uint32_t lm = occupied_levels(P, b, gx, gy, gz);
        if (lm != 0u || !P.skip_empty) cls[0] = lm ? __ffs((int)lm) - 1 : 3;
        e[0].w = __uint_as_float((uint32_t)i | (lm << 28));
    }
    append_to_lists(P, e, cls);
    if (cls[0] < 0 && i < n) P.sigma[i] = __ldg(P.wf32 + oSigmaEmpty);
}

// ------------------------------------------------------------------------------------------------ 2. decoder over the list
// One persistent CTA per SM walks the frame's tiles of TP = 128 list rows.  The CTA is warp-specialised:
//   producer warpgroup (warps 0-3)   warp 0: one elected lane streams the weights with bulk copies into a 4-slot ring (one
//                                     K-step of both N halves and both planes per slot).  Warps 1-3: each tile's list rows,
//                                     their grid coordinates and voxel table (double-buffered, built one tile ahead) and
//                                     layer 3's per-point tile.
//   consumer warpgroups 1 and 2      rows [0, 64) and [64, 128) of a tile: gather layer 0's feature segments of their own rows,
//                                     issue the wgmma and run the epilogues.  Nothing divergent sits between a wgmma and the
//                                     wait that retires it (the gather runs only while none of the warpgroup's wgmma are in
//                                     flight; the other warpgroup's MMAs overlap it), and the K-step after a group is issued
//                                     before that group is waited for (wait_group 1), so the tensor pipe always holds the next
//                                     group.  A warpgroup's A operand is its own rows: a warpgroup-local named barrier (plus
//                                     fence.proxy.async) publishes what its epilogue or gather wrote.
//   activations   the ACT planes hold the current layer's A operand as fp16 (hi plane, and in the 3-pass mode the lo plane):
//                 during layer 0 a ring of four gathered 64-channel feature segments, then h0 / h1 / h2 (written by the
//                 epilogue straight from the accumulator registers), and in layer 3 the per-point tile in the lo plane.
//   accumulators  fp32 in registers (two m64n128 halves per warpgroup), started from the fp32 bias of the layer.
// Barriers (mbarrier phases; every wait is bounded by the watchdog):
//   full[s] / empty[s]   weight slot s: bulk-copy transaction bytes / one arrival per consumer warp
//   rows_full            the tile's list rows and voxel table are ready (every row thread)
//   rows_free            every consumer warp has begun the tile, so the other row buffer is free (one arrival per consumer warp)
//   l2_done, pe_full     the consumers' layer-2 MMAs are complete, so the lo plane is free (one arrival per consumer warp) /
//                        the per-point tile is written (every row thread)
constexpr int NT = 384;                                            // producer warpgroup + two consumer warpgroups
constexpr int NROWT = 96;                                          // the row threads: producer warps 1..3
// setmaxnreg moves registers within the CTA's launch allocation (NT x 168: __launch_bounds__(NT, 1) over the 64 K file); a
// consumer increase the pool cannot cover blocks for ever
constexpr int LAUNCH_REGS = (65536 / NT) / 8 * 8;
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
constexpr int CHUNK_STRIDE = TP * 16 + 16;                         // K-chunk stride (LBO) of an ACT plane: 16 bytes of padding
                                                                   // rotate successive chunks by 4 banks for the gather's stores
constexpr int ACT_CHUNKS = kHidden / 8;
constexpr int PLANE_BYTES = ACT_CHUNKS * CHUNK_STRIDE;             // 66048
constexpr int SEG_BUFS = 4;                                        // layer-0 segment ring inside the ACT planes
constexpr int SLOT_BYTES = 16384, NUM_SLOTS = 4;
constexpr int TILE256 = kHalfTile256 * 2;                          // one K-step, one N half (128 rows) of an N = 256 layer: 4 KB
constexpr int TILE3 = kHalfTile3 * 2;                              // one K-step, one N half (64 rows) of layer 3: 2 KB
constexpr int L3_PUSH = 4;                                         // layer-3 K-steps per push
constexpr int L3_PUSHES = (kStepsL3 + L3_PUSH - 1) / L3_PUSH;
constexpr int HEAD_FLOATS = kHidden + 4 + 3 * kColor + 4 + 3 * kHidden;   // alpha_fc, rgb_fc, then the biases of fc_0..fc_2, fp32
constexpr int H_ALPHA = 0, H_RGBW = kHidden + 4, H_RGBB = H_RGBW + 3 * kColor, H_B0 = H_RGBB + 4;
constexpr int OFF_HI = 0, OFF_LO = PLANE_BYTES;
constexpr int OFF_RING = 2 * PLANE_BYTES;
constexpr int OFF_HEAD = OFF_RING + NUM_SLOTS * SLOT_BYTES;
constexpr int OFF_XF = OFF_HEAD + HEAD_FLOATS * 4;
constexpr int OFF_SCHED = OFF_XF + 128;
constexpr int OFF_ROWS = OFF_SCHED + 64;                           // two tiles' list entries (float4 per row)
// Layer-0 voxel tables of the four levels, li = 3 - level (li 0, 1: the coarse levels 3 and 2, 128 channels each; li 2:
// level 1, 64 channels; li 3: level 0, 32 channels).  A 64-row half tile of neighbouring samples touches a few dozen (coarse)
// to about a hundred (fine) distinct voxels of a level but requests 512 corner vectors; the row warps list the distinct ones
// one tile ahead, and the consumer warpgroup copies each of them once into idle segment buffers of its own ACT-plane rows
// and blends from there.  The row warps also publish each row's grid coordinates, so the consumers do not redo world_to_grid
// (six divisions) in every segment.
constexpr int NV_COARSE = 64, NV_FINE = 128;                       // staged voxels per half tile and level (ACT room, fp32:
                                                                   // 64 x 512 B, 128 x 256 B = 2 segment buffers of both planes)
__host__ __device__ constexpr int level_nv(int li) { return li < 2 ? NV_COARSE : NV_FINE; }
__host__ __device__ constexpr int level_channels(int li) { return li < 2 ? 128 : li == 2 ? 64 : 32; }
// the distinct voxels of level li and half tile `half` start at ids[ids_at(li, half)]
__host__ __device__ constexpr int ids_at(int li, int half) {
    return li < 2 ? (2 * li + half) * NV_COARSE : 4 * NV_COARSE + (2 * (li - 2) + half) * NV_FINE;
}
constexpr int HBITS = 8, HSIZE = 1 << HBITS;                       // open-addressed hash per half tile, reused level by level
constexpr uint32_t HEMPTY = 0xFFFFFFFFu;
struct VoxTable {
    float4 grid[TP];                                               // per row: world_to_grid of the sample (x, y, z, -)
    unsigned char slot[TP][4][8];                                  // per row and level: the staged slot of each corner
    uint32_t ids[ids_at(4, 0)];                                    // the distinct voxels (linear index (z H + y) W + x)
    uint32_t n[8];                                                 // their number, [2 li + half]; > level_nv(li): direct
};
constexpr int OFF_VTAB = OFF_ROWS + 2 * TP * 16;                   // two tiles' tables (double-buffered like the rows)
constexpr int OFF_HKEY = OFF_VTAB + 2 * (int)sizeof(VoxTable);
constexpr int OFF_HVAL = OFF_HKEY + 2 * HSIZE * 4;
constexpr int OFF_HCNT = OFF_HVAL + 2 * HSIZE;
// hcnt: [0, 1] the voxels of the level being built per half tile, then the CTA's half-tile counts: [2] / [3] coarse levels
// staged / direct, [4] fine levels direct
constexpr int NCNT = 5;
constexpr int OFF_BAR = OFF_HCNT + 8 * 4;
enum { B_FULL = 0, B_EMPTY = B_FULL + NUM_SLOTS, B_ROWSFULL = B_EMPTY + NUM_SLOTS, B_L2DONE, B_PEFULL, B_ROWSFREE, NUM_BARS };
constexpr int SMEM_BYTES = OFF_BAR + NUM_BARS * 8;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");
static_assert(OFF_RING % 128 == 0 && OFF_HEAD % 16 == 0 && OFF_ROWS % 16 == 0 && OFF_VTAB % 16 == 0 && OFF_HKEY % 16 == 0 &&
              OFF_BAR % 8 == 0, "alignment");
// a level's staging fits two segment buffers of the warpgroup's rows in both planes; a slot fits a byte with 0xFF = none, and
// the hash never fills (at most NV_FINE + 1 + NROWT keys: an insert stops once the count is past the capacity)
static_assert(NV_COARSE * level_channels(0) * 4 <= 2 * 2 * 8 * 1024 && NV_FINE * level_channels(2) * 4 <= 2 * 2 * 8 * 1024 &&
              NV_FINE < 255 && HSIZE > NV_FINE + 1 + NROWT && NCNT <= 8, "voxel staging");
static_assert(128 * PRODUCER_REGS + 256 * CONSUMER_REGS <= NT * LAUNCH_REGS, "register pool of the CTA");

// weight pushes of a tile whose layer 0 runs l0_ksteps K-steps: one per K-step of layers 0..2, layer 3 in groups of L3_PUSH
__host__ __device__ constexpr int pushes_per_tile(int l0_ksteps) { return l0_ksteps + 2 * kKsL12 + L3_PUSHES; }

__device__ __forceinline__ uint32_t act_off(int row, int k) {      // byte offset of element (row, k) in an ACT plane
    return (uint32_t)((k >> 3) * CHUNK_STRIDE + (row >> 3) * 128 + (row & 7) * 16 + (k & 7) * 2);
}

// The trilinear cell of a sample on one level, as the gather addresses it: its 8 corners are (clamped low corner) + {0, 1}
// per axis.  A cell that straddles the volume boundary (index -1 or size-1 on an axis; zeros padding upstream) is shifted
// inside by one and its in-range voxel's weight moves to the slot that now addresses it; the out-of-range slot gets 0.
// Returns the low corner's voxel index (z H + y) W + x; cn holds the (moved) weights.  The row warps that list a tile's
// voxels and the consumers that blend them both call this, so the two cannot disagree.
__device__ __forceinline__ uint32_t clamped_cell(float gx, float gy, float gz, int W, int H, int D, Corners& cn) {
    corner_setup(unnormalize(gx, W), unnormalize(gy, H), unnormalize(gz, D), W, H, D, cn);
    auto axis = [](int i0, int size, float (&w)[2]) {
        if (i0 < 0) { w[0] = w[1]; w[1] = 0.f; return 0; }                        // i0 == -1: only voxel 0
        if (i0 >= size) { w[0] = w[1] = 0.f; return size - 2; }                   // both neighbours outside
        if (i0 == size - 1) { w[1] = w[0]; w[0] = 0.f; return size - 2; }         // only voxel size-1
        return i0;
    };
    const int xc = axis(cn.x0, W, cn.wx), yc = axis(cn.y0, H, cn.wy), zc = axis(cn.z0, D, cn.wz);
    return (uint32_t)((zc * H + yc) * W + xc);
}

// The decoder over the list: the body of render_tc_list_kernel and, with DENSITY, of density_tc_list_kernel.  DENSITY runs
// layers 0-2 and alpha_fc only: the weight stream stops after layer 2, the row warps write no per-point tile (l2_done and
// pe_full are not used), and the consumers store raw sigma to P.sigma[id] in place of the raw record.
template <int NP, typename VT, bool DENSITY>
__device__ __forceinline__ void decode_list(const RenderParams& P) {
    extern __shared__ __align__(1024) unsigned char smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
    FrameXf* xf = reinterpret_cast<FrameXf*>(smem + OFF_XF);
    float* head = reinterpret_cast<float*>(smem + OFF_HEAD);
    float4* rows_buf = reinterpret_cast<float4*>(smem + OFF_ROWS);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int wgid = warp >> 2;                                     // 0: producer, 1 / 2: consumers
    const int S = P.n_samples;
    const uint32_t s_hi0 = tc::smem_u32(smem + OFF_HI), s_lo0 = tc::smem_u32(smem + OFF_LO), s_ring = tc::smem_u32(smem + OFF_RING);

    if (tid == 0) {
        for (int i = 0; i < NUM_SLOTS; ++i) {
            tc::mbar_init(&bars[B_FULL + i], 1);
            tc::mbar_init(&bars[B_EMPTY + i], 8);
        }
        tc::mbar_init(&bars[B_ROWSFULL], NROWT);
        tc::mbar_init(&bars[B_L2DONE], 8);
        tc::mbar_init(&bars[B_PEFULL], NROWT);
        tc::mbar_init(&bars[B_ROWSFREE], 8);
        tc::fence_mbar_init();
    }
    load_frame_xf(P, P.frame, *xf, tid);
    for (int i = tid; i < HEAD_FLOATS; i += NT) {
        float v;
        if (i < H_RGBW) v = __ldg(P.wf32 + oAlphaW + i);                       // [alpha_w | alpha_b]
        else if (i < H_B0) v = __ldg(P.wf32 + oRgbW + (i - H_RGBW));            // [rgb_w | rgb_b]
        else {
            const int j = i - H_B0, l = j / kHidden, n = j % kHidden;
            v = __ldg(P.wf32 + (l == 0 ? oB0 : l == 1 ? oB1 : oB2) + n);
        }
        head[i] = v;
    }
    for (int i = tid; i < 2 * HSIZE; i += NT) reinterpret_cast<uint32_t*>(smem + OFF_HKEY)[i] = HEMPTY;
    if (tid < NCNT) reinterpret_cast<uint32_t*>(smem + OFF_HCNT)[tid] = 0u;
    struct Sched { unsigned int cnt[4]; int start[4]; int n_tiles; };
    Sched* sched = reinterpret_cast<Sched*>(smem + OFF_SCHED);
    if (tid == 0) {
        int acc = 0;
        for (int c = 0; c < 4; ++c) {
            const unsigned int n = P.list_count[c];                         // written by classify_compact_kernel (previous launch)
            sched->cnt[c] = n;
            sched->start[c] = acc;
            acc += (int)((n + TP - 1) / TP);
        }
        sched->n_tiles = acc;
        if (P.stats) atomicMax(P.frame_clock + 0, ~global_ns());            // min(start) over the CTAs, as max(~start)
    }
    __syncthreads();
    const int n_tiles = sched->n_tiles;
    struct TileRef { int cls, nrows; const float4* ent; };
    auto tile_ref = [&](int tile) {
        TileRef r;
        r.cls = tile >= sched->start[3] ? 3 : tile >= sched->start[2] ? 2 : tile >= sched->start[1] ? 1 : 0;
        const int lt = tile - sched->start[r.cls];
        const unsigned int cnt = sched->cnt[r.cls];
        const long long rem = (long long)cnt - (long long)lt * TP;
        r.nrows = rem <= 0 ? 0 : rem < TP ? (int)rem : TP;
        const float4* buf = r.cls >= 2 ? P.list_a : P.list_b;
        r.ent = buf + ((r.cls & 1) ? (size_t)0 : P.list_cap - (size_t)cnt) + (size_t)lt * TP;
        return r;
    };

    if (wgid == 0) {
        // =============================================================================================== producer warpgroup
        tc::setmaxnreg_dec<PRODUCER_REGS>();
        const uint32_t s_hi = s_hi0, s_lo = s_lo0;
        if (warp == 0) {
            // ---- warp 0: the weight stream (one elected lane).  Push j of a tile goes to slot g % NUM_SLOTS, g = pushes of the
            // CTA so far.  A slot is one K-step of both N halves and both planes (layers 0..2), or L3_PUSH K-steps of both
            // halves of layer 3.  A slot is refilled once every consumer warp has arrived on its empty barrier.
            if (lane == 0) {
                tcr::Tracer tl;
                tl.init(P.trace, 3);
                const unsigned char* seq = reinterpret_cast<const unsigned char*>(P.wf16);
                unsigned long long real_tiles = 0, real_ksteps = 0;
                uint32_t g = 0;
                for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                    const TileRef tref = tile_ref(tile);
                    const int l0_ksteps = class_ksteps(tref.cls);
                    real_tiles += tref.nrows > 0;
                    real_ksteps += tref.nrows > 0 ? l0_ksteps : 0;
                    const int npush = pushes_per_tile(l0_ksteps) - (DENSITY ? L3_PUSHES : 0);
                    for (int j = 0; j < npush; ++j, ++g) {
                        const uint32_t slot = g % NUM_SLOTS;
                        tc::mbar_wait(&bars[B_EMPTY + slot], ((g / NUM_SLOTS) & 1) ^ 1);   // (the first round passes at once)
                        if (j == 0) tl.ev(1);
                        unsigned char* dst = smem + OFF_RING + slot * SLOT_BYTES;
                        uint64_t* bar = &bars[B_FULL + slot];
                        if (j < l0_ksteps + 2 * kKsL12) {                   // layers 0..2: K-step ks, tile (half h, plane pl) at 2 h + pl
                            const int layer = j < l0_ksteps ? 0 : j < l0_ksteps + kKsL12 ? 1 : 2;
                            const int ks = layer == 0 ? j : layer == 1 ? j - l0_ksteps : j - l0_ksteps - kKsL12;
                            const int nks = layer == 0 ? kKsL0 : kKsL12;
                            const unsigned char* base = seq + 2 * (layer == 0 ? sL0 : layer == 1 ? sL1 : sL2);
                            tc::mbar_arrive_expect_tx(bar, (uint32_t)(2 * (NP == 3 ? 2 : 1) * TILE256));
#pragma unroll
                            for (int h = 0; h < 2; ++h)
#pragma unroll
                                for (int pl = 0; pl < (NP == 3 ? 2 : 1); ++pl)
                                    tc::bulk_g2s(dst + (2 * h + pl) * TILE256, base + 2 * pair_step_offset(ks, pl, h, nks), TILE256, bar);
                        } else {                                            // layer 3: steps [g0, g0 + n) of both N halves
                            const int g0 = (j - l0_ksteps - 2 * kKsL12) * L3_PUSH;
                            const int n = min(L3_PUSH, kStepsL3 - g0), common = min(n, kStepsL3 - 1 - g0);
                            const bool last = g0 + n == kStepsL3;
                            tc::mbar_arrive_expect_tx(bar, (uint32_t)(2 * n * TILE3));
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                unsigned char* d = dst + h * (SLOT_BYTES / 2);
                                tc::bulk_g2s(d, seq + 2 * (sL3 + pair_l3_offset(g0, h)), common * TILE3, bar);
                                if (last)                                   // the per-frame step 21 (it carries the frame's bias)
                                    tc::bulk_g2s(d + common * TILE3, reinterpret_cast<const unsigned char*>(P.wframe) + ((size_t)P.frame * 2 + h) * TILE3,
                                                 TILE3, bar);
                            }
                        }
                    }
                    tl.ev(2);
                }
                if (P.stats) {
                    atomicAdd(P.stats + 0, real_tiles);
                    atomicAdd(P.stats + 4, real_ksteps);
                    if (blockIdx.x == 0) atomicAdd(P.stats + 1, (unsigned long long)sched->cnt[0] + sched->cnt[1] + sched->cnt[2] + sched->cnt[3]);
                }
            }
            __syncwarp();
        } else {
            // ---- warps 1..3: the tiles' list rows and voxel tables (double-buffered) and the per-point tile of layer 3
            const int pt = tid - 32;                                    // 0 .. NROWT - 1
            VoxTable* vtabs = reinterpret_cast<VoxTable*>(smem + OFF_VTAB);
            uint32_t* hkey = reinterpret_cast<uint32_t*>(smem + OFF_HKEY);
            unsigned char* hval = smem + OFF_HVAL;
            uint32_t* hcnt = reinterpret_cast<uint32_t*>(smem + OFF_HCNT);
            tcr::Tracer tr;
            tr.init(pt == 0 ? P.trace : nullptr, 0);
            auto pwait = [&](uint64_t* bar, uint32_t parity) { tc::mbar_wait_backoff(bar, parity, 64); };
            // insert voxel `id` into half tile `half`'s hash: its hash position, or 0xFF once the level holds more than nv
            // voxels (the consumers then gather that level directly and never read the slots)
            auto insert = [&](int half, uint32_t id, uint32_t* ids, uint32_t nv) -> uint32_t {
                if (*reinterpret_cast<volatile uint32_t*>(hcnt + half) > nv) return 0xFFu;
                uint32_t* keys = hkey + half * HSIZE;
                uint32_t h = (id * 2654435761u) >> (32 - HBITS);
#pragma unroll 1
                for (int p = 0; p < HSIZE; ++p, h = (h + 1) & (HSIZE - 1)) {
                    uint32_t k = *reinterpret_cast<volatile uint32_t*>(keys + h);
                    if (k == HEMPTY) k = atomicCAS(keys + h, HEMPTY, id);
                    if (k == HEMPTY) {                                  // claimed: the voxel's slot is the next free one
                        const uint32_t s = atomicAdd(hcnt + half, 1u);
                        if (s < nv) ids[s] = id;
                        hval[half * HSIZE + h] = (unsigned char)min(s, 255u);
                        return h;
                    }
                    if (k == id) return h;
                }
                return 0xFFu;                                           // (the hash never fills, see the static_assert)
            };
            // The voxel table of a tile whose rows and grid coordinates are in `rows` / `vt`, level by level in one hash per
            // half tile: the level's distinct corner voxels per half tile and, per row, the slot of each of the 8 corners.
            // Insert (slot bytes = hash positions), then resolve them and clear the hash for the next level.
            auto build_table = [&](VoxTable* vt, const float4* rows, int nrows, int nlev) {
                auto occupied = [&](int row, int lvl) { return row < nrows && ((__float_as_uint(rows[row].w) >> (28 + lvl)) & 1u); };
#pragma unroll 1
                for (int li = 0; li < nlev; ++li) {
                    const int lvl = 3 - li, D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
                    const uint32_t nv = (uint32_t)level_nv(li);
#pragma unroll 1
                    for (int j = pt; j < TP * 8; j += NROWT) {              // corner j % 8 of row j / 8
                        const int row = j >> 3, c = j & 7;
                        uint32_t h = 0xFFu;
                        if (occupied(row, lvl)) {
                            const float4 gq = vt->grid[row];
                            Corners cn;
                            const uint32_t id = clamped_cell(gq.x, gq.y, gq.z, W, H, D, cn) + ((c & 1) ? 1u : 0u) +
                                                ((c & 2) ? (uint32_t)W : 0u) + ((c & 4) ? (uint32_t)(W * H) : 0u);
                            h = insert(row >> 6, id, vt->ids + ids_at(li, row >> 6), nv);
                        }
                        vt->slot[row][li][c] = (unsigned char)h;
                    }
                    tcr::named_bar_sync(3, NROWT);
#pragma unroll 1
                    for (int i = pt; i < TP * 2; i += NROWT) {              // corners 4 (i & 1) .. 4 (i & 1) + 3 of row i / 2
                        const int row = i >> 1;
                        uint32_t* wp = reinterpret_cast<uint32_t*>(&vt->slot[row][li][4 * (i & 1)]);
                        const unsigned char* hv = hval + (row >> 6) * HSIZE;
                        uint32_t out = 0xFFFFFFFFu;
                        if (occupied(row, lvl)) {
                            const uint32_t wd = *wp;
                            out = 0u;
#pragma unroll
                            for (int b = 0; b < 4; ++b) out |= (uint32_t)hv[(wd >> (8 * b)) & 0xFFu] << (8 * b);
                        }
                        *wp = out;
                    }
                    for (int i = pt; i < 2 * HSIZE; i += NROWT) hkey[i] = HEMPTY;   // (the keys are not read past the insert)
                    if (pt < 2) {
                        const uint32_t n = hcnt[pt];
                        vt->n[2 * li + pt] = n;
                        hcnt[pt] = 0u;
                        if (nrows > 64 * pt && (li < 2 || n > nv)) atomicAdd(hcnt + (li < 2 ? (n <= nv ? 2 : 3) : 4), 1u);
                    }
                    tcr::named_bar_sync(3, NROWT);
                }
            };
            // a tile's rows, their grid coordinates and its voxel table into buffer `buf`, published through rows_full
            auto load_rows = [&](int buf, int tile) {
                if (tile < n_tiles) {
                    const TileRef r = tile_ref(tile);
                    float4* dst = rows_buf + buf * TP;
                    VoxTable* vt = vtabs + buf;
                    for (int i = pt; i < TP; i += NROWT) {
                        const float4 e = i < r.nrows ? __ldg(r.ent + i) : make_float4(0.f, 0.f, 0.f, __uint_as_float(0xFFFFFFFFu));
                        dst[i] = e;
                        float gx, gy, gz;
                        world_to_grid(*xf, e.x, e.y, e.z, gx, gy, gz);
                        vt->grid[i] = make_float4(gx, gy, gz, 0.f);
                    }
                    tcr::named_bar_sync(3, NROWT);
                    build_table(vt, dst, r.nrows, 4 - r.cls);               // a class-c tile gathers levels 3 .. c
                }
                tcr::named_bar_sync(3, NROWT);
                tc::mbar_arrive(&bars[B_ROWSFULL]);
            };

            // Tile it: once every consumer warp has begun it (rows_free), the other row buffer's tile is finished; the next
            // tile's rows and voxel table are loaded there while this tile's layers 0-2 run, then comes this tile's per-point
            // tile.  load_rows has one call site: iteration it = -1 only loads the first tile.
            int it = -1;
            for (int tile = (int)blockIdx.x - (int)gridDim.x; tile < n_tiles; tile += gridDim.x, ++it) {
                if (it >= 0) {
                    pwait(&bars[B_ROWSFREE], it & 1);
                    tr.ev(1);
                }
                load_rows((it + 1) & 1, tile + gridDim.x);
                if (DENSITY || it < 0) continue;
                tr.ev(30);
                const TileRef tref = tile_ref(tile);
                const int nrows = tref.nrows;
                const float4* rows = rows_buf + (it & 1) * TP;
                // ---- the per-point tile of layer 3 in the lo plane: [PE(xyz) 63 | 0 | PE(view) 27 | 0 | 1 | 1 | 0 | 0]
                pwait(&bars[B_L2DONE], it & 1);                             // the lo plane's h1 is no longer read
                tr.ev(31);
#pragma unroll 1
                for (int job = pt; job < 2 * TP; job += NROWT) {
                    const int prow = job % TP;
                    const float4 e = rows[prow];
                    auto put = [&](int k, float v) {
                        const __half hv = __float2half_rn(v);
                        asm volatile("st.shared.b16 [%0], %1;" ::"r"(s_lo + act_off(prow, k)), "h"(*reinterpret_cast<const unsigned short*>(&hv)) : "memory");
                    };
                    if (job < TP) {
                        positional_embed_anchored<10, 5>(e.x, e.y, e.z, [&](int j, float v) { put(j, v); });
                        put(63, 0.f);
                    } else {
                        const int smp = (int)(__float_as_uint(e.w) & kListIdMask);
                        const size_t ri = (size_t)P.frame * P.n_rays + (prow < nrows ? smp / S : 0);
                        const float dx = __ldg(P.ray_d + ri * 3), dy = __ldg(P.ray_d + ri * 3 + 1), dz = __ldg(P.ray_d + ri * 3 + 2);
                        const float nrm = ray_norm(dx, dy, dz);
                        positional_embed_anchored<4, 4>(__fdiv_rn(dx, nrm), __fdiv_rn(dy, nrm), __fdiv_rn(dz, nrm), [&](int j, float v) { put(64 + j, v); });
                        put(91, 0.f); put(92, 1.f); put(93, 1.f); put(94, 0.f); put(95, 0.f);
                    }
                }
                tc::fence_proxy_async();
                tc::mbar_arrive(&bars[B_PEFULL]);
                tr.ev(32);
            }
        }
    } else {
        // =============================================================================================== consumer warpgroups
        tc::setmaxnreg_inc<CONSUMER_REGS>();
        uint32_t s_hi, s_lo;                                            // the ACT planes (set per tile, below)
        const int cw = wgid - 1;                                        // rows [64 cw, 64 cw + 64) of a tile
        const bool arr = lane == 0;                                     // the warp's arrival on the consumer-side barriers
        // trace events of the warpgroup (CTA 0, its first thread): only the entry index lives in a register, the buffer is
        // read from the kernel parameters at each event (same records as tcr::Tracer).  DENSITY records none: without them
        // its consumers stay spill-free
        int tn = (!DENSITY && (tid & 127) == 0 && blockIdx.x == 0 && P.trace) ? (1 + cw) * 4096 : -1;
        auto tval = [&](int code, unsigned long long v) {
            if (tn >= 0 && tn < (2 + cw) * 4096) P.trace[tn++] = ((unsigned long long)code << 48) | (v & 0xFFFFFFFFFFFFull);
        };
        auto tev = [&](int code) { tval(code, (unsigned long long)clock64()); };
        // this thread's accumulator fragment: rows r0 and r0 + 8 of the tile, columns 8 c + cq + {0, 1} of each 128-column half
        const int r0 = 64 * cw + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
        float acc0[64], acc1[64];                                      // N halves [0, 128) and [128, 256)
        auto init_bias = [&](const float* b) {
#pragma unroll
            for (int c = 0; c < 16; ++c) {
                const float2 v0 = *reinterpret_cast<const float2*>(b + 8 * c + cq), v1 = *reinterpret_cast<const float2*>(b + 128 + 8 * c + cq);
                acc0[4 * c] = v0.x; acc0[4 * c + 1] = v0.y; acc0[4 * c + 2] = v0.x; acc0[4 * c + 3] = v0.y;
                acc1[4 * c] = v1.x; acc1[4 * c + 1] = v1.y; acc1[4 * c + 2] = v1.x; acc1[4 * c + 3] = v1.y;
            }
        };
        const uint32_t wg_rows = (uint32_t)(cw * 8 * 128);              // this warpgroup's first 8-row group in an ACT plane
        // one K-step of a 256 -> 256 layer from the slot at `slot`: A K-step ka (ACT chunk 2 ka)
        auto mma256 = [&](uint32_t slot, int ka) {
            const uint64_t a_hi = tc::make_smem_desc(s_hi + wg_rows + 2 * ka * CHUNK_STRIDE, CHUNK_STRIDE, 128);
            const uint64_t a_lo = tc::make_smem_desc(s_lo + wg_rows + 2 * ka * CHUNK_STRIDE, CHUNK_STRIDE, 128);
            const uint64_t b0h = tc::make_smem_desc(slot + 0 * TILE256, 128 * 16, 128);
            const uint64_t b0l = tc::make_smem_desc(slot + 1 * TILE256, 128 * 16, 128);
            const uint64_t b1h = tc::make_smem_desc(slot + 2 * TILE256, 128 * 16, 128);
            const uint64_t b1l = tc::make_smem_desc(slot + 3 * TILE256, 128 * 16, 128);
            tc::wgmma_m64n128k16_f16(acc0, a_hi, b0h, true);
            tc::wgmma_m64n128k16_f16(acc1, a_hi, b1h, true);
            if (NP == 3) {                                              // A_lo W_hi + A_hi W_lo
                tc::wgmma_m64n128k16_f16(acc0, a_lo, b0h, true);
                tc::wgmma_m64n128k16_f16(acc1, a_lo, b1h, true);
                tc::wgmma_m64n128k16_f16(acc0, a_hi, b0l, true);
                tc::wgmma_m64n128k16_f16(acc1, a_hi, b1l, true);
            }
        };
        uint32_t g = 0;                                                 // pushes consumed by this CTA
        // cycles waited on weights / rows / the per-point tile; gathering the coarse (segments 0-3) and fine (4, 5) levels
        uint32_t w_stall = 0, r_stall = 0, pe_stall = 0, g_coarse = 0, g_fine = 0;
        // wait for push g, issue `mma(slot address)`, commit
        auto take = [&](auto&& mma) {
            const uint32_t s = g % NUM_SLOTS;
            const uint32_t t0 = (uint32_t)clock();
            tc::mbar_wait(&bars[B_FULL + s], (g / NUM_SLOTS) & 1);
            w_stall += (uint32_t)clock() - t0;
            tc::wgmma_fence();
            mma(s_ring + s * SLOT_BYTES);
            tc::wgmma_commit();
            ++g;
        };
        auto release = [&](uint32_t gp, bool pred) { tc::mbar_arrive_if(&bars[B_EMPTY + gp % NUM_SLOTS], pred); };
        auto release_last = [&]() { release(g - 1, arr); };

        // ---- epilogue of a 256-wide layer: relu -> fp16 (hi, lo) operand of the next layer in the ACT planes (own rows only).
        // h2 (`last`) is rounded to nearest, hi only: layer 3 is a 1-pass layer.  Returns this thread's share of alpha_fc . h2.
        auto convert = [&](bool last) {
            float sig0 = 0.f, sig1 = 0.f;
            auto one = [&](const float (&a)[64], int nh) {
#pragma unroll
                for (int c = 0; c < 16; ++c) {
                    const int col = 128 * nh + 8 * c + cq;
#pragma unroll
                    for (int hr = 0; hr < 2; ++hr) {
                        const float x0 = a[4 * c + 2 * hr], x1 = a[4 * c + 2 * hr + 1];
                        const uint32_t off = act_off(r0 + 8 * hr, col);
                        uint32_t hv;
                        if (last) {
                            const float2 aw = *reinterpret_cast<const float2*>(head + H_ALPHA + col);
                            float& sg = hr ? sig1 : sig0;
                            sg = fmaf(fmaxf(x0, 0.f), aw.x, sg);
                            sg = fmaf(fmaxf(x1, 0.f), aw.y, sg);
                            if (DENSITY) continue;                      // no layer 3 reads h2
                            hv = tc::cvt_relu_f16x2(x0, x1);
                        } else if (NP == 3) {
                            hv = tc::cvt_rz_relu_f16x2(x0, x1);
                            float q0, q1;
                            tc::trunc_residual2(x0, x1, q0, q1);
                            const uint32_t lv = tc::cvt_relu_f16x2(q0, q1);   // negative x: hi = 0 and the residual clamps to 0
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_lo + off), "r"(lv) : "memory");
                        } else {
                            hv = tc::cvt_relu_f16x2(x0, x1);
                        }
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(s_hi + off), "r"(hv) : "memory");
                    }
                }
            };
            one(acc0, 0);
            one(acc1, 1);
            return make_float2(sig0, sig1);
        };
        // the epilogue's stores become the warpgroup's next A operand
        auto publish = [&]() {
            tc::fence_proxy_async();
            tcr::named_bar_sync(1 + cw, 128);
        };

        int it = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
            const TileRef tref = tile_ref(tile);
            const int nrows = tref.nrows, nseg = class_segments(tref.cls);
            const float4* rows = rows_buf + (it & 1) * TP;
            // the plane bases are re-read per tile: otherwise ptxas hoists every K-step's descriptor out of the tile loop and
            // spills them
            asm volatile("mov.u32 %0, %1;" : "=r"(s_hi) : "r"(s_hi0));
            asm volatile("mov.u32 %0, %1;" : "=r"(s_lo) : "r"(s_lo0));
            tev(1);
            // ---- layer-0 gather of this warpgroup's rows: segment seg (64 channels of one level, coarse level first) -> segment
            // buffer seg % SEG_BUFS.  It runs while none of the warpgroup's wgmma are in flight; the other warpgroup's MMAs overlap it.
            // Every level is staged: at a level's first segment the warpgroup copies its half tile's distinct voxels (all of the
            // level's channels) with cp.async into idle segment buffers of its own rows (level 2: buffers 0, 1; levels 3, 1 and 0:
            // buffers 2, 3; the warpgroup's MMAs on them are retired, and no segment of the level writes there), and the level's
            // segments blend from there.  A half tile with more distinct voxels on a level than level_nv holds reads them from
            // global memory and redoes world_to_grid (the direct path).  The blend (weights, corner order, FMA order) is the same
            // on both paths, so the results are bit-identical.
            auto gather = [&](int seg) {
                const unsigned char* volbase = reinterpret_cast<const unsigned char*>(P.volume);
                const VoxTable* vt = reinterpret_cast<const VoxTable*>(smem + OFF_VTAB) + (it & 1);
                const int grp = (tid & 127) >> 3, t = tid & 7;
                const int lvl = seg < 2 ? 3 : seg < 4 ? 2 : seg < 5 ? 1 : 0;
                const int cbase0 = seg < 2 ? seg * 64 : seg < 4 ? (seg - 2) * 64 : 0;
                const int nunits = seg == NUM_SEGS - 1 ? 1 : 2;
                const int C = P.lvl_C[lvl], D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
                const int kb = 64 * (seg % SEG_BUFS);
                // staging: voxel v (VB = 2^lg_vb bytes, all channels of the level) at 1 KB piece v / VPP (the warpgroup's 64 rows of
                // one K chunk), pieces 0-15 in the hi plane and 16-31 in the lo plane, from chunk 0 (level 2) or 16 (the others) on
                const int li = seg < 4 ? seg >> 1 : seg - 2;
                const int lg_vb = (li < 2 ? 7 : li == 2 ? 6 : 5) + (sizeof(VT) == 4 ? 2 : 1), lg_vpp = 10 - lg_vb;
                const bool staged = C == level_channels(li) && vt->n[2 * li + cw] <= (uint32_t)level_nv(li);
                const uint32_t st_base = s_hi + (li == 1 ? 0 : 16) * CHUNK_STRIDE + cw * 1024;
                auto stage_addr = [&](uint32_t v) {
                    const uint32_t p = v >> lg_vpp;
                    return st_base + (p >> 4) * PLANE_BYTES + (p & 15) * CHUNK_STRIDE + ((v & ((1u << lg_vpp) - 1)) << lg_vb);
                };
                if (staged && (seg >= 4 || (seg & 1) == 0)) {                 // the level's first segment
                    const unsigned char* src = volbase + P.lvl_off[lvl] + (size_t)P.frame * P.lvl_bstride[lvl] * sizeof(VT);
                    const uint32_t* ids = vt->ids + ids_at(li, cw);
                    const int lg_ppv = lg_vb - 4;
                    const uint32_t nq = vt->n[2 * li + cw] << lg_ppv;
#pragma unroll 4
                    for (uint32_t i = tid & 127; i < nq; i += 128) {
                        const uint32_t v = i >> lg_ppv, q = i & ((1u << lg_ppv) - 1);
                        tc::cp_async_16(stage_addr(v) + 16 * q, src + ((size_t)ids[v] << lg_vb) + 16 * q);
                    }
                    tc::cp_async_wait_all();
                    tcr::named_bar_sync(1 + cw, 128);
                }
                // a row's trilinear set-up at grid coordinates (gx, gy, gz): the clamped cell's low corner and the 8 corner weights
                auto setup = [&](float gx, float gy, float gz, float (&cw)[8]) {
                    Corners cn;
                    const uint32_t cb = clamped_cell(gx, gy, gz, W, H, D, cn);
#pragma unroll
                    for (int c = 0; c < 8; ++c) cw[c] = __fmul_rn(__fmul_rn(cn.wx[c & 1], cn.wy[(c >> 1) & 1]), cn.wz[c >> 2]);
                    return cb;
                };
                // a row's blended units -> its fp16 operand(s) in the segment buffer
                auto store_row = [&](int row, const float (&acc)[2][4]) {
#pragma unroll
                    for (int uu = 0; uu < 2; ++uu) {
                        if (uu >= nunits) continue;
                        const float (&a)[4] = acc[uu];
                        const uint32_t off = act_off(row, kb + 32 * uu + 4 * t);
                        uint2 hw, lw;
                        if (NP == 3) {
                            // (hi, lo) split with a truncated hi: the residual is exact
                            hw.x = tc::cvt_rz_f16x2(a[0], a[1]); hw.y = tc::cvt_rz_f16x2(a[2], a[3]);
                            float q0, q1, q2, q3;
                            tc::trunc_residual2(a[0], a[1], q0, q1);
                            tc::trunc_residual2(a[2], a[3], q2, q3);
                            lw.x = tc::cvt_f16x2(q0, q1); lw.y = tc::cvt_f16x2(q2, q3);
                            tcr::sts_v2(s_lo + off, lw);
                        } else {
                            hw.x = tc::cvt_f16x2(a[0], a[1]); hw.y = tc::cvt_f16x2(a[2], a[3]);
                        }
                        tcr::sts_v2(s_hi + off, hw);
                    }
                };
                // The warpgroup's 64 rows, 4 per lane group.  Each unit accumulates its corners in order 0..7 and skips zero
                // weights on both paths.  The two paths get a loop each, so neither keeps the other's addressing state live
                // beside the accumulators.
                if (staged) {
                    // Two rows in flight: their set-up (from the grid coordinates the row warps published) and their corner
                    // loads are independent, so each hides the other's shared-memory latency.  An unoccupied row blends voxel 0
                    // with weight 0, which leaves its accumulators at 0.
                    const uint32_t st_off = (cbase0 + 4 * t) * sizeof(VT);       // this lane's channels inside a voxel
#pragma unroll 1
                    for (int row = 64 * cw + grp; row < 64 * cw + 64; row += 32) {
                        float acc[2][2][4] = {};
                        float cw8[2][8];
                        uint2 sl[2];
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            const int rw = row + 16 * r;
                            const bool occ = rw < nrows && ((__float_as_uint(rows[rw].w) >> (28 + lvl)) & 1u);
                            const float4 g = vt->grid[rw];
                            setup(g.x, g.y, g.z, cw8[r]);
                            sl[r] = *reinterpret_cast<const uint2*>(&vt->slot[rw][li][0]);
                            if (!occ) {
                                sl[r] = make_uint2(0u, 0u);
#pragma unroll
                                for (int c = 0; c < 8; ++c) cw8[r][c] = 0.f;
                            }
                        }
#pragma unroll
                        for (int c = 0; c < 8; ++c) {
                            typename Quad<VT>::raw v0[2], v1[2];
#pragma unroll
                            for (int r = 0; r < 2; ++r) {
                                const uint32_t a = stage_addr((((c < 4) ? sl[r].x : sl[r].y) >> (8 * (c & 3))) & 0xFFu) + st_off;
                                v0[r] = Quad<VT>::load_shared(a);
                                v1[r] = nunits > 1 ? Quad<VT>::load_shared(a + 32 * sizeof(VT)) : Quad<VT>::zero();
                            }
#pragma unroll
                            for (int r = 0; r < 2; ++r)
                                if (cw8[r][c] != 0.f) {
                                    Quad<VT>::fma(acc[r][0], v0[r], cw8[r][c]);
                                    Quad<VT>::fma(acc[r][1], v1[r], cw8[r][c]);
                                }
                        }
                        store_row(row, acc[0]);
                        store_row(row + 16, acc[1]);
                    }
                } else {
                    const unsigned char* lvl_ptr = volbase + P.lvl_off[lvl] + ((size_t)P.frame * P.lvl_bstride[lvl] + 4 * t) * sizeof(VT);
                    const uint32_t dX = (uint32_t)(C * sizeof(VT)), dY = dX * W, dZ = dY * H;
                    for (int row = 64 * cw + grp; row < 64 * cw + 64; row += 16) {
                        const float4 e = rows[row];
                        const bool occ = row < nrows && ((__float_as_uint(e.w) >> (28 + lvl)) & 1u);
                        float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
                        if (occ) {
                            float gx, gy, gz;
                            world_to_grid(*xf, e.x, e.y, e.z, gx, gy, gz);
                            float cw8[8];
                            const uint32_t cb = setup(gx, gy, gz, cw8) * dX;
#pragma unroll
                            for (int uu = 0; uu < 2; ++uu) {
                                if (uu >= nunits) continue;
                                const unsigned char* ub = lvl_ptr + (size_t)(cbase0 + 32 * uu) * sizeof(VT);
                                typename Quad<VT>::raw v[8];
#pragma unroll
                                for (int c = 0; c < 8; ++c)
                                    v[c] = Quad<VT>::load_bytes(ub + cb + ((c & 1) ? dX : 0u) + ((c & 2) ? dY : 0u) + ((c & 4) ? dZ : 0u));
#pragma unroll
                                for (int c = 0; c < 8; ++c)
                                    if (cw8[c] != 0.f) Quad<VT>::fma(acc[uu], v[c], cw8[c]);
                            }
                        }
                        store_row(row, acc);
                    }
                }
            };

            {
                const uint32_t t0 = (uint32_t)clock();
                tc::mbar_wait(&bars[B_ROWSFULL], it & 1);
                r_stall += (uint32_t)clock() - t0;
            }
            __syncwarp();                                               // (every lane is past the previous tile)
            tc::mbar_arrive_if(&bars[B_ROWSFREE], arr);                 // done with the previous tile's row buffer
            // ================= layer 0: gather a segment, multiply it (its K-steps pipelined), retire them, gather the next
            init_bias(head + H_B0);
            for (int seg = 0; seg < nseg; ++seg) {
                const uint32_t t0 = (uint32_t)clock();
                gather(seg);
                publish();
                (seg < 4 ? g_coarse : g_fine) += (uint32_t)clock() - t0;
                const int nks = seg == NUM_SEGS - 1 ? 2 : 4, ka = 4 * (seg % SEG_BUFS);
                for (int q = 0; q < nks; ++q) {
                    take([&](uint32_t slot) { mma256(slot, ka + q); });
                    tc::wgmma_wait<1>();
                    tc::acc_fence(acc0); tc::acc_fence(acc1);
                    release(g - 2, arr && q > 0);
                }
                tc::wgmma_wait<0>();
                tc::acc_fence(acc0); tc::acc_fence(acc1);
                release_last();
            }
            tev(20);
            convert(false);                                             // h0
            init_bias(head + H_B0 + kHidden);
            publish();
            // ================= layers 1, 2
            float2 sig = make_float2(0.f, 0.f);
            for (int layer = 1; layer <= 2; ++layer) {
                for (int q = 0; q < kKsL12; ++q) {
                    take([&](uint32_t slot) { mma256(slot, q); });
                    tc::wgmma_wait<1>();
                    tc::acc_fence(acc0); tc::acc_fence(acc1);
                    release(g - 2, arr && q > 0);
                }
                tc::wgmma_wait<0>();
                tc::acc_fence(acc0); tc::acc_fence(acc1);
                release_last();
                tev(20 + layer);
                if (layer == 1) {
                    convert(false);                                     // h1
                    init_bias(head + H_B0 + 2 * kHidden);
                } else {
                    if (!DENSITY) tc::mbar_arrive_if(&bars[B_L2DONE], arr);   // the lo plane is free for the per-point tile
                    sig = convert(true);                                // h2 (not stored by DENSITY), and this thread's share of sigma
                }
                publish();
            }
            if constexpr (DENSITY) {
                float sg[2] = {sig.x, sig.y};
#pragma unroll
                for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
                    for (int o = 1; o <= 2; o <<= 1) sg[hr] += __shfl_xor_sync(0xffffffffu, sg[hr], o);
                    const int row = r0 + 8 * hr;
                    if ((lane & 3) == 0 && row < nrows) {
                        const uint32_t id = __float_as_uint(rows[row].w) & kListIdMask;
                        P.sigma[id] = sg[hr] + head[H_ALPHA + kHidden];
                    }
                }
                continue;
            }
            // ================= layer 3 (the folded colour layer, N = 128 as two halves of 64): A = h2 (hi plane) for K-steps
            // 0..15, the per-point tile (lo plane) for 16..21
            float c3a[32], c3b[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) { c3a[i] = 0.f; c3b[i] = 0.f; }
#pragma unroll
            for (int p = 0; p < L3_PUSHES; ++p) {
                if (p * L3_PUSH == 16) {                              // the first push that reads the per-point tile
                    const uint32_t t0 = (uint32_t)clock();
                    tc::mbar_wait(&bars[B_PEFULL], it & 1);
                    pe_stall += (uint32_t)clock() - t0;
                }
                take([&](uint32_t slot) {
#pragma unroll
                    for (int k = 0; k < L3_PUSH; ++k) {
                        const int ks = p * L3_PUSH + k;
                        if (ks >= kStepsL3) break;
                        const uint32_t a = ks < 16 ? s_hi + 2 * ks * CHUNK_STRIDE : s_lo + 2 * (ks - 16) * CHUNK_STRIDE;
                        const uint64_t ad = tc::make_smem_desc(a + wg_rows, CHUNK_STRIDE, 128);
                        tc::wgmma_m64n64k16_f16(c3a, ad, tc::make_smem_desc(slot + k * TILE3, 64 * 16, 128), true);
                        tc::wgmma_m64n64k16_f16(c3b, ad, tc::make_smem_desc(slot + SLOT_BYTES / 2 + k * TILE3, 64 * 16, 128), true);
                    }
                });
                tc::wgmma_wait<1>();
                tc::acc_fence(c3a); tc::acc_fence(c3b);
                release(g - 2, arr && p > 0);
            }
            tc::wgmma_wait<0>();
            tc::acc_fence(c3a); tc::acc_fence(c3b);
            release_last();
            tev(23);
            // ---- the colour head: rgb = rgb_fc . relu(layer-3 accumulator) + bias, and sigma = alpha_fc . h2 + bias, fp32
            float cr[2] = {0.f, 0.f}, cg[2] = {0.f, 0.f}, cbl[2] = {0.f, 0.f};
            auto color = [&](const float (&a)[32], int nh) {
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int col = 64 * nh + 8 * c + cq;
                    const float2 w0 = *reinterpret_cast<const float2*>(head + H_RGBW + col);
                    const float2 w1 = *reinterpret_cast<const float2*>(head + H_RGBW + kColor + col);
                    const float2 w2 = *reinterpret_cast<const float2*>(head + H_RGBW + 2 * kColor + col);
#pragma unroll
                    for (int hr = 0; hr < 2; ++hr) {
                        const float x0 = fmaxf(a[4 * c + 2 * hr], 0.f), x1 = fmaxf(a[4 * c + 2 * hr + 1], 0.f);
                        cr[hr] = fmaf(x1, w0.y, fmaf(x0, w0.x, cr[hr]));
                        cg[hr] = fmaf(x1, w1.y, fmaf(x0, w1.x, cg[hr]));
                        cbl[hr] = fmaf(x1, w2.y, fmaf(x0, w2.x, cbl[hr]));
                    }
                }
            };
            color(c3a, 0);
            color(c3b, 1);
            float sg[2] = {sig.x, sig.y};
#pragma unroll
            for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    cr[hr] += __shfl_xor_sync(0xffffffffu, cr[hr], o);
                    cg[hr] += __shfl_xor_sync(0xffffffffu, cg[hr], o);
                    cbl[hr] += __shfl_xor_sync(0xffffffffu, cbl[hr], o);
                    sg[hr] += __shfl_xor_sync(0xffffffffu, sg[hr], o);
                }
                const int row = r0 + 8 * hr;
                if ((lane & 3) == 0 && row < nrows) {
                    const int smp = (int)(__float_as_uint(rows[row].w) & kListIdMask);
                    P.raw_ws[smp] = make_float4(cr[hr] + head[H_RGBB], cg[hr] + head[H_RGBB + 1], cbl[hr] + head[H_RGBB + 2],
                                                sg[hr] + head[H_ALPHA + kHidden]);
                }
            }
            tev(24);
            tval(50, w_stall);
            tval(51, r_stall);
            tval(52, pe_stall);
            tval(53, g_coarse);
            tval(54, g_fine);
            w_stall = r_stall = pe_stall = g_coarse = g_fine = 0;
        }
    }
    __syncthreads();
    if (tid == 0 && P.stats) {
        atomicMax(P.frame_clock + 1, global_ns());
        const uint32_t* paths = reinterpret_cast<const uint32_t*>(smem + OFF_HCNT) + 2;
        atomicAdd(P.stats + 5, (unsigned long long)paths[0]);             // coarse-level half tiles gathered from the staging
        atomicAdd(P.stats + 6, (unsigned long long)paths[1]);             // ... and directly (more than NV_COARSE distinct voxels)
        atomicAdd(P.stats + 7, (unsigned long long)paths[2]);             // fine-level half tiles gathered directly
    }
}

template <int NP, typename VT>
__global__ void __launch_bounds__(NT, 1) render_tc_list_kernel(const __grid_constant__ RenderParams P) {
    decode_list<NP, VT, false>(P);
}
template <int NP, typename VT>
__global__ void __launch_bounds__(NT, 1) density_tc_list_kernel(const __grid_constant__ RenderParams P) {
    decode_list<NP, VT, true>(P);
}

// stats[2] / [3]: the device-timed duration of the decoder launch that fed this frame, once the launch is complete
__device__ __forceinline__ void add_decoder_time(const RenderParams& P) {
    const unsigned long long t0 = ~P.frame_clock[0], t1 = P.frame_clock[1];
    atomicAdd(P.stats + 2, t1 > t0 ? t1 - t0 : 0ull);
    atomicAdd(P.stats + 3, 1ull);
}
__global__ void decoder_time_kernel(const __grid_constant__ RenderParams P) { add_decoder_time(P); }

// ------------------------------------------------------------------------------------------------ 3. raw2outputs
constexpr int COMP_WARPS = 8;
__global__ void __launch_bounds__(COMP_WARPS * 32) composite_kernel(const __grid_constant__ RenderParams P) {
    __shared__ float zs[COMP_WARPS][kListMaxSamples];   // rays of up to kListMaxSamples samples (the decoder does not care about S)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ray = blockIdx.x * COMP_WARPS + warp;
    if (blockIdx.x == 0 && threadIdx.x == 0 && P.stats) add_decoder_time(P);
    if (ray >= P.n_rays) return;
    const int S = P.n_samples;
    const size_t rg = (size_t)P.frame * P.n_rays + ray;
    const float near = __ldg(P.near + rg), far = __ldg(P.far + rg);
    for (int s = lane; s < S; s += 32) zs[warp][s] = z_sample(near, far, P.t_vals, s, S, P.t_rand ? P.t_rand + rg * S : nullptr, P.z_user ? P.z_user + rg * S : nullptr);
    __syncwarp();
    const float dx = __ldg(P.ray_d + rg * 3), dy = __ldg(P.ray_d + rg * 3 + 1), dz = __ldg(P.ray_d + rg * 3 + 2);
    float* wout = P.weights ? P.weights + rg * S : nullptr;
    RayOut o = composite_ray(P.raw_ws + (size_t)ray * S, zs[warp], S, ray_norm(dx, dy, dz), wout, lane);
    if (lane == 0) store_ray_outputs(P, rg, o);
}

template <int NP, typename VT, bool DENSITY>
static cudaError_t launch_list(const RenderParams& p, int grid, cudaStream_t stream) {
    void (*kernel)(RenderParams) = DENSITY ? density_tc_list_kernel<NP, VT> : render_tc_list_kernel<NP, VT>;
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return e;
    kernel<<<grid, NT, SMEM_BYTES, stream>>>(p);
    return cudaGetLastError();
}
template <bool DENSITY>
static cudaError_t launch_decoder(const RenderParams& p, int volume_dtype, int passes, int grid, cudaStream_t stream) {
    if (passes == 3) return volume_dtype == NB_DTYPE_F32 ? launch_list<3, float, DENSITY>(p, grid, stream) : launch_list<3, __half, DENSITY>(p, grid, stream);
    return volume_dtype == NB_DTYPE_F32 ? launch_list<1, float, DENSITY>(p, grid, stream) : launch_list<1, __half, DENSITY>(p, grid, stream);
}
// one persistent CTA per SM; the tile count of a frame is only known on the device, so the grid is sized for the worst case
// (every entry listed) and tiles past the end are no-ops
static int decoder_grid(size_t max_entries) {
    const int sms = sm_count();
    const long long max_tiles = ((long long)max_entries + TP - 1) / TP + 4;
    return (int)(max_tiles < sms ? max_tiles : sms);
}

constexpr size_t CTL_BYTES = 32;   // per frame: u32 list counts [4], u64 ~start, u64 end

// A batch's list workspace: one control block per frame, then the two list buffers of cap entries each, which the frames use
// in turn.  lists_bytes is its size; set_frame_lists points p at frame b's part and returns the end of the list buffers.
static size_t lists_bytes(int batch, size_t cap) { return align256((size_t)batch * CTL_BYTES) + 2 * align256(cap * sizeof(float4)); }
static unsigned char* set_frame_lists(RenderParams& p, void* workspace, int b, size_t cap) {
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    unsigned char* list = ws + align256((size_t)p.batch * CTL_BYTES);
    const size_t per_frame = align256(cap * sizeof(float4));
    p.frame = b;
    p.list_a = reinterpret_cast<float4*>(list);
    p.list_b = reinterpret_cast<float4*>(list + per_frame);
    p.list_cap = cap;
    p.list_count = reinterpret_cast<unsigned int*>(ws + (size_t)b * CTL_BYTES);
    p.frame_clock = reinterpret_cast<unsigned long long*>(ws + (size_t)b * CTL_BYTES + 16);
    return list + 2 * per_frame;
}

}  // namespace tcl

bool tc_available() { return true; }

size_t render_tc_list_workspace_bytes(int batch, int n_rays, int n_samples) {
    const size_t cap = (size_t)n_rays * n_samples;
    return tcl::lists_bytes(batch, cap) + align256(cap * sizeof(float4));   // + the raw records
}

// the two frame-level kernels the training path (nb_train.cu) shares with this pipeline
void launch_classify(const RenderParams& p, cudaStream_t stream) {
    const int rays_per_block = kListMaxSamples / p.n_samples;
    tcl::classify_compact_kernel<<<(p.n_rays + rays_per_block - 1) / rays_per_block, tcl::CLS_THREADS, 0, stream>>>(p, rays_per_block);
}
void launch_composite(const RenderParams& p, cudaStream_t stream) {
    tcl::composite_kernel<<<(p.n_rays + tcl::COMP_WARPS - 1) / tcl::COMP_WARPS, tcl::COMP_WARPS * 32, 0, stream>>>(p);
}

int launch_render_tc_list(const RenderParams& p_in, int volume_dtype, int passes, void* workspace, size_t workspace_bytes,
                          cudaStream_t stream) {
    RenderParams p = p_in;
    const int S = p.n_samples;
    if (S > kListMaxSamples || (size_t)p.n_rays * S > (size_t)kListIdMask) {
        set_error("the tensor-core render path supports n_samples <= %d and n_rays * n_samples < 2^28 per frame", kListMaxSamples);
        return NB_ERR_UNSUPPORTED;
    }
    if (!workspace || workspace_bytes < render_tc_list_workspace_bytes(p.batch, p.n_rays, S)) {
        set_error("nb_render_fwd: the tensor-core precisions need nb_render_args.workspace (%zu bytes given, %zu needed; see "
                  "nb_render_fwd_workspace_bytes)", workspace ? workspace_bytes : (size_t)0,
                  render_tc_list_workspace_bytes(p.batch, p.n_rays, S));
        return NB_ERR_BAD_ARG;
    }
    if (p.n_rays == 0) return NB_OK;
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)p.batch * tcl::CTL_BYTES, stream);
    if (e != cudaSuccess) { set_error("render_tc_list: memset failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    const int grid = tcl::decoder_grid((size_t)p.n_rays * S);
    for (int b = 0; b < p.batch; ++b) {
        float4* raw_ws = reinterpret_cast<float4*>(tcl::set_frame_lists(p, workspace, b, (size_t)p.n_rays * S));
        p.raw_ws = p_in.raw ? reinterpret_cast<float4*>(p_in.raw) + (size_t)b * p.n_rays * S : raw_ws;
        launch_classify(p, stream);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = tcl::launch_decoder<false>(p, volume_dtype, passes, grid, stream);
        if (e == cudaSuccess) {
            launch_composite(p, stream);
            e = cudaGetLastError();
        }
        if (e != cudaSuccess) { set_error("render_tc_list launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    }
    return NB_OK;
}

size_t density_tc_list_workspace_bytes(int batch, int n_points) {
    return tcl::lists_bytes(batch, (size_t)n_points);
}

// pts (B, n, 3) and sigma (B, n) of the whole batch
int launch_density_tc_list(const RenderParams& p_in, int volume_dtype, int passes, const float* pts, int n, float* sigma,
                           void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    RenderParams p = p_in;
    p.n_points = n;
    if ((size_t)n > (size_t)kListIdMask) {
        set_error("nb_decode_density_list: n_points = %d; the tensor-core list holds < 2^28 points per frame", n);
        return NB_ERR_UNSUPPORTED;
    }
    if (n == 0) return NB_OK;
    if (!workspace || workspace_bytes < density_tc_list_workspace_bytes(p.batch, n)) {
        set_error("nb_decode_density_list: needs nb_render_args.workspace (%zu bytes given, %zu needed; see "
                  "nb_decode_density_workspace_bytes)", workspace ? workspace_bytes : (size_t)0,
                  density_tc_list_workspace_bytes(p.batch, n));
        return NB_ERR_BAD_ARG;
    }
    cudaError_t e = cudaMemsetAsync(workspace, 0, (size_t)p.batch * tcl::CTL_BYTES, stream);
    if (e != cudaSuccess) { set_error("density_tc_list: memset failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    const int grid = tcl::decoder_grid((size_t)n);
    for (int b = 0; b < p.batch; ++b) {
        tcl::set_frame_lists(p, workspace, b, (size_t)n);
        p.points = pts + (size_t)b * n * 3;
        p.sigma = sigma + (size_t)b * n;
        tcl::classify_points_kernel<<<(n + tcl::CLS_THREADS - 1) / tcl::CLS_THREADS, tcl::CLS_THREADS, 0, stream>>>(p);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = tcl::launch_decoder<true>(p, volume_dtype, passes, grid, stream);
        if (e == cudaSuccess && p.stats) {
            tcl::decoder_time_kernel<<<1, 1, 0, stream>>>(p);
            e = cudaGetLastError();
        }
        if (e != cudaSuccess) { set_error("density_tc_list launch failed: %s", cudaGetErrorString(e)); return NB_ERR_CUDA; }
    }
    return NB_OK;
}

}  // namespace nb
