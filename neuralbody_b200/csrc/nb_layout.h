// Layout of the packed decoder-weight blob shared by nb_pack.cu and the render kernels.
//
// Decoder as written upstream (lib/networks/latent_xyzc.py:99-121):
//   h0 = relu(fc_0 f)   h1 = relu(fc_1 h0)   h2 = relu(fc_2 h1)   sigma = alpha_fc h2
//   u  = feature_fc h2 ; v = latent_fc [u (+) latent] ; w = relu(view_fc [v (+) PE(view) (+) PE(xyz)])
//   rgb = rgb_fc w
// There is no activation between feature_fc, latent_fc and view_fc[:, :256], so they fold
// exactly (SURVEY.md 8a) into one 128x256 matrix Wc and a per-frame bias bc:
//   w = relu(Wc h2 + Wx PE(xyz) + Wv PE(view) + bc)
#pragma once
#include <stddef.h>

namespace nb {

constexpr int kFeat = 352;      // 32 + 64 + 128 + 128
constexpr int kHidden = 256;
constexpr int kColor = 128;
constexpr int kXyzPE = 63;
constexpr int kViewPE = 27;
constexpr int kColorK = 320;    // 256 (h2) + 63 (PE xyz) + 1 zero pad

// ---- per-point activation record the exact kernel saves for the backward pass (floats)
constexpr int kSaveF = 0;                       // gathered features          [352]
constexpr int kSaveH0 = kSaveF + kFeat;         // relu(fc_0)                  [256]
constexpr int kSaveH1 = kSaveH0 + kHidden;      // relu(fc_1)                  [256]
constexpr int kSaveH2 = kSaveH1 + kHidden;      // relu(fc_2) | PE(xyz) 63 | 0 [320]  (input of the folded colour layer)
constexpr int kSaveW = kSaveH2 + kColorK;       // relu(colour hidden)         [128]
constexpr int kSaveDim = kSaveW + kColor;       // 1312
// backward scratch per point (floats): [d_raw 4 | d_wpre 128 | d_h2pre 256 | d_h1pre 256 | d_h0pre 256]
constexpr int kGradRaw = 0, kGradW = 4, kGradH2 = kGradW + kColor, kGradH1 = kGradH2 + kHidden,
              kGradH0 = kGradH1 + kHidden, kGradDim = kGradH0 + kHidden;   // 900

// ---- fp32 section (float offsets). "t" = transposed / K-major: Wt[k][n] = W[n][k]
constexpr size_t oW0t = 0;                                  // [352][256]
constexpr size_t oB0 = oW0t + (size_t)kFeat * kHidden;      // [256]
constexpr size_t oW1t = oB0 + kHidden;                      // [256][256]
constexpr size_t oB1 = oW1t + (size_t)kHidden * kHidden;
constexpr size_t oW2t = oB1 + kHidden;                      // [256][256]
constexpr size_t oB2 = oW2t + (size_t)kHidden * kHidden;
constexpr size_t oAlphaW = oB2 + kHidden;                   // [256]
constexpr size_t oAlphaB = oAlphaW + kHidden;               // [1] (+3 pad)
constexpr size_t oWct = oAlphaB + 4;                        // [320][128]: rows 0..255 Wc^T, 256..318 Wx^T, 319 zero
constexpr size_t oWvt = oWct + (size_t)kColorK * kColor;    // [27][128]  Wv^T (+ pad to 28 rows)
constexpr size_t oRgbW = oWvt + (size_t)28 * kColor;        // [3][128]
constexpr size_t oRgbB = oRgbW + 3 * kColor;                // [3] (+1 pad)
constexpr size_t oWc = oRgbB + 4;                           // [128][256] folded Wc, row-major (backward dgrad)
constexpr size_t oSigmaEmpty = oWc + (size_t)kColor * kHidden;   // [1] (+3 pad): sigma of an all-zero feature vector
constexpr size_t kF32Floats = oSigmaEmpty + 4;

// row of the latent table frame b uses: latent_index[b] clamped into [0, num_train_frame)
__host__ __device__ inline long long clamp_latent(long long li, int num_train_frame) {
    return li < 0 ? 0 : li >= num_train_frame ? num_train_frame - 1 : li;
}

// ---- fp16 section: the tensor-core kernel's weight STREAM, in consumption order.
// One "step" = the B operand of one K=16 MMA: an N x 16 tile in the canonical K-major
// no-swizzle layout: element (n, kk) at half-offset ((kk/8) * (N/8) + n/8) * 64 + (n%8) * 8 + (kk%8),
// i.e. 8x8 core matrices (8 rows x 16 B = 128 B contiguous); stride-byte-offset (next 8 rows) = 128 B,
// leading-byte-offset (next 8-wide K chunk) = N*16 B.
// Steps are stored in GROUPS of up to 4 consecutive K-steps (one bulk copy / one ring slot / one mbarrier
// hand-off per group: the single MMA-issuing thread pays ~300 cycles of wait+commit latency per hand-off).
// Layers 0-2 (the density path) carry every weight as hi = fp16(w) and lo = fp16(w - hi): group g is stored as
// [hi steps of g][lo steps of g]; the 3-pass mode (A_hi W_hi + A_lo W_hi + A_hi W_lo) is ~fp32-accurate, the
// 1-pass mode skips the lo halves.
//   L0  : 22 K-steps of fc_0 (N=256) in groups 4,4,4,4,4,2 (= the gather's 64-channel segments), then 1 bias
//         step (A column of ones x [hi(b), lo(b)])
//   L1,2: 16 K-steps in 4 groups, then 1 bias step
//   L3  : N=144 = 128 colour rows (Wc, fp16) + rows 128/129 = hi/lo(alpha_fc) + 14 zero rows;
//         16 steps over h2, then 6 steps over the per-point tile
//         [PE(xyz) 63 | 0 | PE(view) 27 | 0 | 1 | 1 | 0 | 0]  (weights Wx | 0 | Wv | 0 | hi(bc) | lo(bc));
//         the last step carries the per-frame bias bc => stored once per frame, outside the common stream
//   L4  : N=16: rows 0-2 hi(rgb_fc), rows 3-5 lo(rgb_fc); 8 steps + 1 bias step (one group)
constexpr size_t kF16ByteOffset = ((kF32Floats * 4 + 255) / 256) * 256;
constexpr int kKsL0 = 22, kKsL12 = 16;                     // K-steps of layers 0 and 1/2 (without the bias step)
constexpr int kStepsL3 = 22, kStepsL4 = 9;
constexpr int kN3 = 128, kN4 = 16;                        // (kN4: the former tensor-core rgb head; its slot in the blob is unused)
constexpr int kPeK = 96;                                   // per-point tile width of L3
constexpr size_t kStepHalves256 = 256 * 16, kStepHalves3 = kN3 * 16, kStepHalves4 = kN4 * 16;
constexpr size_t sL0 = 0;
constexpr size_t sL1 = sL0 + (2 * kKsL0 + 1) * kStepHalves256;
constexpr size_t sL2 = sL1 + (2 * kKsL12 + 1) * kStepHalves256;
constexpr size_t sL3 = sL2 + (2 * kKsL12 + 1) * kStepHalves256;
constexpr size_t sL4 = sL3 + kStepsL3 * kStepHalves3;      // (the common copy of L3's last step is unused)
constexpr size_t kF16Halves = sL4 + kStepsL4 * kStepHalves4;

// Layer-0 K order of the tensor-core kernel: COARSE LEVEL FIRST -- [level 3: 128 | level 2: 128 | level 1: 64 | level 0: 32]
// (upstream's feature order, latent_xyzc.py:66-71, is level 0 first).  A tile whose rows have no occupied cell in the fine
// levels then simply stops after the leading K segments: 2 / 4 / 5 / 6 segments of 64 channels for a finest occupied level of
// 3 / 2 / 1 / 0.  Maps a K index of that order to the channel of fc_0's 352-wide input.
__host__ __device__ inline int feat_tc_to_orig(int j) {
    return j < 128 ? 224 + j : j < 256 ? 96 + (j - 128) : j < 320 ? 32 + (j - 256) : j - 320;
}
// layer-0 segments / K-steps a tile of sample class c (= finest occupied level) runs
__host__ __device__ inline int class_segments(int c) { return c == 0 ? 6 : c == 1 ? 5 : c == 2 ? 4 : 2; }
__host__ __device__ inline int class_ksteps(int c) { return c == 0 ? 22 : c == 1 ? 20 : c == 2 ? 16 : 8; }

// The tensor-core decoder multiplies every layer as two N halves (one wgmma per half and K-step), so a step of an N-wide
// layer is stored as two (N/2) x 16 tiles (same canonical K-major layout, N/2 rows), arranged so that the tiles of one half
// and plane are contiguous runs:
//   N = 256 layers: group g of gs K-steps = [half 0: gs hi tiles, gs lo tiles][half 1: gs hi tiles, gs lo tiles]  (4 KB tiles);
//                   bias step = [half 0 tile][half 1 tile]
//   L3 (N = 128)  : the folded colour layer: [half 0: steps 0..20][half 1: steps 0..20] (64 x 16 tiles); the per-frame step 21
//                   is [B][half][tile].  alpha_fc (1 x 256) and rgb_fc (3 x 128) are NOT in the stream: the epilogue applies them
//                   in fp32 to the accumulators it converts anyway (a 1- or 3-wide layer would cost the tensor pipe a full
//                   instruction per K-step for a few hundred FMAs per row).
constexpr int kHalfTile256 = 128 * 16;                     // halves in one (N/2 = 128) x 16 tile
constexpr int kHalfTile3 = (kN3 / 2) * 16;                 // 64 x 16
constexpr int kHalfTile4 = (kN4 / 2) * 16;                 // 8 x 16
// half-offset (from the layer base) of the first tile CTA `half` loads for the group starting at K-step g0
__host__ __device__ inline size_t pair_group_offset(int g0, int half, int nks) {
    const int g = g0 >> 2;
    const int gs = (nks - 4 * g) < 4 ? (nks - 4 * g) : 4;
    return (size_t)8 * g * kStepHalves256 + (size_t)half * 2 * gs * kHalfTile256;
}
// half-offset of K-step ks, hi / lo plane, of CTA `half`
__host__ __device__ inline size_t pair_step_offset(int ks, int lo, int half, int nks) {
    const int g = ks >> 2;
    const int gs = (nks - 4 * g) < 4 ? (nks - 4 * g) : 4;
    return pair_group_offset(4 * g, half, nks) + (size_t)((lo ? gs : 0) + (ks & 3)) * kHalfTile256;
}
__host__ __device__ inline size_t pair_bias_offset(int half, int nks) { return (size_t)2 * nks * kStepHalves256 + (size_t)half * kHalfTile256; }
__host__ __device__ inline size_t pair_l3_offset(int step, int half) { return (size_t)half * (kStepsL3 - 1) * kHalfTile3 + (size_t)step * kHalfTile3; }
__host__ __device__ inline size_t pair_l4_offset(int step, int half) { return (size_t)half * kStepsL4 * kHalfTile4 + (size_t)step * kHalfTile4; }

// N=256 layers: half-offset (from the layer base) of K-step ks, hi or lo plane, with nks K-steps in the layer (single-CTA order)
__host__ __device__ inline size_t step256_offset(int ks, int lo, int nks) {
    const int g = ks >> 2;
    const int gsteps = (nks - 4 * g) < 4 ? (nks - 4 * g) : 4;
    return ((size_t)8 * g + (lo ? gsteps : 0) + (ks & 3)) * kStepHalves256;
}
__host__ __device__ inline size_t bias256_offset(int nks) { return (size_t)2 * nks * kStepHalves256; }

// ---- scratch for the fp64 fold (doubles), then per-frame data
constexpr size_t kScratchByteOffset = ((kF16ByteOffset + kF16Halves * 2 + 255) / 256) * 256;
constexpr size_t kScratchDoubles = (size_t)kColor * kHidden;   // T = view_fc[:, :256] * latent_fc[:, :256]
constexpr size_t kBcByteOffset = kScratchByteOffset + kScratchDoubles * 8;
// after bc[B][128] floats: u[B][256] doubles (fold scratch), then the per-frame L3 step [B][144*16] halves

__host__ __device__ inline size_t u_byte_offset(int batch) {
    size_t b = kBcByteOffset + (size_t)batch * kColor * 4;
    return (b + 255) / 256 * 256;
}
__host__ __device__ inline size_t frame_step_byte_offset(int batch) {
    size_t b = u_byte_offset(batch) + (size_t)batch * kHidden * 8;
    return (b + 255) / 256 * 256;
}
__host__ __device__ inline size_t packed_weights_bytes(int batch) {
    return frame_step_byte_offset(batch) + (size_t)batch * kStepHalves3 * 2;
}

// element (n, kk) of an N x 16 step tile
__host__ __device__ inline size_t step_offset(int n, int kk, int N) {
    return ((size_t)(kk >> 3) * (N >> 3) + (n >> 3)) * 64 + (size_t)(n & 7) * 8 + (kk & 7);
}

__host__ __device__ inline size_t umma_kmajor_offset(int n, int k, int N) {
    return ((size_t)(k >> 3) * (N >> 3) + (n >> 3)) * 64 + (size_t)(n & 7) * 8 + (k & 7);
}

}  // namespace nb
