// Device helpers shared by the exact-fp32, the tensor-core and the training kernels:
// sample generation, the ray norm, world->SMPL->grid transform, trilinear corner set-up and gather,
// positional encoding, the alpha-compositing warp scan and the per-ray map stores.
//
// Parity-critical arithmetic follows the reference's op sequence in fp32 with
// explicit round-to-nearest intrinsics (no FMA contraction) where upstream issues
// separate PyTorch ops, so z_vals / grid coordinates agree to the last bit or ulp.
#pragma once
#include "nb_internal.h"

namespace nb {

// ---------------------------------------------------------------- a2: get_sampling_points
// lib/networks/renderer/if_clight_renderer.py:13-14.  torch.linspace's CPU/CUDA kernels
// fill symmetrically: start + step*i below the midpoint, end - step*(steps-1-i) above.
__device__ __forceinline__ float linspace01(int i, int steps) {
    if (steps == 1) return 0.f;
    float step = __fdiv_rn(1.f, (float)(steps - 1));
    return (i < steps / 2) ? __fmul_rn(step, (float)i) : __fsub_rn(1.f, __fmul_rn(step, (float)(steps - 1 - i)));
}

__device__ __forceinline__ float z_plain(float near, float far, float t) {
    // near[..., None] * (1. - t_vals) + far[..., None] * t_vals
    return __fadd_rn(__fmul_rn(near, __fsub_rn(1.f, t)), __fmul_rn(far, t));
}

// z value of sample s, including the stratified jitter of if_clight_renderer.py:16-23
// when t_rand != nullptr (t_rand points at this ray's S uniforms).
// z_user != nullptr (this ray's S caller-supplied depths, nb_render_args.z_vals): used as they are -- the fine pass of
// hierarchical sampling renders sorted(coarse z + importance samples), which no (near, far, t) formula produces.
__device__ __forceinline__ float z_sample(float near, float far, const float* __restrict__ t_vals, int s, int S,
                                          const float* __restrict__ t_rand, const float* __restrict__ z_user = nullptr) {
    if (z_user) return __ldg(z_user + s);
    float tc = t_vals ? __ldg(t_vals + s) : linspace01(s, S);
    float z = z_plain(near, far, tc);
    if (t_rand) {
        float lower = z, upper = z;
        if (s > 0) {
            float tp = t_vals ? __ldg(t_vals + s - 1) : linspace01(s - 1, S);
            lower = __fmul_rn(.5f, __fadd_rn(z, z_plain(near, far, tp)));
        }
        if (s < S - 1) {
            float tn = t_vals ? __ldg(t_vals + s + 1) : linspace01(s + 1, S);
            upper = __fmul_rn(.5f, __fadd_rn(z_plain(near, far, tn), z));
        }
        z = __fadd_rn(lower, __fmul_rn(__fsub_rn(upper, lower), __ldg(t_rand + s)));
    }
    return z;
}

// d z / d near and d z / d far of sample s as z_sample derives it (no z_user): (1 - t_s, t_s) without jitter; with jitter the
// combination lower (1 - r) + upper r makes of the mids .5 (z_{s-1} + z_s) / .5 (z_s + z_{s+1}), or of z_s at either end
__device__ __forceinline__ void z_sample_coefs(const float* __restrict__ t_vals, int s, int S, const float* __restrict__ t_rand,
                                               float& cn, float& cf) {
    auto tv = [&](int i) { return t_vals ? __ldg(t_vals + i) : linspace01(i, S); };
    const float t = tv(s);
    if (!t_rand) { cn = 1.f - t; cf = t; return; }
    const float tl = s > 0 ? .5f * (tv(s - 1) + t) : t, tu = s < S - 1 ? .5f * (t + tv(s + 1)) : t;
    const float r = __ldg(t_rand + s);
    cf = (1.f - r) * tl + r * tu;
    cn = (1.f - r) * (1.f - tl) + r * (1.f - tu);
}

// torch.norm(ray_d, dim=-1): sqrt(x^2 + y^2 + z^2), summed left to right without contraction
__device__ __forceinline__ float ray_norm(float x, float y, float z) {
    return sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));
}

// Per-frame constants of the world -> grid transform, staged once per CTA work item.
struct FrameXf {
    float R[9];        // sp_input['R'][b]   row-major
    float Th[3];       // sp_input['Th'][b]
    float min_dhw[3];  // bounds[b,0,[2,1,0]]
    float voxel[3];    // cfg.voxel_size (dhw)
    float out_sh[3];   // dhw
};

// Element i of each FrameXf array of frame b: threads 0..8 of a CTA fill a shared FrameXf with i = tid; a thread that needs
// its own copy calls it for i = 0..8.
__device__ __forceinline__ void load_frame_xf(const RenderParams& P, int b, FrameXf& xf, int i) {
    if (i < 9) xf.R[i] = __ldg(P.R + b * 9 + i);
    if (i < 3) {
        xf.Th[i] = __ldg(P.Th + b * 3 + i);
        xf.min_dhw[i] = __ldg(P.bounds + b * 6 + (2 - i));
        xf.voxel[i] = P.voxel_size[i];
        xf.out_sh[i] = P.out_sh[i];
    }
}

// a5 + a6: latent_xyzc.py:41-60.  Input world point, output grid coords (x,y,z) in [-1,1].
__device__ __forceinline__ void world_to_grid(const FrameXf& f, float wx, float wy, float wz, float& gx, float& gy,
                                              float& gz) {
    float px = __fsub_rn(wx, f.Th[0]), py = __fsub_rn(wy, f.Th[1]), pz = __fsub_rn(wz, f.Th[2]);
    // torch.matmul(pts, R): c_j = sum_i p_i R[i][j]
    float cx = fmaf(pz, f.R[6], fmaf(py, f.R[3], __fmul_rn(px, f.R[0])));
    float cy = fmaf(pz, f.R[7], fmaf(py, f.R[4], __fmul_rn(px, f.R[1])));
    float cz = fmaf(pz, f.R[8], fmaf(py, f.R[5], __fmul_rn(px, f.R[2])));
    float d = __fdiv_rn(__fsub_rn(cz, f.min_dhw[0]), f.voxel[0]);
    float h = __fdiv_rn(__fsub_rn(cy, f.min_dhw[1]), f.voxel[1]);
    float w = __fdiv_rn(__fsub_rn(cx, f.min_dhw[2]), f.voxel[2]);
    d = __fsub_rn(__fmul_rn(__fdiv_rn(d, f.out_sh[0]), 2.f), 1.f);
    h = __fsub_rn(__fmul_rn(__fdiv_rn(h, f.out_sh[1]), 2.f), 1.f);
    w = __fsub_rn(__fmul_rn(__fdiv_rn(w, f.out_sh[2]), 2.f), 1.f);
    gx = w; gy = h; gz = d;   // grid_coords = dhw[..., [2,1,0]]
}

// F.grid_sample(align_corners=True) un-normalisation: ((g + 1) / 2) * (size - 1)
__device__ __forceinline__ float unnormalize(float g, int size) {
    return __fmul_rn(__fmul_rn(__fadd_rn(g, 1.f), 0.5f), (float)(size - 1));   // x / 2 == x * 0.5 bit for bit
}

// Trilinear corner set-up for one level (ATen grid_sampler_3d, zeros padding).
struct Corners {
    int x0, y0, z0;        // floor indices (may be -1 or size-1 => partly out of range); -2 = all out
    float wx[2], wy[2], wz[2];
};
__device__ __forceinline__ void corner_setup(float ix, float iy, float iz, int W, int H, int D, Corners& c) {
    float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
    bool ok = (fx >= -1.f) && (fx <= (float)W) && (fy >= -1.f) && (fy <= (float)H) && (fz >= -1.f) && (fz <= (float)D);
    // (NaN coordinates fail the comparisons => all corners skipped => zeros, as ATen's bounds test does)
    c.x0 = ok ? (int)fx : -2; c.y0 = ok ? (int)fy : -2; c.z0 = ok ? (int)fz : -2;
    c.wx[0] = __fsub_rn(__fadd_rn(fx, 1.f), ix); c.wx[1] = __fsub_rn(ix, fx);
    c.wy[0] = __fsub_rn(__fadd_rn(fy, 1.f), iy); c.wy[1] = __fsub_rn(iy, fy);
    c.wz[0] = __fsub_rn(__fadd_rn(fz, 1.f), iz); c.wz[1] = __fsub_rn(iz, fz);
}
// f(voxel index, dx, dy, dz) for the corners (x0 + dx, y0 + dy, z0 + dz) of the cell that lie inside the W x H x D volume,
// in ATen's accumulation order: tnw, tne, tsw, tse, bnw, bne, bsw, bse (x fastest)
template <typename F>
__device__ __forceinline__ void for_each_corner_at(const Corners& c, int W, int H, int D, F&& f) {
#pragma unroll
    for (int dz = 0; dz < 2; ++dz)
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int x = c.x0 + dx, y = c.y0 + dy, z = c.z0 + dz;
                if ((c.x0 != -2) && x >= 0 && x < W && y >= 0 && y < H && z >= 0 && z < D)
                    f(((size_t)z * H + y) * W + x, dx, dy, dz);
            }
}
// f(voxel index, weight) for the same corners in the same order
template <typename F>
__device__ __forceinline__ void for_each_corner(const Corners& c, int W, int H, int D, F&& f) {
    for_each_corner_at(c, W, H, D, [&](size_t vox, int dx, int dy, int dz) {
        f(vox, __fmul_rn(__fmul_rn(c.wx[dx], c.wy[dy]), c.wz[dz]));
    });
}

// Channel quad q (0..87) of the 352-wide feature, level 0 first (latent_xyzc.py:66-71): its level and first channel there
__device__ __forceinline__ int level_feature_base(int lvl) { return lvl == 0 ? 0 : lvl == 1 ? 32 : lvl == 2 ? 96 : 224; }
__device__ __forceinline__ void feature_quad(int q, int& lvl, int& c0) {
    lvl = q < 8 ? 0 : q < 24 ? 1 : q < 56 ? 2 : 3;
    c0 = 4 * q - level_feature_base(lvl);
}

template <typename VT>
__device__ __forceinline__ float4 load4(const VT* p);
template <>
__device__ __forceinline__ float4 load4<float>(const float* p) {
    return __ldg(reinterpret_cast<const float4*>(p));
}
template <>
__device__ __forceinline__ float4 load4<__half>(const __half* p) {
    uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    float2 a = __half22float2(*reinterpret_cast<__half2*>(&u.x));
    float2 b = __half22float2(*reinterpret_cast<__half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

// a7 (latent_xyzc.py:62-72): channel quad q of the trilinear sample (F.grid_sample, align_corners=True, zeros padding) of
// frame b's volumes at grid coordinates (gx, gy, gz) in [-1, 1]
template <typename VT>
__device__ __forceinline__ float4 gather_quad(const RenderParams& P, int b, float gx, float gy, float gz, int q) {
    int lvl, c0;
    feature_quad(q, lvl, c0);
    const int C = P.lvl_C[lvl], D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
    Corners cn;
    corner_setup(unnormalize(gx, W), unnormalize(gy, H), unnormalize(gz, D), W, H, D, cn);
    const VT* vol = reinterpret_cast<const VT*>(reinterpret_cast<const char*>(P.volume) + P.lvl_off[lvl]) + (size_t)b * P.lvl_bstride[lvl];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for_each_corner(cn, W, H, D, [&](size_t vox, float wgt) {
        const float4 v = load4<VT>(vol + vox * C + c0);
        acc.x = fmaf(v.x, wgt, acc.x); acc.y = fmaf(v.y, wgt, acc.y);
        acc.z = fmaf(v.z, wgt, acc.z); acc.w = fmaf(v.w, wgt, acc.w);
    });
    return acc;
}

// Backward of gather_quad with respect to the sample position: sum_c df_c * d f_c / d(i_x, i_y, i_z), where i are the
// level's un-normalised coordinates (ATen's grid_sampler_3d backward for the grid, zeros padding: the weight of corner
// (dx, dy, dz) is w_x[dx] w_y[dy] w_z[dz] with d w_x[0] / d i_x = -1 and d w_x[1] / d i_x = +1; corners outside the volume
// are 0 and contribute nothing).  The caller scales by d i / d g = (size - 1) / 2 and sums the levels.
template <typename VT>
__device__ __forceinline__ float3 gather_quad_dpos(const RenderParams& P, int b, float gx, float gy, float gz, int q, float4 df) {
    int lvl, c0;
    feature_quad(q, lvl, c0);
    const int C = P.lvl_C[lvl], D = P.lvl_D[lvl], H = P.lvl_H[lvl], W = P.lvl_W[lvl];
    Corners cn;
    corner_setup(unnormalize(gx, W), unnormalize(gy, H), unnormalize(gz, D), W, H, D, cn);
    const VT* vol = reinterpret_cast<const VT*>(reinterpret_cast<const char*>(P.volume) + P.lvl_off[lvl]) + (size_t)b * P.lvl_bstride[lvl];
    float3 acc = make_float3(0.f, 0.f, 0.f);
    for_each_corner_at(cn, W, H, D, [&](size_t vox, int dx, int dy, int dz) {
        const float4 v = load4<VT>(vol + vox * C + c0);
        const float s = fmaf(v.w, df.w, fmaf(v.z, df.z, fmaf(v.y, df.y, v.x * df.x)));   // dF . V at this corner
        const float sx = cn.wy[dy] * cn.wz[dz] * s, sy = cn.wx[dx] * cn.wz[dz] * s, sz = cn.wx[dx] * cn.wy[dy] * s;
        acc.x += dx ? sx : -sx;
        acc.y += dy ? sy : -sy;
        acc.z += dz ? sz : -sz;
    });
    return acc;
}

// d loss / d(grid coordinate g) -> d loss / d(canonical point c) for one axis: g = ((c - min) / voxel / out_sh) * 2 - 1
__device__ __forceinline__ float grid_to_can_scale(const FrameXf& f, int axis_dhw) {
    return 2.f / (f.voxel[axis_dhw] * f.out_sh[axis_dhw]);
}

// Frame-transform gradients of one sample (world_to_grid: c = (w - Th) R, c_j = sum_i p_i R[i][j]) from d loss / d c:
// t[3 i + j] = d loss / d R[i][j] = p_i dc_j,  t[9 + i] = d loss / d Th[i] = -sum_j R[i][j] dc_j
__device__ __forceinline__ void frame_grad_terms(const FrameXf& f, float wx, float wy, float wz, float dcx, float dcy, float dcz,
                                                 float (&t)[12]) {
    const float p[3] = {__fsub_rn(wx, f.Th[0]), __fsub_rn(wy, f.Th[1]), __fsub_rn(wz, f.Th[2])};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        t[3 * i + 0] = p[i] * dcx; t[3 * i + 1] = p[i] * dcy; t[3 * i + 2] = p[i] * dcz;
        t[9 + i] = -fmaf(f.R[3 * i + 2], dcz, fmaf(f.R[3 * i + 1], dcy, f.R[3 * i] * dcx));
    }
}

// Per-frame sums of N values across one warp's calls: lane k < N holds element k of the running frame's sum and hands it to
// the caller's flush, which adds it to its destination with one atomic, when the frame changes (and once at the end).
// Callers that visit frames in order (sample lists are frame-major) therefore issue one atomic per warp, frame and element.
struct FrameGradAcc {
    int frame = -1;
    float v = 0.f;
};
// the 12 terms of frame_grad_terms -> dR (B,3,3) / dTh (B,3), either may be null
__device__ __forceinline__ void frame_grad_flush(FrameGradAcc& a, float* __restrict__ dR, float* __restrict__ dTh, int lane) {
    if (a.frame >= 0 && a.v != 0.f) {
        if (lane < 9 && dR) atomicAdd(dR + (size_t)a.frame * 9 + lane, a.v);
        else if (lane >= 9 && lane < 12 && dTh) atomicAdd(dTh + (size_t)a.frame * 3 + lane - 9, a.v);
    }
    a.v = 0.f;
}
// d loss / d(canonical point) -> -d_bounds[frame, 0, :] (get_grid_coords subtracts bounds[:, 0] from the canonical point;
// row 1 is never read)
__device__ __forceinline__ void bounds_grad_flush(FrameGradAcc& a, float* __restrict__ d_bounds, int lane) {
    if (a.frame >= 0 && a.v != 0.f && lane < 3) atomicAdd(d_bounds + (size_t)a.frame * 6 + lane, -a.v);
    a.v = 0.f;
}
// Whole warp: each lane contributes t for frame b (b < 0: nothing).
template <int N, typename Flush>
__device__ __forceinline__ void frame_sum_add(FrameGradAcc& a, int b, const float (&t)[N], int lane, Flush&& flush) {
    constexpr int kNone = 0x7fffffff;
    int f = b < 0 ? kNone : b;
    for (;;) {
        const int fm = __reduce_min_sync(0xffffffffu, f);
        if (fm == kNone) break;
        float mine = 0.f;
#pragma unroll
        for (int k = 0; k < N; ++k) {
            float s = f == fm ? t[k] : 0.f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (lane == k) mine = s;
        }
        if (fm != a.frame) { flush(a); a.frame = fm; }
        a.v += mine;
        if (f == fm) f = kNone;
    }
}

// ---------------------------------------------------------------- f-1: if_clight_renderer_mmsk.py:12-45
// inside = AND over the mask views of msk[round(v)][round(u)], (u, v) = perspective projection of the world
// point, rounded half-to-even (torch.round) and clamped to the image like upstream.
__device__ __forceinline__ int mask_pixel(float r, int size) {
    // torch: .round().long() then clamp(0, size-1); non-finite / out-of-range casts give LONG_MIN on x86 => 0
    if (!(fabsf(r) < 9.0e18f)) return 0;
    const long long q = (long long)rintf(r);
    return (int)(q < 0 ? 0 : (q > size - 1 ? size - 1 : q));
}
// The mesh dataset's rule (multi_view_mesh_dataset.py:131-133): np.round (half to even), then .astype(np.int32), then clip.
// A NaN or a rounded value outside int32 converts to INT_MIN on x86, which the clip turns into 0 (not size - 1).
__device__ __forceinline__ int mask_pixel_i32(float r, int size) {
    const float q = rintf(r);
    if (!(q < 2147483648.f) || q < 0.f) return 0;
    const int i = (int)q;
    return i > size - 1 ? size - 1 : i;
}
// The perspective projection of a world point into one mask view (base_utils.project), fp32: pts @ R^T + T, then @ K^T,
// with RT (3,4) world->camera and K (3,3).  (ix, iy, iz) are the homogeneous pixel coordinates; the callers divide
// (u = ix / iz, v = iy / iz, __fdiv_rn) and round with their own integer rule.
__device__ __forceinline__ void project_view(const float* RT, const float* K, float wx, float wy, float wz, float& ix, float& iy,
                                             float& iz) {
    const float cx = __fadd_rn(fmaf(wz, RT[2], fmaf(wy, RT[1], __fmul_rn(wx, RT[0]))), RT[3]);
    const float cy = __fadd_rn(fmaf(wz, RT[6], fmaf(wy, RT[5], __fmul_rn(wx, RT[4]))), RT[7]);
    const float cz = __fadd_rn(fmaf(wz, RT[10], fmaf(wy, RT[9], __fmul_rn(wx, RT[8]))), RT[11]);
    ix = fmaf(cz, K[2], fmaf(cy, K[1], __fmul_rn(cx, K[0])));
    iy = fmaf(cz, K[5], fmaf(cy, K[4], __fmul_rn(cx, K[3])));
    iz = fmaf(cz, K[8], fmaf(cy, K[7], __fmul_rn(cx, K[6])));
}
// The same two steps for a float64 camera (the monocular mesh dataset's, monocular_mesh_dataset.py:35-48): numpy promotes
// the float32 grid point to float64, so the point is widened exactly and the chain above runs in double, in the same
// product and sum order.
__device__ __forceinline__ int mask_pixel_i32(double r, int size) {
    const double q = rint(r);
    if (!(q < 2147483648.0) || q < 0.0) return 0;
    const int i = (int)q;
    return i > size - 1 ? size - 1 : i;
}
__device__ __forceinline__ void project_view(const double* RT, const double* K, float px, float py, float pz, double& ix,
                                             double& iy, double& iz) {
    const double wx = px, wy = py, wz = pz;
    const double cx = __dadd_rn(fma(wz, RT[2], fma(wy, RT[1], __dmul_rn(wx, RT[0]))), RT[3]);
    const double cy = __dadd_rn(fma(wz, RT[6], fma(wy, RT[5], __dmul_rn(wx, RT[4]))), RT[7]);
    const double cz = __dadd_rn(fma(wz, RT[10], fma(wy, RT[9], __dmul_rn(wx, RT[8]))), RT[11]);
    ix = fma(cz, K[2], fma(cy, K[1], __dmul_rn(cx, K[0])));
    iy = fma(cz, K[5], fma(cy, K[4], __dmul_rn(cx, K[3])));
    iz = fma(cz, K[8], fma(cy, K[7], __dmul_rn(cx, K[6])));
}
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
// The single-view variant (if_clight_renderer_msk.py:17-30) first moves the sample into the world of the snapshot frame:
// can = (p - Th) @ R;  q = can @ R0^T + Th0.
__device__ __forceinline__ bool inside_masks(const RenderParams& P, const FrameXf& f, float wx, float wy, float wz) {
    if (P.mask_R0) {
        const float px = __fsub_rn(wx, f.Th[0]), py = __fsub_rn(wy, f.Th[1]), pz = __fsub_rn(wz, f.Th[2]);
        const float cx = fmaf(pz, f.R[6], fmaf(py, f.R[3], __fmul_rn(px, f.R[0])));
        const float cy = fmaf(pz, f.R[7], fmaf(py, f.R[4], __fmul_rn(px, f.R[1])));
        const float cz = fmaf(pz, f.R[8], fmaf(py, f.R[5], __fmul_rn(px, f.R[2])));
        const float* R0 = P.mask_R0;
        wx = __fadd_rn(fmaf(cz, __ldg(R0 + 2), fmaf(cy, __ldg(R0 + 1), __fmul_rn(cx, __ldg(R0 + 0)))), __ldg(P.mask_Th0 + 0));
        wy = __fadd_rn(fmaf(cz, __ldg(R0 + 5), fmaf(cy, __ldg(R0 + 4), __fmul_rn(cx, __ldg(R0 + 3)))), __ldg(P.mask_Th0 + 1));
        wz = __fadd_rn(fmaf(cz, __ldg(R0 + 8), fmaf(cy, __ldg(R0 + 7), __fmul_rn(cx, __ldg(R0 + 6)))), __ldg(P.mask_Th0 + 2));
    }
    for (int v = 0; v < P.mask_nv; ++v) {
        float ix, iy, iz;
        project_view(P.mask_RT + v * 12, P.mask_Ks + v * 9, wx, wy, wz, ix, iy, iz);
        const int u = mask_pixel(__fdiv_rn(ix, iz), P.mask_W), w = mask_pixel(__fdiv_rn(iy, iz), P.mask_H);
        if (!__ldg(P.mask_msks + ((size_t)v * P.mask_H + w) * P.mask_W + u)) return false;
    }
    return true;
}

// ---------------------------------------------------------------- a9: embedder.py:5-50
// out[0..2] = x; out[3+6f+j] = sin(2^f x_j); out[6+6f+j] = cos(2^f x_j)   (x * freq is exact: freq = 2^f)
template <int L, typename Store>
__device__ __forceinline__ void positional_embed(float x, float y, float z, Store&& store) {
    store(0, x); store(1, y); store(2, z);
    float f = 1.f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        float s, c;
        sincosf(x * f, &s, &c); store(3 + 6 * l + 0, s); store(3 + 6 * l + 3, c);
        sincosf(y * f, &s, &c); store(3 + 6 * l + 1, s); store(3 + 6 * l + 4, c);
        sincosf(z * f, &s, &c); store(3 + 6 * l + 2, s); store(3 + 6 * l + 5, c);
        f *= 2.f;
    }
}

// Backward of positional_embed<L> for input axis a: d = d loss / d(encoding), enc = the encoding itself (its saved sin / cos),
// both in the layout above.  d sin(2^l x) = 2^l cos(2^l x) dx, d cos(2^l x) = -2^l sin(2^l x) dx.
template <int L>
__device__ __forceinline__ float positional_embed_bwd(const float* d, const float* enc, int a) {
    float v = d[a], f = 1.f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        v = fmaf(f, fmaf(d[3 + 6 * l + a], enc[6 + 6 * l + a], -d[6 + 6 * l + a] * enc[3 + 6 * l + a]), v);
        f *= 2.f;
    }
    return v;
}

// Same layout, cheaper: an accurate sincosf only every ANCHOR-th octave, the octaves in between by the
// double-angle recurrence (sin 2a = 2 sin a cos a, cos 2a = 1 - 2 sin^2 a).  Each doubling at most doubles the
// absolute error, so with ANCHOR <= 5 the values stay within ~2e-6 of sincosf -- far below the fp16 rounding
// (2^-11) they get as tensor-core operands.  Used by the tensor-core kernel only (colour path).
template <int L, int ANCHOR, typename Store>
__device__ __forceinline__ void positional_embed_anchored(float x, float y, float z, Store&& store) {
    store(0, x); store(1, y); store(2, z);
    float f = 1.f;
    float sx = 0.f, cx = 1.f, sy = 0.f, cy = 1.f, sz = 0.f, cz = 1.f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        if (l % ANCHOR == 0) {
            sincosf(x * f, &sx, &cx); sincosf(y * f, &sy, &cy); sincosf(z * f, &sz, &cz);
        } else {
            float t;
            t = 2.f * sx * cx; cx = fmaf(-2.f * sx, sx, 1.f); sx = t;
            t = 2.f * sy * cy; cy = fmaf(-2.f * sy, sy, 1.f); sy = t;
            t = 2.f * sz * cz; cz = fmaf(-2.f * sz, sz, 1.f); sz = t;
        }
        store(3 + 6 * l + 0, sx); store(3 + 6 * l + 1, sy); store(3 + 6 * l + 2, sz);
        store(3 + 6 * l + 3, cx); store(3 + 6 * l + 4, cy); store(3 + 6 * l + 5, cz);
        f *= 2.f;
    }
}

// ---------------------------------------------------------------- a10: raw2outputs
// nerf_net_utils.py:6-51, one warp per ray.  raw = (rgb logits x3, sigma) per sample in smem,
// z = perturbed z_vals in smem.  All lanes return the same reduced values.
struct RayOut { float r, g, b, depth, acc; };

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Whole warp, per-ray sums: each lane contributes v to its ray ri (~0u: none); the lanes of one ray are summed first and
// lane 0 hands element k of the sum to put(ray, k, sum).  A warp holds consecutive samples, so that is one atomic per ray and
// element, and a ray inside one warp gets its sum in a single call.
template <int N, typename Put>
__device__ __forceinline__ void ray_sum_add(unsigned int ri, const float (&v)[N], int lane, Put&& put) {
    for (;;) {
        const unsigned int rm = __reduce_min_sync(0xffffffffu, ri);
        if (rm == ~0u) break;
        const bool mine = ri == rm;
#pragma unroll
        for (int k = 0; k < N; ++k) {
            const float s = warp_sum(mine ? v[k] : 0.f);
            if (lane == 0) put(rm, k, s);
        }
        if (mine) ri = ~0u;
    }
}

__device__ __forceinline__ RayOut composite_ray(const float4* __restrict__ raw, const float* __restrict__ z, int S,
                                                float norm_d, float* __restrict__ weights_out, int lane) {
    float T_run = 1.f;
    float ar = 0.f, ag = 0.f, ab = 0.f, ad = 0.f, aa = 0.f;
    for (int base = 0; base < S; base += 32) {
        int s = base + lane;
        float alpha = 0.f, fac = 1.f, zr = 0.f;
        float4 rw = make_float4(0.f, 0.f, 0.f, 0.f);
        if (s < S) {
            rw = raw[s];
            zr = z[s];
            float dist = (s + 1 < S) ? __fsub_rn(z[s + 1], zr) : 1e10f;
            dist = __fmul_rn(dist, norm_d);
            alpha = __fsub_rn(1.f, expf(-__fmul_rn(fmaxf(rw.w, 0.f), dist)));   // 1 - exp(-relu(sigma) * dists)
            fac = __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f);                      // 1 - alpha + 1e-10
        }
        // inclusive product scan over the 32 lanes
        float incl = fac;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            float up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl *= up;
        }
        float excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 1.f;
        float w = alpha * (T_run * excl);
        T_run *= __shfl_sync(0xffffffffu, incl, 31);
        if (s < S) {
            if (weights_out) weights_out[s] = w;
            ar += w * (1.f / (1.f + expf(-rw.x)));   // torch.sigmoid
            ag += w * (1.f / (1.f + expf(-rw.y)));
            ab += w * (1.f / (1.f + expf(-rw.z)));
            ad += w * zr;
            aa += w;
        }
    }
    RayOut o;
    o.r = warp_sum(ar); o.g = warp_sum(ag); o.b = warp_sum(ab); o.depth = warp_sum(ad); o.acc = warp_sum(aa);
    return o;
}

// disp_map = 1 / max(1e-10, depth / acc); torch.max propagates the NaN of 0/0 (nerf_net_utils.py:44-45)
__device__ __forceinline__ float disparity(float depth, float acc) {
    float q = __fdiv_rn(depth, acc);
    float m = (q != q) ? q : fmaxf(1e-10f, q);
    return __fdiv_rn(1.f, m);
}

// the maps of ray ri (frame-major ray index); white_bkgd adds 1 - acc to rgb (nerf_net_utils.py:47-48)
__device__ __forceinline__ void store_ray_outputs(const RenderParams& P, size_t ri, const RayOut& o) {
    const float add = P.white_bkgd ? __fsub_rn(1.f, o.acc) : 0.f;
    P.rgb_map[ri * P.rgb_stride + 0] = o.r + add;
    P.rgb_map[ri * P.rgb_stride + 1] = o.g + add;
    P.rgb_map[ri * P.rgb_stride + 2] = o.b + add;
    P.depth_map[ri * P.map_stride] = o.depth;
    P.acc_map[ri * P.map_stride] = o.acc;
    P.disp_map[ri * P.map_stride] = disparity(o.depth, o.acc);
}

}  // namespace nb
