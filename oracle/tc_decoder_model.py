"""The tensor-core decoder's arithmetic, restated on the CPU row by row (neuralbody_b200/csrc/nb_render_tc_list.cu).

Test infrastructure only; nothing here is product code.  Every rounding the decoder applies is restated:

  * layer-0 features: either the oracle's grid_sample, or `gather_f32`, a float32 restatement of the kernel's own gather
    (world_to_grid's _rn chain, unnormalize, the cell's corners in order 0..7 with zero weights skipped, weights (wx wy) wz,
    one fmaf per corner);
  * operands of layers 0-2: activations split as hi = cvt.rz(x) and lo = cvt.rn(x - (x with 13 mantissa bits cleared)) in
    the 3-pass mode, hi = cvt.rn(x) in the 1-pass mode; weights as hi = rn(w), lo = rn(w - hi) (nb_capi.cu f16_hi / f16_lo);
  * biases of layers 0-2: the accumulators start from the fp32 bias (DESIGN.md 4.1).  The packed stream also holds a bias
    step of fp16 (hi, lo) pairs, but the decoder does not multiply it, so the fp32 bias is what the model adds;
  * h2: one fp16 rounded to nearest; the folded colour layer is 1-pass over [h2 | PE(xyz) 63 | 0 | PE(view) 27 | 0 | 1 | 1 |
    0 | 0] with the per-point tile rounded to nearest from the kernel's fp32 PE (positional_embed_anchored), and the bias
    entering as hi(bc) + lo(bc) through the two columns of ones;
  * heads: sigma = alpha_fc . relu(h2 accumulator) + bias and rgb = rgb_fc . relu(layer-3 accumulator) + bias, in fp32.

Accumulation (`acc`): 'f64' sums each layer in float64 and rounds once; 'rz' adds each K-step's 16 exact products of each
pass, in the kernel's issue order, to a float32 accumulator rounded toward zero.  On an H100 'rz' brings the 3-pass sigma of
the decoder from ~1e-4 to ~1e-5 of the kernel's (tests/test_decoder_rows_gpu.py), so the tensor cores' fp32 accumulation
truncates rather than rounds; what is left is their in-K-step summation order and the rare fp16 rounding it flips.  fmaf
is emulated as a float64 product
(exact for float32 operands) plus a float64 sum rounded to float32; the sum can round twice, which on rare ties differs from
one fused rounding by an ulp.
"""
import math

import numpy as np
import torch

F16_MIN_NORMAL = 2.0 ** -14


# ------------------------------------------------------------------------------------------------ roundings
def f16_rn(x):
    """fp32 -> fp16 (round to nearest even) -> fp32 (cvt.rn.f16.f32)."""
    return x.float().to(torch.float16).to(torch.float32)


def trunc13(x):
    """x with its 13 low mantissa bits cleared (the kernel's `x & 0xFFFFE000`)."""
    bits = x.float().contiguous().view(torch.int32) & torch.tensor(-8192, dtype=torch.int32)
    return bits.view(torch.float32)


def f16_rz(x):
    """fp32 -> fp16 rounded toward zero -> fp32 (cvt.rz.f16.f32), for |x| below fp16's largest finite value.  In fp16's
    normal range this is trunc13(x); below 2^-14 the fp16 subnormal grid of 2^-24 truncates further."""
    x = x.float()
    sub = torch.trunc(x.double() * 2.0 ** 24) * 2.0 ** -24
    return torch.where(x.abs() < F16_MIN_NORMAL, sub.float(), trunc13(x))


def split_act(x):
    """An activation's (hi, lo) operand pair in the 3-pass mode: hi = cvt.rz(x), lo = cvt.rn(x - trunc13(x))."""
    x = x.float()
    return f16_rz(x), f16_rn(x - trunc13(x))


def split_weight(w):
    """A weight's (hi, lo) pair as the packer rounds it: hi = rn(w), lo = rn(w - hi)."""
    w = w.float()
    hi = f16_rn(w)
    return hi, f16_rn(w - hi)


def fma32(a, b, c):
    """fmaf(a, b, c) on float32 tensors: the float64 product is exact, the float64 sum is rounded to float32."""
    return (a.double() * b.double() + c.double()).float()


# ------------------------------------------------------------------------------------------------ layer-0 features
def world_to_grid_f32(wpts, R, Th, bounds, voxel_size, out_sh):
    """nb_device.cuh world_to_grid for one frame: wpts (P,3) float32 -> grid (P,3) (x, y, z) in [-1, 1], float32."""
    w = wpts.float()
    R = R.float().reshape(3, 3)
    Th = Th.float().reshape(3)
    b0 = bounds.float().reshape(2, 3)[0]
    p = w - Th
    c = [fma32(p[:, 2], R[2, j].expand_as(p[:, 2]), fma32(p[:, 1], R[1, j].expand_as(p[:, 1]), p[:, 0] * R[0, j]))
         for j in range(3)]
    vox = torch.tensor([float(v) for v in voxel_size], dtype=torch.float32)
    osh = torch.tensor([float(v) for v in out_sh], dtype=torch.float32)   # (d, h, w)
    g = []
    for axis, dhw in ((0, 2), (1, 1), (2, 0)):                             # x <- w, y <- h, z <- d
        t = (c[axis] - b0[axis]) / vox[axis]
        g.append((t / osh[dhw]) * 2.0 - 1.0)
    return torch.stack(g, 1)


def _unnormalize(g, size):
    return ((g + 1.0) * 0.5) * float(size - 1)


def gather_f32(grid, volumes):
    """The kernel's trilinear gather of ONE frame: grid (P,3) float32, volumes [(C,D,H,W)] levels 0..3 -> (P,352) float32,
    upstream's channel order (level 0 first).  Corners in order 0..7 (x fastest), out-of-range and zero-weight corners
    skipped, weight (wx wy) wz, one fmaf per corner."""
    P = grid.shape[0]
    out = []
    for vol in volumes:
        vol = vol.float()
        C, D, H, W = vol.shape
        flat = vol.reshape(C, -1).t().contiguous()                       # (D H W, C)
        ix, iy, iz = (_unnormalize(grid[:, a], n) for a, n in ((0, W), (1, H), (2, D)))
        fx, fy, fz = torch.floor(ix), torch.floor(iy), torch.floor(iz)
        ok = (fx >= -1) & (fx <= W) & (fy >= -1) & (fy <= H) & (fz >= -1) & (fz <= D)
        wx = ((fx + 1.0) - ix, ix - fx)
        wy = ((fy + 1.0) - iy, iy - fy)
        wz = ((fz + 1.0) - iz, iz - fz)
        x0, y0, z0 = fx.long(), fy.long(), fz.long()
        acc = torch.zeros((P, C), dtype=torch.float32)
        for c in range(8):
            dx, dy, dz = c & 1, (c >> 1) & 1, c >> 2
            x, y, z = x0 + dx, y0 + dy, z0 + dz
            wgt = (wx[dx] * wy[dy]) * wz[dz]
            use = ok & (x >= 0) & (x < W) & (y >= 0) & (y < H) & (z >= 0) & (z < D) & (wgt != 0)
            idx = ((z.clamp(0, D - 1) * H + y.clamp(0, H - 1)) * W + x.clamp(0, W - 1))
            v = flat[idx]
            acc = torch.where(use[:, None], fma32(v, wgt[:, None].expand_as(v), acc), acc)
        out.append(acc)
    return torch.cat(out, 1)


# ------------------------------------------------------------------------------------------------ per-point tile
def positional_embed_anchored(x, L, anchor):
    """nb_device.cuh positional_embed_anchored<L, ANCHOR> on (P,3) float32: sin / cos of every ANCHOR-th octave (correctly
    rounded here; CUDA's sincosf is within an ulp), the octaves between by the fp32 double-angle recurrence."""
    x = x.float()
    out = [x]
    s = c = None
    f = 1.0
    for l in range(L):
        if l % anchor == 0:
            a = (x * f).double()
            s, c = torch.sin(a).float(), torch.cos(a).float()
        else:
            t = (2.0 * s) * c
            c = fma32(-2.0 * s, s, torch.ones_like(s))
            s = t
        out += [s, c]
        f *= 2.0
    return torch.cat(out, -1)


def view_dirs_f32(ray_d):
    """ray_d / ray_norm(ray_d) as the kernel forms it (sum left to right, correctly rounded sqrt and division)."""
    d = ray_d.float()
    n2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    return d / torch.sqrt(n2)[:, None]


# ------------------------------------------------------------------------------------------------ the decoder
def folded_colour_layer(w, latent_index):
    """nb_layout.h: view_fc[:, :256] o latent_fc o (feature_fc (+) latent[idx]) -> Wc (128 x 256), bc (128), in fp64 and
    rounded to fp32 once, as the packer folds them.  Also returns view_fc's PE columns Wv[:, 256:] (27 view + 63 xyz)."""
    d = {k: v.double() for k, v in w.items()}
    Wv = d["view_fc.weight"][:, :, 0]
    Lf = d["latent_fc.weight"][:, :, 0]
    Ff = d["feature_fc.weight"][:, :, 0]
    Wv_h = Wv[:, :256]
    T = Wv_h @ Lf[:, :256]
    Wc = T @ Ff
    lat = d["latent.weight"][latent_index].reshape(-1)
    bc = T @ d["feature_fc.bias"] + Wv_h @ (Lf[:, 256:] @ lat + d["latent_fc.bias"]) + d["view_fc.bias"]
    return Wc.float(), Wv[:, 256:].float(), bc.float()


def _mm(a, w):
    """(P,K) x (N,K)^T of fp16-valued operands with a float64 accumulator (products of fp16 values are exact)."""
    return a.double() @ w.double().t()


def rz32(x):
    """float64 -> float32 rounded toward zero."""
    y = x.float()
    over = y.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(y, torch.zeros_like(y)), y)


# layer-0 K order of the tensor-core kernel: coarse level first (nb_layout.h feat_tc_to_orig)
L0_ORDER = list(range(224, 352)) + list(range(96, 224)) + list(range(32, 96)) + list(range(0, 32))


def _accumulate(start, pairs, acc):
    """The layer's accumulator from `start` (P,N float32) over the K-steps of the operand pairs [(A (P,K), W (N,K)), ...]:
    acc = 'f64' sums everything in float64 and rounds once; acc = 'rz' adds each K-step's 16 products of each pass to a
    float32 accumulator rounded toward zero, passes in the kernel's issue order."""
    if acc == "f64":
        return (sum(_mm(a, w) for a, w in pairs) + start.double()).float()
    out = start.float()
    K = pairs[0][0].shape[1]
    for k in range(0, K, 16):
        for a, w in pairs:
            out = rz32(out.double() + _mm(a[:, k:k + 16], w[:, k:k + 16]))
    return out


def dense_layer(a, W, b, passes, acc="f64"):
    """One of layers 0-2 before relu, float32 out: the fp32 bias plus the pass products of the operand roundings
    (a, W in the kernel's K order)."""
    start = b.float().expand(a.shape[0], -1)
    if passes == 3:
        a_hi, a_lo = split_act(a)
        w_hi, w_lo = split_weight(W)
        return _accumulate(start, [(a_hi, w_hi), (a_lo, w_hi), (a_hi, w_lo)], acc)
    return _accumulate(start, [(f16_rn(a), f16_rn(W))], acc)


def decode_rows(w, latent_index, feats, wpts=None, viewdir=None, passes=3, density=False, pe=None, acc="f64"):
    """The decoder over rows.  feats (P,352) float32 in upstream's channel order; wpts / viewdir (P,3) float32 world points
    and unit view directions (the kernel's: see view_dirs_f32), or `pe` = the (P,90) [PE(view) 27 | PE(xyz) 63] tile in the
    oracle's order.  `acc`: the accumulation model of _accumulate.  Returns sigma (P,) when `density`, else raw (P,4) =
    (rgb logits, sigma), float32."""
    h = feats.float()[:, L0_ORDER]
    for i, name in enumerate(("fc_0", "fc_1", "fc_2")):
        Wt = w[name + ".weight"][:, :, 0]
        h = torch.relu(dense_layer(h, Wt[:, L0_ORDER] if i == 0 else Wt, w[name + ".bias"], passes, acc))
    sigma = (h.double() @ w["alpha_fc.weight"][0, :, 0].double() + float(w["alpha_fc.bias"].double()[0])).float()
    if density:
        return sigma
    Wc, Wpe, bc = folded_colour_layer(w, int(latent_index))
    if pe is None:
        pe = torch.cat([positional_embed_anchored(viewdir, 4, 4), positional_embed_anchored(wpts, 10, 5)], -1)
    P = h.shape[0]
    bc_hi, bc_lo = split_weight(bc)
    zero = torch.zeros((P, 1))
    one = torch.ones((P, 1))
    # the per-point tile [PE(xyz) 63 | 0 | PE(view) 27 | 0 | 1 | 1 | 0 | 0] and its weights [Wx | 0 | Wv | 0 | hi(bc) | lo(bc) | 0 | 0]
    tile = torch.cat([pe[:, 27:], zero, pe[:, :27], zero, one, one, zero, zero], 1)
    zc = torch.zeros((Wc.shape[0], 1))
    wt = torch.cat([Wpe[:, 27:], zc, Wpe[:, :27], zc, bc_hi[:, None], bc_lo[:, None], zc, zc], 1)
    a3 = torch.cat([f16_rn(h), f16_rn(tile)], 1)
    w3 = torch.cat([f16_rn(Wc), f16_rn(wt)], 1)
    col = torch.relu(_accumulate(torch.zeros((P, Wc.shape[0])), [(a3, w3)], acc))
    rgb = (col.double() @ w["rgb_fc.weight"][:, :, 0].double().t() + w["rgb_fc.bias"].double()).float()
    return torch.cat([rgb, sigma[:, None]], -1)


def decode_frame(w, latent_index, wpts, volumes, R, Th, bounds, voxel_size, out_sh, passes=3, density=False, ray_d=None,
                 acc="f64"):
    """decode_rows with the kernel's own layer-0 gather: wpts (P,3) world points of one frame, volumes [(C,D,H,W)],
    ray_d (P,3) the ray direction of each point (render rows)."""
    grid = world_to_grid_f32(wpts, R, Th, bounds, voxel_size, out_sh)
    feats = gather_f32(grid, volumes)
    vd = None if ray_d is None else view_dirs_f32(ray_d)
    return decode_rows(w, latent_index, feats, wpts, vd, passes, density, acc=acc)


def sample_points_f32(ray_o, ray_d, z):
    """o + d z per sample as classify_compact_kernel forms it: ray_o / ray_d (n,3), z (n,S) -> (n,S,3) float32."""
    return ray_o.float()[:, None, :] + ray_d.float()[:, None, :] * z.float()[..., None]
