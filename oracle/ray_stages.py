"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

References and designed inputs for the per-ray stages around the decoder:
  - compositing (raw2outputs, nerf_net_utils.py:6-51) and its backward: float64 autograd through
    oracle.neuralbody_oracle.raw2outputs from the kernels' own float32 depths, plus the same graph in float32 on the CPU,
    whose NaN / zero pattern is the one a float32 kernel must reproduce where float64 and float32 legitimately differ;
  - the importance sampler (nb_sample_pdf): a numpy float32 emulation of sample_pdf_kernel in its exact operation order,
    so that z_out and z_samples can be held to the bit;
  - case builders, each placing one edge (saturating alpha, sigma <= 0, zero-length intervals, the 1e10 last interval,
    disp_map at acc = 0 and at depth / acc = 1e-10, u on a CDF value, empty bins, depth ties) deliberately.
Nothing here touches CUDA."""
import numpy as np
import torch

from oracle import neuralbody_oracle as O

F32 = np.float32
EPS32 = float(np.finfo(np.float32).eps)


# ------------------------------------------------------------------ the kernels' sample depths (nb_device.cuh, z_sample)
def linspace01(i, steps):
    """linspace01: torch.linspace(0, 1, steps)[i] as the kernels compute it (symmetric fill), float32."""
    i = np.asarray(i)
    if steps == 1:
        return np.zeros(i.shape, F32)
    step = F32(1) / F32(steps - 1)
    lo = step * i.astype(F32)
    hi = F32(1) - step * (steps - 1 - i).astype(F32)
    return np.where(i < steps // 2, lo, hi).astype(F32)


def _z_plain(near, far, t):
    return near * (F32(1) - t) + far * t          # every op rounds to float32 (numpy, no contraction)


def z_sample(near, far, S, t_vals=None, t_rand=None):
    """The depths of sample s = 0..S-1 of each ray, float32, bit for bit z_sample: near / far (N,), t_vals (S,) or None,
    t_rand (N,S) or None -> (N,S)."""
    near = np.asarray(near, F32)[:, None]
    far = np.asarray(far, F32)[:, None]
    t = linspace01(np.arange(S), S) if t_vals is None else np.asarray(t_vals, F32)
    z = _z_plain(near, far, t[None])
    if t_rand is None:
        return z.astype(F32)
    zp = np.concatenate([z[:, :1], _z_plain(near, far, t[None, :-1])], 1)      # z of s - 1
    zn = np.concatenate([_z_plain(near, far, t[None, 1:]), z[:, -1:]], 1)      # z of s + 1
    lower = np.where(np.arange(S) > 0, F32(.5) * (z + zp), z).astype(F32)
    upper = np.where(np.arange(S) < S - 1, F32(.5) * (zn + z), z).astype(F32)
    return (lower + (upper - lower) * np.asarray(t_rand, F32)).astype(F32)


def z_sample_torch64(near, far, S, t_vals=None, t_rand=None):
    """The same depths as differentiable float64 functions of near / far (N,): the value is z_sample's float32 result
    exactly, the derivative that of z_sample's formula."""
    z32 = torch.from_numpy(z_sample(near.detach().float().numpy(), far.detach().float().numpy(), S,
                                    None if t_vals is None else np.asarray(t_vals),
                                    None if t_rand is None else np.asarray(t_rand))).double()
    t = torch.from_numpy(linspace01(np.arange(S), S) if t_vals is None else np.asarray(t_vals, F32)).double()
    z = near[:, None] * (1 - t) + far[:, None] * t
    if t_rand is not None:
        r = torch.as_tensor(np.asarray(t_rand, F32)).double()
        mids = .5 * (z[:, 1:] + z[:, :-1])
        lower = torch.cat([z[:, :1], mids], 1)
        upper = torch.cat([mids, z[:, -1:]], 1)
        z = lower + (upper - lower) * r
    return z32 + (z - z.detach())


# ------------------------------------------------------------------ compositing
def raw2outputs(raw, z_vals, rays_d, white_bkgd=False):
    """oracle.neuralbody_oracle.raw2outputs, and for a single sample per ray the kernels' reading of it: upstream builds the
    last interval as 1e10 expanded to the shape of dists[..., :1], which is empty when S = 1 (so are its outputs); the
    kernels give that one sample the 1e10 interval like every last sample."""
    if z_vals.shape[-1] > 1:
        return O.raw2outputs(raw, z_vals, rays_d, white_bkgd)
    dists = torch.full_like(z_vals, 1e10) * torch.norm(rays_d[..., None, :], dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    alpha = 1. - torch.exp(-torch.relu(raw[..., 3]) * dists)
    weights = alpha * 1.
    rgb_map = torch.sum(weights[..., None] * rgb, -2)
    depth_map = torch.sum(weights * z_vals, -1)
    disp_map = 1. / torch.max(1e-10 * torch.ones_like(depth_map), depth_map / torch.sum(weights, -1))
    acc_map = torch.sum(weights, -1)
    if white_bkgd:
        rgb_map = rgb_map + (1. - acc_map[..., None])
    return rgb_map, disp_map, acc_map, weights, depth_map


def composite_reference(raw, ray_d, near=None, far=None, S=None, t_vals=None, t_rand=None, z_vals=None, white_bkgd=False,
                        cot=None, rec=None, dtype=torch.float64):
    """raw2outputs on (N,S,4) float32 records with the kernels' depths, in `dtype`, with autograd.
    Depths: z_vals (N,S) as given, or z_sample(near, far, t_vals, t_rand).  cot: dict of map cotangents (any of rgb (N,3),
    depth, acc, disp (N), weights (N,S)); rec (N,S,8): d loss / d(world point) | d loss / d(view direction) per sample,
    entering through p = o + z d and d / |d| (the decoder's part).  Returns (maps dict, grads dict or None) as float64
    numpy arrays: grads d_raw (N,S,4), d_ray_o, d_ray_d (N,3), d_z (N,S), d_near, d_far (N)."""
    N = raw.shape[0]
    S = raw.shape[1]
    raw_t = torch.as_tensor(np.asarray(raw, F32)).to(dtype).requires_grad_(True)
    rd = torch.as_tensor(np.asarray(ray_d, F32)).to(dtype).requires_grad_(True)
    ro = torch.zeros(N, 3, dtype=dtype, requires_grad=True)
    if z_vals is not None:
        z = torch.as_tensor(np.asarray(z_vals, F32)).to(dtype).requires_grad_(True)
        zleaf, nr, fr = z, None, None
    else:
        nr = torch.as_tensor(np.asarray(near, F32)).double().requires_grad_(True)
        fr = torch.as_tensor(np.asarray(far, F32)).double().requires_grad_(True)
        z = z_sample_torch64(nr, fr, S, t_vals, t_rand)
        if dtype != torch.float64:      # the float32 run starts from the same float32 depths
            z = z.detach().to(dtype).requires_grad_(True)
        z.retain_grad()
        zleaf = z
    rgb, disp, acc, w, depth = raw2outputs(raw_t, z, rd, white_bkgd)
    maps = {"rgb_map": rgb, "disp_map": disp, "acc_map": acc, "weights": w, "depth_map": depth}
    grads = None
    if cot is not None or rec is not None:
        loss = torch.zeros((), dtype=dtype)
        for k, m in (("rgb", rgb), ("depth", depth), ("acc", acc), ("disp", disp), ("weights", w)):
            if cot is not None and cot.get(k) is not None:
                loss = loss + (torch.as_tensor(np.asarray(cot[k], F32)).to(dtype) * m).sum()
        if rec is not None:
            r = torch.as_tensor(np.asarray(rec, F32)).to(dtype)
            pts = ro[:, None] + rd[:, None] * z[..., None]
            vd = rd / torch.norm(rd, dim=-1, keepdim=True)
            loss = loss + (r[..., :3] * pts).sum() + (r[..., 3:6].sum(1) * vd).sum()
        loss.backward()
        g = lambda t: None if t is None or t.grad is None else t.grad.detach().double().numpy()
        grads = {"d_raw": g(raw_t), "d_ray_o": g(ro), "d_ray_d": g(rd), "d_z": g(zleaf), "d_near": g(nr), "d_far": g(fr)}
    return {k: v.detach().double().numpy() for k, v in maps.items()}, grads


def composite_bounds(raw, z, ray_d, white_bkgd=False):
    """Per-element error bounds of a float32 composite against float64, from the float64 terms of each output.
    T_i (exclusive transmittance) carries the float32 errors of every earlier factor f_j = 1 - alpha_j + 1e-10 (a few ulps
    of 1 each, absolute), each scaled by the transmittance T_j in front of it: |dT_i| <~ 5 eps sum_{j<i} T_j + i eps T_i;
    alpha_i = 1 - exp(-x) is good to ~4 eps absolute.  The maps add the warp-sum rounding of their terms.  Every bound is
    4x that estimate plus a floor for subnormal transmittance.  Returns dict of float64 arrays shaped like the outputs."""
    raw = np.asarray(raw, np.float64)
    z = np.asarray(z, np.float64)
    N, S = z.shape
    nrm = np.linalg.norm(np.asarray(ray_d, np.float64), axis=-1)[:, None]
    dist = np.concatenate([z[:, 1:] - z[:, :-1], np.full((N, 1), 1e10)], 1) * nrm
    alpha = 1 - np.exp(-np.maximum(raw[..., 3], 0) * dist)
    f = 1 - alpha + 1e-10
    T = np.concatenate([np.ones((N, 1)), np.cumprod(f, 1)[:, :-1]], 1)
    sumT = np.cumsum(T, 1) - T
    i = np.arange(S)[None]
    w = alpha * T
    tw = 4 * EPS32 * (4 * T + np.abs(alpha) * (5 * sumT + (i + 1) * T)) + 1e-37
    c = 1 / (1 + np.exp(-raw[..., :3]))
    red = 4 * EPS32 * (S / 32 + 6)      # per-lane sums + the 5-step butterfly
    t_acc = tw.sum(1) + red * w.sum(1)
    t_rgb = (tw[..., None] * 1.0).sum(1) + red * (w[..., None] * c).sum(1) + 8 * EPS32 * (w[..., None] * c).sum(1)
    if white_bkgd:
        t_rgb = t_rgb + t_acc[:, None] + EPS32
    t_depth = (tw * np.abs(z)).sum(1) + red * (w * np.abs(z)).sum(1)
    return {"weights": tw, "rgb_map": t_rgb, "acc_map": t_acc, "depth_map": t_depth, "T": T, "sumT": sumT, "alpha": alpha,
            "dist": dist, "w": w, "c": c}


def composite_bwd_bounds(raw, z, ray_d, cot, fwd_bounds, depth, acc):
    """Per-element bounds of the float32 d_raw against float64: the terms of d sigma_i = (g_i T_i - T_i U_i) dist_i e_i,
    g_i = dC . c_i + dD z_i + dA + d_weights_i, U_i = sum_{j>i} g_j alpha_j prod_{i<k<j} f_k, taken in absolute value, times
    the relative error they carry (T_i as in composite_bounds; U by a recurrence of S steps); rgb logits from the bound of
    w_i.  The disp cotangent enters dD / dA with the relative error of depth / acc."""
    b = fwd_bounds
    N, S = b["T"].shape
    z = np.asarray(z, np.float64)
    raw = np.asarray(raw, np.float64)
    zero = np.zeros(N)
    dC = np.zeros((N, 3)) if cot.get("rgb") is None else np.abs(np.asarray(cot["rgb"], np.float64))
    dD = zero if cot.get("depth") is None else np.abs(np.asarray(cot["depth"], np.float64))
    dA = zero if cot.get("acc") is None else np.abs(np.asarray(cot["acc"], np.float64))
    dW = np.zeros((N, S)) if cot.get("weights") is None else np.abs(np.asarray(cot["weights"], np.float64))
    errD, errA = np.zeros(N), np.zeros(N)
    if cot.get("disp") is not None:
        dd = np.abs(np.asarray(cot["disp"], np.float64))
        with np.errstate(all="ignore"):
            x = depth / acc
            r = 1 / np.maximum(1e-10, x)
            dm = dd * r * r
            fD, fA = dm / acc, dm * np.abs(x) / acc
            rel = b["depth_map"] / np.maximum(np.abs(depth), 1e-300) + b["acc_map"] / np.maximum(acc, 1e-300) + 8 * EPS32
            errD, errA = np.nan_to_num(fD * 4 * rel, nan=0, posinf=1e300), np.nan_to_num(fA * 4 * rel, nan=0, posinf=1e300)
            dD = dD + np.nan_to_num(fD, nan=0, posinf=1e300)
            dA = dA + np.nan_to_num(fA, nan=0, posinf=1e300)
    gabs = (dC[:, None, :] * b["c"]).sum(-1) + dD[:, None] * np.abs(z) + dA[:, None] + dW
    gerr = errD[:, None] * np.abs(z) + errA[:, None]
    alpha, T, sumT, dist = b["alpha"], b["T"], b["sumT"], b["dist"]
    f = 1 - alpha + 1e-10
    U = np.zeros((N, S))
    G = np.zeros((N, S))
    u = np.zeros(N)
    gg = np.zeros(N)
    for s in range(S - 1, -1, -1):
        U[:, s], G[:, s] = u, gg
        u = gabs[:, s] * alpha[:, s] + f[:, s] * u
        gg = gabs[:, s] + f[:, s] * gg
    e = np.exp(-np.maximum(raw[..., 3], 0) * dist)
    t_dalpha = 4 * EPS32 * (S + 8) * ((gabs + U + 5 * G) * (4 * T + 5 * sumT) + gerr * T) + 1e-37
    tol = np.zeros((N, S, 4))
    tol[..., 3] = t_dalpha * dist * e + 1e-37
    c = b["c"]
    # d logit = w dC c (1 - c): 1 - c is good to an ulp of 1 (absolute), not of itself, where the sigmoid saturates
    w3, tw3 = b["w"][..., None], b["weights"][..., None]
    tol[..., :3] = 4 * ((tw3 + 8 * EPS32 * w3) * c * (1 - c) + 2 * EPS32 * w3 * c) * dC[:, None, :] + 1e-37
    return {"d_raw": tol, "dalpha": t_dalpha, "e": e, "dD_err": errD, "dD_abs": dD}


# ------------------------------------------------------------------ the importance sampler (nb_sample_pdf.cu)
def _warp_sum32(parts):
    """warp_sum over 32 lane values (N,32), xor butterfly, float32: every lane ends with the same value."""
    v = parts.astype(F32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, np.arange(32) ^ o]).astype(F32)
    assert np.all(v == v[:, :1]) or np.isnan(v).any()
    return v[:, 0]


def sample_pdf_emulate(near, far, weights, S, Ni, t_vals=None, t_rand=None, u=None):
    """sample_pdf_kernel in numpy float32, operation by operation: near / far (N,), weights (N,S), u (N,Ni) or None (det).
    Returns dict: zc (N,S) coarse depths, cdf (N,S-1), u (N,Ni), lo (N,Ni) searchsorted(right) index, denom_branch (N,Ni)
    bool, z_samples (N,Ni), z_out (N,S+Ni) sorted."""
    N = len(near)
    M = S - 1
    zc = z_sample(near, far, S, t_vals, t_rand)
    w = (np.asarray(weights, F32)[:, 1:S - 1] + F32(1e-5)).astype(F32)        # M - 1 values
    parts = np.zeros((N, 32), F32)
    for i in range(M - 1):                                                    # lane i % 32, in lane order
        parts[:, i % 32] = parts[:, i % 32] + w[:, i]
    total = _warp_sum32(parts)
    cdf = np.zeros((N, M), F32)
    acc = np.zeros(N, F32)
    for i in range(1, M):
        acc = (acc + (w[:, i - 1] / total).astype(F32)).astype(F32)
        cdf[:, i] = acc
    if u is None:
        u = np.broadcast_to(linspace01(np.arange(Ni), Ni), (N, Ni))
    u = np.asarray(u, F32)
    lo = np.stack([np.searchsorted(cdf[r], u[r], side="right") for r in range(N)]).astype(np.int64)
    below, above = np.maximum(0, lo - 1), np.minimum(M - 1, lo)
    bins = (F32(.5) * (zc[:, 1:] + zc[:, :-1])).astype(F32)
    c0, c1 = np.take_along_axis(cdf, below, 1), np.take_along_axis(cdf, above, 1)
    b0, b1 = np.take_along_axis(bins, below, 1), np.take_along_axis(bins, above, 1)
    denom = (c1 - c0).astype(F32)
    branch = denom < F32(1e-5)
    denom = np.where(branch, F32(1), denom).astype(F32)
    t = ((u - c0).astype(F32) / denom).astype(F32)
    smp = (b0 + (t * (b1 - b0).astype(F32)).astype(F32)).astype(F32)
    z_out = np.sort(np.concatenate([zc, smp], 1), 1, kind="stable")
    return {"zc": zc, "cdf": cdf, "u": u, "lo": lo, "denom_branch": branch, "z_samples": smp, "z_out": z_out}


# ------------------------------------------------------------------ designed inputs
def _rng(seed):
    return np.random.default_rng(seed)


def ray_dirs(rng, n, unit=False):
    d = rng.normal(size=(n, 3)).astype(F32)
    if unit:
        return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(F32)
    return (d * rng.uniform(0.3, 3.0, size=(n, 1))).astype(F32)      # non-unit: |d| in [~0.1, ~9]


def composite_case(S, n, B, seed, jitter=False, z_user=False, white_bkgd=False):
    """Raw records and rays for one composite run, (B*n) rays, with the edges spread over the rays:
    ray r % 8 == 0: sigma around 1e-10..1e-9 only on the last sample (the 1e10 interval decides the output);
    1: saturating sigma early (T runs into subnormals and to 0); 2: all sigma <= 0 (acc = 0, disp NaN);
    3: sigma exactly 0 and negative mixed with positive (the ReLU kink); 4: repeated depths (zero-length intervals, only with
    z_vals); 5: near = far = 0 (depth 0, so disp_map sits below its 1e-10 kink); 6: unit ray_d; others: moderate random
    sigma and non-unit ray_d.  Returns dict of float32 arrays (rays frame-major, (B*n, ...))."""
    rng = _rng(seed)
    N = B * n
    raw = np.empty((N, S, 4), F32)
    raw[..., :3] = rng.normal(0, 3, size=(N, S, 3))
    sig = rng.normal(0, 1, size=(N, S)) * rng.uniform(0.5, 20, size=(N, 1))
    kind = np.arange(N) % 8
    sig[kind == 0] = 0
    sig[kind == 0, -1] = rng.uniform(1e-10, 1e-9, size=int((kind == 0).sum()))
    k1 = kind == 1
    sig[k1] = np.abs(sig[k1]) + 1e3
    k2 = kind == 2
    sig[k2] = -np.abs(sig[k2])
    sig[k2, ::3] = 0
    k3 = kind == 3
    sig[k3, ::2] = 0
    sig[k3, 1::4] = -1
    raw[..., 3] = sig
    near = rng.uniform(0.5, 2.0, size=N).astype(F32)
    far = (near + rng.uniform(0.5, 3.0, size=N)).astype(F32)
    near[kind == 5] = far[kind == 5] = 0               # a dead ray (near = far = 0): every depth 0, every interval 0 but the last
    ray_d = ray_dirs(rng, N)
    ray_d[kind == 6] = ray_dirs(rng, int((kind == 6).sum()), unit=True)
    t_rand = rng.uniform(0, 1, size=(N, S)).astype(F32) if jitter else None
    z_vals = None
    if z_user:
        z = np.sort(rng.uniform(0.5, 4.0, size=(N, S)).astype(F32), 1)
        rep = kind == 4
        z[rep] = np.repeat(z[rep][:, ::2], 2, axis=1)[:, :S]         # pairs of equal depths
        z[rep] = np.sort(z[rep], 1)
        z_vals = z
    return {"raw": raw, "near": near, "far": far, "ray_d": ray_d, "t_rand": t_rand, "z_vals": z_vals,
            "white_bkgd": white_bkgd, "S": S, "n": n, "B": B}


def case_depths(case, t_vals=None):
    if case["z_vals"] is not None:
        return case["z_vals"]
    return z_sample(case["near"], case["far"], case["S"], t_vals, case["t_rand"])


def disp_tie_case(n=64, S=8):
    """disp_map's max(1e-10, depth / acc) at its kink: one opaque first sample (alpha = 1 in float32, w = 1) at depth 1e-10f,
    every other sample empty, so depth / acc == 1e-10f exactly (torch hands half the gradient to each side); rays with the
    first depth at 1e-12 sit below the kink (no gradient through depth / acc).  z_vals given."""
    rng = _rng(11)
    raw = np.zeros((n, S, 4), F32)
    raw[..., :3] = rng.normal(0, 1, size=(n, S, 3))
    raw[:, 0, 3] = 1e4
    z = np.tile(np.linspace(1.0, 2.0, S, dtype=F32), (n, 1))
    z[:, 0] = np.where(np.arange(n) % 2 == 0, F32(1e-10), F32(1e-12))
    return {"raw": raw, "near": None, "far": None, "ray_d": ray_dirs(rng, n, unit=True), "t_rand": None, "z_vals": z,
            "white_bkgd": False, "S": S, "n": n, "B": 1}


def sampler_weights(kind, N, S, rng):
    """Coarse weights (N,S) of one family: zero, onehot, alternating (every other bin empty), dyadic (powers of two), random."""
    if kind == "zero":
        return np.zeros((N, S), F32)
    if kind == "onehot":
        w = np.zeros((N, S), F32)
        w[np.arange(N), rng.integers(1, max(2, S - 1), size=N)] = 1
        return w
    if kind == "alternating":
        w = rng.uniform(0.2, 1.0, size=(N, S)).astype(F32)
        w[:, ::2] = 0
        return w
    if kind == "dyadic":
        return (2.0 ** -rng.integers(0, 6, size=(N, S))).astype(F32)
    return rng.uniform(0.1, 1.0, size=(N, S)).astype(F32)


def sampler_case(S, Ni, n, kind, u_mode, seed, jitter=False, t_vals=False, tied=False):
    """Inputs of one nb_sample_pdf run.  u_mode: 'det' (linspace), 'rand', 'cdf' (u set to the emulated CDF values, cycled,
    so searchsorted meets exact ties), 'ends' (u in {0, 1} alternately).  tied: near == far (every depth equal)."""
    rng = _rng(seed)
    near = rng.uniform(0.5, 2.0, size=n).astype(F32)
    far = near.copy() if tied else (near + rng.uniform(0.5, 3.0, size=n)).astype(F32)
    w = sampler_weights(kind, n, S, rng)
    tv = np.linspace(0, 1, S, dtype=np.float64).astype(F32) if t_vals else None
    tr = rng.uniform(0, 1, size=(n, S)).astype(F32) if jitter else None
    u = None
    if u_mode == "rand":
        u = rng.uniform(0, 1, size=(n, Ni)).astype(F32)
    elif u_mode == "ends":
        u = np.tile((np.arange(Ni) % 2).astype(F32), (n, 1))
    elif u_mode == "cdf":
        cdf = sample_pdf_emulate(near, far, w, S, 1, tv, tr, np.zeros((n, 1), F32))["cdf"]
        idx = (np.arange(Ni)[None] + rng.integers(0, S, size=(n, 1))) % (S - 1)
        u = np.take_along_axis(cdf, idx, 1).astype(F32)
    return {"near": near, "far": far, "weights": w, "t_vals": tv, "t_rand": tr, "u": u, "S": S, "Ni": Ni, "n": n}
