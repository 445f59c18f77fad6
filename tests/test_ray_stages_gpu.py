"""GPU: the per-ray stages around the decoder, driven directly on inputs built to hit their edges (oracle/ray_stages.py).

  - compositing (composite_kernel through nb_debug_composite): every map and weight per element against float64
    raw2outputs, at a bound built from the float64 terms of that element (oracle.ray_stages.composite_bounds); disp_map
    with the NaN pattern of the same graph run in float32; the same bits as nb_render_fwd on a golden scene;
  - its backward (composite_bwd_kernel / ray_grad_kernel through nb_debug_composite_bwd): d raw for each map cotangent
    alone and all five together, and d ray_o / d ray_d / d near / d far / d z with a random and a zero per-sample record,
    against float64 autograd; exact zeros where sigma <= 0, NaN exactly where float32 autograd has NaN;
  - the importance sampler (nb_sample_pdf / nb_sample_pdf_src): z_out and z_samples bit for bit against the float32
    emulation of the kernel, within 2e-5 of float64 where every bin has mass, and the origin of every sorted entry.

Each bound is reported as err / bound; the worst over a family is printed.  On one H100 SXM (80 GB, default power limit)
the worst ratios observed over the whole grid were:
  forward   weights 0.047, rgb_map 0.020, depth_map 0.017, acc_map 0.015, disp_map 0.0024;
  backward  d raw 0.26 (any single cotangent), 0.09 (all five together);
  rays      d ray_o 0.0057, d ray_d 0.081, d z 0.13, d near 0.0084, d far 0.0045;
  sampler   bit for bit against the emulation everywhere; 8.9e-6 against float64 where every bin has mass (gate 2e-5).
No bound was loosened past its rounding argument (oracle.ray_stages.composite_bounds / composite_bwd_bounds)."""
import ctypes

import numpy as np
import pytest
import torch

from neuralbody_b200 import capi
from oracle import ray_stages as RS

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS = RS.EPS32
SAMPLES_FWD = [1, 2, 31, 32, 33, 64, 255, 256, 1024]
SAMPLES_BWD = [1, 2, 31, 32, 33, 64, 255, 256]
RAYS = [1, 7, 8, 9, 1000]
COTANGENTS = [("rgb",), ("depth",), ("acc",), ("disp",), ("weights",), ("rgb", "depth", "acc", "disp", "weights")]


def _lib():
    return capi.load()


def _dev(x, dtype=torch.float32):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(dtype).cuda()


def _ptr(t):
    return None if t is None else t.data_ptr()


def _options(iS, iN):
    """The grid's other axes, cycled over (S, n) so that every value meets many sizes."""
    k = iS + 2 * iN
    return {"B": 3 if (iS + iN) % 2 else 1, "jitter": k % 3 == 1, "z_user": k % 3 == 2, "white_bkgd": (iS + iN) % 4 >= 2,
            "strided": iN % 2 == 1, "t_vals": iS % 2 == 1}


def _t_vals(S, given):
    return torch.linspace(0., 1., steps=S).numpy() if given else None


class _Call:
    """The device side of one nb_debug_composite(_bwd) call on a case: rays, depths, outputs (kept alive here)."""

    def __init__(self, case, t_vals=None, strided=False):
        B, n, S = case["B"], case["n"], case["S"]
        N = B * n
        self.N, self.S = N, S
        self.raw = _dev(case["raw"])
        self.ray_o = torch.zeros(N, 3, device="cuda")
        self.ray_d = _dev(case["ray_d"])
        self.near = _dev(case["near"] if case["near"] is not None else np.zeros(N, F32))
        self.far = _dev(case["far"] if case["far"] is not None else np.zeros(N, F32))
        self.tv, self.tr, self.zv = _dev(t_vals), _dev(case["t_rand"]), _dev(case["z_vals"])
        if strided:
            self.slab = torch.full((N, 7), -7.0, device="cuda")
            self.rgb, self.disp, self.acc, self.depth = (self.slab[:, 0:3], self.slab[:, 3], self.slab[:, 4], self.slab[:, 5])
        else:
            self.rgb = torch.full((N, 3), -7.0, device="cuda")
            self.disp, self.acc, self.depth = (torch.full((N,), -7.0, device="cuda") for _ in range(3))
        self.weights = torch.full((N, S), -7.0, device="cuda")
        a = capi.nb_render_args()
        a.batch, a.n_rays, a.n_samples = B, n, S
        a.ray_o, a.ray_d, a.near, a.far = _ptr(self.ray_o), _ptr(self.ray_d), _ptr(self.near), _ptr(self.far)
        a.t_vals, a.t_rand, a.z_vals = _ptr(self.tv), _ptr(self.tr), _ptr(self.zv)
        a.rgb_map, a.disp_map, a.acc_map, a.depth_map = (_ptr(self.rgb), _ptr(self.disp), _ptr(self.acc), _ptr(self.depth))
        a.weights = _ptr(self.weights)
        a.out_ray_stride = 7 if strided else 0
        a.white_bkgd = int(case["white_bkgd"])
        self.args = a

    def forward(self):
        capi.check(_lib().nb_debug_composite(ctypes.byref(self.args), _ptr(self.raw), None), "nb_debug_composite")
        torch.cuda.synchronize()
        return {"rgb_map": self.rgb.cpu().double().numpy(), "disp_map": self.disp.cpu().double().numpy(),
                "acc_map": self.acc.cpu().double().numpy(), "depth_map": self.depth.cpu().double().numpy(),
                "weights": self.weights.cpu().double().numpy()}

    def backward(self, cot, rec=None, want=()):
        c = {k: _dev(v) for k, v in cot.items()}
        d_raw = torch.full((self.N, self.S, 4), -7.0, device="cuda")
        g = capi.nb_render_input_grads()
        outs = {}
        for k, n3 in (("d_ray_o", 3), ("d_ray_d", 3), ("d_near", 0), ("d_far", 0), ("d_z_vals", -1)):
            if k in want:
                outs[k] = torch.zeros((self.N, n3) if n3 > 0 else (self.N, self.S) if n3 < 0 else (self.N,), device="cuda")
                setattr(g, k, outs[k].data_ptr())
        r = _dev(rec)
        st = _lib().nb_debug_composite_bwd(ctypes.byref(self.args), _ptr(self.raw), _ptr(c.get("rgb")), _ptr(c.get("depth")),
                                           _ptr(c.get("acc")), _ptr(c.get("disp")), _ptr(c.get("weights")), _ptr(r),
                                           ctypes.byref(g), _ptr(d_raw), None)
        capi.check(st, "nb_debug_composite_bwd")
        torch.cuda.synchronize()
        res = {k: v.cpu().double().numpy() for k, v in outs.items()}
        res["d_raw"] = d_raw.cpu().double().numpy()
        return res


def _ratio(got, ref, tol, mask=None):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = np.abs(got - ref)
    r = err / tol
    if mask is not None:
        r = np.where(mask, r, 0)
    return float(np.nanmax(r)) if r.size else 0.0


def _worst(tag, d):
    print(tag, {k: "%.3g" % v for k, v in d.items()})


def _ref_args(case, t_vals):
    return dict(near=case["near"], far=case["far"], S=case["S"], t_vals=t_vals, t_rand=case["t_rand"], z_vals=case["z_vals"],
                white_bkgd=case["white_bkgd"])


def _check_forward(case, out, t_vals, tag):
    z = RS.case_depths(case, t_vals)
    m64, _ = RS.composite_reference(case["raw"], case["ray_d"], **_ref_args(case, t_vals))
    m32, _ = RS.composite_reference(case["raw"], case["ray_d"], dtype=torch.float32, **_ref_args(case, t_vals))
    b = RS.composite_bounds(case["raw"], z, case["ray_d"], case["white_bkgd"])
    worst = {}
    for k in ("weights", "rgb_map", "acc_map", "depth_map"):
        assert np.isfinite(out[k]).all(), (tag, k)
        worst[k] = _ratio(out[k], m64[k], b[k])
        assert worst[k] <= 1, (tag, k, worst[k])
    # disp_map: NaN exactly where float32 raw2outputs has NaN; elsewhere the relative error of depth / acc
    nan32 = np.isnan(m32["disp_map"])
    assert np.array_equal(np.isnan(out["disp_map"]), nan32), tag
    ok = ~nan32 & np.isfinite(m64["disp_map"])
    with np.errstate(all="ignore"):
        rel = b["depth_map"] / np.abs(m64["depth_map"]) + b["acc_map"] / m64["acc_map"] + 8 * EPS
        tol = np.abs(m64["disp_map"]) * 4 * rel + 1e-30
    worst["disp_map"] = _ratio(out["disp_map"], m64["disp_map"], tol, ok)
    assert worst["disp_map"] <= 1, (tag, worst["disp_map"])
    return worst


@pytest.mark.parametrize("n", RAYS)
@pytest.mark.parametrize("S", SAMPLES_FWD)
def test_composite_forward_vs_float64(S, n):
    o = _options(SAMPLES_FWD.index(S), RAYS.index(n))
    if S == 1024 and n == 1000:
        o["B"] = 1
    case = RS.composite_case(S, n, o["B"], seed=100 + S + n, jitter=o["jitter"], z_user=o["z_user"], white_bkgd=o["white_bkgd"])
    tv = _t_vals(S, o["t_vals"])
    out = _Call(case, tv, o["strided"]).forward()
    _worst("fwd S=%d n=%d %s" % (S, n, o), _check_forward(case, out, tv, (S, n)))


def test_composite_matches_the_render_on_a_golden_scene():
    """nb_render_fwd (tensor cores, skip_empty) with `raw`, then those records through nb_debug_composite: the same bits in
    every map and weight.  The entry point runs the product path's own compositing."""
    from conftest import golden_case
    import gpu_utils as G
    from neuralbody_b200.lib.config import cfg
    scene, rkw, _ = golden_case("eval_s64")
    S = rkw.get("n_samples", 64)
    out = G.render_product(scene, n_samples=S, precision="tc_fp16x3", want_raw=True)
    B, n = scene["ray_o"].shape[:2]
    case = {"raw": out["raw"].reshape(B * n, S, 4).numpy(), "ray_d": scene["ray_d"].reshape(B * n, 3).numpy(),
            "near": scene["near"].reshape(-1).numpy(), "far": scene["far"].reshape(-1).numpy(), "t_rand": None, "z_vals": None,
            "white_bkgd": bool(cfg.white_bkgd), "S": S, "n": n, "B": B}
    mine = _Call(case, torch.linspace(0., 1., steps=S).numpy()).forward()
    for k in ("rgb_map", "disp_map", "acc_map", "depth_map", "weights"):
        ref = out[k].reshape(mine[k].shape).double().numpy()
        assert np.array_equal(np.nan_to_num(ref, nan=-1.0), np.nan_to_num(mine[k], nan=-1.0)), k


def _cotangents(keys, N, S, seed):
    rng = np.random.default_rng(seed)
    c = {}
    for k in keys:
        shape = {"rgb": (N, 3), "weights": (N, S)}.get(k, (N,))
        c[k] = rng.normal(size=shape).astype(F32) * (1e-2 if k == "disp" else 1.0)
    return c


def _check_d_raw(case, t_vals, cot, got, tag):
    z = RS.case_depths(case, t_vals)
    m64, g64 = RS.composite_reference(case["raw"], case["ray_d"], cot=cot, **_ref_args(case, t_vals))
    _, g32 = RS.composite_reference(case["raw"], case["ray_d"], cot=cot, dtype=torch.float32, **_ref_args(case, t_vals))
    b = RS.composite_bounds(case["raw"], z, case["ray_d"])
    tb = RS.composite_bwd_bounds(case["raw"], z, case["ray_d"], cot, b, m64["depth_map"], m64["acc_map"])
    d = got["d_raw"]
    assert np.array_equal(np.isnan(d), np.isnan(g32["d_raw"])), tag
    assert np.all(d[..., 3][case["raw"][..., 3] <= 0] == 0), tag            # relu: exact zeros, never -0 or NaN
    ok = np.isfinite(g64["d_raw"]) & np.isfinite(g32["d_raw"])
    assert np.isfinite(d[ok]).all(), tag
    r = _ratio(d, g64["d_raw"], tb["d_raw"], ok)
    assert r <= 1, (tag, r)
    return r, (m64, g64, b, tb)


@pytest.mark.parametrize("n", RAYS)
@pytest.mark.parametrize("S", SAMPLES_BWD)
def test_composite_backward_vs_float64(S, n):
    o = _options(SAMPLES_BWD.index(S), RAYS.index(n))
    if n == 1000:
        o["B"] = 1
    case = RS.composite_case(S, n, o["B"], seed=200 + S + n, jitter=o["jitter"], z_user=o["z_user"])
    tv = _t_vals(S, o["t_vals"])
    call = _Call(case, tv, o["strided"])
    worst = {}
    for i, keys in enumerate(COTANGENTS):
        cot = _cotangents(keys, case["B"] * n, S, seed=S * 7 + n + i)
        got = call.backward(cot)
        worst["+".join(keys) if len(keys) < 5 else "all"], _ = _check_d_raw(case, tv, cot, got, (S, n, keys))
    _worst("bwd S=%d n=%d %s" % (S, n, o), worst)


def test_disp_map_kink_takes_torchs_half_gradient():
    """depth / acc == 1e-10f exactly (and below it): d z through disp_map is torch's maximum backward in float32 -- half the
    gradient at the tie, none below.  float64 cannot tie there (1e-10 is not 1e-10f), so float32 autograd is the reference."""
    case = RS.disp_tie_case()
    N, S = case["n"], case["S"]
    cot = {"disp": np.full(N, 1e-20, F32)}
    got = _Call(case).backward(cot, rec=np.zeros((N, S, 8), F32), want=("d_z_vals", "d_ray_d"))
    _, g32 = RS.composite_reference(case["raw"], case["ray_d"], z_vals=case["z_vals"], cot=cot,
                                    rec=np.zeros((N, S, 8), F32), dtype=torch.float32)
    dz, ref = got["d_z_vals"], g32["d_z"]
    assert np.all(ref[::2, 0] != 0) and np.all(ref[1::2, 0] == 0)
    assert np.allclose(dz, ref, rtol=1e-5, atol=0), np.abs(dz - ref).max()
    assert np.allclose(got["d_raw"], g32["d_raw"], rtol=1e-5, atol=1e-30)


@pytest.mark.parametrize("record", ["random", "zero"])
@pytest.mark.parametrize("jitter", [False, True])
@pytest.mark.parametrize("S,n", [(1, 9), (2, 7), (31, 8), (33, 9), (64, 1000), (256, 7)])
def test_ray_and_depth_gradients_vs_float64(S, n, jitter, record):
    """d ray_o, d ray_d, d near, d far and d z against float64 autograd through p = o + z d, d / |d| and raw2outputs, with
    every map cotangent.  The record stands in for the decoder's d loss / d(world point, view direction)."""
    B = 3 if n < 100 else 1
    N = B * n
    case = RS.composite_case(S, n, B, seed=300 + S + n + jitter, jitter=jitter)
    cot = _cotangents(COTANGENTS[-1], N, S, seed=S + n)
    rng = np.random.default_rng(S * n)
    rec = rng.normal(size=(N, S, 8)).astype(F32) if record == "random" else np.zeros((N, S, 8), F32)
    rec[..., 6:] = 0
    got = _Call(case).backward(cot, rec=rec, want=("d_ray_o", "d_ray_d", "d_near", "d_far", "d_z_vals"))
    r_draw, (m64, g64, b, tb) = _check_d_raw(case, None, cot, got, (S, n))
    _, g32 = RS.composite_reference(case["raw"], case["ray_d"], cot=cot, rec=rec, dtype=torch.float32, **_ref_args(case, None))
    _, g64 = RS.composite_reference(case["raw"], case["ray_d"], cot=cot, rec=rec, **_ref_args(case, None))
    z = RS.case_depths(case).astype(np.float64)
    rd = case["ray_d"].astype(np.float64)
    nrm = np.linalg.norm(rd, axis=1)
    r64 = rec.astype(np.float64)
    sg = np.maximum(case["raw"][..., 3].astype(np.float64), 0)
    # terms of each gradient in absolute value; the compositing part through the bounds of dalpha
    c_abs = np.abs(g64["d_raw"][..., 3]) * sg / np.where(b["dist"] > 0, b["dist"], np.inf)
    c_err = tb["dalpha"] * sg * tb["e"] + 8 * EPS * c_abs
    red = 8 * EPS * (S + 8)
    tols = {
        "d_ray_o": red * np.abs(r64[..., :3]).sum(1) + 1e-30,
        "d_ray_d": (red * ((np.abs(z)[..., None] * np.abs(r64[..., :3])).sum(1) + 3 * np.abs(r64[..., 3:6]).sum(1)
                           / nrm[:, None]) + ((c_err + red * c_abs) * b["dist"] / nrm[:, None]).sum(1)[:, None] + 1e-30),
    }
    dz_abs = (np.abs(r64[..., :3]) * np.abs(rd)[:, None]).sum(-1)
    dD = tb["dD_abs"][:, None]
    prev = np.concatenate([np.zeros((N, 1)), c_err[:, :-1]], 1)
    cur = np.concatenate([c_err[:, :-1], np.zeros((N, 1))], 1)
    t_dz = (8 * EPS * (dz_abs + dD * b["w"]) + dD * b["weights"] + tb["dD_err"][:, None] * b["w"]
            + nrm[:, None] * (prev + cur) + 1e-30)
    tols["d_z_vals"] = t_dz
    tols["d_near"] = t_dz.sum(1) + red * np.abs(g64["d_z"]).sum(1) + 1e-30
    tols["d_far"] = tols["d_near"]
    refs = {"d_ray_o": g64["d_ray_o"], "d_ray_d": g64["d_ray_d"], "d_z_vals": g64["d_z"], "d_near": g64["d_near"],
            "d_far": g64["d_far"]}
    refs32 = {"d_ray_o": g32["d_ray_o"], "d_ray_d": g32["d_ray_d"], "d_z_vals": g32["d_z"]}
    worst = {"d_raw": r_draw}
    for k, ref in refs.items():
        mine = got[k]
        if k in refs32:
            assert np.array_equal(np.isnan(mine), np.isnan(refs32[k])), k
        ok = np.isfinite(ref) & np.isfinite(mine)
        if k in refs32:
            ok &= np.isfinite(refs32[k])
        worst[k] = _ratio(mine, ref, tols[k], ok)
        assert worst[k] <= 1, (k, worst[k])
    _worst("rays S=%d n=%d jitter=%s rec=%s" % (S, n, jitter, record), worst)


# ---------------------------------------------------------------------------------------------- the importance sampler
FAMILIES = [("zero", "det", False), ("onehot", "rand", False), ("alternating", "cdf", False), ("dyadic", "cdf", False),
            ("random", "ends", False), ("random", "rand", False), ("random", "det", True)]


def _run_sampler(c, src=False):
    n, S, Ni = c["n"], c["S"], c["Ni"]
    near, far, w = _dev(c["near"]), _dev(c["far"]), _dev(c["weights"])
    tv, tr, u = _dev(c["t_vals"]), _dev(c["t_rand"]), _dev(c["u"])
    z_out = torch.full((n, S + Ni), -7.0, device="cuda")
    z_smp = torch.full((n, Ni), -7.0, device="cuda")
    a = capi.nb_importance_args()
    a.n_rays_total, a.n_samples, a.n_importance = n, S, Ni
    a.near, a.far, a.t_vals, a.t_rand, a.weights, a.u = _ptr(near), _ptr(far), _ptr(tv), _ptr(tr), _ptr(w), _ptr(u)
    a.z_out, a.z_samples = _ptr(z_out), _ptr(z_smp)
    zsrc = torch.full((n, S + Ni), -9, dtype=torch.int32, device="cuda") if src else None
    st = _lib().nb_sample_pdf_src(ctypes.byref(a), _ptr(zsrc), None) if src else _lib().nb_sample_pdf(ctypes.byref(a), None)
    capi.check(st, "nb_sample_pdf")
    torch.cuda.synchronize()
    return z_out.cpu().numpy(), z_smp.cpu().numpy(), None if zsrc is None else zsrc.cpu().numpy()


@pytest.mark.parametrize("total", ["S+1", 257, 511, 512])
@pytest.mark.parametrize("S", [3, 4, 33, 64, 255, 256])
def test_sample_pdf_bit_exact_vs_emulation(S, total):
    from oracle import neuralbody_oracle as O
    Ni = 1 if total == "S+1" else total - S
    worst64 = 0.0
    for i, (kind, u_mode, tied) in enumerate(FAMILIES):
        n = (1, 5, 4097)[(i + S) % 3]
        jitter, tv = i % 2 == 1, (i + S) % 2 == 0
        c = RS.sampler_case(S, Ni, n, kind, u_mode, seed=S * 31 + Ni + i, jitter=jitter, t_vals=tv, tied=tied)
        em = RS.sample_pdf_emulate(c["near"], c["far"], c["weights"], S, Ni, c["t_vals"], c["t_rand"], c["u"])
        z_out, z_smp, _ = _run_sampler(c)
        tag = (S, Ni, n, kind, u_mode, tied)
        assert np.array_equal(z_out.view(np.int32), em["z_out"].view(np.int32)), tag
        assert np.array_equal(z_smp.view(np.int32), em["z_samples"].view(np.int32)), tag
        z2, _, src = _run_sampler(c, src=True)
        assert np.array_equal(z2.view(np.int32), z_out.view(np.int32)), tag
        # every coarse index once, at a position holding that coarse depth; the rest importance samples (-1)
        assert np.array_equal(np.sort(src, 1), np.concatenate([np.full((n, Ni), -1), np.tile(np.arange(S), (n, 1))], 1)), tag
        pos = src >= 0
        assert np.array_equal(np.take_along_axis(em["zc"], np.maximum(src, 0), 1)[pos], z_out[pos]), tag
        if kind == "random" and u_mode == "rand":     # every bin has mass: the inverse CDF is well conditioned
            z64, s64 = O.importance_z_vals(torch.from_numpy(em["zc"]).double(), torch.from_numpy(c["weights"]).double(), Ni,
                                           det=False, u=torch.from_numpy(c["u"]).double())
            d = max(float(np.abs(z_out - z64.numpy()).max()), float(np.abs(z_smp - s64.numpy()).max()))
            assert d < 2e-5, (tag, d)
            worst64 = max(worst64, d)
    print("sampler S=%d Ni=%d: bit-exact; worst vs float64 %.3g" % (S, Ni, worst64))
