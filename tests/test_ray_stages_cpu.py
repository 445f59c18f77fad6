"""CPU: the references of tests/test_ray_stages_gpu.py (oracle/ray_stages.py) against the plain oracle, every designed case
really containing its edge, and the argument checks of the two compositing diagnostics (nb_debug_composite /
nb_debug_composite_bwd) and of the sampler's size limits, which reject a call before it enqueues anything."""
import ctypes

import numpy as np
import pytest
import torch

from neuralbody_b200 import capi
from oracle import neuralbody_oracle as O
from oracle import ray_stages as RS

F32 = np.float32


@pytest.mark.parametrize("S", [1, 2, 3, 31, 32, 33, 64, 255, 256, 1024])
def test_linspace01_is_the_kernels_symmetric_fill(S):
    """step * i below the midpoint, 1 - step * (S - 1 - i) above it, each op rounded to float32: exact at both ends and
    within an ulp of torch.linspace (whose vectorised CPU fill steps upwards from the midpoint, so a few entries differ)."""
    t = RS.linspace01(np.arange(S), S)
    assert t[0] == 0 and (S == 1 or t[-1] == 1)
    assert np.all(np.abs(t - torch.linspace(0., 1., steps=S).numpy()) <= np.spacing(F32(1)))
    if S > 1:
        step = F32(1) / F32(S - 1)
        i = np.arange(S)
        assert np.array_equal(t[i < S // 2], (step * i[i < S // 2].astype(F32)).astype(F32))


@pytest.mark.parametrize("jitter", [False, True])
def test_z_sample_matches_the_oracle_sampling(jitter):
    rng = np.random.default_rng(3)
    n, S = 50, 33
    near = rng.uniform(0.5, 2, n).astype(F32)
    far = (near + rng.uniform(0.5, 3, n)).astype(F32)
    tr = rng.uniform(0, 1, (n, S)).astype(F32) if jitter else None
    _, z = O.get_sampling_points(torch.zeros(1, n, 3), torch.ones(1, n, 3), torch.from_numpy(near)[None],
                                 torch.from_numpy(far)[None], S, perturb=1.0 if jitter else 0.0, training=jitter,
                                 t_rand=None if tr is None else torch.from_numpy(tr)[None])
    mine = RS.z_sample(near, far, S, None, tr)
    assert np.abs(mine - z[0].numpy()).max() <= 4e-7 * np.abs(far).max()
    # the float64 twin has the same value and the formula's derivative
    nr, fr = torch.from_numpy(near).double().requires_grad_(True), torch.from_numpy(far).double().requires_grad_(True)
    z64 = RS.z_sample_torch64(nr, fr, S, None, tr)
    assert np.array_equal(z64.detach().numpy(), mine.astype(np.float64))
    z64[:, S // 2].sum().backward()
    t = RS.linspace01(np.arange(S), S).astype(np.float64)[S // 2]
    if not jitter:
        assert np.allclose(nr.grad.numpy(), 1 - t) and np.allclose(fr.grad.numpy(), t)


@pytest.mark.parametrize("det", [True, False])
def test_sampler_emulation_matches_the_oracle_well_conditioned(det):
    """Every bin has mass: the emulation (the kernel's summation order) and oracle.importance_z_vals (torch's) agree to
    rounding, and the emulated CDF is torch's cumsum of the pdf to rounding."""
    rng = np.random.default_rng(4)
    n, S, Ni = 200, 48, 77
    near = rng.uniform(1, 2, n).astype(F32)
    far = (near + 1 + rng.uniform(0, 1, n)).astype(F32)
    w = rng.uniform(0.1, 1.0, (n, S)).astype(F32)
    tr = None if det else rng.uniform(0, 1, (n, S)).astype(F32)
    u = None if det else rng.uniform(0, 1, (n, Ni)).astype(F32)
    em = RS.sample_pdf_emulate(near, far, w, S, Ni, None, tr, u)
    z = torch.from_numpy(RS.z_sample(near, far, S, None, tr))
    z_ref, s_ref = O.importance_z_vals(z, torch.from_numpy(w), Ni, det=det, u=None if u is None else torch.from_numpy(u))
    assert np.abs(em["z_out"] - z_ref.numpy()).max() < 2e-5
    assert np.abs(em["z_samples"] - s_ref.numpy()).max() < 2e-5
    pdf = (w[:, 1:-1] + 1e-5) / (w[:, 1:-1] + 1e-5).sum(1, keepdims=True)
    assert np.abs(em["cdf"][:, 1:] - np.cumsum(pdf, 1)).max() < 1e-6


def test_sampler_cases_contain_their_edges():
    # u exactly on a CDF value, with an empty bin on its left (searchsorted's side decides the sample) ...
    c = RS.sampler_case(64, 64, 64, "alternating", "cdf", seed=1)
    em = RS.sample_pdf_emulate(c["near"], c["far"], c["weights"], 64, 64, None, None, c["u"])
    on_cdf = np.array([[np.any(em["cdf"][r] == x) for x in em["u"][r]] for r in range(64)])
    assert on_cdf.all()
    lo = em["lo"]
    left_gap = np.take_along_axis(em["cdf"], np.clip(lo - 1, 0, 62), 1) - np.take_along_axis(em["cdf"], np.clip(lo - 2, 0, 62), 1)
    assert ((left_gap < 1e-5) & (lo >= 2)).any()
    # ... the `denom < 1e-5 -> 1` branch inside the CDF (one-hot: the empty bins' mass is 1e-5 / (1 + ...) < 1e-5) ...
    c = RS.sampler_case(64, 64, 64, "onehot", "rand", seed=2)
    em = RS.sample_pdf_emulate(c["near"], c["far"], c["weights"], 64, 64, None, None, c["u"])
    inner = em["denom_branch"] & (em["lo"] > 0) & (em["lo"] < 63)
    assert inner.any()
    # ... u = 0 and u = 1 (past the last CDF value: below == above) ...
    c = RS.sampler_case(33, 4, 16, "random", "ends", seed=3)
    em = RS.sample_pdf_emulate(c["near"], c["far"], c["weights"], 33, 4, None, None, c["u"])
    assert (em["u"] == 0).any() and (em["u"] == 1).any() and (em["lo"] == 32).any()
    # ... all-zero weights (uniform pdf) and near == far (every depth tied, every bin of zero width)
    c = RS.sampler_case(16, 8, 8, "zero", "det", seed=4, tied=True)
    em = RS.sample_pdf_emulate(c["near"], c["far"], c["weights"], 16, 8)
    z = em["z_out"].astype(np.float64)
    assert (np.diff(em["z_out"], axis=1) == 0).any() and np.all(z.max(1) - z.min(1) <= 4 * np.spacing(em["z_out"].max(1)))
    assert not em["denom_branch"][:, 1:-1].any()          # uniform pdf: every inner bin has 1 / 14 of the mass


def test_composite_cases_contain_their_edges():
    c = RS.composite_case(64, 64, 1, seed=5, z_user=True)
    z = RS.case_depths(c)
    m, _ = RS.composite_reference(c["raw"], c["ray_d"], z_vals=z, white_bkgd=False)
    m32, _ = RS.composite_reference(c["raw"], c["ray_d"], z_vals=z, dtype=torch.float32)
    b = RS.composite_bounds(c["raw"], z, c["ray_d"])
    kind = np.arange(64) % 8
    # saturating alpha: transmittance below the smallest normal float32 before the last sample, and 0 in float32
    assert (b["T"][kind == 1, -1] < 2.0 ** -126).all()
    w32 = m32["weights"]
    assert (w32[kind == 1, -1] == 0).all()
    # the 1e10 last interval decides the output: sigma * 1e10 |d| of order 1
    x = c["raw"][kind == 0, -1, 3].astype(np.float64) * 1e10 * np.linalg.norm(c["ray_d"][kind == 0], axis=1)
    assert (x > 0.05).all() and (x < 100).all() and ((x > 0.1) & (x < 10)).mean() >= 0.5
    assert (m["acc_map"][kind == 0] > 0.04).all()
    # acc = 0 -> disp NaN; sigma exactly 0 and negative; zero-length intervals
    assert np.isnan(m32["disp_map"][kind == 2]).all() and (m32["acc_map"][kind == 2] == 0).all()
    assert (c["raw"][kind == 3, :, 3] == 0).any() and (c["raw"][kind == 3, :, 3] < 0).any()
    assert (np.diff(z[kind == 4], axis=1) == 0).any()
    c = RS.composite_case(33, 16, 1, seed=6)
    assert (c["near"][np.arange(16) % 8 == 5] == c["far"][np.arange(16) % 8 == 5]).all()
    # disp_map's kink: depth / acc == 1e-10f exactly in float32, and below it
    c = RS.disp_tie_case()
    m32, _ = RS.composite_reference(c["raw"], c["ray_d"], z_vals=c["z_vals"], dtype=torch.float32)
    q = m32["depth_map"].astype(F32) / m32["acc_map"].astype(F32)
    assert (q[::2] == F32(1e-10)).all() and (q[1::2] < F32(1e-10)).all()


def test_composite_reference_gradient_vs_finite_differences():
    """The float64 graph itself: d raw, d ray_d and d near / d far by central differences on well-conditioned samples."""
    c = RS.composite_case(12, 16, 1, seed=7, jitter=True)
    keep = np.arange(16) % 8 >= 6             # moderate sigma, unit and non-unit directions: no edge on these rays
    c = {k: (v[keep] if isinstance(v, np.ndarray) else v) for k, v in c.items()}
    N = int(keep.sum())
    rng = np.random.default_rng(8)
    cot = {"rgb": rng.normal(size=(N, 3)), "depth": rng.normal(size=N), "acc": rng.normal(size=N),
           "disp": rng.normal(size=N) * 1e-2, "weights": rng.normal(size=(N, 12))}
    rec = rng.normal(size=(N, 12, 8))

    def loss(raw, ray_d, near, far):
        nr, fr = torch.from_numpy(near), torch.from_numpy(far)
        z = RS.z_sample_torch64(nr, fr, 12, None, c["t_rand"])
        t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in cot.items()}
        rgb, disp, acc, w, depth = O.raw2outputs(torch.from_numpy(raw), z, torch.from_numpy(ray_d))
        r = torch.from_numpy(rec)
        pts = torch.from_numpy(ray_d)[:, None] * z[..., None]
        vd = torch.from_numpy(ray_d) / torch.norm(torch.from_numpy(ray_d), dim=-1, keepdim=True)
        return float((t["rgb"] * rgb).sum() + (t["depth"] * depth).sum() + (t["acc"] * acc).sum() + (t["disp"] * disp).sum()
                     + (t["weights"] * w).sum() + (r[..., :3] * pts).sum() + (r[..., 3:6].sum(1) * vd).sum())

    _, g = RS.composite_reference(c["raw"], c["ray_d"], c["near"], c["far"], 12, None, c["t_rand"], cot=cot, rec=rec)
    raw0, rd0 = c["raw"].astype(np.float64), c["ray_d"].astype(np.float64)
    # z in the FD loss must vary with near / far: use the float64 formula alone there (z_sample_torch64 pins the value)
    def loss_nf(near, far):
        z = torch.from_numpy(RS.linspace01(np.arange(12), 12).astype(np.float64))
        nr, fr = torch.from_numpy(near), torch.from_numpy(far)
        zz = nr[:, None] * (1 - z) + fr[:, None] * z
        tr = torch.from_numpy(c["t_rand"].astype(np.float64))
        mids = .5 * (zz[:, 1:] + zz[:, :-1])
        zz = torch.cat([zz[:, :1], mids], 1) + (torch.cat([mids, zz[:, -1:]], 1) - torch.cat([zz[:, :1], mids], 1)) * tr
        t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in cot.items()}
        rgb, disp, acc, w, depth = O.raw2outputs(torch.from_numpy(raw0), zz, torch.from_numpy(rd0))
        r = torch.from_numpy(rec)
        pts = torch.from_numpy(rd0)[:, None] * zz[..., None]
        return float((t["rgb"] * rgb).sum() + (t["depth"] * depth).sum() + (t["acc"] * acc).sum() + (t["disp"] * disp).sum()
                     + (t["weights"] * w).sum() + (r[..., :3] * pts).sum())

    h = 1e-6
    for ray in range(3):
        for s in (0, 5, 10):
            for ch in (0, 3):
                if ch == 3 and raw0[ray, s, 3] <= 0.05:
                    continue
                p, m = raw0.copy(), raw0.copy()
                p[ray, s, ch] += h
                m[ray, s, ch] -= h
                fd = (loss(p, rd0, c["near"].astype(np.float64), c["far"].astype(np.float64))
                      - loss(m, rd0, c["near"].astype(np.float64), c["far"].astype(np.float64))) / (2 * h)
                assert abs(fd - g["d_raw"][ray, s, ch]) <= 1e-5 * (1 + abs(fd)), (ray, s, ch, fd, g["d_raw"][ray, s, ch])
        for k in range(3):
            p, m = rd0.copy(), rd0.copy()
            p[ray, k] += h
            m[ray, k] -= h
            fd = (loss(raw0, p, c["near"].astype(np.float64), c["far"].astype(np.float64))
                  - loss(raw0, m, c["near"].astype(np.float64), c["far"].astype(np.float64))) / (2 * h)
            assert abs(fd - g["d_ray_d"][ray, k]) <= 1e-5 * (1 + abs(fd)), (ray, k, fd, g["d_ray_d"][ray, k])
        nf = (c["near"].astype(np.float64), c["far"].astype(np.float64))
        for which, key in ((0, "d_near"), (1, "d_far")):
            p, m = [x.copy() for x in nf], [x.copy() for x in nf]
            p[which][ray] += h
            m[which][ray] -= h
            fd = (loss_nf(*p) - loss_nf(*m)) / (2 * h)
            assert abs(fd - g[key][ray]) <= 1e-5 * (1 + abs(fd)), (ray, key, fd, g[key][ray])


# ---------------------------------------------------------------------------------------------- argument checks
FAKE = 0x10000      # placeholder device address, never dereferenced


def _ray_args(S=8, n=4, B=1):
    a = capi.nb_render_args()
    a.batch, a.n_rays, a.n_samples = B, n, S
    for name in ("ray_o", "ray_d", "near", "far", "rgb_map", "disp_map", "acc_map", "depth_map"):
        setattr(a, name, FAKE)
    return a


def _fwd(a, raw=FAKE):
    return capi.load().nb_debug_composite(ctypes.byref(a), raw, None)


def _bwd(a, raw=FAKE, rec=None, grads=None, d_raw=FAKE):
    return capi.load().nb_debug_composite_bwd(ctypes.byref(a), raw, FAKE, None, None, None, None, rec,
                                              None if grads is None else ctypes.byref(grads), d_raw, None)


def _err():
    return capi.load().nb_last_error().decode()


def test_debug_composite_rejects_bad_calls(built_lib):
    assert _fwd(_ray_args(S=1025)) == -2 and "n_samples <= 1024" in _err()
    assert _fwd(_ray_args(), raw=None) == -1 and _err().startswith("nb_debug_composite:")
    a = _ray_args()
    a.batch = 0
    assert _fwd(a) == -1 and "batch" in _err()
    a = _ray_args()
    a.far = None
    assert _fwd(a) == -1 and _err().startswith("nb_debug_composite:") and "null" in _err()
    a = _ray_args()
    a.n_samples = 0
    assert _fwd(a) == -1
    a = _ray_args()
    a.out_ray_stride = -1
    assert _fwd(a) == -1


def test_debug_composite_bwd_rejects_bad_calls(built_lib):
    assert _bwd(_ray_args(S=257)) == -2 and "n_samples <= 256" in _err()
    assert _bwd(_ray_args(), d_raw=None) == -1 and "d_raw" in _err()
    assert _bwd(_ray_args(), raw=None) == -1
    g = capi.nb_render_input_grads()
    g.d_ray_d = FAKE
    assert _bwd(_ray_args(), grads=g) == -1 and "record" in _err()
    g = capi.nb_render_input_grads()
    g.d_R = FAKE
    assert _bwd(_ray_args(), rec=FAKE, grads=g) == -1 and "d_R" in _err()
    g = capi.nb_render_input_grads()
    g.d_near = FAKE
    a = _ray_args()
    a.z_vals = FAKE
    assert _bwd(a, rec=FAKE, grads=g) == -1 and "z_vals" in _err()
    a = _ray_args()
    a.ray_d = None
    assert _bwd(a) == -1 and _err().startswith("nb_debug_composite_bwd:")


@pytest.mark.parametrize("S,Ni,ok", [(256, 256, True), (256, 257, False), (257, 1, False), (3, 509, True), (2, 1, False),
                                     (4, 0, False)])
def test_sampler_size_limits(built_lib, S, Ni, ok):
    """S + N_importance = 513 and S = 257 are rejected; 512 and S = 256 pass validation (and then fail on the null
    pointers, still before anything is enqueued)."""
    a = capi.nb_importance_args()
    a.n_rays_total, a.n_samples, a.n_importance = 4, S, Ni
    st = capi.load().nb_sample_pdf(ctypes.byref(a), None)
    assert st < 0
    if ok:
        assert "null" in _err(), _err()
    else:
        assert "null" not in _err(), _err()
