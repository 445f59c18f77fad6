"""Every feature-volume precision (cfg.render_volume_dtype) of the render, density and training kernels.

Each kernel that reads the packed feature volume is built twice, for an fp32 and for an fp16 blob.  Both variants widen each
corner to fp32 (load4<__half>, Quad<__half>::fma) and run the same fmaf chain, so on a volume whose values are exactly
representable in fp16 (synth.round_volumes) the two blobs hold the same numbers and the two variants must give the same bits.

TWIN tests render or query such a volume twice, with render_volume_dtype 'fp32' and 'fp16', and compare bit for bit: the
inference maps and `raw` (exact kernel, tc_fp16x3, tc_fp16; skipping on and off), the density decoder, and the training
forward.  Training gradients are accumulated with atomics, whose order changes from run to run: they must agree to
TWIN_GRAD_TOL of each slice's largest entry.  ORACLE tests hold the fp16-blob variants to the float64 oracle on the rounded
volumes at the gates of their fp32-blob twins.

Cases: the golden-sized eval_s64 scene, the B = 3 distinct-frame case (oracle/frames_case.py), their 'subnormal' variant
(level 0 scaled by 2^-20, so its non-zero values are fp16 subnormals), and the full-size 512 x 512 synth-313 view in list
order, where the decoder gathers the coarse levels from its shared-memory staging (stats[5]) for both element sizes.

Also: nb_pack_volume's fp16 rounding at its edges (ties, underflow, subnormals, -0.0, overflow) against torch's
round-to-nearest-even, and training on the exact kernel with render_volume_dtype 'fp16' (its backward reads the fp32
volume, which the renderer packs for such a call)."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import golden_case
from oracle import frames_case as FR
from oracle import neuralbody_oracle as O
from oracle import synth
import test_distinct_frames as TD

MAPS = ("rgb_map", "disp_map", "acc_map", "depth_map", "weights")
# the gather, scatter and frame-gradient kernels of the training path run min(list / 32, 132 * 8) CTAs of 32 list entries:
# a longer list wraps their grid-stride loops
GRID_ENTRIES = 132 * 8 * 32
# fp16-blob vs fp32-blob training gradients: max |a - b| <= TWIN_GRAD_TOL * max |b| per slice (the weight-gradient splits,
# the volume scatter and the frame sums add with atomics).  Measured on an H100 80GB HBM3 (700 W power limit): worst slice
# 1.4e-6 between the blobs, 2.0e-6 between two runs on the fp32 blob
TWIN_GRAD_TOL = 1e-5
# the exact kernel against the float64 oracle on per-sample raw: 2e-4 (tests/test_render_gpu.py) on the rgb logits; sigma
# (|sigma| up to ~30) reaches 2.1e-4 on the rounded eval_s64 scene, on either blob (the twin tests: the same bits)
EXACT_RAW_TOL, EXACT_SIGMA_TOL = 2e-4, 2.5e-4
FP16_MIN_NORMAL = 2.0 ** -14


@pytest.fixture(autouse=True)
def _restore_cfg():
    from neuralbody_b200.lib.config import cfg
    keys = ("render_volume_dtype", "render_precision", "render_skip_empty", "density_precision", "render_train_precision")
    old = {k: (cfg[k] if k in cfg else None) for k in keys}
    yield
    for k, v in old.items():
        if v is None:
            if k in cfg:
                del cfg[k]
        else:
            cfg[k] = v


# ------------------------------------------------------------------------------------------------------------------ cases
_SCENES = {}


def _small(subnormal=False):
    """eval_s64's scene (48 x 48 view, every 9th ray) with fp16-representable volumes."""
    return synth.rounded_scene(golden_case("eval_s64")[0], torch.float16, subnormal)


def _subnormal_only():
    """The subnormal small scene with levels 1-3 zeroed: every occupied sample's only non-zero features are fp16
    subnormals."""
    sc = _small(subnormal=True)
    sc["volumes"] = [sc["volumes"][0]] + [torch.zeros_like(v) for v in sc["volumes"][1:]]
    return sc


def scene(name):
    if name not in _SCENES:
        if name == "small":
            _SCENES[name] = _small()
        elif name == "subnormal":
            _SCENES[name] = _small(subnormal=True)
        elif name == "subnormal_only":
            _SCENES[name] = _subnormal_only()
        elif name == "frames":
            _SCENES[name] = FR.build(volume_dtype=torch.float16)[0]
        elif name == "full":
            _SCENES[name] = synth.rounded_scene(synth.make_scene(H=512, W=512, scale=1.0, all_hit=True))
        else:
            raise KeyError(name)
    return _SCENES[name]


_FR = {}


def frames_case(**kw):
    """frames_case.build(volume_dtype=fp16, **kw), cached: (scene, t_rand, G, Gm)."""
    key = tuple(sorted(kw.items()))
    if key not in _FR:
        _FR[key] = FR.build(volume_dtype=torch.float16, **kw)
    return _FR[key]


_REF = {}


def frames_reference(**kw):
    """frames_case(**kw) + the float64 oracle's (gradients, outputs) on its rounded volumes, cached."""
    key = tuple(sorted(kw.items()))
    if key not in _REF:
        sc, t_rand, G, Gm = frames_case(**kw)
        _REF[key] = (sc, t_rand, G, Gm) + FR.oracle_grads(sc, t_rand, G, Gm, kw.get("n_samples", FR.N_SAMPLES))
    return _REF[key]


def _occupied_samples(sc, t_rand=None, n_samples=64):
    """(B, n*S) bool, float64 oracle: the samples with a non-zero feature (those a kernel must list)."""
    d = FR.to_double(sc)
    if t_rand is None:
        pts, _ = O.get_sampling_points(d["ray_o"], d["ray_d"], d["near"], d["far"], n_samples)
    else:
        pts, _ = O.get_sampling_points(d["ray_o"], d["ray_d"], d["near"], d["far"], t_rand.shape[-1], 1.0, True, t_rand.double())
    B = pts.shape[0]
    sp = O.prepare_sp_input(d)
    grid = O.get_grid_coords(O.pts_to_can_pts(pts.reshape(B, -1, 3), sp["R"], sp["Th"]), sp["bounds"], sp["out_sh"],
                             d["voxel_size"])
    return (O.interpolate_features(grid, d["volumes"]) != 0).any(1)


def _is_fp16(v):
    return torch.equal(v.half().float(), v)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("subnormal", [False, True])
def test_rounded_frames_case_is_fp16_and_well_conditioned(subnormal):
    """The rounded distinct-frame case: every volume holds fp16 values only, the rounding moved the volumes (so the case was
    conditioned on other numbers than the unrounded one), and no sample that carries gradient sits near a cell face or a
    ReLU kink OF THE ROUNDED VOLUMES."""
    sc, t_rand, _, _ = frames_case(subnormal=subnormal)
    assert all(_is_fp16(v) for v in sc["volumes"])
    plain = FR.build()[0]
    assert any(not torch.equal(a, b) for a, b in zip(sc["volumes"], plain["volumes"]))
    assert not bool(FR.fragile_samples(sc, t_rand).any())


def test_subnormal_variants_hold_subnormals():
    """Level 0 of the subnormal variants: its non-zero values are fp16 subnormals (below 2^-14), and most of the unscaled
    volume's non-zero values survive the rounding (nothing is flushed wholesale); levels 1-3 are the rounded ones."""
    for sc, base in ((frames_case(subnormal=True)[0], FR.build()[0]), (scene("subnormal"), golden_case("eval_s64")[0])):
        v0, b0 = sc["volumes"][0], base["volumes"][0]
        nz = v0[v0 != 0]
        assert _is_fp16(v0) and int(nz.numel()) > 0.9 * int((b0 != 0).sum()), (int(nz.numel()), int((b0 != 0).sum()))
        assert float(nz.abs().max()) < FP16_MIN_NORMAL
        assert all(torch.equal(v, b.half().float()) for v, b in zip(sc["volumes"][1:], base["volumes"][1:]))
    only = scene("subnormal_only")
    occ = _occupied_samples(only)
    assert int(occ.sum()) > 100 and not any(bool(v.any()) for v in only["volumes"][1:])


def test_large_case_list_wraps_the_training_grids():
    """The 512-ray, S = 64 rounded case has more samples with a non-zero feature (each of which the training path lists)
    than one pass of the gather / scatter / frame-gradient grids covers."""
    sc, t_rand, _, _ = frames_case(n_samples=64, n_rays=512)
    n = int(_occupied_samples(sc, t_rand).sum())
    print("occupied samples:", n, "one grid pass:", GRID_ENTRIES)
    assert n > GRID_ENTRIES


# ------------------------------------------------------------------------------------------------------------------ GPU
_NETS = {}


def _net(name):
    import gpu_utils as Gu
    if name not in _NETS:
        _NETS.clear()                 # one scene's network (and packed blobs) on the device at a time
        _NETS[name] = Gu.make_net_and_renderer(scene(name))
    return _NETS[name]


def _render(name, precision, vdtype, skip, n_samples=64):
    """Inference render of scene(name) with render_volume_dtype = vdtype -> (outputs + raw on the GPU, stats)."""
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    sc = scene(name)
    net, ren = _net(name)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = n_samples, 0.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.render_skip_empty = precision, vdtype, skip
    net.eval()
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    try:
        batch = {k: sc[k].cuda() for k in Gu.BATCH_KEYS}
        sp = ren.prepare_sp_input(batch)
        with torch.no_grad():
            out = dict(ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"],
                                       net.encode_sparse_voxels(sp), sp, want_raw=True))
        torch.cuda.synchronize()
        stats = ren.stats.cpu()
    finally:
        ren.stats = None
    return out, stats


def _assert_same_bits(a, b, keys, label):
    for k in keys:
        assert a[k].shape == b[k].shape, (label, k)
        assert torch.equal(torch.nan_to_num(a[k], nan=-1.0), torch.nan_to_num(b[k], nan=-1.0)), (label, k)


@pytest.mark.gpu
@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3", "tc_fp16"])
@pytest.mark.parametrize("name", ["small", "frames", "subnormal"])
def test_inference_twins(name, precision, skip):
    """fp16 blob == fp32 blob, bit for bit: the five maps and raw (launch_list<3 / 1, __half> and the exact kernel's
    render_f32_kernel<__half> against their float twins)."""
    a, sa = _render(name, precision, "fp32", skip)
    b, sb = _render(name, precision, "fp16", skip)
    _assert_same_bits(b, a, MAPS + ("raw",), (name, precision, skip))
    # the same tiles over the same list (which half tiles take the staged or the direct gather depends on the list's order,
    # which the classification's atomics vary from run to run: both paths give the same bits)
    assert torch.equal(sa[:2], sb[:2])
    listed = "" if precision == "fp32" else "; listed %d of %d samples" % (int(sb[1]), a["raw"][..., 0].numel())
    print("%s %s skip=%d: bit-identical maps + raw%s" % (name, precision, skip, listed))


@pytest.mark.gpu
@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3", "tc_fp16"])
def test_full_size_view_twins(precision, skip):
    """The full-size 512 x 512 view in list order: the coarse levels of most half tiles come from the shared-memory staging
    (stats[5] > 0) for 4- and 2-byte voxels alike, and the fp16 blob gives the fp32 blob's bits."""
    a, sa = _render("full", precision, "fp32", skip)
    b, sb = _render("full", precision, "fp16", skip)
    _assert_same_bits(b, a, MAPS + ("raw",), ("full", precision, skip))
    if precision == "fp32":
        print("full fp32 skip=%d: bit-identical maps + raw" % skip)
        return
    assert int(sa[5]) > 0 and int(sb[5]) > 0, (sa.tolist(), sb.tolist())
    assert torch.equal(sa[:2], sb[:2])
    print("full %s skip=%d: bit-identical maps + raw; listed %d; staged / direct coarse half tiles fp32 %d / %d, fp16 %d / %d"
          % (precision, skip, int(sb[1]), int(sa[5]), int(sa[6]), int(sb[5]), int(sb[6])))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_subnormal_only_samples_are_listed(precision):
    """A sample whose only non-zero features are fp16 subnormals is listed (the occupancy bitmap does not flush them), with
    either blob; skipping on and off give the same maps."""
    occ = int(_occupied_samples(scene("subnormal_only")).sum())
    for vd in ("fp32", "fp16"):
        on, s_on = _render("subnormal_only", precision, vd, True)
        off, _ = _render("subnormal_only", precision, vd, False)
        _assert_same_bits(on, off, MAPS, ("subnormal_only", precision, vd))
        assert int(s_on[1]) >= occ > 0, (int(s_on[1]), occ)
        print("subnormal_only %s %s: listed %d, occupied (oracle) %d" % (precision, vd, int(s_on[1]), occ))


def _density_case(subnormal):
    """test_density_tc_gpu's 2 x 5000 random points on batch2_s32's scene with fp16-representable volumes."""
    sc = synth.rounded_scene(golden_case("batch2_s32")[0], torch.float16, subnormal)
    g = torch.Generator().manual_seed(5)
    lo, hi = sc["can_bounds"][0, 0], sc["can_bounds"][0, 1]
    return sc, (torch.rand((2, 5000, 3), generator=g) * 1.2 - 0.1) * (hi - lo) + lo


@pytest.mark.gpu
@pytest.mark.parametrize("subnormal", [False, True])
@pytest.mark.parametrize("skip", [True, False])
@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_density_twins(precision, skip, subnormal):
    """calculate_density on the tensor cores (nb_decode_density_list): fp16 blob == fp32 blob, bit for bit."""
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    sc, pts = _density_case(subnormal)
    net, ren = Gu.make_net_and_renderer(sc)
    batch = {k: sc[k].cuda() for k in Gu.BATCH_KEYS}
    sp = ren.prepare_sp_input(batch)
    cfg.density_precision, cfg.render_skip_empty = precision, skip
    got = {}
    for vd in ("fp32", "fp16"):
        cfg.render_volume_dtype = vd
        ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
        got[vd] = ren.calculate_density(pts.cuda(), net.encode_sparse_voxels(sp), sp)
        torch.cuda.synchronize()
        got[vd + "_listed"] = int(ren.stats[1])
        ren.stats = None
    assert torch.equal(got["fp16"], got["fp32"])
    assert got["fp16_listed"] == got["fp32_listed"] > 0
    print("density %s skip=%d subnormal=%d: bit-identical sigma; listed %d of %d points"
          % (precision, skip, subnormal, got["fp16_listed"], pts.shape[0] * pts.shape[1]))


# ------------------------------------------------------------------------------------------------- training (GPU)
def _train(sc, t_rand, G, Gm, train_precision, n_samples, vdtype):
    """test_distinct_frames._train with render_volume_dtype = vdtype and raw -> (maps + raw, grads, listed, packed dtype)."""
    from neuralbody_b200.lib.config import cfg
    net, ren, vols, batch = TD._setup(sc, train_precision, n_samples)
    cfg.render_volume_dtype = vdtype
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda(),
                          want_raw=True)
    FR.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm)).backward()
    torch.cuda.synchronize()
    listed = ren.train_listed_samples()[-1][0] if train_precision == "tc_tf32x3" else None
    maps = {k: v.detach().cpu() for k, v in out.items()}
    return maps, TD._gpu_grads(net, vols, batch), listed, ren._vol_dtype


def _grad_spread(a, b, B, rows):
    """{slice: max |a - b| / max |b|} over the slices of test_distinct_frames._slices; NaN patterns and all-zero slices must
    agree exactly."""
    sa = TD._slices({k: v.detach().cpu().double() for k, v in a.items()}, B, rows)
    sb = TD._slices({k: v.detach().cpu().double() for k, v in b.items()}, B, rows)
    out = {}
    for name, y in sb.items():
        x = sa[name]
        nan = torch.isnan(y)
        assert torch.equal(torch.isnan(x), nan), name
        scale = float(y[~nan].abs().max()) if bool((~nan).any()) else 0.0
        if scale == 0.0:
            assert not bool(x.nan_to_num(0.0).any()), name
            out[name] = 0.0
        else:
            out[name] = float((x[~nan] - y[~nan]).abs().max()) / scale
    return out


def _check_twin_grads(g16, g32, g32b, label):
    rows = sorted(set(FR.LATENT_INDEX))
    d = _grad_spread(g16, g32, 3, rows)
    rerun = _grad_spread(g32b, g32, 3, rows)
    worst = max(d.items(), key=lambda kv: kv[1])
    print("%s: fp16 vs fp32 blob worst slice %s %.1e (fp32 blob run twice: worst %.1e)" % (label, worst[0], worst[1],
                                                                                        max(rerun.values())))
    bad = {k: v for k, v in d.items() if v > TWIN_GRAD_TOL}
    assert not bad, (bad, {k: rerun[k] for k in bad})


@pytest.mark.gpu
@pytest.mark.parametrize("subnormal", [False, True])
def test_training_twins(subnormal):
    """tc_tf32x3 training (gather_kernel<__half>, frame_grad_kernel<__half, *>) on the rounded distinct-frame case: the maps
    and raw of the fp16 blob are the fp32 blob's bits, the gradients agree to TWIN_GRAD_TOL, the lists have one length."""
    sc, t_rand, G, Gm = frames_case(subnormal=subnormal)
    m32, g32, l32, _ = _train(sc, t_rand, G, Gm, "tc_tf32x3", FR.N_SAMPLES, "fp32")
    m32b, g32b, _, _ = _train(sc, t_rand, G, Gm, "tc_tf32x3", FR.N_SAMPLES, "fp32")
    m16, g16, l16, vd = _train(sc, t_rand, G, Gm, "tc_tf32x3", FR.N_SAMPLES, "fp16")
    from neuralbody_b200 import capi
    assert vd == capi.NB_DTYPE_F16
    _assert_same_bits(m16, m32, MAPS + ("raw",), "train")
    assert l16 == l32 > 0
    _check_twin_grads(g16, g32, g32b, "tc_tf32x3 subnormal=%d listed %d" % (subnormal, l16))


@pytest.mark.gpu
def test_exact_training_on_fp16_volume():
    """render_volume_dtype 'fp16' with render_train_precision 'fp32': the exact kernel's backward reads the fp32 volume only,
    so the training call packs that one and loss.backward() completes; maps equal the fp32-volume run's bits, gradients agree
    to TWIN_GRAD_TOL and pass the float64 oracle's per-slice gate."""
    from neuralbody_b200 import capi
    sc, t_rand, G, Gm, ref, ret = frames_reference()
    m32, g32, _, _ = _train(sc, t_rand, G, Gm, "fp32", FR.N_SAMPLES, "fp32")
    m32b, g32b, _, _ = _train(sc, t_rand, G, Gm, "fp32", FR.N_SAMPLES, "fp32")
    m16, g16, _, vd = _train(sc, t_rand, G, Gm, "fp32", FR.N_SAMPLES, "fp16")
    assert vd == capi.NB_DTYPE_F32
    _assert_same_bits(m16, m32, MAPS + ("raw",), "exact train")
    _check_twin_grads(g16, g32, g32b, "fp32 (exact) training, render_volume_dtype fp16")
    TD._check_maps(m16, ret)
    TD._print("fp32 training, fp16 volume setting", TD._check_grads(g16, ref, FR.LATENT_INDEX))


# ------------------------------------------------------------------------------------------------- oracle (GPU)
def _oracle_raw(sc, n_samples=64):
    d = FR.to_double(sc)
    sp = O.prepare_sp_input(d)
    wpts, _ = O.get_sampling_points(d["ray_o"], d["ray_d"], d["near"], d["far"], n_samples)
    vd = d["ray_d"] / d["ray_d"].norm(dim=2, keepdim=True)
    B, n, S = wpts.shape[:3]
    return O.calculate_density_color(d["weights"], wpts.reshape(B, n * S, 3), vd[:, :, None].expand(B, n, S, 3).reshape(B, n * S, 3),
                                     d["volumes"], sp, d["voxel_size"]).view(B, n, S, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
@pytest.mark.parametrize("name", ["small", "frames", "subnormal"])
def test_fp16_blob_inference_vs_oracle(name, precision):
    """The fp16 blob against the float64 oracle on the same (rounded) volumes, every ray and sample: the exact kernel at its
    gates (1e-4 on the maps, EXACT_RAW_TOL / EXACT_SIGMA_TOL on raw), tc_fp16x3 at 1e-3 on the maps and 5e-4 on sigma (2e-2 on
    the rgb logits, as tests/test_render_gpu.py)."""
    import gpu_utils as Gu
    sc = scene(name)
    out, _ = _render(name, precision, "fp16", False)
    out = {k: v.cpu() for k, v in out.items()}
    want = O.render(FR.to_double(sc), n_samples=64)
    tol = {"fp32": 1e-4, "tc_fp16x3": 1e-3}[precision]
    rep = Gu.compare(out, {k: v.numpy() for k, v in want.items()}, tol, label="%s %s fp16 blob" % (name, precision))
    d = (out["raw"].double() - _oracle_raw(sc)).abs()
    sig, logit = float(d[..., 3].max()), float(d[..., :3].max())
    if precision == "fp32":
        assert sig < EXACT_SIGMA_TOL and logit < EXACT_RAW_TOL, (sig, logit)
    else:
        assert sig < 5e-4 and logit < 2e-2, (sig, logit)
    print("%s %s fp16 blob vs float64 oracle: maps %s; raw sigma %.1e, rgb logits %.1e" % (name, precision, rep, sig, logit))


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["S64", "subnormal", "large"])
def test_fp16_blob_training_vs_oracle(case):
    """tc_tf32x3 training on the fp16 blob against the float64 oracle's autograd on the rounded volumes: the maps and every
    gradient slice of test_distinct_frames._check_grads (GATE, TAU, structural zeros exact).  'large' (512 rays, S = 64)
    lists more entries than one pass of the gather / scatter / frame-gradient grids covers."""
    kw = {"S64": dict(n_samples=64), "subnormal": dict(subnormal=True), "large": dict(n_samples=64, n_rays=512)}[case]
    S = kw.get("n_samples", FR.N_SAMPLES)
    sc, t_rand, G, Gm, ref, ret = frames_reference(**kw)
    maps, got, listed, _ = _train(sc, t_rand, G, Gm, "tc_tf32x3", S, "fp16")
    TD._check_maps(maps, ret)
    report = TD._check_grads(got, ref, FR.LATENT_INDEX)
    TD._print("tc_tf32x3 fp16 blob %s (grid pass %d entries)" % (case, GRID_ENTRIES), report, listed)
    assert listed > 0
    if case == "large":
        assert listed > GRID_ENTRIES, listed


# ------------------------------------------------------------------------------------------------- pack edges (GPU)
def _edge_values():
    """float32 values at the edges of fp16 rounding (positive and negative)."""
    g = torch.Generator().manual_seed(17)
    h = torch.arange(1, 0x7C00, dtype=torch.int32).to(torch.int16).view(torch.float16).float()     # every finite fp16 > 0
    ties = (h[:-1] + h[1:]) / 2                                  # exact midpoints (fp32 holds them): round to the even one
    sub = torch.rand(4000, generator=g) * (FP16_MIN_NORMAL - 2.0 ** -24) + 2.0 ** -24               # subnormal range
    tiny = torch.tensor([2.0 ** -25, 2.0 ** -25 * (1 - 2 ** -20), 2.0 ** -25 * (1 + 2 ** -20), 2.0 ** -26, 1e-10, 1e-30,
                         1e-40, 2.0 ** -24, 1.5 * 2.0 ** -24, 2.5 * 2.0 ** -24])     # below half the smallest subnormal, ties
    big = torch.tensor([65504.0, 65519.0, 65519.996, 65520.0, 65536.0, 7e4, 1e10, 3e38])           # above the largest fp16
    rnd = torch.exp(torch.rand(4000, generator=g) * 30 - 20)                                        # all exponents
    pos = torch.cat([ties, sub, tiny, big, rnd])
    return torch.cat([pos, -pos, torch.tensor([-0.0, 0.0])])


@pytest.mark.gpu
def test_pack_volume_fp16_rounding_edges():
    """nb_pack_volume(NB_DTYPE_F16) on fp32 volumes made of rounding edge cases: the packed bits are torch's .half() (round to
    nearest even, subnormals kept, -0.0 kept, overflow to inf), and every voxel with a non-zero fp16 value has all the cell
    bits of the trilinear cells it is a corner of (a bitmap with more bits set is allowed)."""
    import torch.nn.functional as F
    from neuralbody_b200 import capi
    lib = capi.load()
    vals = _edge_values()
    g = torch.Generator().manual_seed(18)
    B, shapes, Cs = 2, ((24, 23, 25), (7, 6, 5), (5, 4, 6), (3, 4, 3)), (8, 16, 32, 8)
    vols, k = [], 0
    for l, ((D, H, W), Cn) in enumerate(zip(shapes, Cs)):
        n = B * Cn * D * H * W
        idx = (torch.arange(n) + k) % vals.numel()
        k += n
        v = vals[idx].view(B, D, H, W, Cn)
        keep = torch.rand((B, D, H, W, 1), generator=g) < 0.5                 # half the voxels are empty
        one = torch.rand((B, D, H, W, 1), generator=g) < 0.3                  # of the rest some hold a single value
        first = torch.arange(Cn).view(1, 1, 1, 1, Cn) == 0
        mask = (keep & (~one | first)).reshape(-1, Cn)                        # (voxel, channel)
        if l == 0:                                                            # level 0 starts with every edge value once
            mask[:(vals.numel() + Cn - 1) // Cn] = True
        mask = mask.view(B, D, H, W, Cn)
        v = torch.where(mask, v, torch.zeros_like(v))
        vols.append(v.permute(0, 4, 1, 2, 3).contiguous())                  # NCDHW
    assert torch.equal(vols[0].permute(0, 2, 3, 4, 1).reshape(-1)[:vals.numel()], vals)
    dev = [v.cuda() for v in vols]
    dims = capi.LevelDims()
    levels = (capi.nb_volume_level * capi.NB_NUM_LEVELS)()
    for l, v in enumerate(dev):
        _, c, d, h, w = v.shape
        dims[l][0], dims[l][1], dims[l][2], dims[l][3] = c, d, h, w
        levels[l].data, levels[l].C, levels[l].D, levels[l].H, levels[l].W = v.data_ptr(), c, d, h, w
    f16 = capi.NB_DTYPE_F16
    nbytes = lib.nb_packed_volume_bytes(dims, B, f16)
    blob = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device="cuda")
    capi.check(lib.nb_pack_volume(levels, B, f16, blob.data_ptr(), nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "nb_pack_volume")
    torch.cuda.synchronize()
    blob = blob.cpu()

    def up(x):
        return (x + 255) // 256 * 256
    occ = lib.nb_packed_volume_level_offset(dims, B, f16, capi.NB_NUM_LEVELS)   # [voxel bits][cell bits] per level from here
    extra_bits = 0
    for l, v in enumerate(vols):
        _, c, D, H, W = v.shape
        off = lib.nb_packed_volume_level_offset(dims, B, f16, l)
        got = blob[off:off + v.numel() * 2].view(torch.int16).view(B, D, H, W, c)
        want = v.permute(0, 2, 3, 4, 1).half()
        assert torch.equal(got, want.view(torch.int16)), ("level", l, int((got != want.view(torch.int16)).sum()))
        vwords = (D * H * W + 31) // 32
        ncell = (D + 1) * (H + 1) * (W + 1)
        cwords = (ncell + 31) // 32
        cell_off = occ + up(B * vwords * 4)
        bits = blob[cell_off:cell_off + B * cwords * 4].view(torch.int32).view(B, cwords).numpy().astype(np.uint32)
        have = ((bits[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(B, -1)[:, :ncell].astype(bool)
        nz = (want != 0).any(-1).float()[:, None]                                              # (B,1,D,H,W)
        need = F.max_pool3d(F.pad(nz, (1, 1, 1, 1, 1, 1)), 2, stride=1).reshape(B, -1).numpy().astype(bool)
        missing = need & ~have
        assert not missing.any(), ("level", l, int(missing.sum()))
        extra_bits += int((have & ~need).sum())
        occ = cell_off + up(B * cwords * 4)
    assert occ == nbytes                                                        # the mirrored layout covers the blob
    # the edges are all there: ties rounded to even both ways, underflow to +-0, subnormals, overflow to +-inf, -0.0
    h = vals.half()
    assert bool(torch.isinf(h).any()) and bool(((h == 0) & (vals != 0)).any()) and bool((h.abs() < FP16_MIN_NORMAL).any())
    assert bool((torch.signbit(h) & (h == 0)).any())
    print("fp16 pack: %d edge values, every bit torch's; %d cell bits set beyond the fp16-occupied cells" % (vals.numel(), extra_bits))
