"""GPU parity tests proper: the product path (make_renderer(cfg, net).render(batch) -> ctypes ->
nb_render_fwd) against (1) the golden vectors made by the unmodified reference and (2) the CPU
oracle on seeded inputs; plus size-independent properties at full size.
Tolerance (the project's parity target): <= 1e-3 abs on rgb_map / depth_map for the tensor-core
path (tc_fp16x3, the default); the exact-fp32 kernel is held to 1e-4.  The 1-pass fp16 mode
(tc_fp16) is an opt-in speed mode that does NOT meet the gate on depth_map (one fp16 rounding of
any density-path operand costs ~1e-3); it is only checked against a documented 6e-3 envelope."""
import numpy as np
import pytest
import torch

from conftest import golden_case, hier_golden_case
from oracle import golden_cases, neuralbody_oracle as O
import gpu_utils as G

pytestmark = pytest.mark.gpu

TOL = {"fp32": 1e-4, "tc_fp16x3": 1e-3, "tc_fp16": 6e-3}
ALL_PREC = ["fp32", "tc_fp16x3", "tc_fp16"]


def _precisions():
    from neuralbody_b200 import capi
    lib = capi.load()
    return ["fp32"] + (["tc_fp16", "tc_fp16x3"] if lib.nb_has_precision(capi.NB_PRECISION_TC_FP16X3) else [])


@pytest.mark.parametrize("name", list(golden_cases.CASES))
@pytest.mark.parametrize("precision", ALL_PREC + ["tc_fp16x3_dense", "tc_fp16_dense"])
def test_golden_parity(name, precision):
    """tensor-core modes run twice: with exact empty-sample skipping (default) and dense."""
    skip_empty = not precision.endswith("_dense")
    precision = precision.replace("_dense", "")
    if precision not in _precisions():
        pytest.skip("precision %s not built" % precision)
    scene, rkw, gold = golden_case(name)
    out = G.render_product(scene, precision=precision, skip_empty=skip_empty, **rkw)
    rep = G.compare(out, gold, TOL[precision], nan_mismatch_frac=0.0 if precision != "tc_fp16" else 0.01,
                    label="%s/%s" % (name, precision))
    print(name, precision, rep)


@pytest.mark.parametrize("precision", ALL_PREC)
def test_raw_decoder_output_vs_oracle(precision):
    """Per-sample (rgb logits, sigma) against calculate_density_color of the oracle."""
    if precision not in _precisions():
        pytest.skip("precision %s not built" % precision)
    scene, rkw, _ = golden_case("eval_s64")
    # dense evaluation: with empty-sample skipping the raw rgb logits of skipped samples are (by design) not computed
    out = G.render_product(scene, precision=precision, want_raw=True, skip_empty=False, **rkw)
    sp = O.prepare_sp_input(scene)
    wpts, z = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], 64)
    vd = scene["ray_d"] / scene["ray_d"].norm(dim=2, keepdim=True)
    B, n, S = wpts.shape[:3]
    raw = O.calculate_density_color(scene["weights"], wpts.view(B, n * S, 3),
                                    vd[:, :, None].repeat(1, 1, S, 1).view(B, n * S, 3), scene["volumes"], sp,
                                    scene["voxel_size"]).view(B, n, S, 4)
    d = (out["raw"] - raw).abs()
    tol = {"fp32": 2e-4, "tc_fp16x3": 2e-2, "tc_fp16": 8e-2}[precision]   # sigma reaches +-30, logits +-8
    if precision == "tc_fp16x3":   # the density path is ~fp32-accurate in the 3-pass mode
        assert float(d[..., 3].max()) < 5e-4, float(d[..., 3].max())
    assert float(d.max()) < tol, float(d.max())


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
@pytest.mark.parametrize("name", ["eval_s64", "train_jitter_white", "batch2_s32", "eval_s48_seed7", "full_313"])
def test_empty_sample_skipping_is_bit_exact(name, precision):
    """Skipping samples whose trilinear cells are all unoccupied changes no output bit (sigma_empty < 0): the same pipeline
    with skip_empty = 0 lists EVERY sample and produces identical maps."""
    scene, rkw, _ = golden_case(name)
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    B, n = scene["ray_o"].shape[:2]
    S = rkw["n_samples"]
    dense = G.render_product(scene, precision=precision, skip_empty=False, renderer=ren, net=net, **rkw)
    assert int(ren.stats[1]) == B * n * S               # every sample went through the decoder
    ren.stats.zero_()
    sparse = G.render_product(scene, precision=precision, skip_empty=True, renderer=ren, net=net, **rkw)
    tiles, occ = int(ren.stats[0]), int(ren.stats[1])
    assert 0 < occ < B * n * S and tiles * 128 >= occ    # some, but not all, samples were evaluated
    assert tiles <= (occ + 127) // 128 + 4 * B           # full tiles but the last of each frame's four class lists
    print(name, precision, "evaluated %.1f%% of the samples in %d tiles" % (100.0 * occ / (B * n * S), tiles))
    for k in ("rgb_map", "depth_map", "acc_map", "weights", "disp_map"):
        assert torch.equal(torch.nan_to_num(dense[k], nan=-1.0), torch.nan_to_num(sparse[k], nan=-1.0)), k


def test_raw_records_of_skipped_samples():
    """want_raw: evaluated samples carry the same (rgb logits, sigma) with and without skipping; skipped ones carry the
    constant (0, 0, 0, min(sigma_empty, 0)) record (documented in the header next to `raw`)."""
    scene, rkw, _ = golden_case("train_jitter_white")
    net, ren = G.make_net_and_renderer(scene)
    a = G.render_product(scene, precision="tc_fp16x3", want_raw=True, renderer=ren, net=net, skip_empty=False, **rkw)
    b = G.render_product(scene, precision="tc_fp16x3", want_raw=True, renderer=ren, net=net, skip_empty=True, **rkw)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert torch.equal(a[k], b[k]), k
    same = (a["raw"] == b["raw"]).all(dim=-1)
    skipped = ~same
    assert 0 < int(skipped.sum()) < skipped.numel()
    rs = b["raw"][skipped]
    assert float(rs[:, :3].abs().max()) == 0.0 and float(rs[:, 3].max()) <= 0.0 and float((rs[:, 3] - rs[0, 3]).abs().max()) == 0.0
    assert float(a["raw"][skipped][:, 3].max()) < 0.0   # the dense run's sigma of those samples is sigma_empty < 0: weight 0


def test_density_only_decoder_matches_oracle():
    """f-3: Network.calculate_density on a voxel grid of world points (mesh extraction, if_mesh_renderer.py)."""
    scene, _, _ = golden_case("batch2_s32")
    net, ren = G.make_net_and_renderer(scene)
    g = torch.Generator().manual_seed(5)
    lo, hi = scene["can_bounds"][0, 0], scene["can_bounds"][0, 1]
    pts = (torch.rand((2, 5000, 3), generator=g) * 1.2 - 0.1) * (hi - lo) + lo          # some points outside the box
    sp = O.prepare_sp_input(scene)
    want = O.calculate_density(scene["weights"], pts, scene["volumes"], sp, scene["voxel_size"])
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    spg = ren.prepare_sp_input(batch)
    got = net.calculate_density(pts.cuda(), net.encode_sparse_voxels(spg), spg).cpu()
    assert got.shape == want.shape == (2, 5000, 1)
    assert float((got - want).abs().max()) < 2e-4
    assert float(want.max()) > 5.0 and float(want.min()) < -5.0          # not vacuous


def test_long_rays():
    """N_samples > 128 (e.g. 64 coarse + 128 importance merged, SURVEY 8f-4) stays on the tensor cores: the decoder works on a
    sample list and does not care about S."""
    scene, rkw, _ = golden_case("eval_s64")
    sub = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sub[k] = scene[k][:, :64].contiguous()
    ref = O.render(sub, n_samples=192)
    net, ren = G.make_net_and_renderer(sub)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    out = G.render_product(sub, precision="tc_fp16x3", n_samples=192, renderer=ren, net=net)
    assert int(ren.stats[3]) == 1 and int(ren.stats[0]) > 0          # one decoder launch of the list pipeline ran
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k] - ref[k]).abs().max()) < 1e-3, k


def test_chunked_equals_single_launch():
    scene, rkw, _ = golden_case("eval_s64")
    a = G.render_product(scene, precision="fp32", **rkw)
    b = G.render_product(scene, precision="fp32", chunk=100, **rkw)
    for k in a:
        assert torch.equal(torch.nan_to_num(a[k]), torch.nan_to_num(b[k])), k


def test_fp16_volume_with_exact_mlp_is_close():
    """Volume pack in fp16 (what the tensor-core path gathers from) only perturbs at the 1e-3 level."""
    from neuralbody_b200.lib.config import cfg
    scene, rkw, gold = golden_case("eval_s64")
    net, ren = G.make_net_and_renderer(scene)
    cfg.render_volume_dtype = "fp16"
    try:
        cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.render_precision, cfg.chunk = 64, 0.0, False, "fp32", 0
        net.eval()
        batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
        with torch.no_grad():
            out = {k: v.cpu() for k, v in ren.render(batch).items()}
    finally:
        cfg.render_volume_dtype = "auto"
    G.compare(out, gold, 1e-3, nan_mismatch_frac=0.01, label="fp16vol")


def test_full_size_properties():
    """512x512 x 64 samples on the full synth-313 body (config 2): properties that need no oracle
    run.  Empty rays give exact zeros and NaN disparity, weights sum to acc, acc in [0,1], and the
    result does not depend on how rays are grouped into launches (permutation invariance)."""
    from oracle import synth
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    assert scene["ray_o"].shape[1] == 512 * 512
    net, ren = G.make_net_and_renderer(scene)
    out = G.render_product(scene, precision="fp32", renderer=ren, net=net)
    acc, w = out["acc_map"], out["weights"]
    assert torch.isfinite(out["rgb_map"]).all() and torch.isfinite(out["depth_map"]).all()
    assert float(acc.min()) >= 0.0 and float(acc.max()) <= 1.0 + 1e-5
    assert float((w.sum(-1) - acc).abs().max()) < 1e-5
    assert float((w.min())) >= 0.0
    empty = acc == 0
    assert torch.isnan(out["disp_map"][empty]).all() and not torch.isnan(out["disp_map"][~empty]).any()
    assert float(out["rgb_map"][empty].abs().max()) == 0.0
    assert 0.2 < float(acc.mean()) < 0.8
    # permutation invariance: rays are independent units
    perm = torch.randperm(512 * 512, generator=torch.Generator().manual_seed(0))
    sc2 = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sc2[k] = scene[k][:, perm].contiguous()
    out2 = G.render_product(sc2, precision="fp32", renderer=ren, net=net)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert torch.equal(out[k][:, perm], out2[k]), k
    # and a strided subset agrees with the reference's golden vectors for the same rays
    gold = golden_case("full_313")[2]
    idx = torch.arange(0, 512 * 512, 521)
    sub = {k: (v[:, idx] if v.shape[1] == 512 * 512 else v) for k, v in out.items()}
    G.compare(sub, gold, 1e-4, label="full_313 subset")


def test_product_path_fails_loudly_on_cpu_tensors():
    scene, rkw, _ = golden_case("eval_s64")
    net, ren = G.make_net_and_renderer(scene)
    batch = {k: scene[k] for k in G.BATCH_KEYS}   # CPU tensors
    net.set_feature_volume(scene["volumes"])
    with pytest.raises(RuntimeError):
        with torch.no_grad():
            ren.render(batch)


# ---------------------------------------------------------------------------------------------- f-4 hierarchical sampling
@pytest.mark.parametrize("name", list(golden_cases.HIER_CASES))
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
def test_hierarchical_render_matches_reference_pieces(name, precision):
    """Coarse pass -> nb_sample_pdf -> fine pass (nb_render_args.z_vals, S + N_importance samples per ray, on the tensor
    cores through the frame-compacting pipeline) against the composition of the reference's own functions."""
    from neuralbody_b200.lib.config import cfg
    scene, rkw, gold = hier_golden_case(name)
    net, ren = G.make_net_and_renderer(scene)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd = rkw["n_samples"], float(rkw.get("perturb", 0.)), bool(rkw.get("white_bkgd", False))
    cfg.raw_noise_std, cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = 0, precision, "auto", 0
    cfg.render_skip_empty, cfg.render_importance = True, rkw["n_importance"]
    net.train(bool(rkw.get("training", False)))
    try:
        batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
        sp = ren.prepare_sp_input(batch)
        vol = net.encode_sparse_voxels(sp)
        tr = rkw.get("t_rand")
        u = rkw.get("u")
        with torch.no_grad():
            # the depths first: bit-for-bit the reference's sort(cat(z_vals, sample_pdf(...))) up to the summation order of the pdf
            coarse = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp,
                                     t_rand=None if tr is None else tr.cuda(), want_weights=True)
            z_all, z_smp = ren.importance_z_vals(batch["near"], batch["far"], coarse["weights"], rkw["n_samples"],
                                                 rkw["n_importance"], t_rand=None if tr is None else tr.cuda(),
                                                 u=None if u is None else u.cuda())
            out = ren.render_rays_hierarchical(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp,
                                               t_rand=None if tr is None else tr.cuda(), u=None if u is None else u.cuda())
        torch.cuda.synchronize()
    finally:
        cfg.render_importance = 0
    zg = torch.from_numpy(gold["z_vals"])
    assert torch.all(z_all[..., 1:] >= z_all[..., :-1])
    # The depths follow the reference's sort(cat(z_vals, sample_pdf(...))).  The inverse CDF is ill-conditioned where the
    # coarse weights vanish (pdf = 1e-5 / sum: dz/du ~ 300 m), so a 1e-6 difference in a weight moves a sample that sits in
    # EMPTY space by up to ~1e-3 m without touching any output; everywhere else the depths agree to rounding.
    dz = (z_all.cpu() - zg).abs()
    ztol = 2e-5 if precision == "fp32" else 2e-3
    assert float((dz < ztol).float().mean()) > 0.97, float((dz < ztol).float().mean())
    assert float(dz.max()) < (5e-3 if precision == "fp32" else 5e-2), float(dz.max())
    out = {k: v.detach().cpu() for k, v in out.items()}
    tol = TOL[precision]
    for k in ("rgb_map", "depth_map", "acc_map", "rgb0", "acc0"):
        d = float((out[k] - torch.from_numpy(gold[k])).abs().max())
        assert d < tol, (k, d)
    assert float((out["z_std"] - torch.from_numpy(gold["z_std"])).abs().max()) < (1e-3 if precision == "fp32" else 1e-2)
    assert out["weights"].shape[-1] == rkw["n_samples"] + rkw["n_importance"]


def test_sample_pdf_kernel_vs_oracle_random():
    """nb_sample_pdf alone on random weights / jitter / uniforms against oracle.importance_z_vals (no rendering involved)."""
    torch.manual_seed(5)
    from oracle import synth
    scene = synth.make_scene(H=8, W=8, scale=0.25)
    net, ren = G.make_net_and_renderer(scene)
    B, n, S, Ni = 2, 300, 48, 77
    near = torch.rand(B, n) + 1.0
    far = near + 1.0 + torch.rand(B, n)
    # every bin carries mass, so the inverse CDF is well conditioned (where weights vanish the reference's formula jumps by
    # a whole bin on a 1-ulp change of the CDF: `denom < 1e-5 -> 1`), plus rays without any weight (uniform pdf: the +1e-5)
    w = torch.rand(B, n, S) * 0.9 + 0.1
    w[:, ::7] = 0.
    t_rand, u = torch.rand(B, n, S), torch.rand(B, n, Ni)
    ro, rd = torch.zeros(B, n, 3), torch.ones(B, n, 3)
    for det in (True, False):
        _, z = O.get_sampling_points(ro, rd, near, far, S, perturb=0.0 if det else 1.0, training=not det, t_rand=None if det else t_rand)
        z_ref, s_ref = O.importance_z_vals(z.view(B * n, S), w.view(B * n, S), Ni, det=det, u=None if det else u.view(B * n, Ni))
        z_all, z_smp = ren.importance_z_vals(near.cuda(), far.cuda(), w.cuda(), S, Ni, t_rand=None if det else t_rand.cuda(),
                                             u=None if det else u.cuda())
        torch.cuda.synchronize()
        assert float((z_all.cpu().view(B * n, -1) - z_ref).abs().max()) < 2e-5
        assert float((z_smp.cpu().view(B * n, -1) - s_ref).abs().max()) < 2e-5


def test_strided_outputs_equal_dense_outputs():
    """nb_render_args.out_ray_stride: the four maps written as columns of one 24-byte-per-ray record (the slab a ray-sharded
    render all-gathers) hold the same bits as the dense maps -- tensor-core pipeline and exact kernel."""
    from neuralbody_b200 import dist as nbdist
    scene, rkw, _ = golden_case("batch2_s32")
    net, ren = G.make_net_and_renderer(scene)
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    for precision in ("tc_fp16x3", "fp32"):
        from neuralbody_b200.lib.config import cfg
        cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.render_precision = 32, 0.0, False, precision
        net.eval()
        sp = ren.prepare_sp_input(batch)
        vol = net.encode_sparse_voxels(sp)
        with torch.no_grad():
            dense = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp)
            slab, views = nbdist.new_slab(batch["ray_o"].shape[0], batch["ray_o"].shape[1], "cuda")
            slab.fill_(-7.0)
            ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vol, sp, out=views)
        torch.cuda.synchronize()
        for k in ("rgb_map", "disp_map", "acc_map", "depth_map"):
            assert torch.equal(torch.nan_to_num(dense[k], nan=-1.0), torch.nan_to_num(views[k], nan=-1.0)), (precision, k)


def test_two_frames_through_one_renderer():
    """The pack caches must not serve frame k's latent code / volumes to frame k+1 (fresh tensors that may land on recycled
    addresses): two frames with different latent_index and different volumes through ONE Renderer equal fresh renderers."""
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    frames = [synth.make_scene(H=24, W=24, scale=0.25, all_hit=True, latent_index=li, volume_seed=vs)
              for li, vs in ((3, 313), (11, 999))]
    net, ren = G.make_net_and_renderer(frames[0])
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.render_precision = 64, 0.0, False, "tc_fp16x3"
    net.eval()
    got = []
    for rep in range(2):
        for f in frames:
            net.set_feature_volume([v.clone().cuda() for v in f["volumes"]])     # fresh device tensors every frame
            batch = {k: f[k].clone().cuda() for k in G.BATCH_KEYS}
            with torch.no_grad():
                got.append({k: v.cpu() for k, v in ren.render(batch).items()})
            del batch
    for i, f in enumerate(frames):
        want = O.render(f, n_samples=64)
        for rep in range(2):
            for k in ("rgb_map", "depth_map", "acc_map"):
                assert float((got[2 * rep + i][k] - want[k]).abs().max()) < 1e-3, (i, rep, k)
    assert float((got[0]["rgb_map"] - got[1]["rgb_map"]).abs().max()) > 1e-2      # the frames do differ


def test_config5_shape_batch_of_frames_128_samples():
    """BASELINE config 5's shape at test size: B = 2 frames with their own pose and volume, 256x256 rays, 128 samples, one
    Renderer batch; compared with the oracle on a strided subset of the rays (rays are independent)."""
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    poses = [synth.make_scene(H=256, W=256, scale=0.3, all_hit=True, azimuth_deg=20.0 + 50.0 * p, Rh=(0.3 - 0.2 * p, -0.2, 0.1 + 0.3 * p),
                              Th=(0.1 + 0.05 * p, 0.2, 1.0), volume_seed=313 + 5 * p, latent_index=2 + 3 * p) for p in range(2)]
    scene = {k: torch.cat([q[k] for q in poses], 0) for k in G.BATCH_KEYS}
    scene["volumes"] = [torch.cat([q["volumes"][l] for q in poses], 0) for l in range(4)]
    scene["weights"], scene["voxel_size"] = poses[0]["weights"], poses[0]["voxel_size"]
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    out = G.render_product(scene, precision="tc_fp16x3", n_samples=128, renderer=ren, net=net)
    assert int(ren.stats[3]) == 2 and out["rgb_map"].shape == (2, 65536, 3)
    idx = torch.arange(0, 65536, 97)
    sub = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sub[k] = scene[k][:, idx].contiguous()
    want = O.render(sub, n_samples=128)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k][:, idx] - want[k]).abs().max()) < 1e-3, k
    assert 0.05 < float(want["acc_map"].mean()) < 0.95


def test_largest_frame_the_sample_ids_allow():
    """1024 x 1024 rays x 128 samples = 2^27 samples in one frame: the list entries carry 28-bit sample ids (the renderer
    leaves the tensor cores at 2^28); a strided subset is compared with the oracle."""
    from oracle import synth
    scene = synth.make_scene(H=1024, W=1024, scale=0.3, all_hit=True)
    assert scene["ray_o"].shape[1] * 128 == 1 << 27
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    out = G.render_product(scene, precision="tc_fp16x3", n_samples=128, renderer=ren, net=net)
    assert int(ren.stats[3]) == 1 and int(ren.stats[0]) > 0          # the tensor-core pipeline ran
    idx = torch.arange(0, 1 << 20, 2053)
    sub = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sub[k] = scene[k][:, idx].contiguous()
    want = O.render(sub, n_samples=128)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k][:, idx] - want[k]).abs().max()) < 1e-3, k
    # one sample more per ray would not fit the ids: the renderer then takes the exact kernel instead of failing
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.config import cfg
    assert (1 << 20) * 256 >= (1 << 28)
