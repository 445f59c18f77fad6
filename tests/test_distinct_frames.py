"""Multi-frame batches whose frames differ in pose, camera, volumes, latent code and bounds (oracle/frames_case.py), so that
a kernel reading or writing another frame's slice -- volume block, R / Th, bounds, folded colour bias, latent row -- cannot
pass.  Every other multi-frame case of the suite replicates one frame, and there such a mix-up cancels exactly.

CPU: the float32 oracle reproduces the unmodified reference's gradients on this case (tests/golden/grad_frames_b3_s33.npz,
tools/frames_grad_case.py), and giving one frame frame 0's R / Th, volume, latent row or bounds moves that frame's outputs
or gradients by far more than the GPU gate.

GPU: the training render (both training precisions, everything training, the loss over all five maps) against the
oracle's autograd in float64, PER FRAME SLICE: R[b], Th[b], bounds[b, 0], vol_l[b], the rays / near / far of frame b,
latent rows 2 and 5, and the shared decoder tensors whole.  Each slice must have the reference's NaN pattern, a rel-L2
<= GATE over its finite entries and max |g - r| <= TAU max |r|.  The case keeps every sample that carries gradient off the
trilinear cell faces and the decoder's ReLU kinks (frames_case.well_conditioned), so these are functions of the inputs a
float32 kernel can be held to.  Gradients that are zero by construction (latent rows no
frame uses, bounds[:, 1], every gradient of a frame with no listed sample) must be exactly zero.  The cases cover
S = 33 / 64 / 256 (the backward's limit), an odd ray count, an empty frame between two occupied ones, a batch with nothing
listed, a list shorter than one 32-entry block and than the weight-gradient splits, a list of many blocks, and a chunked
render.  Also per frame: the inference maps, the packed volume and its occupancy bitmap, the folded colour bias of
nb_pack_weights and Network.calculate_density."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import frames_case as FR
from oracle import grad_case
from tools import frames_grad_case as FG
from tools import map_grad_case as MC

GATE = 1e-3          # rel-L2 per slice over its finite entries (the gate of tests/test_backward.py)
# max |g - r| <= TAU * max |r| per slice.  Measured on an H100 80GB HBM3 (700 W power limit): the worst slice of any case
# was vol0[0] of the 512-ray case on tc_tf32x3 at 1.1e-4.
TAU = 2e-3
# giving one frame frame 0's R / Th, volume, latent row or bounds must move that frame by more than this (rel-L2)
FRAME_MARGIN = 10 * GATE
WGRAD_SPLITS = 74    # the weight-gradient GEMMs split the list over 74 CTAs (nb_train.cu)
TRAIN_PRECISIONS = ["tc_tf32x3", "fp32"]


@pytest.fixture(scope="module")
def golden():
    from oracle import synth
    scene, t_rand, G, Gm = FR.build()
    gold = load_golden(FG.GOLDEN)
    assert synth.scene_checksum(scene) == gold["input_sha256"]
    return scene, t_rand, G, Gm, gold


_REF = {}


def reference(**kw):
    """(scene, t_rand, G, Gm, float64 oracle gradients, float64 oracle outputs) of frames_case.build(**kw), cached."""
    key = tuple(sorted(kw.items()))
    if key not in _REF:
        scene, t_rand, G, Gm = FR.build(**kw)
        _REF[key] = (scene, t_rand, G, Gm) + FR.oracle_grads(scene, t_rand, G, Gm, kw.get("n_samples", FR.N_SAMPLES))
    return _REF[key]


def _rel_l2(a, b):
    return MC.rel_l2_finite(a, b)


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_distinct_frames_match_reference(golden):
    """The float32 oracle reproduces the reference's per-frame gradients (latent per frame, bounds per frame) and its
    decoder / volume fingerprints."""
    scene, t_rand, G, Gm, gold = golden
    g, ret = FR.oracle_grads(scene, t_rand, G, Gm, FR.N_SAMPLES, dtype=torch.float32)
    np.testing.assert_array_equal((ret["acc_map"] == 0).numpy(), gold["empty_rays"])
    got = FG.summaries(g)
    for k in FG.FULL:
        np.testing.assert_array_equal(np.isnan(got["d_" + k]), np.isnan(gold["d_" + k]), err_msg=k)
        np.testing.assert_allclose(got["d_" + k], gold["d_" + k], rtol=1e-5, atol=1e-5, err_msg=k)
    np.testing.assert_allclose(got["d_latent"], gold["d_latent"], rtol=1e-5, atol=1e-6)
    used = sorted(set(FR.LATENT_INDEX))
    assert [r for r in range(gold["d_latent"].shape[0]) if gold["d_latent"][r].any()] == used
    for k in [k for k in gold if k.startswith(("sum:", "abs:", "head:"))]:
        np.testing.assert_allclose(got[k], gold[k], rtol=1e-4, atol=1e-6, err_msg=k)
    assert not gold["d_bounds"][:, 1].any() and float(np.abs(gold["d_bounds"][:, 0]).min()) > 0


def _swap(scene, field, b):
    """A copy of the scene in which frame b has frame 0's `field`."""
    sc = dict(scene)
    if field == "volume":
        sc["volumes"] = [v.clone() for v in scene["volumes"]]
        for v in sc["volumes"]:
            v[b] = v[0]
        return sc
    keys = {"R_Th": ("R", "Th"), "latent": ("latent_index",), "bounds": ("bounds",)}[field]
    for k in keys:
        sc[k] = scene[k].clone()
        sc[k][b] = scene[k][0]
    return sc


@pytest.mark.parametrize("field", ["R_Th", "volume", "latent", "bounds"])
def test_case_tells_the_frames_apart(golden, field):
    """A kernel that read frame 0's R / Th, volume block, latent row or bounds for frame 1 would fail the GPU gate: in the
    float64 oracle that substitution moves frame 1's maps or gradients by more than FRAME_MARGIN (rel-L2)."""
    scene, t_rand, G, Gm, _ = golden
    base, ret0 = FR.oracle_grads(scene, t_rand, G, Gm, FR.N_SAMPLES)
    g, ret = FR.oracle_grads(_swap(scene, field, 1), t_rand, G, Gm, FR.N_SAMPLES)
    b = 1
    moved = {k: _rel_l2(ret[k][b], ret0[k][b]) for k in ("rgb_map", "depth_map", "acc_map", "weights")}
    moved.update({k: _rel_l2(g[k][b], base[k][b]) for k in FR.FRAME_GRADS})
    moved["latent"] = max(_rel_l2(g["latent.weight"][r], base["latent.weight"][r]) for r in (2, 5))
    print(field, {k: round(v, 4) for k, v in moved.items()})
    assert max(moved.values()) > FRAME_MARGIN, moved
    # the frame's own outputs move, not only a gradient
    assert max(moved[k] for k in ("rgb_map", "depth_map", "acc_map", "weights")) > FRAME_MARGIN, moved


def test_case_is_well_conditioned(golden):
    """No sample that carries gradient sits within FACE_MARGIN cells of a trilinear cell face or within RELU_MARGIN of a
    ReLU kink (frames_case.well_conditioned), and such samples were there before the redraw: the condition is not vacuous."""
    scene, t_rand, _, _, _ = golden
    assert not bool(FR.fragile_samples(scene, t_rand).any())
    raw = torch.rand(t_rand.shape, generator=torch.Generator().manual_seed(77))
    assert int(FR.fragile_samples(scene, raw).sum()) > 10


def test_case_variants_are_what_they_say():
    """middle_empty / all_empty: the emptied frames' samples all have zero features, so nothing of them is listed and all
    their rays have acc_map == 0; the distinct case has every frame occupied."""
    from oracle import neuralbody_oracle as O
    for variant, empty in (("distinct", ()), ("middle_empty", (1,)), ("all_empty", (0, 1, 2))):
        scene, t_rand, _, _ = FR.build(n_samples=16, variant=variant)
        pts, _ = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], 16, 1.0, True, t_rand)
        sp = O.prepare_sp_input(scene)
        B = pts.shape[0]
        grid = O.get_grid_coords(O.pts_to_can_pts(pts.view(B, -1, 3), sp["R"], sp["Th"]), sp["bounds"], sp["out_sh"],
                                 scene["voxel_size"])
        occupied = (O.interpolate_features(grid, scene["volumes"]) != 0).any(1).sum(1)
        for b in range(B):
            assert (int(occupied[b]) == 0) == (b in empty), (variant, b, occupied.tolist())


# ------------------------------------------------------------------------------------------------------------------ GPU
def _setup(scene, train_precision, n_samples, chunk=0, perturb=1.0):
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    dev = "cuda:0"
    net, ren = Gu.make_net_and_renderer(scene, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = n_samples, perturb, True, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = "tc_fp16x3", "auto", chunk
    cfg.render_train_precision = train_precision
    cfg.render_importance = 0
    net.train()
    for p in net.parameters():
        p.requires_grad_(True)
    vols = [v.to(dev).requires_grad_(True) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].to(dev) for k in Gu.BATCH_KEYS}
    for k in FR.LEAVES:
        batch[k] = batch[k].clone().requires_grad_(True)
    return net, ren, vols, batch


def _gpu_grads(net, vols, batch):
    got = {k: batch[k].grad for k in FR.LEAVES}
    got.update({k: p.grad for k, p in net.named_parameters() if k in grad_case.GRAD_KEYS})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return got


def _train(scene, t_rand, G, Gm, train_precision, n_samples):
    """Render (training precision, everything training), backward the loss over all five maps -> (maps, grads, listed)."""
    net, ren, vols, batch = _setup(scene, train_precision, n_samples)
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())
    FR.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm)).backward()
    torch.cuda.synchronize()
    listed = ren.train_listed_samples()[-1][0] if train_precision == "tc_tf32x3" else None
    maps = {k: v.detach().cpu() for k, v in out.items()}
    return maps, _gpu_grads(net, vols, batch), listed


def _check_maps(maps, ret):
    for k in ("rgb_map", "depth_map", "acc_map", "weights"):
        for b in range(ret[k].shape[0]):
            d = float((maps[k][b].double() - ret[k][b]).abs().max())
            assert d < 1e-4, (k, b, d)
    np.testing.assert_allclose(maps["disp_map"].numpy(), ret["disp_map"].numpy(), rtol=1e-3, atol=1e-4)  # NaN: same rays


def _slices(g, B, rows):
    """name -> tensor: every per-frame gradient per frame (bounds: row 0 only), the latent rows in `rows`, the other
    decoder tensors whole."""
    out = {}
    for k in FR.FRAME_GRADS:
        for b in range(B):
            out["%s[%d]" % (k, b)] = g[k][b][0] if k == "bounds" else g[k][b]
    for r in rows:
        out["latent[%d]" % r] = g["latent.weight"][r]
    for k in grad_case.GRAD_KEYS:
        if k != "latent.weight":
            out[k] = g[k]
    return out


def _check_grads(got, ref, latent_index, empty=()):
    """Per-slice comparison (see the module doc); returns {slice: (rel-L2, max err / max |r|)} of the compared slices."""
    B = len(latent_index)
    for k, r in ref.items():
        assert got[k] is not None, k
        assert got[k].shape == r.shape, (k, tuple(got[k].shape), tuple(r.shape))
    got = {k: v.detach().cpu().double() for k, v in got.items()}
    rows = sorted({latent_index[b] for b in range(B) if b not in empty})
    # structural zeros, exactly: the latent rows no occupied frame uses, bounds[:, 1], every gradient of an empty frame
    unused = [r for r in range(got["latent.weight"].shape[0]) if r not in rows]
    assert not bool(got["latent.weight"][unused].any()), [r for r in unused if got["latent.weight"][r].any()]
    assert not bool(got["bounds"][:, 1].any())
    for b in empty:
        for k in FR.FRAME_GRADS:
            g, r = got[k][b], ref[k][b]
            assert torch.equal(torch.isnan(g), torch.isnan(r)), (k, b)
            assert not bool(g.nan_to_num(0.0).any()) and not bool(r.nan_to_num(0.0).any()), (k, b)
    ref_s = _slices(ref, B, rows)
    got_s = _slices(got, B, rows)
    report, bad = {}, {}
    for name, r in ref_s.items():
        if any(name.endswith("[%d]" % b) and not name.startswith("latent") for b in empty):
            continue
        g = got_s[name]
        nan = torch.isnan(r)
        if not torch.equal(torch.isnan(g), nan):
            bad[name] = ("NaN pattern", int(torch.isnan(g).sum()), int(nan.sum()))
            continue
        fin = ~nan
        scale = float(r[fin].abs().max())
        assert scale > 0, name                   # every compared slice carries gradient on these cases
        e, m = _rel_l2(g, r), float((g[fin] - r[fin]).abs().max()) / scale
        report[name] = (e, m)
        if not (e <= GATE and m <= TAU):
            bad[name] = (e, m)
    assert not bad, bad
    return report


def _print(label, report, listed=None):
    worst = max(report.items(), key=lambda kv: kv[1][1])
    print(label, "listed:", listed, "worst max-err slice: %s %.2e;" % (worst[0], worst[1][1]),
          "(rel-L2 / max err)", {k: "%.1e/%.1e" % v for k, v in report.items()})


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
@pytest.mark.parametrize("n_samples", [33, 64, 256])
def test_distinct_frames_grads(train_precision, n_samples):
    """Three distinct frames, 83 rays each (odd against the backward's 4-warp ray blocks), S = 33 / 64 / 256 (256 is the
    backward's limit): maps and every gradient slice against the float64 oracle."""
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=n_samples)
    maps, got, listed = _train(scene, t_rand, G, Gm, train_precision, n_samples)
    _check_maps(maps, ret)
    report = _check_grads(got, ref, FR.LATENT_INDEX)
    _print("%s S=%d" % (train_precision, n_samples), report, listed)
    if listed is not None:
        assert 0 < listed < 3 * FR.N_RAYS * n_samples


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_middle_frame_empty(train_precision):
    """Frame 1 lists no sample, frames 0 and 2 do: frame 1's gradients are exactly zero (NaN where the oracle's are), the
    others pass the per-slice gate, and the batch lists exactly what frames 0 and 2 list without frame 1."""
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=64, variant="middle_empty")
    maps, got, listed = _train(scene, t_rand, G, Gm, train_precision, 64)
    _check_maps(maps, ret)
    assert not bool(maps["acc_map"][1].any())
    report = _check_grads(got, ref, FR.LATENT_INDEX, empty=(1,))
    if listed is not None:
        sub = FR.build(n_samples=64, variant="middle_empty", frames=(0, 2))     # frames 0 and 2 of this very batch
        _, _, listed_02 = _train(*sub, train_precision, 64)
        assert listed > 0 and listed == listed_02, (listed, listed_02)
    _print("%s middle_empty" % train_precision, report, listed)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_all_frames_empty(train_precision):
    """Nothing listed (the GEMMs and column sums see zero rows): backward completes, every gradient is a tensor of exact
    zeros (NaN where the oracle's is: d ray_d / near / far of rays with acc_map == 0), the maps are the oracle's."""
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=FR.N_SAMPLES, variant="all_empty")
    maps, got, listed = _train(scene, t_rand, G, Gm, train_precision, FR.N_SAMPLES)
    _check_maps(maps, ret)
    assert not bool(maps["acc_map"].any())
    for k, r in ref.items():
        g = got[k]
        assert g is not None and g.shape == r.shape, k
        g = g.detach().cpu()
        assert torch.equal(torch.isnan(g), torch.isnan(r)), k
        assert not bool(g.nan_to_num(0.0).any()), k
    if listed is not None:
        assert listed == 0
    print(train_precision, "all_empty listed:", listed)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_single_ray(train_precision):
    """B = 1, one ray, 33 samples: a list shorter than one 32-entry block and than the weight-gradient splits."""
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=FR.N_SAMPLES, n_rays=1, batch=1)
    maps, got, listed = _train(scene, t_rand, G, Gm, train_precision, FR.N_SAMPLES)
    _check_maps(maps, ret)
    report = _check_grads(got, ref, FR.LATENT_INDEX[:1])
    if listed is not None:
        assert 0 < listed < 32, listed
    _print("%s one ray" % train_precision, report, listed)


@pytest.mark.gpu
def test_many_rays_list():
    """512 rays per frame at S = 64 (tc_tf32x3): a list of many blocks per weight-gradient split, whose length is not a
    multiple of the 128-row GEMM tiles."""
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=64, n_rays=512)
    maps, got, listed = _train(scene, t_rand, G, Gm, "tc_tf32x3", 64)
    assert listed > WGRAD_SPLITS * 16 and listed % 128 != 0, listed
    _check_maps(maps, ret)
    report = _check_grads(got, ref, FR.LATENT_INDEX)
    _print("tc_tf32x3 512 rays", report, listed)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_chunked_render(train_precision):
    """render(batch) with cfg.chunk = 29: three launches of 29, 29 and 25 rays, each drawing its own jitter (as upstream does
    per chunk; here the draws serve the case's jitter chunk by chunk), against the float64 oracle of the whole batch."""
    from neuralbody_b200.lib.config import cfg
    scene, t_rand, G, Gm, ref, ret = reference(n_samples=FR.N_SAMPLES)
    chunk, n = 29, scene["ray_o"].shape[1]
    draws = [t_rand[:, i:i + chunk] for i in range(0, n, chunk)]
    try:
        net, ren, vols, batch = _setup(scene, train_precision, FR.N_SAMPLES, chunk=chunk)

        def draw(B, m, S, dev):
            d = draws.pop(0)
            assert tuple(d.shape) == (B, m, S)
            return d.to(dev).contiguous()
        ren._draw_t_rand = draw
        out = ren.render(batch)
        FR.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm)).backward()
        torch.cuda.synchronize()
    finally:
        cfg.chunk = 0
    assert not draws
    _check_maps({k: v.detach().cpu() for k, v in out.items()}, ret)
    report = _check_grads(_gpu_grads(net, vols, batch), ref, FR.LATENT_INDEX)
    _print("%s chunk=29" % train_precision, report)


@pytest.mark.gpu
@pytest.mark.parametrize("precision,skip", [("fp32", True), ("tc_fp16x3", True), ("tc_fp16x3", False), ("tc_fp16", True)])
def test_inference_maps_per_frame(precision, skip):
    """The inference render of the distinct case, per frame, against the float64 oracle at tests/test_render_gpu.py's TOL."""
    import gpu_utils as Gu
    from oracle import neuralbody_oracle as O
    tol = {"fp32": 1e-4, "tc_fp16x3": 1e-3, "tc_fp16": 6e-3}[precision]
    scene, _, _, _ = FR.build()
    out = Gu.render_product(scene, n_samples=64, precision=precision, skip_empty=skip)
    want = O.render(FR.to_double(scene), n_samples=64)
    for b in range(3):
        gold = {k: want[k][b:b + 1].numpy() for k in want}
        rep = Gu.compare({k: v[b:b + 1] for k, v in out.items()}, gold, tol,
                         nan_mismatch_frac=0.0 if precision != "tc_fp16" else 0.01, label="frame %d %s" % (b, precision))
        print(precision, skip, b, rep)
    assert float((want["rgb_map"][0] - want["rgb_map"][2]).abs().max()) > 1e-2


@pytest.mark.gpu
def test_pack_volume_per_frame():
    """nb_pack_volume on three distinct frames: each frame's channels-last block and its last-level cell-occupancy bitmap."""
    import gpu_utils as Gu
    from neuralbody_b200 import capi
    scene, _, _, _ = FR.build()
    net, ren = Gu.make_net_and_renderer(scene)
    vols = [v.cuda() for v in scene["volumes"]]
    B = vols[0].shape[0]
    for dtype, tdt in ((capi.NB_DTYPE_F32, torch.float32), (capi.NB_DTYPE_F16, torch.float16)):
        ren._vol_key = None
        blob, dims = ren.pack_volume(vols, dtype)
        torch.cuda.synchronize()
        for l, v in enumerate(vols):
            off = ren.lib.nb_packed_volume_level_offset(dims, B, dtype, l)
            got = blob[off:off + v.numel() * (4 if dtype == capi.NB_DTYPE_F32 else 2)].view(tdt).view(B, *v.shape[2:], v.shape[1])
            for b in range(B):
                assert torch.equal(got[b], v[b].permute(1, 2, 3, 0).to(tdt)), (l, dtype, b)
    # the last level's cell bitmap (the blob's last region): bit (cx,cy,cz) = OR of the 8 voxels of that trilinear cell
    v = vols[3]
    occ = (v != 0).any(dim=1, keepdim=True).float()
    cell = torch.nn.functional.max_pool3d(torch.nn.functional.pad(occ, (1, 1, 1, 1, 1, 1)), 2, stride=1)
    D, H, W = v.shape[2:]
    ncell = (D + 1) * (H + 1) * (W + 1)
    words = (ncell + 31) // 32
    total = ren.lib.nb_packed_volume_bytes(dims, B, capi.NB_DTYPE_F16)
    region = ((B * words * 4 + 255) // 256) * 256
    bits = blob[total - region: total - region + B * words * 4].view(torch.int32).view(B, words).cpu().numpy().astype(np.uint32)
    unpacked = ((bits[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(B, -1)[:, :ncell]
    want = cell.reshape(B, -1).cpu().numpy().astype(np.uint32)
    for b in range(B):
        np.testing.assert_array_equal(unpacked[b], want[b], err_msg="frame %d" % b)
    assert not torch.equal(vols[3][0], vols[3][1]) and not torch.equal(vols[3][0], vols[3][2])   # the frames' features differ


def _bc_byte_offset():
    """kBcByteOffset of csrc/nb_layout.h: the per-frame folded colour bias bc[B][128] (fp32).  Mirrors the header's fp32
    section (oW0t .. kF32Floats, nb_layout.h:34-48), its fp16 stream (kF16ByteOffset .. kF16Halves, :73-84) and the fold
    scratch (kScratchByteOffset, kBcByteOffset, :134-136); test_pack_weights_folded_bias_per_frame checks the mirror against
    nb_packed_weights_bytes first."""
    def up(x):
        return (x + 255) // 256 * 256
    f32_floats = 352 * 256 + 256 + 2 * (256 * 256 + 256) + 256 + 4 + 320 * 128 + 28 * 128 + 3 * 128 + 4 + 128 * 256 + 4
    f16_halves = (2 * 22 + 1) * 4096 + 2 * (2 * 16 + 1) * 4096 + 22 * 2048 + 9 * 256
    return up(up(f32_floats * 4) + f16_halves * 2) + 128 * 256 * 8


@pytest.mark.gpu
def test_pack_weights_folded_bias_per_frame():
    """nb_pack_weights folds each frame's latent row into its own colour bias bc[b] = T feature_fc.b + view_fc[:, :256]
    (latent_fc [0 (+) latent[li[b]]] + latent_fc.b) + view_fc.b: against fp64 torch for latent indices [2, 5, 2]."""
    import gpu_utils as Gu
    scene, _, _, _ = FR.build()
    net, ren = Gu.make_net_and_renderer(scene)
    li = scene["latent_index"].cuda()
    assert li.tolist() == list(FR.LATENT_INDEX)
    B = li.shape[0]
    blob = ren.pack_weights(li, torch.device("cuda:0"))
    torch.cuda.synchronize()
    off = _bc_byte_offset()

    def up(x):
        return (x + 255) // 256 * 256
    # packed_weights_bytes (nb_layout.h:139-149) from the mirrored kBcByteOffset: a layout change fails here, by name
    mirrored = up(up(off + B * 128 * 4) + B * 256 * 8) + B * 128 * 16 * 2
    assert mirrored == ren.lib.nb_packed_weights_bytes(B), ("csrc/nb_layout.h changed: update _bc_byte_offset",
                                                           mirrored, ren.lib.nb_packed_weights_bytes(B))
    got = blob[off:off + B * 128 * 4].view(torch.float32).view(B, 128).cpu().double()
    w = {k: v.double() for k, v in scene["weights"].items()}
    Wv, Wl = w["view_fc.weight"][:, :, 0], w["latent_fc.weight"][:, :, 0]
    T = Wv[:, :256] @ Wl[:, :256]
    u = w["latent.weight"][scene["latent_index"]] @ Wl[:, 256:].t() + w["latent_fc.bias"]
    want = (T @ w["feature_fc.bias"])[None] + u @ Wv[:, :256].t() + w["view_fc.bias"]
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-6, atol=1e-6)
    assert torch.equal(got[0], got[2]) and float((got[0] - got[1]).abs().max()) > 1e-2


@pytest.mark.gpu
@pytest.mark.parametrize("precision,tol", [("fp32", 2e-4), ("tc_fp16x3", 5e-4)])
def test_calculate_density_per_frame(precision, tol):
    """Network.calculate_density (cfg.density_precision) on points around each frame's own body, per frame, against the
    float64 oracle."""
    import gpu_utils as Gu
    from oracle import neuralbody_oracle as O
    from neuralbody_b200.lib.config import cfg
    scene, _, _, _ = FR.build()
    net, ren = Gu.make_net_and_renderer(scene)
    g = torch.Generator().manual_seed(6)
    lo, hi = scene["can_bounds"][:, :1], scene["can_bounds"][:, 1:]
    pts = (torch.rand((3, 4000, 3), generator=g) * 1.2 - 0.1) * (hi - lo) + lo       # some points outside the box
    sc = FR.to_double(scene)
    want = O.calculate_density(sc["weights"], pts.double(), sc["volumes"], O.prepare_sp_input(sc), sc["voxel_size"])
    batch = {k: scene[k].cuda() for k in Gu.BATCH_KEYS}
    sp = ren.prepare_sp_input(batch)
    old = cfg["density_precision"] if "density_precision" in cfg else None
    cfg.density_precision = precision
    try:
        got = net.calculate_density(pts.cuda(), net.encode_sparse_voxels(sp), sp).cpu().double()
    finally:
        if old is None:
            del cfg["density_precision"]
        else:
            cfg.density_precision = old
    assert got.shape == want.shape == (3, 4000, 1)
    for b in range(3):
        d = float((got[b] - want[b]).abs().max())
        assert d < tol, (b, d)
        assert float(want[b].max()) > 5.0 and float(want[b].min()) < -5.0          # not vacuous
