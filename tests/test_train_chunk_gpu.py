"""The training step bench.py --config c3 times, at its full size, against float64 (oracle/train_chunk_case.py): the
full-size synth-313 body, one 1024-ray chunk, 64 coarse + 128 importance samples (a 192-sample fine pass), the loss
mse(rgb_map) + mse(rgb0), through Renderer.get_pixel_value and loss.backward(), for both training precisions.  Every other
gradient test runs a 24 x 24 scene at a quarter of the body's size; here the sample lists are ~1e5 entries long (each of
the 74 weight-gradient splits reduces several thousand rows), the trilinear scatter and the gradient blob run at the full
level dims, and one Renderer's buffer pool holds the two passes' activation records and hands them to the next step.

The fine depths are fixed before the step: the coarse pass is run once at the training precision on a separate Renderer,
its weights give the fine depths through ray_stages.sample_pdf_emulate (bit-exact with nb_sample_pdf), and the importance
uniforms of every fragile fine sample are redrawn.  The step itself must then merge exactly those depths (the coarse
forward is deterministic per sample), which the test checks bit for bit before comparing gradients.

Per slice -- each decoder tensor, the used latent row, each volume level -- rel-L2 <= GATE and max |g - r| <= TAU max |r|;
the maps within MAP_TOL; the latent rows no frame uses exactly zero.  Also: a differentiable render of more samples per ray
than the backward takes is refused by the forward, before anything is enqueued."""
import time

import pytest
import torch

from oracle import grad_case
from oracle import train_chunk_case as TC
from tools import map_grad_case as MC

GATE = 1e-3          # rel-L2 per slice (the gate of tests/test_backward.py and tests/test_distinct_frames.py)
# max |g - r| <= TAU * max |r| per slice: ~3x the worst slice measured on an H100 80GB HBM3 (700 W power limit), alpha_fc.bias
# of chunk A on tc_tf32x3 at 5.4e-5 (fp32: vol0 at 1.3e-5).  Weight-gradient GEMMs run as one TF32 pass instead of three
# measured 7.3e-4 here (rel-L2 6.6e-4, under GATE): this bound is what tells them apart.
TAU = 1.6e-4
MAP_TOL = 1e-4
WGRAD_SPLITS = 74    # the weight-gradient GEMMs split the list over 74 CTAs (nb_train.cu)
TRAIN_PRECISIONS = ["tc_tf32x3", "fp32"]
CFG = {"N_samples": TC.N_SAMPLES, "perturb": 1.0, "white_bkgd": False, "raw_noise_std": 0, "render_precision": "tc_fp16x3",
       "render_volume_dtype": "auto", "chunk": 0, "render_skip_empty": True, "render_return_weights": True,
       "render_importance": TC.N_IMPORTANCE}

_CASES = {}
_REF = {}


@pytest.fixture
def c3_cfg():
    """run_c3's configuration for the duration of a test (the config is global: restore what was there)."""
    from neuralbody_b200.lib.config import cfg
    keys = list(CFG) + ["render_train_precision"]
    old = {k: cfg[k] for k in keys if k in cfg}
    for k, v in CFG.items():
        cfg[k] = v
    yield cfg
    for k in keys:
        if k in old:
            cfg[k] = old[k]
        elif k in cfg:
            del cfg[k]


def _case(chunk):
    if chunk not in _CASES:
        if "scene" not in _CASES:
            _CASES["scene"] = TC.full_scene()
        _CASES[chunk] = TC.build(chunk, _CASES["scene"])
    return _CASES[chunk]


def _net(scene):
    """run_c3's network: train mode, every decoder tensor and volume a leaf."""
    import gpu_utils as Gu
    net, ren = Gu.make_net_and_renderer(scene)
    net.train()
    for p in net.parameters():
        p.requires_grad_(True)
    vols = [v.cuda().requires_grad_(True) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    return net, ren, vols


def _batch(ren, scene):
    import gpu_utils as Gu
    batch = {k: scene[k].cuda() for k in Gu.BATCH_KEYS}
    return batch, ren.prepare_sp_input(batch)


def _counts(stats):
    return {k: v for k, v in stats.items() if k != "scale"}


def reference(chunk, train_precision, cfg):
    """(case, u, Z, float64 grads, float64 maps) of `chunk` at `train_precision`, cached: the coarse weights come from the
    training precision's own forward (a Renderer of its own, so the tested one's pool starts empty)."""
    from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer
    key = (chunk, train_precision)
    if key not in _REF:
        case = _case(chunk)
        net, _, vols = _net(case["scene"])
        side = make_renderer(cfg, net)
        batch, sp = _batch(side, case["scene"])
        coarse = side.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp,
                                  t_rand=case["t_rand"].cuda(), want_weights=True)
        assert coarse["weights"].grad_fn is not None            # the training precision's forward, not inference
        weights = coarse["weights"].detach().cpu()
        del coarse
        side.release()
        t0 = time.perf_counter()
        u, Z, stats = TC.fine_depths(case, weights)
        t_cond = time.perf_counter() - t0
        grads, maps, t_ref = TC.oracle_step(case, Z)
        print("chunk %s %s: coarse conditioning %s, fine conditioning %s (%.1f s), float64 oracle step %.1f s on %d threads" % (
            chunk, train_precision, _counts(case["stats"]["coarse"]), _counts(stats), t_cond, t_ref, torch.get_num_threads()))
        _REF[key] = (case, u, Z, grads, maps)
    return _REF[key]


def _step(ren, net, vols, case, u):
    """One c3 step through ren.get_pixel_value (cfg.render_importance = 128) with the case's jitter and uniforms, then
    loss.backward().  Returns (maps, grads, the z_all the fine pass ran on)."""
    batch, sp = _batch(ren, case["scene"])
    seen = []
    z_vals_of = ren.importance_z_vals
    hierarchical = ren.render_rays_hierarchical

    def spy(*a, **kw):
        z_all, z_smp = z_vals_of(*a, **kw)
        seen.append(z_all.detach().cpu())
        return z_all, z_smp
    ren.importance_z_vals = spy
    ren.render_rays_hierarchical = lambda *a, **kw: hierarchical(*a, t_rand=case["t_rand"].cuda(), u=u.cuda(), **kw)
    try:
        for p in net.parameters():
            p.grad = None
        for v in vols:
            v.grad = None
        out = ren.get_pixel_value(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, batch)
        TC.loss_of(out, case["target"].cuda()).backward()
        torch.cuda.synchronize()
    finally:
        del ren.importance_z_vals, ren.render_rays_hierarchical
    assert len(seen) == 1
    maps = {k: out[k].detach().cpu() for k in ("rgb_map", "rgb0", "acc_map", "depth_map", "weights")}
    grads = {k: p.grad for k, p in net.named_parameters() if k in grad_case.GRAD_KEYS}
    grads.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return maps, grads, seen[0]


def _check(label, maps, got, z_all, case, Z, ref, ref_maps):
    """z_all == Z bit for bit, the maps, then every gradient slice; returns {slice: (rel-L2, max err / max |r|)}."""
    assert torch.equal(z_all.view(torch.int32), Z.view(torch.int32)), \
        (label, "the step's merged depths differ from the emulated ones", int((z_all != Z).sum()))
    for k in ("rgb_map", "rgb0", "acc_map", "depth_map", "weights"):
        d = float((maps[k].double() - ref_maps[k]).abs().max())
        assert d < MAP_TOL, (label, k, d)
    for k, r in ref.items():
        assert got[k] is not None and got[k].shape == r.shape, k
    got = {k: v.detach().cpu().double() for k, v in got.items()}
    rows = sorted(set(case["scene"]["latent_index"].tolist()))
    unused = [r for r in range(got["latent.weight"].shape[0]) if r not in rows]
    assert not bool(got["latent.weight"][unused].any()), [r for r in unused if got["latent.weight"][r].any()]
    names = {"latent[%d]" % r: ("latent.weight", r) for r in rows}
    names.update({k: (k, None) for k in ref if k != "latent.weight"})
    report, bad = {}, {}
    for name, (k, row) in names.items():
        g, r = (got[k], ref[k]) if row is None else (got[k][row], ref[k][row])
        assert bool(torch.isfinite(g).all()) and bool(torch.isfinite(r).all()), name
        scale = float(r.abs().max())
        assert scale > 0, name
        e, m = MC.rel_l2_finite(g, r), float((g - r).abs().max()) / scale
        report[name] = (e, m)
        if not (e <= GATE and m <= TAU):
            bad[name] = (e, m)
    worst = max(report.items(), key=lambda kv: kv[1][1])
    print(label, "worst max-err slice: %s %.2e;" % (worst[0], worst[1][1]), "(rel-L2 / max err)",
          {k: "%.1e/%.1e" % v for k, v in report.items()})
    assert not bad, (label, bad)
    return report


def _check_listed(label, listed, case, Z):
    """The list lengths of the coarse and the fine pass against the float64 count of samples with a non-zero feature."""
    for name, depths, (count, total) in (("coarse", TC.coarse_depths(case["scene"], case["t_rand"]), listed[0]),
                                         ("fine", Z, listed[1])):
        assert total == TC.N_RAYS * depths.shape[-1], (name, total)
        occupied, near_face = TC.listed_bounds(case, depths)
        print(label, name, "listed %d of %d; float64: %d with a non-zero feature off the cell faces, %d within FACE_MARGIN of "
              "one (left out)" % (count, total, occupied, near_face))
        assert occupied <= count <= occupied + near_face, (label, name, count, occupied, near_face)
        # several 128-row tiles per weight-gradient split, and a last tile the list does not fill
        assert count > WGRAD_SPLITS * 16 * 8 and count % 128 != 0, (label, name, count)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_train_chunk_step(c3_cfg, train_precision):
    """run_c3's step on chunk A through a fresh Renderer: the merged depths, the maps, every gradient slice and (tc_tf32x3)
    the list lengths of both passes."""
    c3_cfg.render_train_precision = train_precision
    case, u, Z, ref, ref_maps = reference("A", train_precision, c3_cfg)
    net, ren, vols = _net(case["scene"])
    maps, got, z_all = _step(ren, net, vols, case, u)
    _check("%s chunk A" % train_precision, maps, got, z_all, case, Z, ref, ref_maps)
    if train_precision == "tc_tf32x3":
        listed = ren.train_listed_samples()
        assert len(listed) == 2, listed
        _check_listed("%s chunk A" % train_precision, listed, case, Z)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", TRAIN_PRECISIONS)
def test_steps_through_one_renderer(c3_cfg, train_precision):
    """Chunk A, chunk B, chunk A again through the same Renderer and network, gradients set to None in between as bench.py's
    step does: each step reuses the pooled activation records and backward scratch of the one before with other list
    lengths -- one transition lengthens a pass's list and the other shortens it, leaving the longer list's tail in the
    buffer -- and each step must match its own reference."""
    c3_cfg.render_train_precision = train_precision
    refs = {c: reference(c, train_precision, c3_cfg) for c in ("A", "B")}
    net, ren, vols = _net(refs["A"][0]["scene"])
    listed = []
    for i, chunk in enumerate(("A", "B", "A")):
        # the chunks share the frame: only the rays differ (the volumes and the network are the same leaves)
        case, u, Z, ref, ref_maps = refs[chunk]
        maps, got, z_all = _step(ren, net, vols, case, u)
        _check("%s step %d (chunk %s)" % (train_precision, i + 1, chunk), maps, got, z_all, case, Z, ref, ref_maps)
        if train_precision == "tc_tf32x3":
            listed.append([c for c, _ in ren.train_listed_samples()[-2:]])
    if listed:
        for p, name in enumerate(("coarse", "fine")):
            n = [step[p] for step in listed]
            print(train_precision, name, "list lengths A -> B -> A: %d -> %d -> %d (%s, then %s)" % (
                n[0], n[1], n[2], "grew" if n[1] > n[0] else "shrank", "grew" if n[2] > n[1] else "shrank"))
            assert n[0] != n[1] and n[2] == n[0], (name, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n_samples,n_importance", [(257, 0), (64, 256)])
def test_differentiable_render_over_the_backward_limit_refused(c3_cfg, n_samples, n_importance):
    """S = 257, and a hierarchical 64 + 256: the backward takes rays of at most 256 samples, so the forward raises before it
    packs, draws or launches anything; the same call without autograd still renders."""
    from oracle import synth
    scene = synth.make_scene(H=24, W=24, scale=0.25, all_hit=True)
    c3_cfg.N_samples, c3_cfg.render_importance = n_samples, n_importance
    net, ren, vols = _net(scene)
    batch, sp = _batch(ren, scene)
    args = (batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, batch)
    rng = torch.get_rng_state()
    with pytest.raises(NotImplementedError, match="at most 256 samples per ray"):
        ren.get_pixel_value(*args)
    torch.cuda.synchronize()
    assert ren.launches == 0 and ren._vol_key is None and ren._w_key is None and "_pool" not in ren.__dict__
    assert torch.equal(torch.get_rng_state(), rng)             # no jitter / uniforms drawn either
    with torch.no_grad():
        out = ren.get_pixel_value(*args)
    torch.cuda.synchronize()
    S = n_samples + n_importance
    assert out["weights"].shape == (1, scene["ray_o"].shape[1], S) and bool(torch.isfinite(out["rgb_map"]).all())
    assert ren.launches > 0
