"""Gradients of the rays ray_o / ray_d (camera refinement).  CPU: the oracle's autograd reproduces the unmodified reference's
d ray_o / d ray_d (tests/golden/grad_rays_b2_s32.npz, tools/ray_grad_case.py), every path from the rays to the loss carries
gradient on this case, and the C entry point is exported, bound and validates its arguments.  GPU: Renderer + loss.backward()
against the oracle's autograd on the 2-frame case, both training precisions; rel-L2 <= 1e-3 per tensor, the gate of
tests/test_backward.py and tests/test_frame_grad.py."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import grad_case
from tools import ray_grad_case as RC

GATE = 1e-3
# Cutting one path (tools/ray_grad_case.render_detached) must move d ray_o or d ray_d by more than this (rel-L2).  Measured
# on this case: view direction 1.4e-2 and |ray_d| in raw2outputs 1.4e-2 of d ray_d; points into PE(xyz) 0.45 and points into
# the grid 0.85 of both.  5e-3 is five times the GPU gate, so a kernel that dropped any one path fails that gate.
PATH_MARGIN = 5e-3


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def case():
    from oracle import synth
    scene, t_rand, G = RC.build()
    gold = load_golden(RC.GOLDEN)
    assert synth.scene_checksum(scene) == gold["input_sha256"]
    return scene, t_rand, G, gold


def test_oracle_ray_grads_match_reference(case):
    scene, t_rand, G, gold = case
    g, _ = RC.oracle_ray_grads(scene, t_rand, G)
    assert g["ray_o"].shape == scene["ray_o"].shape and g["ray_d"].shape == scene["ray_d"].shape
    np.testing.assert_allclose(g["ray_o"].numpy(), gold["d_ray_o"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(g["ray_d"].numpy(), gold["d_ray_d"], rtol=1e-5, atol=1e-5)
    assert float(np.abs(gold["d_ray_o"]).max()) > 1.0 and float(np.abs(gold["d_ray_d"]).max()) > 1.0   # not vacuous


def test_every_ray_path_carries_gradient(case):
    """Detaching, in turn, the view direction, the norm in raw2outputs, the points fed to PE(xyz) and the points fed to the
    grid each moves the ray gradients by more than PATH_MARGIN; with nothing detached the restatement is the oracle's."""
    scene, t_rand, G, gold = case
    o0, d0, raw = RC.render_detached(scene, t_rand, G)
    np.testing.assert_allclose(o0.numpy(), gold["d_ray_o"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(d0.numpy(), gold["d_ray_d"], rtol=1e-5, atol=1e-5)
    # The last sample's delta is 1e10 |ray_d|, so its |ray_d| term relu(sigma) 1e10 exp(-relu(sigma) 1e10 |ray_d|) is
    # ill-conditioned for a tiny positive sigma (upstream has the same expression).  On this case every last sample is
    # empty (sigma < 0), so that term is exactly 0 here.
    assert float(raw[:, -1, 3].max()) < 0.
    for path in RC.PATHS:
        o, d, _ = RC.render_detached(scene, t_rand, G, detach=(path,))
        moved = max(_rel_l2(o, o0), _rel_l2(d, d0))
        assert moved > PATH_MARGIN, (path, moved)


def test_ray_entry_point_exported_and_bound(built_lib):
    from neuralbody_b200 import capi
    lib = ctypes.CDLL(built_lib)
    assert hasattr(lib, "nb_render_bwd_rays")
    assert "nb_render_bwd_rays" in capi.EXPORTS
    bound = capi.load()
    assert bound.nb_abi_version() == 5
    assert bound.nb_render_bwd_rays.restype is ctypes.c_int
    assert len(bound.nb_render_bwd_rays.argtypes) == 6


def test_ray_entry_point_rejects_null_args(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_render_bwd_rays(None, None, None, None, None, None) == -1      # NB_ERR_BAD_ARG, before any CUDA call
    err = lib.nb_last_error().decode()
    assert err.startswith("nb_render_bwd:") and "null" in err, err
    ba = capi.nb_render_bwd_args()                                                # fwd / save / raw / ... unset
    assert lib.nb_render_bwd_rays(ctypes.byref(ba), None, None, None, None, None) == -1


# ------------------------------------------------------------------------------------------------------------------ GPU
def _setup(scene, train_precision, decoder=False, frame=False, importance=0, chunk=0, perturb=1.0):
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    dev = "cuda:0"
    net, ren = Gu.make_net_and_renderer(scene, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = RC.N_SAMPLES, perturb, True, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = "tc_fp16x3", "auto", chunk
    cfg.render_train_precision = train_precision
    cfg.render_importance = importance
    net.train()
    for p in net.parameters():
        p.requires_grad_(decoder)
    vols = [v.to(dev).requires_grad_(decoder) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].to(dev) for k in Gu.BATCH_KEYS}
    batch["R"].requires_grad_(frame)
    batch["Th"].requires_grad_(frame)
    batch["ray_o"] = batch["ray_o"].clone().requires_grad_(True)
    batch["ray_d"] = batch["ray_d"].clone().requires_grad_(True)
    return net, ren, vols, batch


def _render(ren, vols, batch, t_rand):
    sp = ren.prepare_sp_input(batch)
    return ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())


def _check(report):
    bad = {k: e for k, e in report.items() if not e <= GATE}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_ray_grads_match_oracle(case, train_precision):
    """Decoder, volumes, frame transform and rays all train: every gradient within the gate in one backward."""
    scene, t_rand, G, _ = case
    ref, ret_ref = RC.oracle_ray_grads(scene, t_rand, G, decoder=True, frame=True)
    net, ren, vols, batch = _setup(scene, train_precision, decoder=True, frame=True)
    out = _render(ren, vols, batch, t_rand)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    ro, rd = batch["ray_o"], batch["ray_d"]
    assert ro.grad.shape == ro.shape and rd.grad.shape == rd.shape and rd.grad.dtype == torch.float32
    got = {"ray_o": ro.grad, "ray_d": rd.grad, "R": batch["R"].grad, "Th": batch["Th"].grad}
    got.update({k: p.grad for k, p in net.named_parameters() if k in grad_case.GRAD_KEYS})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    assert set(got) == set(ref)
    report = {k: _rel_l2(got[k].cpu(), ref[k]) for k in ref}
    print(train_precision, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_ray_grads_only(case, train_precision):
    """Only the rays require grad: the outputs still require grad, backward works, and no parameter, volume or frame tensor
    gets a .grad."""
    scene, t_rand, G, gold = case
    net, ren, vols, batch = _setup(scene, train_precision)
    out = _render(ren, vols, batch, t_rand)
    assert out["rgb_map"].requires_grad
    grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    report = {"ray_o": _rel_l2(batch["ray_o"].grad.cpu(), torch.from_numpy(gold["d_ray_o"])),
              "ray_d": _rel_l2(batch["ray_d"].grad.cpu(), torch.from_numpy(gold["d_ray_d"]))}
    print(train_precision, report)
    _check(report)
    assert all(p.grad is None for p in net.parameters())
    assert all(v.grad is None for v in vols)
    assert batch["R"].grad is None and batch["Th"].grad is None


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_hierarchical_ray_grads(case, train_precision):
    """Coarse + fine pass (render_importance = 48): both _FusedRender nodes add into ray_o.grad / ray_d.grad; the fine pass
    takes the merged depths as given and the importance samples stay detached.  The oracle's fine pass is evaluated at the
    depths the GPU's importance sampling produced: they follow the coarse weights, and a 1e-6 relative shift of them moves
    the ray gradients by ~9e-4 on this case (the 2^9 octave of PE(xyz)), which is forward sensitivity, not the backward."""
    from neuralbody_b200.lib.config import cfg
    scene, t_rand, G, _ = case
    u, rgb0 = RC.hier_inputs(scene)
    G = dict(G, rgb0=rgb0)
    try:
        net, ren, vols, batch = _setup(scene, train_precision, importance=RC.N_IMPORTANCE)
        sampled = {}
        importance_z_vals = ren.importance_z_vals

        def keep_depths(*a, **k):
            r = importance_z_vals(*a, **k)
            sampled["z_all"] = r[0]
            return r
        ren.importance_z_vals = keep_depths
        sp = ren.prepare_sp_input(batch)
        out = ren.render_rays_hierarchical(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp,
                                           t_rand=t_rand.cuda(), u=u.cuda())
    finally:
        cfg.render_importance = 0
    ref, ret_ref = RC.oracle_hier_ray_grads(scene, t_rand, u, G, z_all=sampled["z_all"].cpu())
    for k in ("rgb_map", "depth_map", "acc_map", "rgb0"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    grad_case.hier_loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    report = {k: _rel_l2(batch[k].grad.cpu(), ref[k]) for k in ("ray_o", "ray_d")}
    print(train_precision, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_chunked_render_ray_grads(case, train_precision):
    """render(batch) with cfg.chunk < n (sliced ray views, one launch each) gives the ray gradients of one launch.  No jitter:
    render() draws it per chunk."""
    scene, _, G, _ = case
    grads = []
    for chunk in (0, 40):
        net, ren, vols, batch = _setup(scene, train_precision, chunk=chunk, perturb=0.0)
        out = ren.render(batch)
        grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
        torch.cuda.synchronize()
        grads.append({k: batch[k].grad.cpu() for k in ("ray_o", "ray_d")})
    assert batch["ray_o"].shape[1] > 2 * 40
    report = {k: _rel_l2(grads[1][k], grads[0][k]) for k in ("ray_o", "ray_d")}
    print(train_precision, report)
    _check(report)
    assert float(grads[0]["ray_d"].abs().max()) > 1.0


@pytest.mark.gpu
def test_mask_views_reject_ray_grads(case):
    """The mask-view renderers are inference only: rays that require grad raise, as R / Th do."""
    scene, t_rand, _, _ = case
    net, ren, vols, batch = _setup(scene, "tc_tf32x3")
    sp = ren.prepare_sp_input(batch)
    with pytest.raises(NotImplementedError, match="mask views are an inference feature"):
        ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, masks={})


def _backward_kernel_names(scene, t_rand, G, train_precision, rays):
    import gpu_utils as Gu
    net, ren, vols, batch = _setup(scene, train_precision, decoder=True)
    if not rays:
        batch["ray_o"].requires_grad_(False)
        batch["ray_d"].requires_grad_(False)
    out = _render(ren, vols, batch, t_rand)
    return Gu.backward_kernel_names(grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}))


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_no_ray_kernel_unless_asked(case, train_precision):
    """A backward that asks for no ray gradient enqueues no ray-gradient kernel; one that does, does, and otherwise runs the
    same kernels."""
    scene, t_rand, G, _ = case
    without = _backward_kernel_names(scene, t_rand, G, train_precision, rays=False)
    assert any("dgrad" in n or "gemm" in n for n in without), sorted(without)     # the profiler saw the backward
    assert not any("ray_grad" in n or "pe_grad" in n or "frame_grad" in n for n in without), sorted(without)
    with_rays = _backward_kernel_names(scene, t_rand, G, train_precision, rays=True)
    assert any("ray_grad_kernel" in n for n in with_rays), sorted(with_rays)
    if train_precision == "tc_tf32x3":
        assert without <= with_rays, sorted(without - with_rays)
    else:   # the fp32 dgrad kernel is instantiated with the grid part of the ray gradients
        assert {n for n in without if "decoder_dgrad" not in n} <= with_rays
