"""Gradients of the frame transform sp_input['R'] / ['Th'] (pose refinement).  CPU: the oracle's autograd reproduces the
unmodified reference's dR / dTh (tests/golden/grad_frame_b2_s32.npz, tools/frame_grad_case.py), and the C entry point is
exported, bound and validates its arguments.  GPU: Renderer.render_rays + loss.backward() against the oracle's autograd on
the 2-frame case, both training precisions; rel-L2 <= 1e-3 per tensor, the gate of tests/test_backward.py."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import grad_case
from tools import frame_grad_case as FC

GATE = 1e-3


@pytest.fixture(scope="module")
def case():
    from oracle import synth
    scene, t_rand, G = FC.build()
    gold = load_golden(FC.GOLDEN)
    assert synth.scene_checksum(scene) == gold["input_sha256"]
    return scene, t_rand, G, gold


def test_oracle_frame_grads_match_reference(case):
    scene, t_rand, G, gold = case
    dR, dTh, _, _, _ = FC.oracle_frame_grads(scene, t_rand, G, decoder=False)
    assert dR.shape == (2, 3, 3) and dTh.shape == (2, 1, 3)
    np.testing.assert_allclose(dR.numpy(), gold["dR"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(dTh.numpy(), gold["dTh"], rtol=1e-5, atol=1e-5)
    assert float(np.abs(gold["dR"]).max()) > 1.0 and float(np.abs(gold["dTh"]).max()) > 1.0   # not vacuous
    assert not np.allclose(gold["dR"][0], gold["dR"][1])                                          # per frame


def test_frame_entry_point_exported_and_bound(built_lib):
    from neuralbody_b200 import capi
    lib = ctypes.CDLL(built_lib)
    assert hasattr(lib, "nb_render_bwd_frame")
    assert "nb_render_bwd_frame" in capi.EXPORTS
    bound = capi.load()
    assert bound.nb_abi_version() == 5
    assert bound.nb_render_bwd_frame.restype is ctypes.c_int
    assert len(bound.nb_render_bwd_frame.argtypes) == 4


def test_frame_entry_point_rejects_null_args(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_render_bwd_frame(None, None, None, None) == -1      # NB_ERR_BAD_ARG, before any CUDA call
    assert b"null" in lib.nb_last_error()
    ba = capi.nb_render_bwd_args()                                     # fwd / save / raw / ... unset
    assert lib.nb_render_bwd_frame(ctypes.byref(ba), None, None, None) == -1


# ------------------------------------------------------------------------------------------------------------------ GPU
def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _setup(scene, train_precision, th_shape, decoder, importance=0):
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    dev = "cuda:0"
    net, ren = Gu.make_net_and_renderer(scene, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = FC.N_SAMPLES, 1.0, True, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = "tc_fp16x3", "auto", 0
    cfg.render_train_precision = train_precision
    cfg.render_importance = importance
    net.train()
    for p in net.parameters():
        p.requires_grad_(decoder)
    vols = [v.to(dev).requires_grad_(decoder) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].to(dev) for k in Gu.BATCH_KEYS}
    B = scene["R"].shape[0]
    batch["R"] = batch["R"].clone().requires_grad_(True)
    batch["Th"] = batch["Th"].reshape((B,) + tuple(th_shape)).clone().requires_grad_(True)
    return net, ren, vols, batch


@pytest.mark.gpu
@pytest.mark.parametrize("th_shape", [(1, 3), (3,)], ids=["Th_B13", "Th_B3"])
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_frame_grads_match_oracle(case, train_precision, th_shape):
    """Decoder, volumes and frame transform all train: every gradient within the gate in one backward."""
    scene, t_rand, G, _ = case
    dR_ref, dTh_ref, pg, vg, ret_ref = FC.oracle_frame_grads(scene, t_rand, G, th_shape=th_shape)
    net, ren, vols, batch = _setup(scene, train_precision, th_shape, decoder=True)
    sp = ren.prepare_sp_input(batch)
    assert sp["R"] is batch["R"] and sp["Th"] is batch["Th"]
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    R, Th = batch["R"], batch["Th"]
    assert R.grad.shape == R.shape and Th.grad.shape == Th.shape and R.grad.dtype == torch.float32
    report = {"dR": _rel_l2(R.grad.cpu(), dR_ref), "dTh": _rel_l2(Th.grad.cpu(), dTh_ref)}
    sd = dict(net.named_parameters())
    for k in grad_case.GRAD_KEYS:
        report[k] = _rel_l2(sd[k].grad.cpu(), pg[k])
    for l, v in enumerate(vols):
        report["vol%d" % l] = _rel_l2(v.grad.cpu(), vg[l])
    print(train_precision, th_shape, report)
    bad = {k: e for k, e in report.items() if not e <= GATE}
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_frame_grads_only(case, train_precision):
    """Only R / Th require grad (frozen decoder and volumes): the call still records an autograd node, backward works,
    and no parameter gets a .grad."""
    scene, t_rand, G, gold = case
    net, ren, vols, batch = _setup(scene, train_precision, (1, 3), decoder=False)
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())
    assert out["rgb_map"].requires_grad
    grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    report = {"dR": _rel_l2(batch["R"].grad.cpu(), torch.from_numpy(gold["dR"])),
              "dTh": _rel_l2(batch["Th"].grad.cpu(), torch.from_numpy(gold["dTh"]))}
    print(train_precision, report)
    assert all(e <= GATE for e in report.values()), report
    assert all(p.grad is None for p in net.parameters())
    assert all(v.grad is None for v in vols)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_hierarchical_frame_grads(case, train_precision):
    """Coarse + fine pass (render_importance = 48): both _FusedRender nodes add into R.grad / Th.grad."""
    from neuralbody_b200.lib.config import cfg
    scene, t_rand, G, _ = case
    u, rgb0 = FC.hier_inputs(scene)
    G = dict(G, rgb0=rgb0)
    dR_ref, dTh_ref, ret_ref = FC.oracle_hier_frame_grads(scene, t_rand, u, G)
    try:
        net, ren, vols, batch = _setup(scene, train_precision, (1, 3), decoder=False, importance=FC.N_IMPORTANCE)
        sp = ren.prepare_sp_input(batch)
        out = ren.render_rays_hierarchical(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp,
                                           t_rand=t_rand.cuda(), u=u.cuda())
    finally:
        cfg.render_importance = 0
    for k in ("rgb_map", "depth_map", "acc_map", "rgb0"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    grad_case.hier_loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    report = {"dR": _rel_l2(batch["R"].grad.cpu(), dR_ref), "dTh": _rel_l2(batch["Th"].grad.cpu(), dTh_ref)}
    print(train_precision, report)
    assert all(e <= GATE for e in report.values()), report


def _backward_kernel_names(scene, t_rand, G, frame):
    import gpu_utils as Gu
    net, ren, vols, batch = _setup(scene, "tc_tf32x3", (1, 3), decoder=True)
    if not frame:
        batch["R"].requires_grad_(False)
        batch["Th"].requires_grad_(False)
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())
    return Gu.backward_kernel_names(grad_case.loss_of(out, {k: v.cuda() for k, v in G.items()}))


@pytest.mark.gpu
def test_no_frame_kernel_unless_asked(case):
    """A backward that asks for no frame-transform gradient enqueues no frame-gradient kernel; one that does, does."""
    scene, t_rand, G, _ = case
    without = _backward_kernel_names(scene, t_rand, G, frame=False)
    assert any("scatter_kernel" in n for n in without), sorted(without)          # the profiler saw the backward
    assert not any("frame_grad" in n for n in without), sorted(without)
    with_frame = _backward_kernel_names(scene, t_rand, G, frame=True)
    assert any("frame_grad_kernel" in n for n in with_frame), sorted(with_frame)
