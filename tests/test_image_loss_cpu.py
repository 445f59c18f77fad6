"""CPU: the training wrapper drop-in without a GPU -- upstream's make_trainer._wrapper_factory loads it by path and builds
a NetworkWrapper, the binding validates its arguments before any CUDA call, and a restatement of nb_image_loss's
reduction (csrc/nb_image_loss.cu: per-thread grid-stride sums in float64, a fixed tree per CTA, the CTAs in order) and of
its cotangent rounding agrees with float64 (loss) and with torch autograd bit for bit (cotangent).  The GPU tests
(test_image_loss_gpu.py) hold the kernel to the same restatements."""
import ctypes
import importlib.machinery
import importlib.util
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

THREADS, MAX_CTAS = 256, 2 * 132      # kLossThreads, kLossMaxCtas


def restate_loss(pred, gt, mask=None):
    """nb_image_loss_fwd in numpy: (loss float32, count).  The kernel's per-thread sum is an fma chain; here d*d is rounded
    before the add, which moves the float64 sum by ulps only."""
    x = np.asarray(pred, np.float32).reshape(-1).astype(np.float64)
    y = np.asarray(gt, np.float32).reshape(-1).astype(np.float64)
    elems = x.size
    keep = np.ones(elems, bool) if mask is None else np.repeat(np.asarray(mask).reshape(-1) != 0, 3)
    ctas = int(min(max(1, -(-elems // THREADS)), MAX_CTAS))
    stride = ctas * THREADS
    d2 = np.where(keep, (x - y) ** 2, 0.0)
    pad = -(-elems // stride) * stride
    d2 = np.concatenate([d2, np.zeros(pad - elems)]).reshape(-1, stride)      # row k: iteration k of every thread
    cnt = np.concatenate([keep, np.zeros(pad - elems, bool)]).reshape(-1, stride)
    per_thread = np.zeros(stride)
    for row in d2:                                                          # each thread's chain, in its order
        per_thread = per_thread + row
    per_thread_c = cnt.sum(0)

    def tree(v):          # the CTA's fixed tree: shuffle-down within each warp, then over the warps
        v = v.reshape(-1, 32).copy()
        for o in (16, 8, 4, 2, 1):
            v[:, :o] = v[:, :o] + v[:, o:2 * o]
        w = np.concatenate([v[:, 0], np.zeros(32 - v.shape[0])])
        for o in (16, 8, 4, 2, 1):
            w[:o] = w[:o] + w[o:2 * o]
        return w[0]
    partial = [tree(per_thread[b * THREADS:(b + 1) * THREADS]) for b in range(ctas)]
    count = int(per_thread_c.sum())
    lanes = np.zeros(THREADS)
    for i, p in enumerate(partial):                                          # the finishing CTA: thread i % 256
        lanes[i % THREADS] += p
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.float32(tree(lanes) / np.float64(count)), count


def restate_cotangent(pred, gt, mask, g, count):
    """nb_image_loss_bwd in torch float32 ops: g * (1 / N), times 2 * (pred - gt); 0 + v on a masked call; 0 off the mask."""
    x, y = torch.as_tensor(pred, dtype=torch.float32), torch.as_tensor(gt, dtype=torch.float32)
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(count), dtype=torch.float32)
    v = (torch.as_tensor(g, dtype=torch.float32) * inv) * (2.0 * (x - y))
    if mask is None:
        return v
    m = torch.as_tensor(mask).bool()[..., None]
    return torch.where(m, torch.zeros_like(v) + v, torch.zeros_like(v))


def _case(B, n, kind, seed):
    rng = np.random.RandomState(seed)
    pred = rng.rand(B, n, 3).astype(np.float32)
    gt = rng.rand(B, n, 3).astype(np.float32)
    mask = {"all": np.ones((B, n), bool), "partial": rng.rand(B, n) < 0.6, "empty": np.zeros((B, n), bool)}[kind]
    if kind == "partial":
        mask.flat[0] = True
    return pred, gt, mask


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("kind", ["all", "partial", "empty"])
@pytest.mark.parametrize("n", [1, 1024, 70001])
def test_restated_reduction_matches_float64(B, kind, n):
    pred, gt, mask = _case(B, n, kind, 7 * B + n)
    loss, count = restate_loss(pred, gt, mask)
    m = np.repeat(mask.reshape(-1), 3)
    d = (pred.astype(np.float64) - gt).reshape(-1)[m]
    assert count == d.size
    if kind == "empty":
        assert np.isnan(loss)
        return
    ref = np.mean(d ** 2)
    assert abs(float(loss) - ref) <= 1e-6 * ref
    l0, c0 = restate_loss(pred, gt)                       # img_loss0: no mask
    assert c0 == pred.size and abs(float(l0) - np.mean((pred.astype(np.float64) - gt) ** 2)) <= 1e-6 * float(l0)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("kind", ["all", "partial", "empty"])
@pytest.mark.parametrize("g", [1.0, 0.5])
def test_restated_cotangent_is_autograds(B, kind, g):
    """Bit for bit against autograd through upstream's expression.  torch's CPU division by a scalar divides where its CUDA
    kernel multiplies by the reciprocal; for the power-of-two g of loss.backward() both give the same bits (the GPU test
    takes arbitrary g against CUDA autograd)."""
    pred, gt, mask = _case(B, 1024, kind, 11 * B)
    x = torch.from_numpy(pred).requires_grad_(True)
    y, m = torch.from_numpy(gt), torch.from_numpy(mask)
    loss = torch.mean((x[m] - y[m]) ** 2)
    loss.backward(torch.tensor(g))
    _, count = restate_loss(pred, gt, mask)
    got = restate_cotangent(pred, gt, mask, g, count)
    assert torch.equal(got.view(torch.int32), x.grad.view(torch.int32))
    x0 = torch.from_numpy(pred).requires_grad_(True)
    torch.mean((x0 - y) ** 2).backward(torch.tensor(g))
    assert torch.equal(restate_cotangent(pred, gt, None, g, pred.size).view(torch.int32), x0.grad.view(torch.int32))


def test_wrapper_factory_loads_the_dropin(built_lib):
    """upstream's make_trainer._wrapper_factory: imp.load_source(cfg.trainer_module, cfg.trainer_path).NetworkWrapper(net)
    (SourceFileLoader, which imp.load_source wraps)."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import make_network
    from neuralbody_b200.lib.networks.renderer import if_nerf_renderer
    cfg.num_train_frame = 4
    net = make_network(cfg)
    trainer_module = "lib.train.trainers.if_nerf_clight"
    trainer_path = os.path.join(ROOT, "neuralbody_b200", "lib", "train", "trainers", "if_nerf_clight.py")
    loader = importlib.machinery.SourceFileLoader(trainer_module, trainer_path)
    mod = importlib.util.module_from_spec(importlib.util.spec_from_loader(trainer_module, loader))
    loader.exec_module(mod)
    wrapper = mod.NetworkWrapper(net)
    assert isinstance(wrapper, torch.nn.Module) and wrapper.net is net
    assert isinstance(wrapper.renderer, if_nerf_renderer.Renderer) and wrapper.renderer.net is net
    assert {n for n, _ in wrapper.named_parameters()} == {"net." + n for n, _ in net.named_parameters()}


def test_binding_validates_before_any_cuda_call(built_lib):
    from neuralbody_b200 import capi, image_loss
    lib = capi.load()
    assert "nb_image_loss_fwd" in capi.EXPORTS and "nb_image_loss_bwd" in capi.EXPORTS
    assert lib.nb_image_loss_workspace_bytes() >= 2 * MAX_CTAS * 8
    a = capi.nb_image_loss_args()
    assert lib.nb_image_loss_fwd(None, None) < 0 and b"null" in lib.nb_last_error()
    a.rays = -1
    a.count = 8
    assert lib.nb_image_loss_fwd(ctypes.byref(a), None) < 0 and b"rays" in lib.nb_last_error()
    a.rays = 1 << 30
    assert lib.nb_image_loss_bwd(ctypes.byref(a), None, None, None) < 0
    x = torch.zeros(4, 3)
    with pytest.raises(ValueError, match="CUDA"):
        image_loss.image_mse(x, x)
