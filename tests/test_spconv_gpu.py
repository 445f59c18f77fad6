"""GPU: the sparse CUDA encoder (nb_spconv_fwd / nb_spconv_bwd, CudaSparseConvNet) against float64 references -- the
brute-force restatement of spconv (oracle/spconv_oracle.py) on small blobs, and the dense emulation DenseSparseConvNet run in
float64 on the synth-313 body (6890 vertices, one frame and a batch of two poses) -- forward in train and eval mode, the
running statistics, the backward into the code, every conv weight and every BatchNorm weight and bias, one training step
through the trainer drop-in, and the absence of host synchronisation."""
import os

import numpy as np
import pytest
import torch

from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet
from oracle import spconv_oracle as SO
from oracle import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _blob_coords(B, shape, n_vert, seed):
    """(B * n_vert, 4) frame-major coords of a blob (so neighbours exist and several vertices share sites), plus points on
    the first and last plane of every axis."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for b in range(B):
        c = torch.stack([torch.randint(0, s, (n_vert,), generator=g) for s in shape], 1)
        for ax, s in enumerate(shape):
            c[:, ax] = (c[:, ax] // 2 + s // 4).clamp(0, s - 1)
        for ax, s in enumerate(shape):
            c[2 * ax, ax], c[2 * ax + 1, ax] = 0, s - 1
        rows.append(torch.cat([torch.full((n_vert, 1), b), c], 1))
    return torch.cat(rows).to(torch.int32)


def _synth_coords(poses):
    """The synth-313 body (6890 vertices, 5 mm voxels) in each pose: (B * 6890, 4) coords and out_sh = the max over the
    frames, as prepare_sp_input builds them."""
    coords, shs = [], []
    for b, rh in enumerate(poses):
        s = synth.make_scene(H=8, W=8, Rh=rh)
        c = s["coord"][0].long()
        coords.append(torch.cat([torch.full((c.shape[0], 1), b), c], 1))
        shs.append(s["out_sh"][0])
    return torch.cat(coords).to(torch.int32), torch.stack(shs).max(0).values.tolist()


def _nets(seed, running=False):
    """A float64 DenseSparseConvNet with non-trivial BatchNorm parameters (and running statistics), and a CudaSparseConvNet
    holding the same values in float32."""
    torch.manual_seed(seed)
    ref = DenseSparseConvNet()
    with torch.no_grad():
        for m in ref.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                if running:
                    m.running_mean.uniform_(-0.5, 0.5)
                    m.running_var.uniform_(0.5, 2.0)
    ours = CudaSparseConvNet()
    ours.load_state_dict(ref.state_dict())
    return ref.double().to(DEV), ours.to(DEV)


def _code(n_vert, seed):
    return torch.randn(n_vert, 16, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _masks(coord, out_sh, B):
    """The active set of every level, from the emulation's own rules (float64 masks)."""
    D, H, W = out_sh
    c = coord.long().to(DEV)
    m = torch.zeros((B, 1, D, H, W), dtype=torch.float64, device=DEV)
    m[c[:, 0], 0, c[:, 1], c[:, 2], c[:, 3]] = 1.0
    out = []
    for _ in range(4):
        m = torch.nn.functional.max_pool3d(m, 3, stride=2, padding=1)
        out.append(m)
    return out


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-300))


def _compare_forward(vols, ref, masks, counts, label):
    assert counts[0] > 0
    for lvl, (v, r, m) in enumerate(zip(vols, ref, masks)):
        assert v.shape == r.shape, (label, lvl)
        assert int(counts[lvl + 1]) == int(m.sum()), "%s level %d: %d active rows, the reference has %d" % (
            label, lvl + 1, int(counts[lvl + 1]), int(m.sum()))
        assert float((v.double() * (1 - m)).abs().max()) == 0.0, "%s level %d: non-zero off the active set" % (label, lvl)
        rel, mx = _rel_l2(v, r), float((v.double() - r).abs().max())
        assert rel <= 1e-5 and mx <= 1e-4 * float(r.abs().max()), "%s level %d: rel-L2 %.2e, max-abs %.2e (max %.2e)" % (
            label, lvl, rel, mx, float(r.abs().max()))


# BatchNorm over a handful of rows divides the float32 rounding of the conv outputs by their small spread: on a grid whose
# coarsest level holds 4 active sites the float32 dense emulation itself is 1e-5 from float64 there.  These grids keep every
# level's batch large enough for the gate to measure the kernels (the float32 emulation stays under 3.1e-6).
@pytest.mark.parametrize("B,shape,seed", ((1, (9, 12, 10), 0), (2, (21, 30, 19), 2), (2, (24, 32, 22), 1)))
def test_blobs_match_the_sparse_restatement(built_lib, B, shape, seed):
    n_vert = 150
    coord = _blob_coords(B, shape, n_vert, seed)
    ref, ours = _nets(seed)
    code = _code(n_vert, seed)
    params = {k: v.detach().cpu().numpy() for k, v in ref.state_dict().items()}
    want = SO.sparse_conv_net(params, code.double().cpu().repeat(B, 1).numpy(), coord.numpy(), shape, B)
    ours.train()
    with torch.no_grad():
        vols = ours.encode(code, coord.to(DEV), list(shape), B)
    _compare_forward(vols, [torch.from_numpy(w).to(DEV) for w in want], _masks(coord, shape, B), ours.last_row_counts.cpu(),
                     "blob")


def _active_sets_case(coord, out_sh, B, n_vert, seed):
    """With beta = 3 and gamma = 0.01 every active output is > 0 after the ReLU, so the non-zero pattern of each volume is
    exactly its active set."""
    ref, ours = _nets(seed)
    with torch.no_grad():
        for _, bn in ours.convs_and_batchnorms():
            bn.weight.fill_(0.01)
            bn.bias.fill_(3.0)
        vols = ours.train().encode(_code(n_vert, seed), coord.to(DEV), out_sh, B)
    for lvl, (v, m) in enumerate(zip(vols, _masks(coord, out_sh, B))):
        nz = (v != 0).any(1, keepdim=True)
        assert torch.equal(nz, m > 0), "level %d: active sets differ" % (lvl + 1)


def test_active_sets_are_identical(built_lib):
    _active_sets_case(_blob_coords(2, (16, 24, 16), 172, 3), [16, 24, 16], 2, 172, 3)
    coord, out_sh = _synth_coords(POSES["B2"])
    _active_sets_case(coord, out_sh, 2, 6890, 4)


POSES = {"B1": [(0.3, -0.2, 0.1)], "B2": [(0.3, -0.2, 0.1), (-0.4, 0.9, 0.2)]}


@pytest.mark.parametrize("mode", ("train", "eval"))
@pytest.mark.parametrize("batch", sorted(POSES))
def test_synth313_matches_the_float64_emulation(built_lib, batch, mode):
    coord, out_sh = _synth_coords(POSES[batch])
    B = len(POSES[batch])
    ref, ours = _nets(5, running=True)
    code = _code(6890, 5)
    ref.train(mode == "train")
    ours.train(mode == "train")
    with torch.no_grad():
        want = ref.encode(code.double(), coord.to(DEV), out_sh, B)
        vols = ours.encode(code, coord.to(DEV), out_sh, B)
    torch.cuda.synchronize()
    _compare_forward(vols, want, _masks(coord, out_sh, B), ours.last_row_counts.cpu(), "synth %s %s" % (batch, mode))
    # running statistics: updated in train mode exactly as the emulation updates them, untouched in eval mode
    sd_ref, sd_ours = ref.state_dict(), ours.state_dict()
    for k in sd_ref:
        if "running" in k:
            assert _rel_l2(sd_ours[k], sd_ref[k]) <= 1e-5, k
        if "num_batches_tracked" in k:
            assert int(sd_ours[k]) == int(sd_ref[k]) == (1 if mode == "train" else 0), k


def _f32_emulation_grads(ours, code, coord, out_sh, B, cot):
    """Gradients of the float32 dense emulation (exact float32 cuDNN convolutions, no TF32) with ours' parameters."""
    f32 = DenseSparseConvNet().to(DEV)
    f32.load_state_dict(ours.state_dict())
    f32.train(ours.training)
    c = code.clone().requires_grad_(True)
    saved = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        torch.autograd.backward(f32.encode(c, coord.to(DEV), out_sh, B), cot)
    finally:
        torch.backends.cudnn.allow_tf32 = saved
    return dict([("code", c.grad)] + [(k, p.grad) for k, p in f32.named_parameters()])


# Train-mode BatchNorm on the full-size body: float32 arithmetic itself is ~1e-3 from float64 there (the float32 dense
# emulation is 1.4e-3 to 3e-3 off on almost every gradient), so that case is held to twice the float32 emulation's own
# error, tensor by tensor, and to 1e-4 where that is larger.  Every other case is held to 1e-4.
@pytest.mark.parametrize("mode", ("train", "eval"))
@pytest.mark.parametrize("case", ("blob_B2", "synth_B1"))
def test_backward_matches_float64_autograd(built_lib, case, mode):
    if case == "blob_B2":
        B, out_sh, n_vert = 2, [16, 24, 16], 150
        coord = _blob_coords(B, out_sh, n_vert, 6)
    else:
        coord, out_sh = _synth_coords(POSES["B1"])
        B, n_vert = 1, 6890
    ref, ours = _nets(7, running=True)
    ref.train(mode == "train")
    ours.train(mode == "train")
    code = _code(n_vert, 7)
    code64 = code.double().requires_grad_(True)
    code32 = code.clone().requires_grad_(True)
    want = ref.encode(code64, coord.to(DEV), out_sh, B)
    vols = ours.encode(code32, coord.to(DEV), out_sh, B)
    g = torch.Generator(device=DEV).manual_seed(8)
    cot = [torch.randn(v.shape, generator=g, device=DEV) for v in vols]
    torch.autograd.backward(want, [c.double() for c in cot])
    torch.autograd.backward(vols, cot)
    pairs = [("code", code32.grad, code64.grad)]
    named_ref = dict(ref.named_parameters())
    for k, p in ours.named_parameters():
        pairs.append((k, p.grad, named_ref[k].grad))
    assert len(pairs) == 1 + 17 * 3
    f32 = _f32_emulation_grads(ours, code, coord, out_sh, B, cot) if (case, mode) == ("synth_B1", "train") else None
    for k, a, b in pairs:
        assert a is not None and torch.isfinite(a).all(), k
        gate = 1e-4 if f32 is None else max(1e-4, 2 * _rel_l2(f32[k], b))
        assert _rel_l2(a, b) <= gate, "%s: rel-L2 %.2e > %.2e" % (k, _rel_l2(a, b), gate)


def test_encode_does_not_wait_for_the_host(built_lib):
    coord, out_sh = _synth_coords(POSES["B2"])
    _, ours = _nets(9)
    code = _code(6890, 9).requires_grad_(True)
    coord = coord.to(DEV)
    cot = None
    ours.train()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        vols = ours.encode(code, coord, out_sh, 2)
        cot = [torch.ones_like(v) for v in vols]
        torch.autograd.backward(vols, cot)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert code.grad is not None and torch.isfinite(code.grad).all()
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "neuralbody_b200", "lib", "networks",
                            "sparse_encode_cuda.py")).read()
    for call in (".item(", ".tolist(", ".cpu(", "synchronize"):
        assert call not in src, call


def _train_setup(scene, n_rays=1024):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from neuralbody_b200.lib.networks.make_network import make_network
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(scene["ray_o"].shape[1], generator=g)[:n_rays]
    batch = {k: scene[k][:, idx].contiguous().to(DEV) for k in ("ray_o", "ray_d", "near", "far")}
    batch.update({k: scene[k].to(DEV) for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")})
    batch["rgb"] = torch.rand((1, n_rays, 3), generator=g).to(DEV)
    batch["mask_at_box"] = torch.ones((1, n_rays), dtype=torch.bool, device=DEV)
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.voxel_size = list(scene["voxel_size"])
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.render_importance = "tc_fp16x3", "auto", 0
    cfg.render_train_precision, cfg.render_return_weights = "tc_tf32x3", True
    net = make_network(cfg)
    net.load_state_dict(scene["weights"], strict=False)
    mod = load_source("lib.train.trainers.if_nerf_clight", os.path.join(
        os.path.dirname(os.path.abspath(__file__)), "..", "neuralbody_b200", "lib", "train", "trainers", "if_nerf_clight.py"))
    return net, mod, batch


@pytest.fixture
def cuda_cfg():
    """sparse_encode = 'cuda' for one test, in this package's cfg (which the yaml test merges into) and in the one the
    network reads when it is built (get_active_cfg(): upstream's once the reference's lib.config is loaded); both are
    restored after the test."""
    from neuralbody_b200.lib.config import cfg, get_active_cfg
    saved = cfg.clone()
    active = get_active_cfg()
    had, old = "sparse_encode" in active, active.get("sparse_encode")
    dict.__setitem__(cfg, "sparse_encode", "cuda")
    dict.__setitem__(active, "sparse_encode", "cuda")
    yield cfg
    cfg.clear()
    cfg.update(saved)
    if active is not cfg:
        dict.pop(active, "sparse_encode", None)
        if had:
            dict.__setitem__(active, "sparse_encode", old)


def test_training_step_through_the_trainer_matches_the_float64_encode(built_lib, cuda_cfg):
    scene = synth.make_scene(H=256, W=256, scale=1.0, all_hit=True)
    net, mod, batch = _train_setup(scene)
    ref, _ = _nets(11)
    net.xyzc_net.load_state_dict(ref.state_dict())
    net = net.to(DEV).train()
    ref.train()
    wrapper = mod.NetworkWrapper(net)
    # the reference: the float64 emulation's volumes, rounded to float32, through the same render and loss
    sp = wrapper.renderer.prepare_sp_input(batch)
    code64 = net.c.weight.detach().double().requires_grad_(True)
    vols64 = ref.encode(code64, sp["coord"], sp["out_sh"], sp["batch_size"])
    vols_ref = [v.detach().float().requires_grad_(True) for v in vols64]
    net.set_feature_volume(vols_ref)
    ret_ref, loss_ref, _, _ = wrapper(dict(batch))
    loss_ref.backward()
    torch.autograd.backward(vols64, [v.grad.double() for v in vols_ref])
    fc0_ref = net.fc_0.weight.grad.clone()
    maps_ref = {k: ret_ref[k].detach() for k in ("rgb_map", "acc_map", "depth_map")}
    net.zero_grad(set_to_none=True)
    net.set_feature_volume(None)
    # the CUDA encoder: encode_sparse_voxels runs it inside the render
    ret, loss, _, _ = wrapper(dict(batch))
    loss.backward()
    torch.cuda.synchronize()
    for k, v in maps_ref.items():
        d = float((ret[k].detach() - v).abs().max())
        assert d <= 1e-4, "%s differs by %.2e" % (k, d)
    assert _rel_l2(net.c.weight.grad, code64.grad) <= 1e-3, _rel_l2(net.c.weight.grad, code64.grad)
    assert _rel_l2(net.fc_0.weight.grad, fc0_ref) <= 1e-3, _rel_l2(net.fc_0.weight.grad, fc0_ref)
    assert float(net.xyzc_net.conv0[0].weight.grad.abs().sum()) > 0


def test_yaml_driven_training_loop(built_lib, cuda_cfg):
    """train_net.py's loop, with the encoder chosen by the yaml key alone: the loss stays finite and every part of the
    network trains, the SparseConvNet included."""
    from neuralbody_b200.lib.config import make_cfg
    here = os.path.dirname(os.path.abspath(__file__))
    make_cfg(os.path.join(here, "..", "neuralbody_b200", "configs", "synth_313.yaml"), ["sparse_encode", "cuda"])
    scene = synth.make_scene(H=256, W=256, scale=1.0, all_hit=True)
    net, mod, batch = _train_setup(scene)
    assert type(net.xyzc_net).__name__ == "CudaSparseConvNet"
    net = net.to(DEV).train()
    wrapper = mod.NetworkWrapper(net)
    opt = torch.optim.Adam(net.parameters(), lr=5e-4)
    w0 = net.xyzc_net.conv2[3].weight.detach().clone()
    losses = []
    for _ in range(3):
        opt.zero_grad()
        _, loss, _, _ = wrapper(dict(batch))
        loss.backward()
        torch.nn.utils.clip_grad_value_(net.parameters(), 40)
        opt.step()
        losses.append(float(loss))
    assert all(np.isfinite(losses)), losses
    assert not torch.equal(w0, net.xyzc_net.conv2[3].weight.detach())
    assert int(net.xyzc_net.conv4[7].num_batches_tracked) == 3
