"""Gradients of near, far, the sample depths and bounds, the last float inputs of the render upstream's autograd reaches.
CPU: the oracle's autograd reproduces the unmodified reference's d near / d far / d bounds (tests/golden/grad_depths_b2_s32.npz,
tools/depth_grad_case.py), each of z's three paths carries gradient on this case, and the C entry points are exported, bound
and validate their arguments.  GPU: Renderer + loss.backward() against the oracle's autograd, both training precisions;
rel-L2 <= 1e-3 per tensor over its finite entries (the gate of tests/test_backward.py)."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import grad_case
from tools import depth_grad_case as DC
from tools import map_grad_case as MC

GATE = 1e-3
# Cutting one of z's paths (tools/depth_grad_case.render_detached) must move d near or d far by more than this (rel-L2):
# five times the GPU gate, so a kernel that dropped any one path fails that gate.
PATH_MARGIN = 5e-3


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def case():
    from oracle import synth
    scene, t_rand, G = DC.build()
    gold = load_golden(DC.GOLDEN)
    assert synth.scene_checksum(scene) == gold["input_sha256"]
    return scene, t_rand, G, gold


def test_oracle_depth_grads_match_reference(case):
    scene, t_rand, G, gold = case
    g, _ = DC.oracle_depth_grads(scene, t_rand, lambda r: grad_case.loss_of(r, G))
    for k in ("near", "far", "bounds", "ray_o", "ray_d"):
        assert g[k].shape == scene[k].shape, k
        np.testing.assert_allclose(g[k].numpy(), gold["d_" + k], rtol=1e-5, atol=1e-5, err_msg=k)
    for k in ("near", "far"):                                                       # not vacuous
        assert float(np.abs(gold["d_" + k]).max()) > 1.0 and np.count_nonzero(gold["d_" + k]) > gold["d_" + k].size // 2, k
    assert float(np.abs(gold["d_bounds"][:, 0]).max()) > 1.0
    assert not gold["d_bounds"][:, 1].any()


def test_every_depth_path_carries_gradient(case):
    """Detaching z, in turn, in the sample points, the dists and the depth map each moves d near / d far by more than
    PATH_MARGIN; with nothing detached the restatement is the oracle's."""
    scene, t_rand, G, gold = case
    n0, f0 = DC.render_detached(scene, t_rand, G)
    np.testing.assert_allclose(n0.numpy(), gold["d_near"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(f0.numpy(), gold["d_far"], rtol=1e-5, atol=1e-5)
    for path in DC.PATHS:
        n, f = DC.render_detached(scene, t_rand, G, detach=(path,))
        moved = max(_rel_l2(n, n0), _rel_l2(f, f0))
        assert moved > PATH_MARGIN, (path, moved)


def test_depth_entry_points_exported_and_bound(built_lib):
    from neuralbody_b200 import capi
    lib = ctypes.CDLL(built_lib)
    for name in ("nb_render_bwd_inputs", "nb_sample_pdf_src"):
        assert hasattr(lib, name) and name in capi.EXPORTS, name
    bound = capi.load()
    assert bound.nb_abi_version() == 5
    assert bound.nb_render_bwd_inputs.restype is ctypes.c_int and len(bound.nb_render_bwd_inputs.argtypes) == 5
    assert bound.nb_sample_pdf_src.restype is ctypes.c_int and len(bound.nb_sample_pdf_src.argtypes) == 3
    assert [f[0] for f in capi.nb_render_input_grads._fields_] == ["d_R", "d_Th", "d_ray_o", "d_ray_d", "d_near", "d_far",
                                                                    "d_z_vals", "d_bounds"]


def test_depth_entry_points_reject_bad_args(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    ig = capi.nb_render_input_grads()
    assert lib.nb_render_bwd_inputs(None, None, None, ctypes.byref(ig), None) == -1      # NB_ERR_BAD_ARG, before any CUDA call
    err = lib.nb_last_error().decode()
    assert err.startswith("nb_render_bwd:") and "null" in err, err
    ba = capi.nb_render_bwd_args()                                                       # fwd / save / raw / ... unset
    assert lib.nb_render_bwd_inputs(ctypes.byref(ba), None, None, ctypes.byref(ig), None) == -1
    assert lib.nb_sample_pdf_src(None, None, None) == -1
    # d_near after a forward that was given its depths (z_vals): rejected before anything is enqueued.  The pointers are
    # dummies that are never dereferenced: the check comes first.
    f = capi.nb_render_args()
    f.z_vals = 16
    ba.fwd = ctypes.pointer(f)
    ba.save = ba.raw = ba.workspace = 16
    w = capi.nb_decoder_weights()
    ba.weights, ba.grads = ctypes.pointer(w), ctypes.pointer(w)
    for field in ("d_near", "d_far"):
        ig = capi.nb_render_input_grads()
        setattr(ig, field, 16)
        assert lib.nb_render_bwd_inputs(ctypes.byref(ba), None, None, ctypes.byref(ig), None) == -1, field
        err = lib.nb_last_error().decode()
        assert "z_vals" in err and "d_near" in err, err


# ------------------------------------------------------------------------------------------------------------------ GPU
def _setup(scene, train_precision, decoder=False, frame=False, rays=False, near_far=True, bounds=True, importance=0, chunk=0,
           perturb=1.0):
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    dev = "cuda:0"
    net, ren = Gu.make_net_and_renderer(scene, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = DC.N_SAMPLES, perturb, True, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = "tc_fp16x3", "auto", chunk
    cfg.render_train_precision = train_precision
    cfg.render_importance = importance
    net.train()
    for p in net.parameters():
        p.requires_grad_(decoder)
    vols = [v.to(dev).requires_grad_(decoder) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].to(dev) for k in Gu.BATCH_KEYS}
    for k, on in (("R", frame), ("Th", frame), ("ray_o", rays), ("ray_d", rays), ("near", near_far), ("far", near_far),
                  ("bounds", bounds)):
        batch[k] = batch[k].clone().requires_grad_(on)
    return net, ren, vols, batch


def _render(ren, vols, batch, t_rand):
    sp = ren.prepare_sp_input(batch)
    return ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())


def _gpu_grads(net, vols, batch, keys):
    got = {k: batch[k].grad for k in ("ray_o", "ray_d", "R", "Th", "near", "far", "bounds")}
    got.update({k: p.grad for k, p in net.named_parameters() if k in grad_case.GRAD_KEYS})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return {k: got[k] for k in keys}


def _compare(got, ref, nan_keys=("ray_d", "near", "far")):
    """rel-L2 per tensor over the finite entries; the NaN pattern must be the reference's, and only nan_keys may have any."""
    report = {}
    for k, r in ref.items():
        g = got[k]
        assert g is not None, k
        g = g.detach().cpu()
        r = r.reshape(g.shape) if k == "Th" else r
        assert g.shape == r.shape and g.dtype == r.dtype, (k, g.shape, r.shape, g.dtype)
        assert torch.equal(torch.isnan(g), torch.isnan(r)), (k, int(torch.isnan(g).sum()), int(torch.isnan(r).sum()))
        if k not in nan_keys:
            assert torch.isfinite(g).all(), k
        report[k] = MC.rel_l2_finite(g, r)
    return report


def _check(report):
    bad = {k: e for k, e in report.items() if not e <= GATE}
    assert not bad, bad


def _loss(G, dev=None):
    G = {k: v.to(dev) for k, v in G.items()} if dev else G
    return lambda r: grad_case.loss_of(r, G)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_depth_grads_everything_training(case, train_precision):
    """Decoder, volumes, R / Th, the rays, near / far and bounds all train: every gradient within the gate."""
    scene, t_rand, G, _ = case
    ref, ret_ref = DC.oracle_depth_grads(scene, t_rand, _loss(G), decoder=True, frame=True)
    net, ren, vols, batch = _setup(scene, train_precision, decoder=True, frame=True, rays=True)
    out = _render(ren, vols, batch, t_rand)
    for k in ("rgb_map", "depth_map", "acc_map"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    _loss(G, "cuda")(out).backward()
    torch.cuda.synchronize()
    report = _compare(_gpu_grads(net, vols, batch, ref), ref)
    print(train_precision, report)
    _check(report)
    assert not bool(batch["bounds"].grad[:, 1].any())            # exactly zero: get_grid_coords reads bounds[:, 0] only


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
@pytest.mark.parametrize("which", ["near_far", "bounds"])
def test_depth_grads_alone(case, train_precision, which):
    """Only near / far, or only bounds, require grad: the call still takes the training path, backward works, the gradients
    match the golden and nothing else gets a .grad."""
    scene, t_rand, G, gold = case
    net, ren, vols, batch = _setup(scene, train_precision, near_far=which == "near_far", bounds=which == "bounds")
    out = _render(ren, vols, batch, t_rand)
    assert out["rgb_map"].requires_grad
    _loss(G, "cuda")(out).backward()
    torch.cuda.synchronize()
    keys = ("near", "far") if which == "near_far" else ("bounds",)
    report = {k: _rel_l2(batch[k].grad.cpu(), torch.from_numpy(gold["d_" + k])) for k in keys}
    print(train_precision, which, report)
    _check(report)
    for k in {"near", "far", "bounds"} - set(keys):
        assert batch[k].grad is None, k
    assert all(p.grad is None for p in net.parameters()) and all(v.grad is None for v in vols)
    assert batch["ray_o"].grad is None and batch["R"].grad is None
    if which == "bounds":
        assert batch["bounds"].grad.dtype == batch["bounds"].dtype and not bool(batch["bounds"].grad[:, 1].any())


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_depth_grads_with_disp_loss(case, train_precision):
    """The loss reads every map, disp_map and weights included: d near / d far are NaN on exactly the oracle's rays (those
    with acc_map == 0), d bounds stays finite, everything within the gate."""
    scene, t_rand, G, _ = case
    Gm = MC.map_cotangents(scene)
    ref, ret_ref = DC.oracle_depth_grads(scene, t_rand, lambda r: MC.loss_of(r, G, Gm))
    nan_rays = torch.isnan(ref["near"])
    assert bool(nan_rays.any()) and torch.equal(nan_rays, ret_ref["acc_map"] == 0)
    net, ren, vols, batch = _setup(scene, train_precision, rays=True)
    out = _render(ren, vols, batch, t_rand)
    MC.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm)).backward()
    torch.cuda.synchronize()
    report = _compare(_gpu_grads(net, vols, batch, ref), ref)
    print(train_precision, report)
    _check(report)
    assert torch.isfinite(batch["bounds"].grad).all()


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_hierarchical_depth_grads(case, train_precision):
    """Coarse + fine pass (render_importance = 48) with near / far training: the fine pass's merged depths route their
    gradient back to the coarse depths and on to near / far; the importance samples get none.  The oracle's fine pass
    renders sort(cat(z_coarse, z_imp.detach())) at the GPU's importance depths (forward sensitivity, see
    tests/test_ray_grad.py::test_hierarchical_ray_grads)."""
    from oracle import neuralbody_oracle as O
    from neuralbody_b200.lib.config import cfg
    scene, t_rand, G, _ = case
    u, rgb0 = DC.hier_inputs(scene)
    G = dict(G, rgb0=rgb0)
    try:
        net, ren, vols, batch = _setup(scene, train_precision, importance=DC.N_IMPORTANCE)
        sampled = {}
        importance_z_vals = ren.importance_z_vals

        def keep_depths(*a, **k):
            r = importance_z_vals(*a, **k)
            sampled["z_all"], sampled["z_imp"] = r
            return r
        ren.importance_z_vals = keep_depths
        sp = ren.prepare_sp_input(batch)
        out = ren.render_rays_hierarchical(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp,
                                           t_rand=t_rand.cuda(), u=u.cuda())
    finally:
        cfg.render_importance = 0
    assert sampled["z_all"].requires_grad
    sc = DC.leaves(scene)
    spo, w, vs = O.prepare_sp_input(sc), sc["weights"], sc["voxel_size"]
    _, z_c = O.get_sampling_points(sc["ray_o"], sc["ray_d"], sc["near"], sc["far"], DC.N_SAMPLES, 1.0, True, t_rand)
    z_all, _ = torch.sort(torch.cat([z_c, sampled["z_imp"].detach().cpu()], -1), -1)
    np.testing.assert_allclose(z_all.detach().numpy(), sampled["z_all"].detach().cpu().numpy(), rtol=1e-6, atol=1e-6)
    ties = int((z_all[..., 1:] == z_all[..., :-1]).sum())
    coarse = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_c, sc["volumes"], spo, vs, True)
    ret = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_all, sc["volumes"], spo, vs, True)
    ret["rgb0"] = coarse["rgb_map"]
    grad_case.hier_loss_of(ret, G).backward()
    ref = {k: sc[k].grad for k in ("near", "far")}
    for k in ("rgb_map", "depth_map", "acc_map", "rgb0"):
        assert float((out[k].detach().cpu() - ret[k].detach()).abs().max()) < 1e-4, k
    grad_case.hier_loss_of(out, {k: v.cuda() for k, v in G.items()}).backward()
    torch.cuda.synchronize()
    report = _compare({k: batch[k].grad for k in ref}, ref)
    print(train_precision, "ties:", ties, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_user_z_vals_grad(case, train_precision):
    """A caller-supplied z_vals that requires grad gets d z_vals (B,n,S) within the gate; near / far are not read."""
    from oracle import neuralbody_oracle as O
    scene, t_rand, G, _ = case
    _, z0 = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], DC.N_SAMPLES, 1.0, True, t_rand)
    sc = dict(scene, z=z0.clone().requires_grad_(True))
    ret = O.get_pixel_value_at(sc["weights"], sc["ray_o"], sc["ray_d"], sc["z"], sc["volumes"], O.prepare_sp_input(sc),
                               sc["voxel_size"], True)
    grad_case.loss_of(ret, G).backward()
    net, ren, vols, batch = _setup(scene, train_precision, near_far=True, bounds=False)
    z = z0.cuda().requires_grad_(True)
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, z_vals=z)
    _loss(G, "cuda")(out).backward()
    torch.cuda.synchronize()
    assert batch["near"].grad is None and batch["far"].grad is None
    report = _compare({"z": z.grad}, {"z": sc["z"].grad})
    print(train_precision, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_chunked_render_depth_grads(case, train_precision):
    """render(batch) with cfg.chunk = 40 gives the near / far / bounds gradients of one launch.  No jitter: render() draws
    it per chunk."""
    scene, _, G, _ = case
    grads = []
    for chunk in (0, 40):
        net, ren, vols, batch = _setup(scene, train_precision, chunk=chunk, perturb=0.0)
        out = ren.render(batch)
        _loss(G, "cuda")(out).backward()
        torch.cuda.synchronize()
        grads.append({k: batch[k].grad.cpu() for k in ("near", "far", "bounds")})
    assert batch["near"].shape[1] > 2 * 40
    report = _compare(grads[1], grads[0])
    print(train_precision, report)
    _check(report)


def _get_near_far(box, ray_o, ray_d):
    """Upstream's get_near_far (lib/utils/if_nerf/if_nerf_data_utils.py:54-69) in torch, per frame, for rays that all hit
    the box: box (B,2,3), rays (B,n,3) -> near, far (B,n)."""
    norm_d = torch.norm(ray_d, dim=-1, keepdim=True)
    viewdir = ray_d / norm_d
    viewdir = torch.where((viewdir < 1e-5) & (viewdir > -1e-10), torch.full_like(viewdir, 1e-5), viewdir)
    viewdir = torch.where((viewdir > -1e-5) & (viewdir < 1e-10), torch.full_like(viewdir, -1e-5), viewdir)
    tmin = (box[:, None, 0] - ray_o) / viewdir
    tmax = (box[:, None, 1] - ray_o) / viewdir
    near = torch.minimum(tmin, tmax).max(-1).values
    far = torch.maximum(tmin, tmax).min(-1).values
    return near / norm_d[..., 0], far / norm_d[..., 0]


def _camera_chain(scene, cam_t, cam_w, box):
    """Rays of per-frame refined cameras: ray_o + cam_t, ray_d rotated by exp([cam_w]x); near / far = the box intersection
    of the refined rays."""
    B = cam_w.shape[0]
    K = torch.zeros((B, 3, 3), dtype=cam_w.dtype, device=cam_w.device)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -cam_w[:, 2], cam_w[:, 1], -cam_w[:, 0]
    Rc = torch.matrix_exp(K - K.transpose(1, 2))
    ray_o = scene["ray_o"].to(cam_t.device) + cam_t[:, None]
    ray_d = torch.matmul(scene["ray_d"].to(cam_t.device), Rc.transpose(1, 2))
    near, far = _get_near_far(box.to(cam_t.device), ray_o, ray_d)
    return ray_o, ray_d, near, far


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_camera_refinement_chain(case, train_precision):
    """Camera refinement end to end: rays from per-frame camera parameters, near / far recomputed in torch from those rays
    (box intersection), and .grad on the camera parameters against the oracle's autograd through the same chain."""
    from oracle import neuralbody_oracle as O
    scene, t_rand, G, _ = case
    pts = torch.cat([scene["ray_o"] + scene["ray_d"] * scene[k][..., None] for k in ("near", "far")], 1)
    box = torch.stack([pts.min(1).values - 0.05, pts.max(1).values + 0.05], 1)      # (B,2,3) world box around the body
    B = scene["ray_o"].shape[0]
    cam = {"t": torch.full((B, 3), 0.01), "w": torch.full((B, 3), 0.02)}

    ref_p = {k: v.clone().requires_grad_(True) for k, v in cam.items()}
    sc = dict(scene)
    sc["ray_o"], sc["ray_d"], sc["near"], sc["far"] = _camera_chain(scene, ref_p["t"], ref_p["w"], box)
    assert bool((sc["near"] < sc["far"]).all())
    ret = O.render(sc, n_samples=DC.N_SAMPLES, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand)
    grad_case.loss_of(ret, G).backward()

    net, ren, vols, batch = _setup(scene, train_precision, near_far=False, bounds=False)
    gpu_p = {k: v.cuda().requires_grad_(True) for k, v in cam.items()}
    ray_o, ray_d, near, far = _camera_chain(scene, gpu_p["t"], gpu_p["w"], box)
    sp = ren.prepare_sp_input(batch)
    out = ren.render_rays(ray_o, ray_d, near, far, vols, sp, t_rand=t_rand.cuda())
    _loss(G, "cuda")(out).backward()
    torch.cuda.synchronize()
    report = {k: _rel_l2(gpu_p[k].grad.cpu(), ref_p[k].grad) for k in cam}
    print(train_precision, report, {k: ref_p[k].grad for k in cam})
    _check(report)


def _backward_kernel_names(scene, t_rand, G, train_precision, depths):
    import gpu_utils as Gu
    net, ren, vols, batch = _setup(scene, train_precision, decoder=True, rays=True, near_far=depths, bounds=depths)
    out = _render(ren, vols, batch, t_rand)
    return Gu.backward_kernel_names(_loss(G, "cuda")(out))


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_depth_kernels_only_when_asked(case, train_precision):
    """Without a depth input the backward enqueues the kernels of nb_render_bwd_maps (no depth variant); with them the
    depth variants run instead."""
    scene, t_rand, G, _ = case
    without = _backward_kernel_names(scene, t_rand, G, train_precision, depths=False)
    ours = lambda names: {n for n in names if "nb::" in n or "_ZN2nb" in n}   # noqa: E731
    assert any("ray_grad_kernel" in n for n in ours(without)), sorted(ours(without))
    assert not any("<true>" in n and "ray_grad_kernel" in n for n in ours(without)), sorted(ours(without))
    with_depths = _backward_kernel_names(scene, t_rand, G, train_precision, depths=True)
    assert any("ray_grad_kernel<true>" in n or "ray_grad_kernelILb1E" in n for n in ours(with_depths)), sorted(ours(with_depths))


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_no_depth_inputs_null_and_same_as_maps_entry(case, train_precision):
    """Without near / far / bounds requiring grad the binding calls nb_render_bwd_inputs with the four depth pointers NULL;
    on the same forward record, that gives the ray gradients of nb_render_bwd_maps (bit for bit on fp32)."""
    from neuralbody_b200 import capi
    scene, t_rand, G, _ = case
    net, ren, vols, batch = _setup(scene, train_precision, rays=True, near_far=False, bounds=False)
    lib = ren.lib
    seen = {}

    class Spy:
        def __getattr__(self, name):
            return getattr(lib, name)

        def nb_render_bwd_maps(self, *a):
            seen["maps"] = True
            return lib.nb_render_bwd_maps(*a)

        def nb_render_bwd_inputs(self, ba_ref, d_disp, d_weights, ig_ref, stream):
            ig = ig_ref._obj
            seen["depth_ptrs"] = [ig.d_near, ig.d_far, ig.d_bounds, ig.d_z_vals]
            B, n = batch["ray_o"].shape[:2]
            twin = {k: torch.zeros((B, n, 3), dtype=torch.float32, device="cuda") for k in ("ray_o", "ray_d")}
            ba = capi.nb_render_bwd_args.from_buffer_copy(ba_ref._obj)
            assert lib.nb_render_bwd_maps(ctypes.byref(ba), d_disp, d_weights, None, None, twin["ray_o"].data_ptr(),
                                          twin["ray_d"].data_ptr(), stream) == 0
            seen["twin"] = twin
            return lib.nb_render_bwd_inputs(ba_ref, d_disp, d_weights, ig_ref, stream)
    ren.lib = Spy()
    out = _render(ren, vols, batch, t_rand)
    _loss(G, "cuda")(out).backward()
    torch.cuda.synchronize()
    assert "maps" not in seen and "twin" in seen
    assert seen["depth_ptrs"] == [None] * 4, seen["depth_ptrs"]
    for k in ("ray_o", "ray_d"):
        if train_precision == "fp32":
            assert torch.equal(batch[k].grad, seen["twin"][k]), k
        else:
            assert MC.rel_l2_finite(batch[k].grad, seen["twin"][k]) <= 1e-5, k


@pytest.mark.gpu
def test_sample_pdf_src_routes_and_matches(case):
    """nb_sample_pdf_src writes the same z_out as nb_sample_pdf, bit for bit, and each entry's source index holds that
    entry's depth: the coarse depth it names, or an importance sample (-1)."""
    from neuralbody_b200 import capi
    scene, t_rand, _, _ = case
    net, ren, vols, batch = _setup(scene, "tc_tf32x3", near_far=False, bounds=False)
    B, n = batch["ray_o"].shape[:2]
    S, Ni = DC.N_SAMPLES, DC.N_IMPORTANCE
    gen = torch.Generator().manual_seed(5)
    weights = torch.rand((B, n, S), generator=gen).cuda()
    u = torch.rand((B, n, Ni), generator=gen).cuda()
    tr = t_rand.cuda()
    outs = []
    for src in (None, torch.empty((B, n, S + Ni), dtype=torch.int32, device="cuda")):
        z_all = torch.empty((B, n, S + Ni), device="cuda")
        a = capi.nb_importance_args()
        a.n_rays_total, a.n_samples, a.n_importance = B * n, S, Ni
        a.near, a.far, a.t_vals = batch["near"].data_ptr(), batch["far"].data_ptr(), ren._t_vals(S, "cuda").data_ptr()
        a.t_rand, a.weights, a.u, a.z_out, a.z_samples = tr.data_ptr(), weights.data_ptr(), u.data_ptr(), z_all.data_ptr(), None
        st = ren.lib.nb_sample_pdf(ctypes.byref(a), None) if src is None else \
            ren.lib.nb_sample_pdf_src(ctypes.byref(a), src.data_ptr(), None)
        assert st == 0
        torch.cuda.synchronize()
        outs.append((z_all, src))
    assert torch.equal(outs[0][0], outs[1][0])
    z_all, src = outs[1]
    src = src.long()
    # every coarse index exactly once per ray, the rest -1
    assert torch.equal(torch.sort(src, -1).values, torch.cat([torch.full((B, n, Ni), -1, device="cuda"),
                                                              torch.arange(S, device="cuda").expand(B, n, S)], -1))
    zc = ren._coarse_z(batch["near"], batch["far"], S, tr, "cuda")
    picked = zc.gather(-1, src.clamp(min=0))
    torch.testing.assert_close(picked[src >= 0], z_all[src >= 0], rtol=1e-6, atol=1e-6)
