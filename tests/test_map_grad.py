"""Gradients through disp_map and weights, the last two outputs of the render.  CPU: the oracle's autograd reproduces the
unmodified reference's gradients on the map-loss case (tests/golden/grad_maps_b2_s32.npz, tools/map_grad_case.py), NaN
positions included, and the C entry point is exported, bound and validates its arguments.  GPU: Renderer + loss.backward()
against the oracle's autograd, both training precisions; rel-L2 <= 1e-3 per tensor over its finite entries (the gate of
tests/test_backward.py), the NaN pattern of d ray_d equal to the oracle's and every other gradient finite."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import grad_case
from tools import map_grad_case as MC

GATE = 1e-3


def _loss(kind, G, Gm):
    """The losses the tests differentiate: everything (the golden's), weights alone, disp_map alone, or no map term."""
    def disp_term(r):
        return (torch.where(r["acc_map"] > 0, r["disp_map"], torch.zeros_like(r["disp_map"])) * Gm[0]).sum()
    return {"all": lambda r: MC.loss_of(r, G, Gm),
            "weights": lambda r: (r["weights"] * Gm[1]).sum(),
            "disp": disp_term,
            "none": lambda r: MC.loss_of(r, G, Gm, terms=False)}[kind]


@pytest.fixture(scope="module")
def case():
    from oracle import synth
    scene, t_rand, G = MC.build()
    gold = load_golden(MC.GOLDEN)
    assert synth.scene_checksum(scene) == gold["input_sha256"]
    return scene, t_rand, G, MC.map_cotangents(scene), gold


def test_oracle_map_grads_match_reference(case):
    scene, t_rand, G, Gm, gold = case
    g, ret = MC.oracle_map_grads(scene, t_rand, _loss("all", G, Gm))
    empty = (ret["acc_map"] == 0).numpy()
    np.testing.assert_array_equal(empty, gold["empty_rays"])
    assert empty.any()
    nan_d = np.isnan(g["ray_d"].numpy())
    np.testing.assert_array_equal(nan_d, np.isnan(gold["d_ray_d"]))            # NaN positions equal: every axis of the empty rays
    np.testing.assert_array_equal(nan_d.any(-1), empty)
    np.testing.assert_allclose(g["ray_d"].numpy(), gold["d_ray_d"], rtol=1e-5, atol=1e-5)   # NaN == NaN here
    np.testing.assert_allclose(g["ray_o"].numpy(), gold["d_ray_o"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(g["R"].numpy(), gold["dR"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(g["Th"].numpy(), gold["dTh"].reshape(g["Th"].shape), rtol=1e-5, atol=1e-5)
    for k in list(grad_case.GRAD_KEYS) + ["vol%d" % l for l in range(4)]:
        t = g[k].double()
        assert torch.isfinite(t).all(), k
        np.testing.assert_allclose(float(t.sum()), gold["sum:" + k], rtol=1e-4, atol=1e-6, err_msg=k)
        np.testing.assert_allclose(float(t.abs().sum()), gold["abs:" + k], rtol=1e-4, err_msg=k)
        if "head:" + k in gold:
            np.testing.assert_allclose(g[k].reshape(-1)[:64].numpy(), gold["head:" + k], rtol=1e-4, atol=1e-6, err_msg=k)


def test_map_entry_point_exported_and_bound(built_lib):
    from neuralbody_b200 import capi
    lib = ctypes.CDLL(built_lib)
    assert hasattr(lib, "nb_render_bwd_maps")
    assert "nb_render_bwd_maps" in capi.EXPORTS
    bound = capi.load()
    assert bound.nb_abi_version() == 6
    assert bound.nb_render_bwd_maps.restype is ctypes.c_int
    assert len(bound.nb_render_bwd_maps.argtypes) == 8


def test_map_entry_point_rejects_null_args(built_lib):
    from neuralbody_b200 import capi
    lib = capi.load()
    assert lib.nb_render_bwd_maps(None, None, None, None, None, None, None, None) == -1   # NB_ERR_BAD_ARG, before any CUDA call
    err = lib.nb_last_error().decode()
    assert err.startswith("nb_render_bwd:") and "null" in err, err
    ba = capi.nb_render_bwd_args()                                                      # fwd / save / raw / ... unset
    assert lib.nb_render_bwd_maps(ctypes.byref(ba), None, None, None, None, None, None, None) == -1


# ------------------------------------------------------------------------------------------------------------------ GPU
def _setup(scene, train_precision, decoder=True, frame=True, importance=0, chunk=0, perturb=1.0):
    import gpu_utils as Gu
    from neuralbody_b200.lib.config import cfg
    dev = "cuda:0"
    net, ren = Gu.make_net_and_renderer(scene, dev)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = MC.N_SAMPLES, perturb, True, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = "tc_fp16x3", "auto", chunk
    cfg.render_train_precision = train_precision
    cfg.render_importance = importance
    net.train()
    for p in net.parameters():
        p.requires_grad_(decoder)
    vols = [v.to(dev).requires_grad_(decoder) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].to(dev) for k in Gu.BATCH_KEYS}
    batch["R"] = batch["R"].clone().requires_grad_(frame)
    batch["Th"] = batch["Th"].clone().requires_grad_(frame)
    batch["ray_o"] = batch["ray_o"].clone().requires_grad_(True)
    batch["ray_d"] = batch["ray_d"].clone().requires_grad_(True)
    return net, ren, vols, batch


def _render(ren, vols, batch, t_rand):
    sp = ren.prepare_sp_input(batch)
    return ren.render_rays(batch["ray_o"], batch["ray_d"], batch["near"], batch["far"], vols, sp, t_rand=t_rand.cuda())


def _gpu_grads(net, vols, batch, keys):
    got = {"ray_o": batch["ray_o"].grad, "ray_d": batch["ray_d"].grad, "R": batch["R"].grad, "Th": batch["Th"].grad}
    got.update({k: p.grad for k, p in net.named_parameters() if k in grad_case.GRAD_KEYS})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return {k: got[k] for k in keys}


def _compare(got, ref):
    """rel-L2 per tensor over the finite entries; asserts the NaN pattern is the reference's and only d ray_d has NaNs.
    A tensor the reference's autograd never reached (None) must come back None or all zero."""
    report = {}
    for k, r in ref.items():
        g = got[k]
        if r is None:
            assert g is None or not bool(g.any()), k
            continue
        g = g.detach().cpu()
        assert g.shape == r.shape, (k, g.shape, r.shape)
        assert torch.equal(torch.isnan(g), torch.isnan(r)), (k, int(torch.isnan(g).sum()), int(torch.isnan(r).sum()))
        if k != "ray_d":
            assert torch.isfinite(g).all(), k
        report[k] = MC.rel_l2_finite(g, r)
    return report


def _check(report):
    bad = {k: e for k, e in report.items() if not e <= GATE}
    assert not bad, bad


class _Spy:
    """Stands in for Renderer.lib and records what each nb_render_bwd_inputs call was given."""

    def __init__(self, lib, twin=None):
        self._lib, self._twin, self.calls = lib, twin, []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def nb_render_bwd_inputs(self, ba_ref, d_disp, d_weights, ig_ref, stream):
        ba = ba_ref._obj
        self.calls.append({"d_rgb": ba.d_rgb_map, "d_depth": ba.d_depth_map, "d_acc": ba.d_acc_map,
                           "d_disp": d_disp.value, "d_weights": d_weights.value})
        if self._twin is not None:
            self._twin(ba, ig_ref._obj, stream)
        return self._lib.nb_render_bwd_inputs(ba_ref, d_disp, d_weights, ig_ref, stream)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_map_grads_match_oracle(case, train_precision):
    """Decoder, volumes, frame transform and rays all train, the loss reads every map: every gradient within the gate, the
    NaN rays of d ray_d the oracle's, everything else finite."""
    scene, t_rand, G, Gm, _ = case
    ref, ret_ref = MC.oracle_map_grads(scene, t_rand, _loss("all", G, Gm))
    net, ren, vols, batch = _setup(scene, train_precision)
    out = _render(ren, vols, batch, t_rand)
    assert out["disp_map"].requires_grad and out["weights"].requires_grad
    for k in ("rgb_map", "depth_map", "acc_map", "weights"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    np.testing.assert_allclose(out["disp_map"].detach().cpu().numpy(), ret_ref["disp_map"].detach().numpy(), rtol=1e-3,
                               atol=1e-4)                                       # NaN on the same (empty) rays
    _loss("all", {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm))(out).backward()
    torch.cuda.synchronize()
    report = _compare(_gpu_grads(net, vols, batch, ref), ref)
    print(train_precision, report)
    _check(report)
    assert int(torch.isnan(batch["ray_d"].grad).any(-1).sum()) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
@pytest.mark.parametrize("kind", ["weights", "disp"])
def test_single_map_loss_inputs_entry(case, train_precision, kind):
    """A loss that reads only weights, or only disp_map: backward runs with the rgb / depth / acc cotangents NULL (and the
    other new one NULL too) and every gradient is within the gate."""
    scene, t_rand, G, Gm, _ = case
    ref, _ = MC.oracle_map_grads(scene, t_rand, _loss(kind, G, Gm))
    net, ren, vols, batch = _setup(scene, train_precision)
    spy = ren.lib = _Spy(ren.lib)
    out = _render(ren, vols, batch, t_rand)
    _loss(kind, G, tuple(t.cuda() for t in Gm))(out).backward()
    torch.cuda.synchronize()
    assert len(spy.calls) == 1
    c = spy.calls[0]
    assert c["d_rgb"] is None and c["d_depth"] is None and c["d_acc"] is None, c
    assert (c["d_weights"] is not None) == (kind == "weights") and (c["d_disp"] is not None) == (kind == "disp"), c
    report = _compare(_gpu_grads(net, vols, batch, ref), ref)
    print(train_precision, kind, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_hierarchical_map_grads(case, train_precision):
    """Coarse + fine pass (render_importance = 48) with disp0 (the coarse node's disp_map) and the fine weights in the loss,
    rays training.  The importance samples take the coarse weights detached, as upstream; the oracle's fine pass runs at
    the GPU's importance depths (see tests/test_ray_grad.py::test_hierarchical_ray_grads)."""
    from neuralbody_b200.lib.config import cfg
    scene, t_rand, G, Gm, _ = case
    u, rgb0 = MC.FC.hier_inputs(scene)
    G = dict(G, rgb0=rgb0)
    B, n = scene["ray_o"].shape[:2]
    gen = torch.Generator().manual_seed(102)
    Gh = (Gm[0], torch.randn((B, n, MC.N_SAMPLES + MC.N_IMPORTANCE), generator=gen) * 0.5)
    try:
        net, ren, vols, batch = _setup(scene, train_precision, decoder=False, frame=False, importance=MC.N_IMPORTANCE)
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
    assert out["disp0"].requires_grad and out["weights"].requires_grad
    ref, ret_ref = MC.oracle_hier_map_grads(scene, t_rand, G, Gh, sampled["z_all"].cpu())
    for k in ("rgb_map", "depth_map", "acc_map", "rgb0", "acc0", "weights"):
        assert float((out[k].detach().cpu() - ret_ref[k].detach()).abs().max()) < 1e-4, k
    MC.hier_loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gh)).backward()
    torch.cuda.synchronize()
    report = _compare({k: batch[k].grad for k in ("ray_o", "ray_d")}, ref)
    print(train_precision, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_chunked_render_map_grads(case, train_precision):
    """render(batch) with cfg.chunk = 40 (the maps joined by torch.cat) gives the gradients of one launch.  No jitter:
    render() draws it per chunk."""
    scene, _, G, Gm, _ = case
    grads = []
    for chunk in (0, 40):
        net, ren, vols, batch = _setup(scene, train_precision, chunk=chunk, perturb=0.0)
        out = ren.render(batch)
        MC.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm)).backward()
        torch.cuda.synchronize()
        keys = ["ray_o", "ray_d", "R", "Th", "fc_0.weight", "alpha_fc.weight", "vol0"]
        grads.append({k: g.cpu() for k, g in _gpu_grads(net, vols, batch, keys).items()})
    assert batch["ray_o"].shape[1] > 2 * 40
    report = _compare(grads[1], grads[0])
    print(train_precision, report)
    _check(report)


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_no_map_terms_inputs_entry_matches_ray_entry(case, train_precision):
    """A loss without disp_map or weights: the binding passes NULL for both, and on the same forward record the gradients are
    those of nb_render_bwd_rays.  The spy runs nb_render_bwd_rays first, into its own zeroed buffers, then the binding's
    call: so the record is also shown to be read-only to a backward.  On fp32 the ray gradients are deterministic and are
    compared bit for bit.  Everything else is summed with float atomics in an order that varies from run to run, even
    between two calls of the same entry point: on tc_tf32x3 that includes the ray gradients (frame_grad_kernel adds each
    listed sample's level terms with shared-memory atomics), compared to 1e-5; the decoder, volume and frame gradients are
    compared to 1e-4 (a scalar bias gradient is a sum over every sample, with cancellation)."""
    from neuralbody_b200 import capi
    from neuralbody_b200.lib.networks.renderer.if_nerf_renderer import _DECODER_FIELDS
    scene, t_rand, G, Gm, _ = case
    net, ren, vols, batch = _setup(scene, train_precision)
    lib = ren.lib
    twin = {}

    def rays_twin(ba, ig, stream):
        t = capi.nb_render_bwd_args.from_buffer_copy(ba)
        g = capi.nb_decoder_weights.from_buffer_copy(ba.grads.contents)
        twin["params"] = [torch.zeros(p.shape, dtype=torch.float32, device="cuda") for p in net.decoder_tensors()]
        for name, p in zip(_DECODER_FIELDS, twin["params"]):
            setattr(g, name, p.data_ptr())
        twin["vols"] = [torch.zeros(v.shape, dtype=torch.float32, device="cuda") for v in vols]
        for l in range(capi.NB_NUM_LEVELS):
            t.d_volumes[l] = twin["vols"][l].data_ptr() if ba.d_volumes[l] else None
        t.grads = ctypes.pointer(g)
        B, n = batch["ray_o"].shape[:2]
        shapes = {"R": (B, 3, 3), "Th": (B, 3), "ray_o": (B, n, 3), "ray_d": (B, n, 3)}
        ptrs = []
        for k in ("R", "Th", "ray_o", "ray_d"):
            twin[k] = torch.zeros(shapes[k], dtype=torch.float32, device="cuda") if getattr(ig, "d_" + k) else None
            ptrs.append(ctypes.c_void_p(twin[k].data_ptr() if twin[k] is not None else 0))
        assert lib.nb_render_bwd_rays(ctypes.byref(t), *ptrs, stream) == 0, lib.nb_last_error()
    spy = ren.lib = _Spy(lib, rays_twin)
    out = _render(ren, vols, batch, t_rand)
    MC.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm), terms=False).backward()
    torch.cuda.synchronize()
    assert len(spy.calls) == 1
    assert spy.calls[0]["d_disp"] is None and spy.calls[0]["d_weights"] is None, spy.calls[0]
    for k in ("ray_o", "ray_d"):
        if train_precision == "fp32":
            assert torch.equal(batch[k].grad, twin[k]), k
        else:
            assert MC.rel_l2_finite(batch[k].grad, twin[k]) <= 1e-5, k
    got = {"R": batch["R"].grad, "Th": batch["Th"].grad.reshape(twin["Th"].shape)}
    got.update({k: p.grad for k, p in zip(grad_case.GRAD_KEYS, net.decoder_tensors())})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    want = {"R": twin["R"], "Th": twin["Th"]}
    want.update({k: p.view_as(t) for k, p, t in zip(grad_case.GRAD_KEYS, twin["params"], net.decoder_tensors())})
    want.update({"vol%d" % l: v for l, v in enumerate(twin["vols"])})
    report = {k: MC.rel_l2_finite(got[k], want[k]) for k in want}
    print(train_precision, report)
    assert all(e <= 1e-4 for e in report.values()), report


def _backward_kernel_names(scene, t_rand, G, Gm, train_precision, terms):
    import gpu_utils as Gu
    net, ren, vols, batch = _setup(scene, train_precision)
    out = _render(ren, vols, batch, t_rand)
    return Gu.backward_kernel_names(MC.loss_of(out, {k: v.cuda() for k, v in G.items()}, tuple(t.cuda() for t in Gm),
                                               terms=terms))


@pytest.mark.gpu
@pytest.mark.parametrize("train_precision", ["tc_tf32x3", "fp32"])
def test_map_terms_add_no_kernel(case, train_precision):
    """The disp_map and weights cotangents enter kernels that run anyway: the backward enqueues the same kernels with and
    without them."""
    scene, t_rand, G, Gm, _ = case
    # two captures per configuration, united: on a shared host the profiler can miss a kernel of one capture, while a kernel
    # that only one configuration enqueues is in both of its captures and in neither of the other's
    names = lambda terms: set().union(*(_backward_kernel_names(scene, t_rand, G, Gm, train_precision, terms=terms)  # noqa: E731
                                        for _ in range(2)))
    without = names(False)
    assert any("composite_bwd_kernel" in n for n in without) and any("ray_grad_kernel" in n for n in without), sorted(without)
    with_terms = names(True)
    ours = lambda names: {n for n in names if "nb::" in n or "_ZN2nb" in n}   # noqa: E731  (the loss's torch kernels differ)
    assert ours(with_terms) == ours(without), sorted(ours(with_terms) ^ ours(without))
