"""nb_mask_views: the demo and mesh datasets' mask views after decoding on the GPU, bit for bit with OpenCV's outputs in
the goldens and with the numpy restatement (tools/mask_views_case.py, pinned to OpenCV by test_mask_views_cpu); every
drop-in's 'device' item gives the host item's masks, the masked renderers' maps and the mesh renderer's cube, mesh and
inside test are the host batch's, and Renderer.mask_views does not synchronise with the host."""
import numpy as np
import pytest
import torch

from conftest import golden_case
from tools import mask_views_case as MC

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _run(msks_u8, Ks, Ds, H, W, binarise, dil):
    from neuralbody_b200 import images
    cams = [images.item_camera(K, D) for K, D in zip(Ks, Ds)]
    out = images.mask_views(torch.from_numpy(np.ascontiguousarray(msks_u8)).to(DEV), np.stack([c for _, c in cams]),
                            max(n for n, _ in cams), H, W, binarise, dil)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_goldens_equal_opencv():
    """Each recipe on a batch of views with different cameras (and distortion models) in one call."""
    for g in MC.load_golden():
        binarise, dil, _ = MC.RECIPES[g["recipe"]]
        H, W = g["msks"].shape[1:]
        got = _run(g["msks_u8"], g["Ks"], g["Ds"], H, W, binarise, dil)
        assert np.array_equal(got, g["msks"]), g["recipe"]


FULL = [((1024, 1024), 0.5, ("d5", "k1", "rational8", "d4"), "01", "multi_view_perform"),
        ((1024, 1024), 1.0, ("d5", "zero"), "0255", "multi_view_mesh"),
        ((1080, 1080), 0.5, ("rational8",), "any", "monocular_demo"),
        ((1080, 1080), 1.0, ("k1",), "any", "monocular_mesh"),
        ((1002, 1000), 0.5, ("d4", "d5"), "any", "multi_view_demo"),
        ((1002, 1000), 1.0, ("k1",), "any", "monocular_mesh")]


@pytest.mark.parametrize("case", FULL, ids=["%dx%d_r%g_%s" % (c[0] + (c[1], c[4])) for c in FULL])
def test_full_size_equals_the_restatement(case):
    (H0, W0), ratio, dists, values, recipe = case
    binarise, dil, _ = MC.RECIPES[recipe]
    msks_u8, Ks, Ds = MC.case(H0, W0, dists, values, H0 + len(dists))
    H, W = MC.out_size(H0, W0, ratio)
    got = _run(msks_u8, Ks, Ds, H, W, binarise, dil)
    for v in range(len(dists)):
        want, tie = MC.mask_view(msks_u8[v], Ks[v], Ds[v], H, W, binarise, dil)
        bad = got[v] != want
        print("%s view %d: %d flagged pixels, %d of them differ" % (recipe, v, tie.sum(), (bad & tie).sum()))
        assert not bad.any(), (recipe, v, int(bad.sum()))


# ----------------------------------------------------------------------------- the drop-ins' items and the renderers
def _renderer(mod, net):
    import os
    from conftest import ROOT
    from neuralbody_b200.lib.networks.make_network import load_source
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", mod + ".py")
    return load_source("neuralbody_b200.lib.networks.renderer." + mod, path).Renderer(net)


def _collate(item, keys):
    """What upstream's visualize loop hands the renderer: every key but 'meta' batched on the GPU, 'meta' on the host."""
    b = {k: torch.as_tensor(np.asarray(item[k]))[None].to(DEV) for k in keys}
    b["meta"] = {k: torch.as_tensor(np.asarray(v))[None] for k, v in item["meta"].items()}
    return b


@pytest.mark.parametrize("kind", list(MC.DROP_INS))
def test_dropin_device_item_gives_the_host_masks(kind):
    from neuralbody_b200.lib.networks.renderer import if_nerf_renderer
    ratio = 1.0 if kind == "multi_view_mesh" else 0.5
    host, dev = MC.item_pair(kind, 120, 160, 3, ratio, seed=5, values="any")
    ren = if_nerf_renderer.Renderer.__new__(if_nerf_renderer.Renderer)
    if kind == "monocular_demo":
        ren.MASK_VIEWS_KEY = "msk"
    b = _collate(dev, ["msks_u8"])
    ren.mask_views(b)
    torch.cuda.synchronize()
    key = ren.MASK_VIEWS_KEY
    want = np.asarray(host[key])[None]
    got = b[key].cpu().numpy()
    assert got.dtype == np.uint8 and got.shape == want.shape and np.array_equal(got, want), kind


def _decoded(views, seed):
    """Decoded masks for processed views (nv,H,W): the views with part labels, and a mild camera per view."""
    rng = np.random.RandomState(seed)
    nv, H, W = views.shape
    dec = np.where(views != 0, rng.randint(1, 256, views.shape), 0).astype(np.uint8)
    cams = []
    for v in range(nv):
        K = np.array([[1.2 * W, 0., W / 2 + 0.3], [0., 1.2 * W, H / 2 - 0.2], [0., 0., 1.]])
        cams.append((K, np.array([0.03, -0.01, 0.001, -0.001, 0.002])[:, None] * (1 + v)))
    return dec, cams


@pytest.mark.parametrize("single", [False, True], ids=["mmsk", "msk"])
def test_masked_renderer_maps_equal_the_host_batch(single):
    """The _mmsk (multi-view recipe) and _msk (single-view recipe) renderers on a 'device' batch give the host batch's
    maps bit for bit."""
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.datasets import mask_item
    import gpu_utils as G
    scene, rkw, _ = golden_case("msk_s64" if single else "mmsk_s64")
    masks = rkw["masks"]
    key = "msk" if single else "msks"
    views = masks[key].numpy().reshape(-1, int(masks["mask_H"]), int(masks["mask_W"]))
    dec, cams = _decoded(views, 3)
    binarise, dil = (False, 0) if single else (True, 5)
    H, W = views.shape[1:]
    host_views = np.stack([MC.mask_view(d, K, D, H, W, binarise, dil)[0] for d, (K, D) in zip(dec, cams)])
    assert (host_views != 0).mean() > 0.05
    keys, meta = mask_item.mask_fields(dec, [K for K, _ in cams], [D for _, D in cams], H, W, binarise, dil)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 0.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.render_skip_empty = "fp32", "auto", True
    cfg.H, cfg.W, cfg.ratio = H, W, 1.0
    net, _ = G.make_net_and_renderer(scene)
    net.eval()
    ren = _renderer("if_nerf_renderer_msk" if single else "if_nerf_renderer_mmsk", net)
    outs = []
    for device in (False, True):
        b = {k: scene[k].to(DEV) for k in G.BATCH_KEYS}
        b.update({k: masks[k].to(DEV) for k in (("R0_snap", "Th0_snap", "RT", "K") if single else ("RT", "Ks"))})
        if device:
            b["msks_u8"] = torch.from_numpy(keys["msks_u8"])[None].to(DEV)
            b["meta"] = {k: torch.as_tensor(np.asarray(v))[None] for k, v in meta.items()}
        else:
            b[key] = torch.from_numpy(host_views if single else host_views[None]).to(DEV)
        with torch.no_grad():
            out = ren.render(b)
        torch.cuda.synchronize()
        outs.append((b[key].cpu(), {k: v.cpu() for k, v in out.items()}))
    (m0, o0), (m1, o1) = outs
    assert torch.equal(m0, m1)
    assert float(o0["acc_map"].max()) > 0
    for k in o0:
        assert o0[k].shape == o1[k].shape and torch.equal(o0[k].contiguous().view(torch.uint8),
                                                          o1[k].contiguous().view(torch.uint8)), k


def test_mesh_renderer_equals_the_host_batch():
    """The mesh renderer on a 'device' batch (multi-view mesh recipe) gives the host batch's inside test, cube and mesh."""
    import os
    from conftest import ROOT
    from oracle import mesh_case
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.datasets import mask_item
    from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer
    import gpu_utils as G
    scene, masks, batch = mesh_case.build_case("mesh_s03")
    views = masks["msks"].numpy().reshape(-1, *masks["msks"].shape[-2:])
    dec, cams = _decoded(views, 4)
    H, W = views.shape[1:]
    host_views = np.stack([MC.mask_view(d, K, D, H, W, True, 5)[0] for d, (K, D) in zip(dec, cams)])
    keys, meta = mask_item.mask_fields(dec, [K for K, _ in cams], [D for _, D in cams], H, W, True, 5)
    net, _ = G.make_net_and_renderer(scene)
    old = cfg.renderer_module, cfg.renderer_path, cfg.mesh_th
    cfg.renderer_module = "neuralbody_b200.lib.networks.renderer.if_mesh_renderer"
    cfg.renderer_path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", "if_mesh_renderer.py")
    cfg.mesh_th = 10.0
    try:
        ren = make_renderer(cfg, net)
        outs = []
        for device in (False, True):
            b = {k: v.to(DEV) for k, v in batch.items() if k not in ("pts", "inside")}
            b.update(wbounds=scene["can_bounds"].to(DEV), RT=masks["RT"].to(DEV), Ks=masks["Ks"].to(DEV))
            if device:
                b["msks_u8"] = torch.from_numpy(keys["msks_u8"])[None].to(DEV)
                b["meta"] = {k: torch.as_tensor(np.asarray(v))[None] for k, v in meta.items()}
            else:
                b["msks"] = torch.from_numpy(host_views)[None].to(DEV)
            out = ren.render(b)
            _, inside = ren.grid_from_masks(b)
            torch.cuda.synchronize()
            outs.append((inside.cpu(), out["cube"], np.asarray(out["mesh"].vertices), np.asarray(out["mesh"].faces)))
    finally:
        cfg.renderer_module, cfg.renderer_path, cfg.mesh_th = old
    (i0, c0, v0, f0), (i1, c1, v1, f1) = outs
    assert torch.equal(i0, i1) and int(i0.sum()) > 0
    assert np.array_equal(c0, c1)
    assert np.array_equal(v0.view(np.int64), v1.view(np.int64)) and np.array_equal(f0, f1) and len(f0) > 0


def test_mask_views_does_not_synchronise():
    """Under torch's sync debug mode "error", Renderer.mask_views on a batch whose views are on the GPU runs to the end."""
    from neuralbody_b200.lib.networks.renderer import if_nerf_renderer
    _, dev = MC.item_pair("multi_view_perform", 120, 160, 3, 0.5, seed=6, values="any")
    ren = if_nerf_renderer.Renderer.__new__(if_nerf_renderer.Renderer)
    ren.mask_views(_collate(dev, ["msks_u8"]))          # the first call configures the kernel
    torch.cuda.synchronize()
    b = _collate(dev, ["msks_u8"])
    try:
        torch.cuda.set_sync_debug_mode("error")
        ren.mask_views(b)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    want, _ = MC.restate_item(dev)
    assert np.array_equal(b["msks"][0].cpu().numpy(), want)
