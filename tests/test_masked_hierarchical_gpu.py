"""GPU: coarse + fine sampling (cfg.render_importance) through the masked demo renderers and into the ray-sharded view
render's slabs.  The _mmsk / _msk renderers against the goldens made from the unmodified reference's masked renderer,
sample_pdf and sort-merge (oracle/masked_hier_case.py); masked-out samples weigh nothing in either pass; render_importance
= 0 is the coarse-only render it always was; a view rendered rank by rank into FrameGatherer slabs is the unsharded view
bit for bit; and a masked hierarchical view with perturb = 0 does not synchronise with the host."""
import os

import pytest
import torch

from conftest import ROOT, load_golden
from oracle import masked_hier_case as MH, neuralbody_oracle as O, synth
import gpu_utils as G

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = {"fp32": 1e-4, "tc_fp16x3": 1e-3, "tc_fp16": 6e-3}


def _masked_renderer(net, single):
    from neuralbody_b200.lib.networks.make_network import load_source
    mod = "if_nerf_renderer_msk" if single else "if_nerf_renderer_mmsk"
    path = os.path.join(ROOT, "neuralbody_b200", "lib", "networks", "renderer", mod + ".py")
    return load_source("neuralbody_b200.lib.networks.renderer." + mod, path).Renderer(net)


def _setup(scene, masks, precision, importance, skip_empty=True):
    """(net, masked renderer, device batch with the mask keys, sp_input, volumes, the masks as render_rays takes them)."""
    from neuralbody_b200.lib.config import cfg
    net, _ = G.make_net_and_renderer(scene)
    net.train(False)
    single = "R0_snap" in masks
    ren = _masked_renderer(net, single)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = 64, 0.0, False, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.chunk = precision, "auto", 0
    cfg.render_skip_empty, cfg.render_importance = skip_empty, importance
    cfg.H, cfg.W, cfg.ratio = int(masks["mask_H"]), int(masks["mask_W"]), 1.0
    batch = {k: scene[k].to(DEV) for k in G.BATCH_KEYS}
    batch.update({k: masks[k].to(DEV) for k in (("R0_snap", "Th0_snap", "RT", "K", "msk") if single else ("RT", "Ks", "msks"))})
    sp = ren.prepare_sp_input(batch)
    vol = net.encode_sparse_voxels(sp)
    if single:      # what if_nerf_renderer_msk.get_pixel_value hands render_rays
        rmasks = {"msks": batch["msk"][:, None], "RT": batch["RT"][:, None], "Ks": batch["K"][:, None],
                  "R0_snap": batch["R0_snap"], "Th0_snap": batch["Th0_snap"]}
    else:
        rmasks = batch
    return net, ren, batch, sp, vol, rmasks


def _oracle_masks(scene, masks):
    """The mask views as the oracle's predicate takes them: the single-view one also reads the frame's R and Th."""
    return dict(masks, R=scene["R"], Th=scene["Th"]) if "R0_snap" in masks else masks


def _rays(batch):
    return batch["ray_o"], batch["ray_d"], batch["near"], batch["far"]


@pytest.fixture(autouse=True)
def _coarse_only_afterwards():
    yield
    from neuralbody_b200.lib.config import cfg
    cfg.render_importance = 0


def _case(name):
    scene, rkw = MH.build_case(name)
    gold = load_golden(name)
    assert synth.scene_checksum(scene) == gold["input_sha256"], "rebuilt inputs differ from the golden generator's"
    return scene, rkw, gold


@pytest.mark.parametrize("name", list(MH.CASES))
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3", "tc_fp16"])
def test_masked_hierarchical_render_matches_reference_pieces(name, precision):
    """The masked renderer's render(batch) with render_importance = 128: both passes masked, the fine pass over the merged
    depths of the masked coarse weights.  fp32 / tc_fp16x3 at the gates of the plain hierarchical render (maps at the usual
    tolerance, depths 97 % within 2e-5 / 2e-3); tc_fp16 at its 6e-3 envelope on the maps.
    The mask predicate is a step in the sample's position.  A fine sample near a mask edge can sit on the other side of it
    after the small depth difference the plain hierarchical render already allows, and then the decoder runs on a sample
    the reference masked out, or the reverse.  So the fine maps are held
    at the usual tolerance twice: against the reference on every ray whose fine samples all get the reference's verdict,
    and against the oracle's masked fine pass at this render's own depths on every ray."""
    scene, rkw, gold = _case(name)
    S, Ni = rkw["n_samples"], rkw["n_importance"]
    net, ren, batch, sp, vol, rmasks = _setup(scene, rkw["masks"], precision, Ni)
    with torch.no_grad():
        out = ren.render(batch)
        coarse = ren.render_rays(*_rays(batch), vol, sp, masks=rmasks, want_weights=True)
        z_all, _ = ren.importance_z_vals(batch["near"], batch["far"], coarse["weights"], S, Ni)
    torch.cuda.synchronize()
    out, z_all = {k: v.cpu() for k, v in out.items()}, z_all.cpu()
    assert set(out) == {"rgb_map", "disp_map", "acc_map", "depth_map", "weights", "rgb0", "disp0", "acc0", "z_std"}
    assert out["weights"].shape[-1] == S + Ni
    tol = TOL[precision]
    for k in ("rgb0", "acc0"):
        d = float((out[k] - torch.from_numpy(gold[k])).abs().max())
        assert d < tol, (k, d)
    masks = _oracle_masks(scene, rkw["masks"])
    ro, rd = scene["ray_o"], scene["ray_d"]
    z_gold = torch.from_numpy(gold["z_vals"])
    edge = (MH.inside_at(ro, rd, z_all, masks) != MH.inside_at(ro, rd, z_gold, masks)).view(z_all.shape).any(-1)
    at_own = MH.get_pixel_value_masked_at(scene["weights"], ro, rd, z_all, scene["volumes"], O.prepare_sp_input(scene),
                                          scene["voxel_size"], masks)
    print(name, precision, "%d of %d rays have a fine sample on the other side of a mask edge" % (int(edge.sum()), edge.numel()))
    assert float(edge.float().mean()) < 0.02
    for k in ("rgb_map", "depth_map", "acc_map"):
        d_own = float((out[k] - at_own[k]).abs().max())
        d_ref = float((out[k] - torch.from_numpy(gold[k]))[~edge].abs().max())
        assert d_own < tol and d_ref < tol, (k, d_own, d_ref)
    # the rays every sample of which is masked out, in both passes: nothing to composite, as upstream (acc 0, disp NaN)
    dead = torch.from_numpy(gold["acc_map"] == 0) & torch.from_numpy(gold["acc0"] == 0)
    assert dead.any() and bool((out["acc_map"][dead] == 0).all()) and bool(torch.isnan(out["disp_map"][dead]).all())
    if precision == "tc_fp16":
        return
    assert torch.all(z_all[..., 1:] >= z_all[..., :-1])
    dz = (z_all - z_gold).abs()
    ztol = 2e-5 if precision == "fp32" else 2e-3
    assert float((dz < ztol).float().mean()) > 0.97, float((dz < ztol).float().mean())
    assert float(dz.max()) < (5e-3 if precision == "fp32" else 5e-2), float(dz.max())
    assert float((out["z_std"] - torch.from_numpy(gold["z_std"])).abs().max()) < (1e-3 if precision == "fp32" else 1e-2)


@pytest.mark.parametrize("name", list(MH.CASES))
@pytest.mark.parametrize("precision", ["fp32", "tc_fp16x3"])
def test_masked_out_samples_weigh_nothing_in_either_pass(name, precision):
    """Every pass evaluated densely (no empty-sample skipping): a sample the mask views remove has the raw record of a
    removed sample (rgb logits exactly 0, sigma <= 0) and weight exactly 0, in the coarse pass and in the fine pass; the
    predicate is the oracle's (upstream's) at the same depths; and render_rays_hierarchical's fine weights are those of the
    masked fine pass over the depths the masked coarse weights give."""
    scene, rkw, _ = _case(name)
    S, Ni = rkw["n_samples"], rkw["n_importance"]
    net, ren, batch, sp, vol, rmasks = _setup(scene, rkw["masks"], precision, Ni, skip_empty=False)
    with torch.no_grad():
        coarse = ren.render_rays(*_rays(batch), vol, sp, masks=rmasks, want_raw=True, want_weights=True)
        z_all, _ = ren.importance_z_vals(batch["near"], batch["far"], coarse["weights"], S, Ni)
        fine = ren.render_rays(*_rays(batch), vol, sp, masks=rmasks, z_vals=z_all, want_raw=True, want_weights=True)
        hier = ren.render_rays_hierarchical(*_rays(batch), vol, sp, masks=rmasks)
    torch.cuda.synchronize()
    masks = _oracle_masks(scene, rkw["masks"])
    _, z0 = O.get_sampling_points(scene["ray_o"], scene["ray_d"], scene["near"], scene["far"], S)
    for label, ret, z in (("coarse", coarse, z0), ("fine", fine, z_all.cpu())):
        raw, w = ret["raw"].cpu(), ret["weights"].cpu()
        removed = (raw[..., :3] == 0).all(-1)
        assert bool((raw[..., 3][removed] <= 0).all()) and bool((w[removed] == 0).all()), label
        inside = MH.inside_at(scene["ray_o"], scene["ray_d"], z, masks).view(removed.shape)
        print(name, precision, label, "removed %.1f%% of the samples" % (100.0 * float(removed.float().mean())))
        assert 0 < float(removed.float().mean()) < 1, label
        assert torch.equal(inside, ~removed), label
        assert float(w[~removed].max()) > 1e-2, label          # the samples kept do carry the body
    assert torch.equal(hier["weights"], fine["weights"])
    for k in ("rgb_map", "acc_map", "depth_map"):
        assert torch.equal(hier[k], fine[k]), k
    assert torch.equal(hier["acc0"], coarse["acc_map"])


@pytest.mark.parametrize("name", list(MH.CASES))
def test_importance_zero_is_the_coarse_render(name):
    """render_importance = 0 (the default): the masked renderers return what render_rays with the mask views returns, bit for
    bit and with the same keys."""
    scene, rkw, _ = _case(name)
    net, ren, batch, sp, vol, rmasks = _setup(scene, rkw["masks"], "tc_fp16x3", 0)
    with torch.no_grad():
        got = ren.render(batch)
        want = ren.render_rays(*_rays(batch), vol, sp, masks=rmasks)
    torch.cuda.synchronize()
    assert set(got) == set(want) == {"rgb_map", "disp_map", "acc_map", "depth_map", "weights"}
    for k in want:
        assert torch.equal(got[k].view(torch.int32), want[k].view(torch.int32)), k     # bits: disp_map has NaN


def _orbit_scene(single):
    """A 64 x 64 view (4096 rays, sixteen 256-ray chunks) with mask views that cut through the body."""
    scene = synth.make_scene(H=64, W=64, scale=0.3, all_hit=True, th_shape=(3,) if single else (1, 3))
    masks = synth.make_snapshot_view(scene, H=96, W=96, radius=2) if single else synth.make_mask_views(scene, nv=4, H=96,
                                                                                                       W=96, radius=2)
    return scene, masks


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("kind", ["plain", "mmsk"])
@pytest.mark.parametrize("precision", ["tc_fp16x3", "fp32"])
def test_sharded_hierarchical_render_is_bit_identical(world, kind, precision):
    """Each rank's interleaved shard rendered with coarse + fine sampling into its slab (render_rays_hierarchical(out=...)),
    rank by rank on one GPU; the stacked slabs un-permuted by dist.unpack_slab hold the unsharded render's bits."""
    from neuralbody_b200 import dist as nbdist
    scene, masks = _orbit_scene(False)
    net, ren, batch, sp, vol, rmasks = _setup(scene, masks, precision, 128)
    if kind == "plain":
        ren, rmasks = _plain(net), None
    n = batch["ray_o"].shape[1]
    plan = nbdist.ShardPlan.get(n, world, 256, DEV)
    with torch.no_grad():
        want = ren.render_rays_hierarchical(*_rays(batch), vol, sp, masks=rmasks)
        slabs = []
        for rank in range(world):
            local = plan.shard(batch, rank)
            slab, views = nbdist.new_slab(1, plan.per, DEV)
            slab.fill_(-7.0)
            ret = ren.render_rays_hierarchical(*_rays(local), vol, sp, masks=rmasks, out=views)
            assert ret["rgb_map"].data_ptr() == views["rgb_map"].data_ptr() and "rgb0" in ret
            slabs.append(slab)
        got = nbdist.unpack_slab(torch.stack(slabs), n, 256)
    torch.cuda.synchronize()
    assert 0 < float(want["acc_map"].mean()) < 1
    for k in ("rgb_map", "disp_map", "acc_map", "depth_map"):
        assert torch.equal(got[k].contiguous().view(torch.int32), want[k].view(torch.int32)), (kind, world, k)


def _plain(net):
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.renderer.make_renderer import make_renderer
    return make_renderer(cfg, net)


@pytest.mark.parametrize("single", [False, True], ids=["mmsk", "msk"])
def test_masked_hierarchical_view_does_not_synchronise(single):
    """perturb = 0, mask views and rays on the device: the view's coarse pass, sampler and fine pass (into dense maps, and
    into a slab) are enqueued without one host synchronisation."""
    from neuralbody_b200 import dist as nbdist
    scene, masks = _orbit_scene(single)
    net, ren, batch, sp, vol, rmasks = _setup(scene, masks, "tc_fp16x3", 128)
    args = _rays(batch) + (vol, sp, batch)
    _, views = nbdist.new_slab(1, batch["ray_o"].shape[1], DEV)
    with torch.no_grad():
        ren.get_pixel_value(*args)                                                  # warm: packs, t_vals, workspace
        ren.render_rays_hierarchical(*_rays(batch), vol, sp, masks=rmasks, out=views)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ret = ren.get_pixel_value(*args)
            ren.render_rays_hierarchical(*_rays(batch), vol, sp, masks=rmasks, out=views)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert "rgb0" in ret and ret["weights"].shape[-1] == 64 + 128
    assert torch.equal(views["rgb_map"], ret["rgb_map"])
