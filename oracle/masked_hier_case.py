"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

f-1 x f-4: the masked demo renderers (if_clight_renderer_mmsk.py / if_clight_renderer_msk.py) with coarse + fine sampling.
Upstream never combines them: its masked renderers have no fine pass, and its fine pass lives in the NeRF-baseline renderer
(volume_renderer.py:60-118).  The spec is that renderer with upstream's masked get_pixel_value as its coarse network and the
same masked pass at the merged depths as its fine network: the coarse weights that drive sample_pdf are the masked ones, and
the mask predicate is applied to the fine samples too.

  * the cases: the scenes and mask views of golden_cases' `mmsk_s64` / `msk_s64` (the masks cut through the body, and some
    rays are masked out entirely) with N_importance = 128, eval mode (det = perturb == 0);
  * `render_hierarchical_masked`: the oracle's restatement (neuralbody_oracle's masked predicate, decoder, raw2outputs,
    sample_pdf / sort-merge), composed like neuralbody_oracle.render_hierarchical;
  * `reference_render_hierarchical_masked`: the same composition of the UNMODIFIED reference's functions (its masked
    Renderer's get_pixel_value for the coarse pass, its prepare_inside_pts / get_density_color at the merged depths for the
    fine pass, nerf_net_utils.sample_pdf / raw2outputs); needs the reference tree (oracle/ref_harness.py);
  * `python -m oracle.masked_hier_case` writes tests/golden/<case>.npz from the latter.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name -> (golden_cases.CASES entry whose scene, rays and mask views it reuses, N_importance)
CASES = {
    "mmsk_hier_s64_i128": ("mmsk_s64", 128),     # 4 mask views (if_clight_renderer_mmsk)
    "msk_hier_s64_i128": ("msk_s64", 128),       # one snapshot view, Th as (B,3) (if_clight_renderer_msk)
}
KEYS = ("rgb_map", "disp_map", "acc_map", "weights", "depth_map", "rgb0", "disp0", "acc0", "z_std", "z_vals", "weights0")


def build_case(name):
    """-> (scene, render kwargs: n_samples, n_importance, masks)."""
    from oracle import golden_cases
    base, n_importance = CASES[name]
    scene, rkw = golden_cases.build_case(base)
    return scene, dict(rkw, n_importance=n_importance)


def mask_checksum(scene, masks):
    """sha256 over the mask-view tensors (the scene's own checksum covers the rest), as make_golden.py stores it."""
    from oracle import synth
    mk = ("R0_snap", "Th0_snap", "RT", "K", "msk") if "R0_snap" in masks else ("RT", "Ks", "msks")
    return synth.scene_checksum({**scene, "weights": {}, "volumes": [masks[k].float() for k in mk]})


# ------------------------------------------------------------------ the oracle's restatement
def inside_at(ray_o, ray_d, z_vals, masks):
    """The masked renderer's predicate (multi-view or, with R0_snap, single view: then `masks` also carries the frame's R
    and Th) at pts = ray_o + ray_d * z: (1,n,S) -> (1, n*S) bool."""
    from oracle import neuralbody_oracle as O
    wpts = ray_o[:, :, None] + ray_d[:, :, None] * z_vals[..., None]
    if "R0_snap" in masks:
        return O.prepare_inside_pts_msk(wpts, masks, masks["mask_H"], masks["mask_W"])
    return O.prepare_inside_pts(wpts, masks, masks["mask_H"], masks["mask_W"])


def get_pixel_value_masked_at(w, ray_o, ray_d, z_vals, feature_volume, sp_input, voxel_size, masks, white_bkgd=False):
    """neuralbody_oracle.get_pixel_value_mmsk at given depths (B = 1): pts = ray_o + ray_d * z, the masked renderer's
    predicate, the decoder on inside samples only, raw = 0 elsewhere."""
    from oracle import neuralbody_oracle as O
    wpts = ray_o[:, :, None] + ray_d[:, :, None] * z_vals[..., None]
    inside = inside_at(ray_o, ray_d, z_vals, masks)
    viewdir = ray_d / torch.norm(ray_d, dim=2, keepdim=True)
    n_batch, n_pixel, n_sample = wpts.shape[:3]
    wp = wpts.view(n_batch, n_pixel * n_sample, -1)
    vd = viewdir[:, :, None].repeat(1, 1, n_sample, 1).contiguous().view(n_batch, n_pixel * n_sample, -1)
    full_raw = torch.zeros([n_batch, n_pixel * n_sample, 4]).to(wp)
    if inside.sum() > 0:
        raw = O.calculate_density_color(w, wp[inside][None], vd[inside][None], feature_volume, sp_input, voxel_size)
        full_raw[inside] = raw[0]
    raw = full_raw.reshape(-1, n_sample, 4)
    rgb_map, disp_map, acc_map, weights, depth_map = O.raw2outputs(raw, z_vals.view(-1, n_sample), ray_d.reshape(-1, 3),
                                                                   white_bkgd)
    return {'rgb_map': rgb_map.view(n_batch, n_pixel, -1), 'disp_map': disp_map.view(n_batch, n_pixel),
            'acc_map': acc_map.view(n_batch, n_pixel), 'weights': weights.view(n_batch, n_pixel, -1),
            'depth_map': depth_map.view(n_batch, n_pixel), 'inside': inside.view(n_batch, n_pixel, n_sample)}


def render_hierarchical_masked(scene, masks, n_samples=64, n_importance=128, white_bkgd=False, chunk=2048):
    """neuralbody_oracle.render_hierarchical (eval mode) with the masked pass at both depths.  Returns the fine maps and
    weights, rgb0 / disp0 / acc0 / z_std / z_vals as render_hierarchical does, the coarse weights (`weights0`) and both
    passes' inside predicates (`inside0`, `inside`)."""
    from oracle import neuralbody_oracle as O
    sp_input = O.prepare_sp_input(scene)
    if "R0_snap" in masks:
        masks = dict(masks, R=scene['R'], Th=scene['Th'])
    w, vols, vs = scene['weights'], scene['volumes'], scene['voxel_size']
    outs = []
    for i in range(0, scene['ray_o'].shape[1], chunk):
        ro, rd = scene['ray_o'][:, i:i + chunk], scene['ray_d'][:, i:i + chunk]
        near, far = scene['near'][:, i:i + chunk], scene['far'][:, i:i + chunk]
        _, z_vals = O.get_sampling_points(ro, rd, near, far, n_samples)
        coarse = get_pixel_value_masked_at(w, ro, rd, z_vals, vols, sp_input, vs, masks, white_bkgd)
        B, n = z_vals.shape[:2]
        z_all, z_samples = O.importance_z_vals(z_vals.view(B * n, -1), coarse['weights'].view(B * n, -1), n_importance,
                                               det=True)
        fine = get_pixel_value_masked_at(w, ro, rd, z_all.view(B, n, -1), vols, sp_input, vs, masks, white_bkgd)
        fine.update({'rgb0': coarse['rgb_map'], 'disp0': coarse['disp_map'], 'acc0': coarse['acc_map'],
                     'weights0': coarse['weights'], 'inside0': coarse['inside'],
                     'z_std': torch.std(z_samples, dim=-1, unbiased=False).view(B, n), 'z_vals': z_all.view(B, n, -1)})
        outs.append(fine)
    return {k: torch.cat([r[k] for r in outs], dim=1) for k in outs[0]}


# ------------------------------------------------------------------ the unmodified reference's functions
def reference_render_hierarchical_masked(scene, masks, n_samples=64, n_importance=128, white_bkgd=False, chunk=2048):
    """The composition above, run on the reference's own code: its masked Renderer (if_clight_renderer_mmsk.Renderer, or
    if_clight_renderer_msk.Renderer with R0_snap) drives the coarse pass through its unmodified get_pixel_value; the fine
    pass is that renderer's prepare_inside_pts + get_density_color at the merged depths followed by raw2outputs, i.e. its
    get_pixel_value with the depths of volume_renderer.py:84-93 (sample_pdf, det = True, and the sort-merge)."""
    from oracle import ref_harness
    cfg, latent_xyzc, _, nerf_net_utils = ref_harness.load_reference()
    if "torchsearchsorted" not in sys.modules:       # nerf_net_utils.py:56; same semantics as torch.searchsorted
        import types
        tss = types.ModuleType("torchsearchsorted")
        tss.searchsorted = lambda a, v, side="left": torch.searchsorted(a, v, right=(side == "right"))
        sys.modules["torchsearchsorted"] = tss
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std = int(n_samples), 0.0, bool(white_bkgd), 0
    cfg.voxel_size = [float(v) for v in scene["voxel_size"]]
    cfg.num_train_frame = int(scene["weights"]["latent.weight"].shape[0])
    cfg.H, cfg.W, cfg.ratio = int(masks["mask_H"]), int(masks["mask_W"]), 1.0
    net = latent_xyzc.Network()
    missing, unexpected = net.load_state_dict(scene["weights"], strict=False)
    assert not unexpected and all(k.startswith("xyzc_net") or k.startswith("c.") for k in missing)
    net.train(False)
    batch = {k: scene[k] for k in ("coord", "out_sh", "bounds", "R", "Th", "latent_index")}
    if "R0_snap" in masks:
        from lib.networks.renderer import if_clight_renderer_msk as ref_mod
        batch.update({k: masks[k] for k in ("R0_snap", "Th0_snap", "RT", "K", "msk")})
    else:
        from lib.networks.renderer import if_clight_renderer_mmsk as ref_mod
        batch.update({k: masks[k] for k in ("RT", "Ks", "msks")})
    renderer = ref_mod.Renderer(net)
    sp_input = renderer.prepare_sp_input(batch)
    vols = [v.clone() for v in scene["volumes"]]
    decoder = lambda x, vd: net.calculate_density_color(x, vd, vols, sp_input)
    outs = []
    assert chunk == 2048     # the reference hard-codes it (if_clight_renderer.py:107)
    with torch.no_grad():
        for i in range(0, scene["ray_o"].shape[1], chunk):
            ro, rd = scene["ray_o"][:, i:i + chunk], scene["ray_d"][:, i:i + chunk]
            near, far = scene["near"][:, i:i + chunk], scene["far"][:, i:i + chunk]
            B, n = ro.shape[:2]
            coarse = renderer.get_pixel_value(ro, rd, near, far, vols, sp_input, batch)
            _, z_vals = renderer.get_sampling_points(ro, rd, near, far)      # the depths get_pixel_value sampled at
            z_vals = z_vals.view(-1, n_samples)
            weights0 = coarse['weights'].view(-1, n_samples)
            # volume_renderer.py:84-93
            z_vals_mid = .5 * (z_vals[..., 1:] + z_vals[..., :-1])
            z_samples = nerf_net_utils.sample_pdf(z_vals_mid, weights0[..., 1:-1], n_importance, det=True).detach()
            z_all, _ = torch.sort(torch.cat([z_vals, z_samples], -1), -1)
            S2 = n_samples + n_importance
            pts = ro[:, :, None] + rd[:, :, None] * z_all.view(B, n, S2)[..., None]
            inside = renderer.prepare_inside_pts(pts, batch)
            viewdir = rd / torch.norm(rd, dim=2, keepdim=True)
            raw = renderer.get_density_color(pts, viewdir, inside, decoder).reshape(-1, S2, 4)
            rgb, disp, acc, w2, depth = nerf_net_utils.raw2outputs(raw, z_all, rd.reshape(-1, 3), cfg.raw_noise_std,
                                                                   cfg.white_bkgd)
            outs.append({"rgb_map": rgb.view(B, n, 3), "disp_map": disp.view(B, n), "acc_map": acc.view(B, n),
                         "weights": w2.view(B, n, S2), "depth_map": depth.view(B, n), "rgb0": coarse['rgb_map'],
                         "disp0": coarse['disp_map'], "acc0": coarse['acc_map'], "weights0": coarse['weights'],
                         "z_std": torch.std(z_samples, dim=-1, unbiased=False).view(B, n), "z_vals": z_all.view(B, n, S2)})
    return {k: torch.cat([o[k] for o in outs], dim=1).detach() for k in outs[0]}


def main():
    import numpy as np
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import synth
    for name in CASES:
        scene, rkw = build_case(name)
        ret = reference_render_hierarchical_masked(scene, rkw["masks"], rkw["n_samples"], rkw["n_importance"])
        arrays = {k: v.numpy().astype(np.float32) for k, v in ret.items()}
        arrays["input_sha256"] = np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8)
        arrays["mask_sha256"] = np.frombuffer(mask_checksum(scene, rkw["masks"]).encode(), dtype=np.uint8)
        arrays["torch_version"] = np.frombuffer(torch.__version__.encode(), dtype=np.uint8)
        path = os.path.join(ROOT, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **arrays)
        acc = ret["acc_map"]
        print("%-20s rays=%-4d acc.mean=%.3f empty rays=%d |rgb - rgb0|max=%.3f -> %s (%d KB)" % (
            name, acc.numel(), float(acc.mean()), int((acc == 0).sum()), float((ret["rgb_map"] - ret["rgb0"]).abs().max()),
            path, os.path.getsize(path) // 1024))


if __name__ == "__main__":
    main()
