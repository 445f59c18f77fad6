"""Diagnostics (GPU): BASELINE config 3 -- one N_rand = 1024 training chunk on the synth-313 body, 64 coarse samples +
128 importance samples (cfg.render_importance), gradient path on: forward (the training precision cfg.render_train_precision,
default tc_tf32x3: sample list + TF32x3 GEMM chains, with activation record, coarse + fine) + nb_sample_pdf + backward through
both passes.  Prints one JSON line (rays/s for fwd+bwd).
With --frame-grads the same process alternates steps without and with gradients for the frame transform
(sp_input['R'] / ['Th'] requiring grad, as pose refinement does) and reports both step times; --ray-grads does the same
with ray_o / ray_d requiring grad (camera refinement), --map-grads with a loss that also reads disp_map, disp0 and the fine
weights (an entropy regulariser on the ray weights and a disparity term, as distortion / smoothness losses do),
--depth-grads with near, far and sp_input['bounds'] requiring grad (the box-intersection near / far of refined cameras).
Usage: python tools/bench_train_chunk.py [n_importance=128] [iters=30] [--frame-grads] [--ray-grads] [--map-grads]
                                         [--depth-grads] [--precision tc_tf32x3|fp32]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402


def main():
    args = sys.argv[1:]
    frame_grads = "--frame-grads" in args
    ray_grads = "--ray-grads" in args
    map_grads = "--map-grads" in args
    depth_grads = "--depth-grads" in args
    precision = "tc_tf32x3"
    if "--precision" in args:
        precision = args[args.index("--precision") + 1]
        del args[args.index("--precision"):args.index("--precision") + 2]
    pos = [a for a in args if not a.startswith("--")]
    ni = int(pos[0]) if len(pos) > 0 else 128
    iters = int(pos[1]) if len(pos) > 1 else 30
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    import gpu_utils as G
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(scene["ray_o"].shape[1], generator=g)[:1024]
    for k in ("ray_o", "ray_d", "near", "far"):
        scene[k] = scene[k][:, idx].contiguous()
    net, ren = G.make_net_and_renderer(scene)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype, cfg.render_importance = "tc_fp16x3", "auto", ni
    cfg.render_train_precision = precision
    net.train()
    vols = [v.cuda().requires_grad_(True) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    sp = ren.prepare_sp_input(batch)
    pose = dict(batch, R=batch["R"].clone().requires_grad_(True), Th=batch["Th"].clone().requires_grad_(True))
    sp_pose = ren.prepare_sp_input(pose)
    cam = dict(batch, ray_o=batch["ray_o"].clone().requires_grad_(True), ray_d=batch["ray_d"].clone().requires_grad_(True))
    depth = dict(batch, near=batch["near"].clone().requires_grad_(True), far=batch["far"].clone().requires_grad_(True),
                 bounds=batch["bounds"].clone().requires_grad_(True))
    sp_depth = ren.prepare_sp_input(depth)
    target = torch.rand((1, 1024, 3), device="cuda")

    def step(mode):
        for p in net.parameters():
            p.grad = None
        for v in vols:
            v.grad = None
        s, b = {"plain": (sp, batch), "frame": (sp_pose, pose), "rays": (sp, cam), "maps": (sp, batch), "depths": (sp_depth, depth)}[mode]
        b["R"].grad = b["Th"].grad = b["ray_o"].grad = b["ray_d"].grad = None
        b["near"].grad = b["far"].grad = b["bounds"].grad = None
        out = ren.get_pixel_value(b["ray_o"], b["ray_d"], b["near"], b["far"], vols, s, b)
        loss = ((out["rgb_map"] - target) ** 2).mean()
        if "rgb0" in out:
            loss = loss + ((out["rgb0"] - target) ** 2).mean()          # img_loss0, if_nerf_clight.py:29-32
        if mode == "maps":
            w = out["weights"]
            loss = loss + 1e-3 * -(w * torch.log(w + 1e-10)).sum(-1).mean()
            for d, a in (("disp_map", "acc_map"), ("disp0", "acc0")):
                loss = loss + 1e-3 * torch.where(out[a] > 0, out[d], torch.zeros_like(out[d])).mean()
        loss.backward()

    modes = ("plain",) + (("frame",) if frame_grads else ()) + (("rays",) if ray_grads else ()) + (("maps",) if map_grads else ()) + \
        (("depths",) if depth_grads else ())
    for _ in range(5):
        for m in modes:
            step(m)
    torch.cuda.synchronize()
    # alternate the modes step by step so that both see the same clocks and host load; one event pair per step
    ev = {m: [] for m in modes}
    for _ in range(iters):
        for m in modes:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(m)
            e1.record()
            ev[m].append((e0, e1))
    torch.cuda.synchronize()
    ms = {m: sum(a.elapsed_time(b) for a, b in ev[m]) / iters for m in modes}
    res = {"config": "c3: 1024-ray training chunk, 64 + %d samples, fwd + bwd, %s" % (ni, precision),
           "gpu": torch.cuda.get_device_name(0),
           "ms_per_step": ms["plain"], "rays_per_s_fwd_bwd": 1024 / (ms["plain"] * 1e-3),
           "grad_norm_fc0": float(dict(net.named_parameters())["fc_0.weight"].grad.norm())}
    if frame_grads:
        res["ms_per_step_frame_grads"] = ms["frame"]
        res["frame_grads_overhead_ms"] = ms["frame"] - ms["plain"]
        res["dR_norm"], res["dTh_norm"] = float(pose["R"].grad.norm()), float(pose["Th"].grad.norm())
    if ray_grads:
        res["ms_per_step_ray_grads"] = ms["rays"]
        res["ray_grads_overhead_ms"] = ms["rays"] - ms["plain"]
        res["d_ray_o_norm"], res["d_ray_d_norm"] = float(cam["ray_o"].grad.norm()), float(cam["ray_d"].grad.norm())
    if map_grads:
        res["ms_per_step_map_grads"] = ms["maps"]
        res["map_grads_overhead_ms"] = ms["maps"] - ms["plain"]
    if depth_grads:
        res["ms_per_step_depth_grads"] = ms["depths"]
        res["depth_grads_overhead_ms"] = ms["depths"] - ms["plain"]
        res["d_near_norm"], res["d_far_norm"] = float(depth["near"].grad.norm()), float(depth["far"].grad.norm())
        res["d_bounds_norm"] = float(depth["bounds"].grad.norm())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
