"""Diagnostics (GPU): what upstream's image loss costs inside a training step, and what the drop-in wrapper
(lib/train/trainers/if_nerf_clight.py, nb_image_loss_fwd / _bwd) saves.  The c3-like step -- one N_rand = 1024 chunk of
the synth-313 frame, 64 coarse + 128 importance samples, perturb = 1, forward, loss, backward,
clip_grad_value_(40) over the network's parameters and an Adam step, as Trainer.train runs it -- two ways in one process,
alternating step by step so that both see the same clocks and host load:
  upstream: this renderer with upstream's wrapper expression torch.mean((rgb_map[mask] - rgb[mask]) ** 2) + img_loss0;
  dropin:   the drop-in NetworkWrapper.
Reported per way: ms per step (CUDA events around the step, mean and median over the timed steps), and how often the host
queued the backward's first launch before the forward pass had finished on the device (an event recorded after the
render, queried when loss.backward() is called: not yet complete = the host ran ahead).  Prints one JSON line.
Usage: python tools/bench_trainer.py [iters=50] [--precision tc_tf32x3|fp32] [--importance 128]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402


def main():
    args = sys.argv[1:]
    opts = {"--precision": "tc_tf32x3", "--importance": "128"}
    for k in list(opts):
        if k in args:
            i = args.index(k)
            opts[k] = args[i + 1]
            del args[i:i + 2]
    iters = int(args[0]) if args else 50
    if not torch.cuda.is_available():
        raise SystemExit("bench_trainer needs a CUDA device")
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    import gpu_utils as G
    torch.set_num_threads(1)         # as under torchrun (OMP_NUM_THREADS=1): the step's few CPU ops stay on this thread
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    g = torch.Generator().manual_seed(0)
    idx = torch.randperm(scene["ray_o"].shape[1], generator=g)[:1024]
    for k in ("ray_o", "ray_d", "near", "far"):
        scene[k] = scene[k][:, idx].contiguous()
    net, _ = G.make_net_and_renderer(scene)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype = "tc_fp16x3", "auto"
    cfg.render_importance, cfg.render_train_precision, cfg.render_return_weights = int(opts["--importance"]), opts["--precision"], True
    net.train()
    vols = [v.cuda().requires_grad_(True) for v in scene["volumes"]]
    net.set_feature_volume(vols)
    batch = {k: scene[k].cuda() for k in G.BATCH_KEYS}
    batch["rgb"] = torch.rand((1, 1024, 3), generator=g).cuda()
    batch["mask_at_box"] = torch.ones((1, 1024), dtype=torch.bool, device="cuda")     # the training items' all-True mask
    mod = load_source("lib.train.trainers.if_nerf_clight",
                      os.path.join(ROOT, "neuralbody_b200", "lib", "train", "trainers", "if_nerf_clight.py"))
    wrapper = mod.NetworkWrapper(net)
    ren = wrapper.renderer
    optimizer = torch.optim.Adam(net.parameters(), lr=5e-4)

    def upstream_forward(b, marks):
        ret = ren.render(b)
        marks.append(torch.cuda.Event())
        marks[-1].record()
        mask = b["mask_at_box"]
        loss = 0
        loss += torch.mean((ret["rgb_map"][mask] - b["rgb"][mask]) ** 2)
        if "rgb0" in ret:
            loss += torch.mean((ret["rgb0"] - b["rgb"]) ** 2)
        return loss

    def dropin_forward(b, marks):
        orig = ren.render

        def render(bb):
            out = orig(bb)
            marks.append(torch.cuda.Event())
            marks[-1].record()
            return out
        ren.render = render
        try:
            return wrapper(b)[1]
        finally:
            ren.render = orig

    ways = {"upstream": upstream_forward, "dropin": dropin_forward}
    ahead = {w: 0 for w in ways}

    def step(way, count):
        marks = []
        optimizer.zero_grad()
        for v in vols:
            v.grad = None
        loss = ways[way](dict(batch), marks)
        before_bwd = not marks[-1].query()        # the forward pass still running on the device when backward is queued
        loss.backward()
        torch.nn.utils.clip_grad_value_(wrapper.parameters(), 40)
        optimizer.step()
        if count:
            ahead[way] += int(before_bwd)
        return loss

    for _ in range(5):
        for w in ways:
            step(w, False)
    torch.cuda.synchronize()
    ev = {w: [] for w in ways}
    for _ in range(iters):
        for w in ways:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(w, True)
            e1.record()
            ev[w].append((e0, e1))
    torch.cuda.synchronize()
    res = {"config": "c3-like training step: 1024 rays, 64 + %s samples, perturb 1, %s, forward + loss + backward + "
                     "clip_grad_value_(40) + Adam, alternating" % (opts["--importance"], opts["--precision"]),
           "gpu": torch.cuda.get_device_name(0), "iters": iters}
    for w in ways:
        ms = sorted(a.elapsed_time(b) for a, b in ev[w])
        res[w] = {"ms_per_step": sum(ms) / iters, "median_ms": ms[iters // 2], "min_ms": ms[0],
                  "host_ahead_of_forward_at_backward": "%d of %d steps" % (ahead[w], iters)}
    res["dropin_saves_ms"] = res["upstream"]["ms_per_step"] - res["dropin"]["ms_per_step"]
    res["dropin_saves_median_ms"] = res["upstream"]["median_ms"] - res["dropin"]["median_ms"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
