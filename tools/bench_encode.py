"""Diagnostics (GPU): the SparseConvNet encode on the synth-313 frame (6890 vertices, 5 mm voxels, out_sh 96 x 352 x 192),
two ways in one process, alternating call by call so both see the same clocks and host load:
  dense: DenseSparseConvNet (lib/networks/sparse_encode.py), the dense-PyTorch emulation, float32 (cuDNN convolutions
         with PyTorch's default TF32 setting for them);
  cuda:  CudaSparseConvNet (lib/networks/sparse_encode_cuda.py, nb_spconv_fwd / nb_spconv_bwd).
Timed with CUDA events: the forward in train mode, the forward + backward (a fixed random cotangent on the four volumes,
gradients into the code, the conv weights and the BatchNorm parameters), and the c3-like training step of
tools/bench_trainer.py (1024 rays, 64 + --importance samples, perturb 1, forward + loss + backward + clip_grad_value_(40) +
Adam through the trainer drop-in) with the encode inside it.  Also: the peak memory of one forward + backward above what
was allocated before it, and the active rows of every level.  Reports the median, min and max over the timed calls, the
card, its power limit and its maximum SM clock.  Prints one JSON line.
Usage: python tools/bench_encode.py [iters=20] [--importance 128]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402


def _card():
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:          # the numbers are reported without them, and say so
        out["power_limit"] = out["max_sm_clock"] = "not read (%s)" % type(e).__name__
    return out


def _stats(ms):
    ms = sorted(ms)
    return {"median_ms": ms[len(ms) // 2], "min_ms": ms[0], "max_ms": ms[-1]}


def _alternate(fns, iters, warmup=3):
    for _ in range(warmup):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    ev = {k: [] for k in fns}
    for _ in range(iters):
        for k, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            ev[k].append((e0, e1))
    torch.cuda.synchronize()
    return {k: _stats([a.elapsed_time(b) for a, b in v]) for k, v in ev.items()}


def main():
    args = sys.argv[1:]
    importance = "128"
    if "--importance" in args:
        i = args.index("--importance")
        importance = args[i + 1]
        del args[i:i + 2]
    iters = int(args[0]) if args else 20
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode needs a CUDA device")
    from oracle import synth
    from neuralbody_b200.lib.config import cfg
    from neuralbody_b200.lib.networks.make_network import load_source
    from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
    from neuralbody_b200.lib.networks.sparse_encode_cuda import CudaSparseConvNet
    import gpu_utils as G
    torch.set_num_threads(1)
    dev = "cuda:0"
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    torch.manual_seed(0)
    dense = DenseSparseConvNet()
    cuda = CudaSparseConvNet()
    cuda.load_state_dict(dense.state_dict())
    dense, cuda = dense.to(dev).train(), cuda.to(dev).train()
    coord = torch.cat([torch.zeros((6890, 1), dtype=torch.int32), scene["coord"][0]], 1).to(dev)
    out_sh = scene["out_sh"][0].tolist()
    code = torch.randn(6890, 16, device=dev, requires_grad=True)
    g = torch.Generator(device=dev).manual_seed(1)
    with torch.no_grad():
        shapes = [tuple(v.shape) for v in cuda.encode(code, coord, out_sh, 1)]
    cot = [torch.randn(s, generator=g, device=dev) for s in shapes]
    encoders = {"dense": dense, "cuda": cuda}

    def fwd(m):
        with torch.no_grad():
            m.encode(code, coord, out_sh, 1)

    def fwd_bwd(m):
        torch.autograd.backward(m.encode(code, coord, out_sh, 1), cot)

    res = {"config": "synth-313 frame, B = 1, out_sh %s, train mode; dense and cuda alternating" % (out_sh,),
           "iters": iters}
    res.update(_card())
    res["forward"] = _alternate({k: (lambda m=m: fwd(m)) for k, m in encoders.items()}, iters)
    res["forward_backward"] = _alternate({k: (lambda m=m: fwd_bwd(m)) for k, m in encoders.items()}, iters)
    peak = {}
    for k, m in encoders.items():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fwd_bwd(m)
        torch.cuda.synchronize()
        peak[k] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    res["peak_mem_mib_forward_backward"] = peak
    res["active_rows"] = dict(zip(("input", "level1", "level2", "level3", "level4"), cuda.last_row_counts.tolist()))
    res["grid_sites"] = [out_sh[0] * out_sh[1] * out_sh[2]] + [s[2] * s[3] * s[4] for s in shapes]

    # the c3-like training step with the encode inside it
    idx = torch.randperm(scene["ray_o"].shape[1], generator=torch.Generator().manual_seed(0))[:1024]
    for k in ("ray_o", "ray_d", "near", "far"):
        scene[k] = scene[k][:, idx].contiguous()
    net, _ = G.make_net_and_renderer(scene)
    net.set_feature_volume(None)
    cfg.N_samples, cfg.perturb, cfg.white_bkgd, cfg.raw_noise_std, cfg.chunk = 64, 1.0, False, 0, 0
    cfg.render_precision, cfg.render_volume_dtype = "tc_fp16x3", "auto"
    cfg.render_importance, cfg.render_train_precision, cfg.render_return_weights = int(importance), "tc_tf32x3", True
    net.train()
    batch = {k: scene[k].to(dev) for k in G.BATCH_KEYS}
    batch["rgb"] = torch.rand((1, 1024, 3), generator=torch.Generator().manual_seed(2)).to(dev)
    batch["mask_at_box"] = torch.ones((1, 1024), dtype=torch.bool, device=dev)
    mod = load_source("lib.train.trainers.if_nerf_clight",
                      os.path.join(ROOT, "neuralbody_b200", "lib", "train", "trainers", "if_nerf_clight.py"))
    wrapper = mod.NetworkWrapper(net)
    net.xyzc_net = dense
    optimizer = torch.optim.Adam(list(net.parameters()) + list(cuda.parameters()), lr=5e-4)

    def step(m):
        net.xyzc_net = m
        optimizer.zero_grad()
        loss = wrapper(dict(batch))[1]
        loss.backward()
        torch.nn.utils.clip_grad_value_(wrapper.parameters(), 40)
        optimizer.step()

    res["train_step"] = _alternate({k: (lambda m=m: step(m)) for k, m in encoders.items()}, iters)
    res["train_step"]["config"] = "c3-like: 1024 rays, 64 + %s samples, perturb 1, tc_tf32x3, encode included" % importance
    print(json.dumps(res))


if __name__ == "__main__":
    main()
