"""Training-chunk case: the step bench.py --config c3 times, at its full size, as test infrastructure.
TEST INFRASTRUCTURE ONLY (tests/test_train_chunk_cpu.py, tests/test_train_chunk_gpu.py).

The scene is bench.build_scene()'s: the full-size synth-313 body (synth.make_scene(H=512, W=512, scale=1.0, all_hit=True),
a 137 MB float32 volume), of which a step renders one 1024-ray chunk: N_SAMPLES coarse samples, then N_IMPORTANCE importance
samples drawn from the coarse weights, and a fine pass over the merged 192 depths; the loss is run_c3's,
mse(rgb_map) + mse(rgb0), against a seeded target.  Two chunks, A and B, are drawn with different seeds, so that one
Renderer driven through both sees list lengths change from one step to the next.

As in oracle/frames_case.py, every sample that carries gradient is kept off the trilinear cell faces and the decoder's
ReLU kinks, where float32 and float64 can legitimately disagree by O(1):
  - the coarse jitter t_rand is redrawn where a coarse sample is fragile (build);
  - the importance uniforms u are redrawn where a fine sample is fragile (fine_depths).  The fine depths depend on the coarse
    weights, which only the kernel under test produces bit for bit, so this runs once the coarse pass has run: the depths
    come from ray_stages.sample_pdf_emulate, which is bit-exact with nb_sample_pdf.
A redraw moves only the sample redrawn (a coarse sample's depth depends on its own jitter; an importance sample on its own
uniform and the CDF), so only the redrawn samples are evaluated again, held to the margins of the whole pass
(frames_case.sample_conditions' `scale`).

The depths of both passes are the kernels' float32 values (ray_stages.z_sample for the coarse pass, the emulated merge for
the fine one); the float64 reference (oracle_step) evaluates the decoder at exactly those depths."""
import time

import numpy as np
import torch

H = W = 512
N_RAYS = 1024
N_SAMPLES = 64
N_IMPORTANCE = 128
CHUNK_SEEDS = {"A": 0, "B": 1}     # "A" is run_c3's own chunk (torch.randperm with seed 0)
MAX_REDRAWS = 40


def full_scene():
    """bench.build_scene(): the full-size synth-313 frame, every pixel's ray."""
    from oracle import synth
    return synth.make_scene(H=H, W=W, scale=1.0, all_hit=True)


def t_vals(S):
    """The renderer's t_vals (Renderer._t_vals: torch.linspace on the CPU), as the float32 the kernels read."""
    return torch.linspace(0., 1., steps=S).numpy()


def coarse_depths(scene, t_rand):
    """(1,n,S) float32: the coarse pass's depths as the kernels compute them (ray_stages.z_sample)."""
    from oracle import ray_stages as RS
    near, far = scene["near"][0].numpy(), scene["far"][0].numpy()
    z = RS.z_sample(near, far, t_rand.shape[-1], t_vals(t_rand.shape[-1]), t_rand[0].numpy())
    return torch.from_numpy(z)[None]


def _rays_of(scene, rows):
    """The scene with one ray per entry of `rows` (ray indices, repeats allowed)."""
    sub = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sub[k] = scene[k][:, rows].contiguous()
    return sub


def condition(scene, depths_of, draws, gen, what):
    """Redraw the entries of `draws` (1,n,K) whose sample is fragile until none is left.  depths_of(draws) -> (1,n,K) float32
    depths.  The first pass evaluates every sample; a later one only those just redrawn, against the first pass's margins.
    Returns (draws, stats): the number of fragile samples found on the first pass, the redraw passes it took and the margins
    scale (the first pass's rms pre-activations, which every later pass and a check of the result are held to)."""
    from oracle import frames_case as FR
    draws = draws.clone()
    cond = FR.sample_conditions(scene, depths_of(draws))
    bad, scale = cond["fragile"], cond["scale"]
    first = int(bad.sum())
    for it in range(MAX_REDRAWS):
        if not bool(bad.any()):
            return draws, {"fragile_first_pass": first, "redraw_passes": it, "scale": scale}
        rows, cols = bad[0].nonzero(as_tuple=True)
        draws[0, rows, cols] = torch.rand(len(rows), generator=gen)
        z = depths_of(draws)[0, rows, cols]
        again = FR.sample_conditions(_rays_of(scene, rows), z.view(1, -1, 1), scale=scale)["fragile"].view(-1)
        bad = torch.zeros_like(bad)
        bad[0, rows[again], cols[again]] = True
    raise AssertionError("%s: could not keep the samples off the cell faces and ReLU kinks" % what)


def build(chunk="A", scene=None):
    """Chunk `chunk` of the c3 step: dict(scene (1024 rays), idx, t_rand (1,n,S), u0 (1,n,Ni) uniforms before the fine
    conditioning, target (1,n,3), stats: what the coarse conditioning found)."""
    if scene is None:
        scene = full_scene()
    seed = CHUNK_SEEDS[chunk]
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(scene["ray_o"].shape[1], generator=g)[:N_RAYS]            # run_c3's draw
    sc = _rays_of(scene, idx)
    g = torch.Generator().manual_seed(1000 + seed)
    target = torch.rand((1, N_RAYS, 3), generator=g)
    t_rand = torch.rand((1, N_RAYS, N_SAMPLES), generator=g)
    u0 = torch.rand((1, N_RAYS, N_IMPORTANCE), generator=g)
    t_rand, stats = condition(sc, lambda tr: coarse_depths(sc, tr), t_rand, g, "coarse jitter")
    return {"chunk": chunk, "scene": sc, "idx": idx, "t_rand": t_rand, "u0": u0, "target": target,
            "stats": {"coarse": stats}}


def importance(case, weights, u):
    """ray_stages.sample_pdf_emulate on the chunk: coarse weights (1,n,S) float32 -> its dict (z_out (n, S + Ni), ...)."""
    from oracle import ray_stages as RS
    sc = case["scene"]
    return RS.sample_pdf_emulate(sc["near"][0].numpy(), sc["far"][0].numpy(), np.asarray(weights, np.float32).reshape(N_RAYS, -1),
                                 N_SAMPLES, N_IMPORTANCE, t_vals(N_SAMPLES), case["t_rand"][0].numpy(), u[0].numpy())


def fine_depths(case, weights):
    """The fine pass's depths from the coarse pass's weights (1,n,S): (u (1,n,Ni) with every fragile fine sample's uniform
    redrawn, Z (1,n,S+Ni) float32 sorted, stats).  Deterministic: the same weights give the same u and Z."""
    g = torch.Generator().manual_seed(2000 + CHUNK_SEEDS[case["chunk"]])

    def smp(u):
        return torch.from_numpy(importance(case, weights, u)["z_samples"])[None]
    u, stats = condition(case["scene"], smp, case["u0"], g, "importance uniforms")
    Z = torch.from_numpy(importance(case, weights, u)["z_out"])[None]
    return u, Z, stats


def listed_bounds(case, depths):
    """What the training forward's sample list must hold for one pass at `depths` (1,n,K): the float64 count of samples with a
    non-zero feature, leaving out every sample within FACE_MARGIN cells of a cell face of any level (occupied or not: float32
    may put it in the neighbouring cell), and the number left out.  The list length lies in [count, count + near_face]."""
    from oracle import frames_case as FR
    cond = FR.sample_conditions(case["scene"], depths, kinks=False)
    near_face = cond["face"] < FR.FACE_MARGIN
    return int((cond["occupied"] & ~near_face).sum()), int(near_face.sum())


def loss_of(ret, target):
    """run_c3's loss: mse(rgb_map) + mse(rgb0) (img_loss + img_loss0, lib/train/trainers/if_nerf_clight.py:29-32)."""
    return ((ret["rgb_map"] - target) ** 2).mean() + ((ret["rgb0"] - target) ** 2).mean()


def oracle_step(case, Z, rays_per_chunk=128):
    """Autograd of loss_of through the oracle in float64, decoder tensors and volumes the leaves: the coarse pass at the
    kernels' coarse depths, the fine pass at Z (detached, as upstream).  Run by rays, `rays_per_chunk` at a time (the loss is a
    sum over rays, so the chunks' gradients add up to the whole step's), to bound the float64 activations.
    Returns ({name: grad} (GRAD_KEYS, vol0..3), {map: (1,n,...)} (the fine maps, rgb0 / acc0, weights of both passes),
    seconds)."""
    from oracle import frames_case as FR
    from oracle import grad_case
    from oracle import neuralbody_oracle as O
    t0 = time.perf_counter()
    sc = FR.to_double(case["scene"])
    w = {k: v.clone().requires_grad_(True) for k, v in sc["weights"].items()}
    vols = [v.clone().requires_grad_(True) for v in sc["volumes"]]
    sp = O.prepare_sp_input(sc)
    zc = coarse_depths(case["scene"], case["t_rand"]).double()
    Zd = Z.double()
    tgt = case["target"].double()
    n = zc.shape[1]
    outs = []
    for i in range(0, n, rays_per_chunk):
        r = slice(i, i + rays_per_chunk)
        ro, rd = sc["ray_o"][:, r], sc["ray_d"][:, r]
        coarse = O.get_pixel_value_at(w, ro, rd, zc[:, r], vols, sp, sc["voxel_size"])
        fine = O.get_pixel_value_at(w, ro, rd, Zd[:, r], vols, sp, sc["voxel_size"])
        ret = {"rgb_map": fine["rgb_map"], "rgb0": coarse["rgb_map"]}
        # the whole step's mean over n rays, restricted to these rays
        loss = (((ret["rgb_map"] - tgt[:, r]) ** 2).sum() + ((ret["rgb0"] - tgt[:, r]) ** 2).sum()) / (n * 3)
        loss.backward()
        outs.append({"rgb_map": fine["rgb_map"], "acc_map": fine["acc_map"], "depth_map": fine["depth_map"],
                     "weights": fine["weights"], "rgb0": coarse["rgb_map"], "acc0": coarse["acc_map"],
                     "weights0": coarse["weights"]})
    maps = {k: torch.cat([o[k].detach() for o in outs], 1) for k in outs[0]}
    grads = {k: w[k].grad for k in grad_case.GRAD_KEYS}
    grads.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return grads, maps, time.perf_counter() - t0
