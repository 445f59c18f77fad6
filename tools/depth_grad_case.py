"""Depth gradient case: the 2-frame case of tools/frame_grad_case.py (32 samples, jitter, white background, the loss of
oracle/grad_case.py) with near, far (B,n) and bounds (B,2,3) requiring grad.  TEST INFRASTRUCTURE ONLY
(tests/test_depth_grad.py).

    python -m tools.depth_grad_case

writes tests/golden/grad_depths_b2_s32.npz from the UNMODIFIED reference (oracle/ref_harness.py): its autograd d near,
d far and d bounds in full (with the rays training too, their gradients), plus the sha256 of the inputs.  Existing golden
files are not touched.

`render_detached` restates the oracle's get_pixel_value with z cut on one of its three paths to the loss at a time (the
sample points ray_o + ray_d z, the dists of raw2outputs, the depth map sum w z), so the test can show that each carries
gradient to near / far on this case."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import grad_case  # noqa: E402
from tools import frame_grad_case as FC  # noqa: E402
from tools import ray_grad_case as RC  # noqa: E402

N_SAMPLES = FC.N_SAMPLES
N_IMPORTANCE = FC.N_IMPORTANCE
GOLDEN = "grad_depths_b2_s32"
PATHS = ("points", "dists", "depth")
DEPTH_KEYS = ("near", "far", "bounds")

build = FC.build
hier_inputs = FC.hier_inputs


def leaves(scene, decoder=False, frame=False):
    """A copy of the scene whose rays, near, far and bounds (and optionally decoder + volumes, R + Th) are fresh leaves
    requiring grad."""
    sc = RC.leaves(scene, decoder, frame)
    for k in DEPTH_KEYS:
        sc[k] = scene[k].clone().requires_grad_(True)
    return sc


def grads_of(sc, decoder=False, frame=False):
    out = RC._grads(sc, decoder, frame)
    out.update({k: sc[k].grad for k in DEPTH_KEYS})
    return out


def oracle_depth_grads(scene, t_rand, loss, decoder=False, frame=False):
    """Autograd of loss(outputs) through the oracle restatement -> ({'near', 'far', 'bounds', 'ray_o', 'ray_d'[, 'R', 'Th',
    params..., 'vol0'..]: grad}, outputs)."""
    from oracle import neuralbody_oracle as O
    sc = leaves(scene, decoder, frame)
    ret = O.render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand)
    loss(ret).backward()
    return grads_of(sc, decoder, frame), ret


def render_detached(scene, t_rand, G, detach=()):
    """get_pixel_value of the oracle, composed from its functions, with z detached on the paths named in `detach` (a subset
    of PATHS) -> (d near, d far); with detach=() these are oracle_depth_grads' under grad_case.loss_of."""
    import torch.nn.functional as F
    from oracle import neuralbody_oracle as O
    sc = leaves(scene)
    w, sp, vs = sc["weights"], O.prepare_sp_input(sc), sc["voxel_size"]
    ray_o, ray_d = sc["ray_o"], sc["ray_d"]
    cut = lambda t, path: t.detach() if path in detach else t   # noqa: E731
    _, z_vals = O.get_sampling_points(ray_o, ray_d, sc["near"], sc["far"], N_SAMPLES, 1.0, True, t_rand)
    wpts = ray_o[:, :, None] + ray_d[:, :, None] * cut(z_vals, "points")[..., None]
    viewdir = ray_d / torch.norm(ray_d, dim=2, keepdim=True)
    B, n, S = wpts.shape[:3]
    vd = viewdir[:, :, None].repeat(1, 1, S, 1).contiguous().view(B, n * S, 3)
    raw = O.calculate_density_color(w, wpts.view(B, n * S, 3), vd, sc["volumes"], sp, vs).reshape(-1, S, 4)
    # raw2outputs (nerf_net_utils.py:6-51) with z's two uses in it separated
    z = z_vals.view(-1, S)
    zd = cut(z, "dists")
    dists = zd[..., 1:] - zd[..., :-1]
    dists = torch.cat([dists, torch.Tensor([1e10]).expand(dists[..., :1].shape).to(dists)], -1)
    dists = dists * torch.norm(ray_d.reshape(-1, 3)[..., None, :], dim=-1)
    rgb = torch.sigmoid(raw[..., :3])
    alpha = 1. - torch.exp(-F.relu(raw[..., 3]) * dists)
    weights = alpha * torch.cumprod(torch.cat([torch.ones((alpha.shape[0], 1)).to(alpha), 1. - alpha + 1e-10], -1), -1)[:, :-1]
    acc_map = torch.sum(weights, -1)
    rgb_map = torch.sum(weights[..., None] * rgb, -2) + (1. - acc_map[..., None])
    depth_map = torch.sum(weights * cut(z, "depth"), -1)
    ret = {"rgb_map": rgb_map.view(B, n, 3), "depth_map": depth_map.view(B, n), "acc_map": acc_map.view(B, n)}
    grad_case.loss_of(ret, G).backward()
    return sc["near"].grad, sc["far"].grad


def make_golden():
    from oracle import ref_harness, synth
    scene, t_rand, G = build()
    sc = leaves(scene)
    ret, _, _ = ref_harness.reference_render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True,
                                             t_rand=t_rand, grad=True)
    grad_case.loss_of(ret, G).backward()
    got = grads_of(sc)
    for k, g in got.items():
        assert g is not None and torch.isfinite(g).all(), k
    assert not bool(got["bounds"][:, 1].any())          # get_grid_coords reads bounds[:, 0] only
    arrays = {"input_sha256": np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8),
              "torch_version": np.frombuffer(torch.__version__.encode(), dtype=np.uint8)}
    arrays.update({"d_" + k: g.numpy().astype(np.float32) for k, g in got.items()})
    path = os.path.join(ROOT, "tests", "golden", GOLDEN + ".npz")
    np.savez_compressed(path, **arrays)
    print("depth gradients ->", path, {k: "max |d| = %.4e" % float(g.abs().max()) for k, g in got.items()})


if __name__ == "__main__":
    make_golden()
