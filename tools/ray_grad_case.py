"""Ray gradient case (camera refinement): the 2-frame case of tools/frame_grad_case.py (32 samples, jitter, the loss of
oracle/grad_case.py) with ray_o and ray_d (B,n,3) requiring grad.  TEST INFRASTRUCTURE ONLY (tests/test_ray_grad.py).

    python -m tools.ray_grad_case

writes tests/golden/grad_rays_b2_s32.npz from the UNMODIFIED reference (oracle/ref_harness.py): its autograd d ray_o and
d ray_d in full, plus the sha256 of the inputs.  Existing golden files are not touched.

`render_detached` restates the oracle's get_pixel_value with one path from the rays to the loss cut at a time, so the test
can show that every path carries gradient on this case."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import grad_case  # noqa: E402
from tools import frame_grad_case as FC  # noqa: E402

N_SAMPLES = FC.N_SAMPLES
N_IMPORTANCE = FC.N_IMPORTANCE
GOLDEN = "grad_rays_b2_s32"
PATHS = ("viewdir", "norm", "pe", "grid")   # view direction, |ray_d| in raw2outputs, points into PE(xyz), points into the grid

build = FC.build
hier_inputs = FC.hier_inputs


def leaves(scene, decoder=False, frame=False):
    """A copy of the scene whose rays (and optionally decoder + volumes, R + Th) are fresh leaves requiring grad."""
    sc = dict(scene)
    sc["ray_o"] = scene["ray_o"].clone().requires_grad_(True)
    sc["ray_d"] = scene["ray_d"].clone().requires_grad_(True)
    if decoder:
        sc["weights"] = {k: v.clone().requires_grad_(True) for k, v in scene["weights"].items()}
        sc["volumes"] = [v.clone().requires_grad_(True) for v in scene["volumes"]]
    if frame:
        sc["R"] = scene["R"].clone().requires_grad_(True)
        sc["Th"] = scene["Th"].clone().requires_grad_(True)
    return sc


def oracle_ray_grads(scene, t_rand, G, decoder=False, frame=False):
    """Autograd through the oracle restatement -> ({'ray_o', 'ray_d'[, 'R', 'Th', params..., 'vol0'..]: grad}, outputs)."""
    from oracle import neuralbody_oracle as O
    sc = leaves(scene, decoder, frame)
    ret = O.render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand)
    grad_case.loss_of(ret, G).backward()
    return _grads(sc, decoder, frame), ret


def oracle_hier_ray_grads(scene, t_rand, u, G, z_all=None):
    """The same through the oracle's coarse + detached sample_pdf + fine pass (loss + the coarse image term).  z_all
    (B,n,S+N_IMPORTANCE): render the fine pass at these depths instead of the oracle's own importance samples."""
    from oracle import neuralbody_oracle as O
    sc = leaves(scene)
    if z_all is None:
        ret = O.render_hierarchical(sc, n_samples=N_SAMPLES, n_importance=N_IMPORTANCE, perturb=1.0, training=True,
                                    white_bkgd=True, t_rand=t_rand, u=u)
    else:   # render_hierarchical's two passes (one chunk here) with the fine depths given
        sp, w, vs = O.prepare_sp_input(sc), sc["weights"], sc["voxel_size"]
        _, z_vals = O.get_sampling_points(sc["ray_o"], sc["ray_d"], sc["near"], sc["far"], N_SAMPLES, 1.0, True, t_rand)
        coarse = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_vals, sc["volumes"], sp, vs, True)
        ret = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_all, sc["volumes"], sp, vs, True)
        ret["rgb0"] = coarse["rgb_map"]
    grad_case.hier_loss_of(ret, G).backward()
    return _grads(sc, False, False), ret


def _grads(sc, decoder, frame):
    out = {"ray_o": sc["ray_o"].grad, "ray_d": sc["ray_d"].grad}
    if frame:
        out["R"], out["Th"] = sc["R"].grad, sc["Th"].grad
    if decoder:
        out.update({k: sc["weights"][k].grad for k in grad_case.GRAD_KEYS})
        out.update({"vol%d" % l: v.grad for l, v in enumerate(sc["volumes"])})
    return out


def render_detached(scene, t_rand, G, detach=()):
    """get_pixel_value + calculate_density_color of the oracle, composed from its functions, with the rays detached on the
    paths named in `detach` (a subset of PATHS).  -> (d ray_o, d ray_d, raw (B*n, S, 4)); with detach=() the gradients are
    those of oracle_ray_grads."""
    import torch.nn.functional as F
    from oracle import neuralbody_oracle as O
    sc = leaves(scene)
    w, sp, vs = sc["weights"], O.prepare_sp_input(sc), sc["voxel_size"]
    ray_o, ray_d = sc["ray_o"], sc["ray_d"]
    cut = lambda t, path: t.detach() if path in detach else t   # noqa: E731
    wpts, z_vals = O.get_sampling_points(ray_o, ray_d, sc["near"], sc["far"], N_SAMPLES, 1.0, True, t_rand)
    d_view = cut(ray_d, "viewdir")
    viewdir = d_view / torch.norm(d_view, dim=2, keepdim=True)
    B, n, S = wpts.shape[:3]
    wp = wpts.view(B, n * S, 3)
    vd = viewdir[:, :, None].repeat(1, 1, S, 1).contiguous().view(B, n * S, 3)
    # calculate_density_color (latent_xyzc.py:91-126) with its two uses of the world points separated
    grid = O.get_grid_coords(O.pts_to_can_pts(cut(wp, "grid"), sp['R'], sp['Th']), sp['bounds'], sp['out_sh'], vs)
    net = O.interpolate_features(grid, sc["volumes"])
    for name in ("fc_0", "fc_1", "fc_2"):
        net = F.relu(O._conv(w, name, net))
    alpha = O._conv(w, "alpha_fc", net)
    features = O._conv(w, "feature_fc", net)
    latent = w["latent.weight"][sp['latent_index']]
    features = torch.cat((features, latent[..., None].expand(*latent.shape, net.size(2))), dim=1)
    features = O._conv(w, "latent_fc", features)
    features = torch.cat((features, O.positional_embed(vd, 4).transpose(1, 2),
                          O.positional_embed(cut(wp, "pe"), 10).transpose(1, 2)), dim=1)
    rgb = O._conv(w, "rgb_fc", F.relu(O._conv(w, "view_fc", features)))
    raw = torch.cat((rgb, alpha), dim=1).transpose(1, 2).reshape(-1, S, 4)
    rgb_map, _, acc_map, _, depth_map = O.raw2outputs(raw, z_vals.view(-1, S), cut(ray_d, "norm").reshape(-1, 3),
                                                      white_bkgd=True)
    ret = {"rgb_map": rgb_map.view(B, n, 3), "depth_map": depth_map.view(B, n), "acc_map": acc_map.view(B, n)}
    grad_case.loss_of(ret, G).backward()
    return ray_o.grad, ray_d.grad, raw.detach()


def make_golden():
    from oracle import ref_harness, synth
    scene, t_rand, G = build()
    sc = leaves(scene)
    ret, _, _ = ref_harness.reference_render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True,
                                             t_rand=t_rand, grad=True)
    grad_case.loss_of(ret, G).backward()
    arrays = {"input_sha256": np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8),
              "torch_version": np.frombuffer(torch.__version__.encode(), dtype=np.uint8),
              "d_ray_o": sc["ray_o"].grad.numpy().astype(np.float32), "d_ray_d": sc["ray_d"].grad.numpy().astype(np.float32)}
    path = os.path.join(ROOT, "tests", "golden", GOLDEN + ".npz")
    np.savez_compressed(path, **arrays)
    print("ray gradients ->", path, "max |d ray_o| = %.4e, max |d ray_d| = %.4e" % (
        float(sc["ray_o"].grad.abs().max()), float(sc["ray_d"].grad.abs().max())))


if __name__ == "__main__":
    make_golden()
