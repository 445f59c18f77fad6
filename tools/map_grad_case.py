"""Map gradient case: the 2-frame case of tools/frame_grad_case.py (32 samples, jitter, white background) with a loss that also
reads disp_map and weights, and every input training: decoder, volumes, R / Th and the rays.  TEST INFRASTRUCTURE ONLY
(tests/test_map_grad.py).

    python -m tools.map_grad_case

writes tests/golden/grad_maps_b2_s32.npz from the UNMODIFIED reference (oracle/ref_harness.py): its autograd d ray_o,
d ray_d (NaNs included), dR and dTh in full, the sum / abs / head summaries of the decoder and volume gradients (as
grad_train_s32), plus the sha256 of the inputs.  Existing golden files are not touched.

The loss is grad_case.loss_of + sum(where(acc > 0, disp, 0) G_disp) + sum(weights G_w).  The where() keeps the loss finite,
but on a ray with acc == 0 the gradient of disp_map is still NaN (0 * NaN): upstream's relu keeps it out of sigma, so only
d ray_d (through dists * relu(sigma)) is NaN, on exactly those rays.  The generator asserts that, and that the two new terms
move the gradients by far more than the GPU gate."""
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
GOLDEN = "grad_maps_b2_s32"
# the new terms must move each of these gradients by more than this (rel-L2, finite entries): ten times the GPU gate.
# The colour path (rgb_fc, view_fc, latent_fc, feature_fc, latent) does not see disp_map or weights at all.
TERM_MARGIN = 1e-2
TERM_KEYS = ("fc_0.weight", "fc_1.weight", "fc_2.weight", "alpha_fc.weight", "vol0", "R", "Th", "ray_o", "ray_d")

build = FC.build


def map_cotangents(scene):
    """(G_disp (B,n), G_w (B,n,S)), seed 101."""
    B, n = scene["ray_o"].shape[:2]
    g = torch.Generator().manual_seed(101)
    return torch.randn((B, n), generator=g) * 0.2, torch.randn((B, n, N_SAMPLES), generator=g) * 0.5


def loss_of(ret, G, Gm, terms=True):
    """grad_case.loss_of plus, with `terms`, the disparity and weights terms; Gm = (G_disp, G_w) on ret's device."""
    loss = grad_case.loss_of(ret, G)
    if terms:
        disp = torch.where(ret["acc_map"] > 0, ret["disp_map"], torch.zeros_like(ret["disp_map"]))
        loss = loss + (disp * Gm[0]).sum() + (ret["weights"] * Gm[1]).sum()
    return loss


def oracle_map_grads(scene, t_rand, loss):
    """Autograd of loss(outputs) through the oracle restatement, everything training -> ({'ray_o', 'ray_d', 'R', 'Th',
    params..., 'vol0'..: grad}, outputs)."""
    from oracle import neuralbody_oracle as O
    sc = RC.leaves(scene, decoder=True, frame=True)
    ret = O.render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand)
    loss(ret).backward()
    return RC._grads(sc, True, True), ret


def oracle_hier_map_grads(scene, t_rand, G, Gm, z_all):
    """Coarse + fine pass of the oracle with the fine depths given (z_all (B,n,S+N_IMPORTANCE)), rays training; the loss is
    hier_loss_of + the disp term on the coarse disp0 + the weights term on the fine weights (Gm[1] (B,n,S+N_IMPORTANCE))."""
    from oracle import neuralbody_oracle as O
    sc = RC.leaves(scene)
    sp, w, vs = O.prepare_sp_input(sc), sc["weights"], sc["voxel_size"]
    _, z_vals = O.get_sampling_points(sc["ray_o"], sc["ray_d"], sc["near"], sc["far"], N_SAMPLES, 1.0, True, t_rand)
    coarse = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_vals, sc["volumes"], sp, vs, True)
    ret = O.get_pixel_value_at(w, sc["ray_o"], sc["ray_d"], z_all, sc["volumes"], sp, vs, True)
    ret.update(rgb0=coarse["rgb_map"], disp0=coarse["disp_map"], acc0=coarse["acc_map"])
    hier_loss_of(ret, G, Gm).backward()
    return RC._grads(sc, False, False), ret


def hier_loss_of(ret, G, Gm):
    disp0 = torch.where(ret["acc0"] > 0, ret["disp0"], torch.zeros_like(ret["disp0"]))
    return grad_case.hier_loss_of(ret, G) + (disp0 * Gm[0]).sum() + (ret["weights"] * Gm[1]).sum()


def rel_l2_finite(a, b):
    """rel-L2 of a against b over the entries finite in both."""
    a, b = a.double(), b.double()
    m = torch.isfinite(a) & torch.isfinite(b)
    return float((a[m] - b[m]).norm() / b[m].norm().clamp_min(1e-30))


def _reference_grads(scene, t_rand, G, Gm, terms):
    from oracle import ref_harness
    sc = RC.leaves(scene, frame=True)
    ret, net, vols = ref_harness.reference_render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True,
                                                  t_rand=t_rand, grad=True)
    loss_of(ret, G, Gm, terms).backward()
    sd = dict(net.named_parameters())
    out = {"ray_o": sc["ray_o"].grad, "ray_d": sc["ray_d"].grad, "R": sc["R"].grad, "Th": sc["Th"].grad}
    out.update({k: sd[k].grad for k in grad_case.GRAD_KEYS})
    out.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    return out, ret


def make_golden():
    from oracle import synth
    scene, t_rand, G = build()
    Gm = map_cotangents(scene)
    got, ret = _reference_grads(scene, t_rand, G, Gm, terms=True)
    empty = (ret["acc_map"] == 0).detach()
    nan_rays = torch.isnan(got["ray_d"]).any(-1)
    assert torch.equal(nan_rays, empty), (int(nan_rays.sum()), int(empty.sum()))
    assert torch.equal(torch.isnan(got["ray_d"]).all(-1), empty)
    assert int(empty.sum()) > 0                                    # the case has empty rays
    for k, g in got.items():
        if k != "ray_d":
            assert torch.isfinite(g).all(), k
    base, _ = _reference_grads(scene, t_rand, G, Gm, terms=False)
    moved = {k: rel_l2_finite(got[k], base[k]) for k in TERM_KEYS}
    assert min(moved.values()) > TERM_MARGIN, moved
    arrays = {"input_sha256": np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8),
              "torch_version": np.frombuffer(torch.__version__.encode(), dtype=np.uint8),
              "d_ray_o": got["ray_o"].numpy().astype(np.float32), "d_ray_d": got["ray_d"].numpy().astype(np.float32),
              "dR": got["R"].numpy().astype(np.float32), "dTh": got["Th"].numpy().astype(np.float32),
              "empty_rays": empty.numpy()}
    for k in list(grad_case.GRAD_KEYS) + ["vol%d" % l for l in range(4)]:
        g = got[k]
        arrays["sum:" + k] = np.float64(g.double().sum())
        arrays["abs:" + k] = np.float64(g.double().abs().sum())
        if not k.startswith("vol"):
            arrays["head:" + k] = g.reshape(-1)[:64].numpy().astype(np.float32)
    path = os.path.join(ROOT, "tests", "golden", GOLDEN + ".npz")
    np.savez_compressed(path, **arrays)
    print("map gradients ->", path, "%d empty rays;" % int(empty.sum()),
          "rel-L2 moved by the disp / weights terms:", {k: round(v, 4) for k, v in moved.items()})


if __name__ == "__main__":
    make_golden()
