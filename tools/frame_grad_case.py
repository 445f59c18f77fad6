"""Frame-transform gradient case (pose refinement): the gradient parity case of oracle/grad_case.py on a 2-frame batch, with
sp_input['R'] (B,3,3) and ['Th'] (B,1,3) requiring grad.  Same jitter recipe and loss as grad_case; each frame sees the body
from its own camera azimuth.  TEST INFRASTRUCTURE ONLY (tests/test_frame_grad.py).

    python -m tools.frame_grad_case

writes tests/golden/grad_frame_b2_s32.npz from the UNMODIFIED reference (oracle/ref_harness.py): its autograd dR and dTh
in full, plus the sha256 of the inputs.  Existing golden files are not touched."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import grad_case  # noqa: E402

N_SAMPLES = grad_case.N_SAMPLES
N_IMPORTANCE = grad_case.N_IMPORTANCE
GOLDEN = "grad_frame_b2_s32"


def build():
    """(scene, t_rand, G): every 5th ray of a 24 x 24 view per frame, 32 samples, jitter and cotangents from seed 99."""
    from oracle import synth
    scene = synth.make_scene(H=24, W=24, scale=0.25, all_hit=True, latent_index=3, batch=2)
    idx = torch.arange(0, scene["ray_o"].shape[1], 5)
    for k in ("ray_o", "ray_d", "near", "far"):
        scene[k] = scene[k][:, idx].contiguous()
    B, n = scene["ray_o"].shape[:2]
    g = torch.Generator().manual_seed(99)
    t_rand = torch.rand((B, n, N_SAMPLES), generator=g)
    G = {"rgb_map": torch.randn((B, n, 3), generator=g), "depth_map": torch.randn((B, n), generator=g) * 0.3,
         "acc_map": torch.randn((B, n), generator=g) * 0.5}
    return scene, t_rand, G


def hier_inputs(scene):
    """Uniforms of sample_pdf and the coarse image's cotangent for the coarse + fine variant (seed 100, as grad_case)."""
    B, n = scene["ray_o"].shape[:2]
    g = torch.Generator().manual_seed(100)
    return torch.rand((B, n, N_IMPORTANCE), generator=g), torch.randn((B, n, 3), generator=g)


def _leaves(scene, th_shape, decoder):
    sc = dict(scene)
    B = scene["R"].shape[0]
    sc["R"] = scene["R"].clone().requires_grad_(True)
    sc["Th"] = scene["Th"].reshape((B,) + tuple(th_shape)).clone().requires_grad_(True)
    if decoder:
        sc["weights"] = {k: v.clone().requires_grad_(True) for k, v in scene["weights"].items()}
        sc["volumes"] = [v.clone().requires_grad_(True) for v in scene["volumes"]]
    return sc


def oracle_frame_grads(scene, t_rand, G, th_shape=(1, 3), decoder=True):
    """Autograd through the oracle restatement -> (dR, dTh, {param: grad} or None, [volume grads] or None, outputs)."""
    from oracle import neuralbody_oracle as O
    sc = _leaves(scene, th_shape, decoder)
    ret = O.render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True, t_rand=t_rand)
    grad_case.loss_of(ret, G).backward()
    pg = {k: sc["weights"][k].grad for k in grad_case.GRAD_KEYS} if decoder else None
    vg = [v.grad for v in sc["volumes"]] if decoder else None
    return sc["R"].grad, sc["Th"].grad, pg, vg, ret


def oracle_hier_frame_grads(scene, t_rand, u, G):
    """The same through the oracle's coarse + detached sample_pdf + fine pass (loss + the coarse image term)."""
    from oracle import neuralbody_oracle as O
    sc = _leaves(scene, (1, 3), decoder=False)
    ret = O.render_hierarchical(sc, n_samples=N_SAMPLES, n_importance=N_IMPORTANCE, perturb=1.0, training=True,
                                white_bkgd=True, t_rand=t_rand, u=u)
    grad_case.hier_loss_of(ret, G).backward()
    return sc["R"].grad, sc["Th"].grad, ret


def make_golden():
    from oracle import ref_harness, synth
    scene, t_rand, G = build()
    sc = _leaves(scene, (1, 3), decoder=False)
    ret, _, _ = ref_harness.reference_render(sc, n_samples=N_SAMPLES, perturb=1.0, training=True, white_bkgd=True,
                                             t_rand=t_rand, grad=True)
    grad_case.loss_of(ret, G).backward()
    arrays = {"input_sha256": np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8),
              "torch_version": np.frombuffer(torch.__version__.encode(), dtype=np.uint8),
              "dR": sc["R"].grad.numpy().astype(np.float32), "dTh": sc["Th"].grad.numpy().astype(np.float32)}
    path = os.path.join(ROOT, "tests", "golden", GOLDEN + ".npz")
    np.savez_compressed(path, **arrays)
    print("frame-transform gradients ->", path, "max |dR| = %.4e, max |dTh| = %.4e" % (
        float(sc["R"].grad.abs().max()), float(sc["Th"].grad.abs().max())))


if __name__ == "__main__":
    make_golden()
