"""Golden of the distinct-frame case (oracle/frames_case.py: three frames with their own pose, camera, volumes, latent code
[2, 5, 2] and bounds, 33 samples, 83 rays per frame, jitter, the loss over all five maps).  TEST INFRASTRUCTURE ONLY
(tests/test_distinct_frames.py).

    python -m tools.frames_grad_case

writes tests/golden/grad_frames_b3_s33.npz from the UNMODIFIED reference (oracle/ref_harness.py) in float32, every float
input training: the per-frame gradients in full (R, Th, bounds, rays, near, far; NaNs included), latent.weight in full, the
sum / abs / head summaries of the other decoder gradients and the per-frame sum / abs of the volume gradients, plus the
sha256 of the inputs.  Existing golden files are not touched."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import frames_case as FR  # noqa: E402
from oracle import grad_case  # noqa: E402

GOLDEN = "grad_frames_b3_s33"
FULL = ("R", "Th", "bounds", "ray_o", "ray_d", "near", "far")


def summaries(g):
    """The arrays the golden stores from a gradient dict (frames_case.grads_of's keys), float32 / float64 numpy."""
    out = {"d_" + k: g[k].detach().numpy().astype(np.float32) for k in FULL}
    out["d_latent"] = g["latent.weight"].detach().numpy().astype(np.float32)
    for k in grad_case.GRAD_KEYS:
        t = g[k].detach().double()
        out["sum:" + k] = np.float64(t.sum())
        out["abs:" + k] = np.float64(t.abs().sum())
        out["head:" + k] = t.reshape(-1)[:64].numpy().astype(np.float32)
    for l in range(4):
        t = g["vol%d" % l].detach().double()
        out["sum:vol%d" % l] = t.flatten(1).sum(1).numpy()
        out["abs:vol%d" % l] = t.flatten(1).abs().sum(1).numpy()
    return out


def make_golden():
    from oracle import ref_harness, synth
    scene, t_rand, G, Gm = FR.build()
    sc = FR.leaves(scene)
    sc["volumes"] = scene["volumes"]          # the harness makes its own leaves of the volumes (and the net's parameters)
    ret, net, vols = ref_harness.reference_render(sc, n_samples=FR.N_SAMPLES, perturb=1.0, training=True, white_bkgd=True,
                                                  t_rand=t_rand, grad=True)
    FR.loss_of(ret, G, Gm).backward()
    sd = dict(net.named_parameters())
    got = {k: sc[k].grad for k in FR.LEAVES}
    got.update({k: sd[k].grad for k in grad_case.GRAD_KEYS})
    got.update({"vol%d" % l: v.grad for l, v in enumerate(vols)})
    empty = (ret["acc_map"] == 0).detach()
    assert bool(empty.any()) and not bool(empty.all(1).any())          # every frame has hit and empty rays
    assert torch.equal(torch.isnan(got["near"]), empty) and torch.equal(torch.isnan(got["ray_d"]).any(-1), empty)
    assert not got["bounds"][:, 1].any()
    rows = got["latent.weight"].abs().sum(1).nonzero().flatten().tolist()
    assert rows == sorted(set(FR.LATENT_INDEX)), rows
    arrays = {"input_sha256": np.frombuffer(synth.scene_checksum(scene).encode(), dtype=np.uint8),
              "torch_version": np.frombuffer(torch.__version__.encode(), dtype=np.uint8),
              "empty_rays": empty.numpy()}
    arrays.update(summaries(got))
    path = os.path.join(ROOT, "tests", "golden", GOLDEN + ".npz")
    np.savez_compressed(path, **arrays)
    print("distinct-frame gradients ->", path, "%d empty rays;" % int(empty.sum()),
          {k: "max |d| = %.4e" % float(np.nanmax(np.abs(arrays["d_" + k]))) for k in FULL})


if __name__ == "__main__":
    make_golden()
