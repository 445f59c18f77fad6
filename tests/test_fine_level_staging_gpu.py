"""GPU: the tensor-core decoder stages the fine levels 1 and 0 of layer 0's gather in shared memory, like the coarse ones.

In list order a 64-row half tile touches at most about a hundred distinct voxels of a fine level, which fits the 128 the
staging holds, so the unpermuted full-size view gathers its fine levels from shared memory.  stats[7] counts the fine-level
half tiles that were gathered directly from global memory instead.  A random ray permutation destroys the locality and sends
the fine-level half tiles direct, which gives their number to compare against.  (test_gather_staging_gpu.py checks that the
two renders agree bit for bit.)"""
import pytest
import torch

import gpu_utils as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_fine_levels_are_staged(precision):
    from oracle import synth
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    G.render_product(scene, precision=precision, renderer=ren, net=net)
    direct = int(ren.stats[7])

    perm = torch.randperm(512 * 512, generator=torch.Generator().manual_seed(0))
    sc2 = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sc2[k] = scene[k][:, perm].contiguous()
    ren.stats.zero_()
    G.render_product(sc2, precision=precision, renderer=ren, net=net)
    direct_permuted = int(ren.stats[7])
    print(precision, "fine-level half tiles gathered directly: %d unpermuted, %d permuted" % (direct, direct_permuted))
    assert direct_permuted > 0
    assert direct * 1000 <= direct_permuted
