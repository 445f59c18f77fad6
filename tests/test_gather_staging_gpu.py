"""GPU: the tensor-core decoder's two layer-0 gather paths for the coarse levels 3 and 2 give the same bits.

A 64-row half tile whose samples touch at most NV distinct voxels of a coarse level blends them from a shared-memory copy
(staged path); one that touches more reads the corners from global memory (direct path).  In list order the rows of a tile
are neighbouring rays at neighbouring depths, so the unpermuted full-size view is gathered almost entirely from the staging.
A random ray permutation destroys that locality and sends coarse half tiles through the direct path.  Rays are independent,
so both renders must agree bit for bit after un-permuting.  stats[5] / stats[6] count the half tiles of each path."""
import pytest
import torch

import gpu_utils as G

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["tc_fp16x3", "tc_fp16"])
def test_staged_and_direct_gather_are_bit_identical(precision):
    from oracle import synth
    scene = synth.make_scene(H=512, W=512, scale=1.0, all_hit=True)
    net, ren = G.make_net_and_renderer(scene)
    ren.stats = torch.zeros(8, dtype=torch.int64, device="cuda")
    out = G.render_product(scene, precision=precision, renderer=ren, net=net)
    staged, direct = int(ren.stats[5]), int(ren.stats[6])
    print(precision, "unpermuted: %d staged / %d direct coarse half tiles" % (staged, direct))
    assert staged > 0 and direct < staged

    perm = torch.randperm(512 * 512, generator=torch.Generator().manual_seed(0))
    sc2 = dict(scene)
    for k in ("ray_o", "ray_d", "near", "far"):
        sc2[k] = scene[k][:, perm].contiguous()
    ren.stats.zero_()
    out2 = G.render_product(sc2, precision=precision, renderer=ren, net=net)
    staged2, direct2 = int(ren.stats[5]), int(ren.stats[6])
    print(precision, "permuted: %d staged / %d direct coarse half tiles" % (staged2, direct2))
    assert direct2 > 0
    for k in ("rgb_map", "depth_map", "acc_map", "disp_map", "weights"):
        a, b = out[k][:, perm], out2[k]
        assert torch.equal(torch.nan_to_num(a, nan=-1.0), torch.nan_to_num(b, nan=-1.0)), k
