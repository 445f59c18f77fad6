"""CPU: the sparse encoder's edge cases (oracle/spconv_cases.py) build the row counts they promise, the absolute-value twin
bounds a float32 run of the emulation, and the element-wise comparator sees one dropped neighbour term, one row missing
from a weight gradient and a SubM data gradient with its offset mirror wrong -- so the GPU gate is neither vacuous nor
too loose to catch the kernel's indexing mistakes."""
import pytest
import torch
import torch.nn.functional as F

from neuralbody_b200.lib.networks.sparse_encode import DenseSparseConvNet
from oracle import spconv_cases as S

CASES = S.all_cases()
OFFSETS = [(k // 9 - 1, (k // 3) % 3 - 1, k % 3 - 1) for k in range(27)]


@pytest.mark.parametrize("name", sorted(CASES))
def test_builders_produce_their_promised_counts(name):
    c = CASES[name]
    assert c["promise"] or name.startswith("extent"), name
    for level, n in c["promise"].items():
        assert c["counts"][level] == n, (name, level, c["counts"], c["promise"])
    assert all(n >= 1 for n in c["counts"]), c["counts"]
    caps = S.row_bounds(c["B"], c["coord"].shape[0], c["out_sh"])
    assert all(n <= cap for n, cap in zip(c["counts"], caps)), (c["counts"], caps)


def test_cases_reach_the_tile_slab_and_bound_edges():
    level0 = {c["counts"][0] for c in CASES.values()}
    assert {1, 63, 64, 65, 255, 256, 257, 288, 289} <= level0
    deeper = {n for c in CASES.values() for n in c["counts"][1:]}
    assert {63, 64, 65} <= deeper
    odd = CASES["odd40"]
    assert odd["counts"][1] == 8 * odd["coord"].shape[0] == S.row_bounds(1, 40, odd["out_sh"])[1]
    full = CASES["filled_b2"]
    sites = [full["B"] * s[0] * s[1] * s[2] for s in S.level_shapes(full["out_sh"])]
    assert full["counts"] == sites == S.row_bounds(full["B"], full["coord"].shape[0], full["out_sh"])
    shapes = {tuple(c["out_sh"]) for c in CASES.values()}
    assert {(1, 1, 1), (1, 5, 2), (2, 3, 7), (33, 1, 17)} <= shapes


def test_batches_have_an_empty_middle_frame_and_duplicates_interleave():
    for name, empty in (("batch3", 1), ("batch5", 2)):
        c = CASES[name]
        frames = set(c["coord"][:, 0].tolist())
        assert frames == set(range(c["B"])) - {empty}, (name, frames)
        per_frame = S.masks(c["coord"], c["out_sh"], c["B"])[0].sum(dim=(1, 2, 3, 4))
        assert per_frame[empty] == 0 and len(set(per_frame.tolist())) == c["B"], per_frame
    c = CASES["duplicates"]
    co = c["coord"].long()
    assert c["coord"].shape[0] > c["counts"][0] > c["n_vert"]
    for b in range(c["B"]):
        idx = (co[:, 0] == b).nonzero()[:, 0]
        keys = [tuple(co[i, 1:].tolist()) for i in idx]
        winners = {k: int(i) for k, i in zip(keys, idx)}                  # the highest index of each site
        dup = [k for k in winners if keys.count(k) > 1]
        assert dup and any(winners[k] != int(idx[-1]) for k in dup)
        assert any(keys.index(k) < len(keys) - 1 - keys[::-1].index(k) for k in dup)


def _affine_net(seed):
    """gamma in [0.005, 0.015] and beta in [2.5, 3.5]: every pre-activation stays far above zero (the affine regime)."""
    torch.manual_seed(seed)
    net = DenseSparseConvNet()
    with torch.no_grad():
        for _, bn in S.layers(net):
            bn.weight.uniform_(0.005, 0.015)
            bn.bias.uniform_(2.5, 3.5)
            bn.running_mean.uniform_(-0.5, 0.5)
            bn.running_var.uniform_(0.5, 2.0)
    return net.eval()


def _inputs(c, seed):
    g = torch.Generator().manual_seed(seed)
    code = torch.randn(c["n_vert"], 16, generator=g)
    cots = [torch.randn((c["B"], ch) + s, generator=g) for ch, s in zip((32, 64, 128, 128), S.level_shapes(c["out_sh"])[1:])]
    return code, cots


_refs = {}


def _reference(name):
    if name not in _refs:
        c = CASES[name]
        net = _affine_net(1)
        code, cots = _inputs(c, 2)
        want, t, margin = S.reference_and_twin(net, code, c["coord"], c["out_sh"], c["B"], cots)
        _refs[name] = (c, net, code, cots, want, t, margin)
    return _refs[name]


def _flagged(got, want, t, counts):
    out = []
    for k in want:
        try:
            S.check_elementwise(got[k], want[k], t[k], S.kappa(k, counts), k)
        except AssertionError:
            out.append(k)
    return out


@pytest.mark.parametrize("name", ("odd40", "tile65", "batch3"))
def test_twin_bounds_the_float32_emulation(name):
    c, net, code, cots, want, t, margin = _reference(name)
    assert margin > 10, margin
    f32 = S.emulation(net, torch.float32).eval()
    got = S.run(f32, code, c["coord"], c["out_sh"], c["B"], cots)
    ratios = S.compare_all(got, want, t, c["counts"], name)
    assert max(ratios.values()) < 0.1, max(ratios.items(), key=lambda kv: kv[1])
    assert min(ratios[k] for k in ("net1", "net2", "net3", "net4")) > 0, "the float32 run is bit-exact: the check says nothing"


def _last_row_with_neighbour(mask):
    """(site, k, neighbour site) of the level's last active site and its first active non-centre neighbour."""
    D, H, W = mask.shape[2:]
    b, z, y, x = (int(v) for v in mask[:, 0].nonzero()[-1])
    for k, (dz, dy, dx) in enumerate(OFFSETS):
        n = (b, z + dz, y + dy, x + dx)
        if k != 13 and 0 <= n[1] < D and 0 <= n[2] < H and 0 <= n[3] < W and mask[n[0], 0, n[1], n[2], n[3]] > 0:
            return (b, z, y, x), k, n
    raise AssertionError("the level's last row has no neighbour")


@pytest.mark.parametrize("layer", (4, 8, 12, 16))
def test_comparator_sees_one_dropped_neighbour_term(layer):
    c, net, code, cots, want, t, _ = _reference("odd40")

    def drop(j, x_in, x_out, conv, m_in, m_out):
        if j != layer:
            return x_out
        r, k, n = _last_row_with_neighbour(m_out)
        term = x_in[n[0], :, n[1], n[2], n[3]] @ conv.weight.reshape(27, *conv.weight.shape[3:])[k]
        x_out = x_out.clone()
        x_out[r[0], :, r[1], r[2], r[3]] -= term
        return x_out
    emu = S.emulation(net).eval()
    emu.conv_hook = drop
    got = S.run(emu, code.double(), c["coord"], c["out_sh"], c["B"], cots)
    assert _flagged(got, want, t, c["counts"]), "dropping one term of layer %d passes the gate" % layer


# The layers whose output is a volume, on levels of 63 to 65 rows.  Deeper in the network the twin's cotangent has passed
# through |W| several times while the real one cancels, so the element-wise gate of a weight far from every volume is loose;
# the GPU test holds those gradients to a relative L2 of 1e-4 as well.
@pytest.mark.parametrize("name,layer", (("lattice4_63", 4), ("tile65", 4), ("lattice8_65", 8), ("lattice16_64", 12),
                                        ("lattice16_64", 16)))
def test_comparator_sees_one_row_missing_from_a_weight_gradient(name, layer):
    """The level's last row's centre-offset product in_j^T dx_j left out of dW_j[13] (what a weight-gradient kernel that
    stops one row short of its slab computes)."""
    c, net, code, cots, want, t, _ = _reference(name)
    seen = {}

    def keep(j, x_in, x_out, conv, m_in, m_out):
        if j == layer:
            x_out.retain_grad()
            seen.update(x_in=x_in, x_out=x_out, mask=m_out)
        return x_out
    emu = S.emulation(net).eval()
    emu.conv_hook = keep
    S.run(emu, code.double(), c["coord"], c["out_sh"], c["B"], cots)
    b, z, y, x = (int(v) for v in seen["mask"][:, 0].nonzero()[-1])
    name_w = S.param_names()[layer]
    got = dict(want)
    got[name_w] = want[name_w].clone()
    got[name_w][1, 1, 1] -= torch.outer(seen["x_in"][b, :, z, y, x], seen["x_out"].grad[b, :, z, y, x])
    assert _flagged(got, want, t, c["counts"]) == [name_w]


class _WrongMirror(torch.autograd.Function):
    """A SubM convolution whose data gradient reads the cotangent at +offset_k instead of -offset_k (k for 26 - k)."""

    @staticmethod
    def forward(ctx, x, w, m_out):
        ctx.save_for_backward(x, w, m_out)
        return F.conv3d(x, w.permute(4, 3, 0, 1, 2), padding=1) * m_out

    @staticmethod
    def backward(ctx, dy):
        x, w, m_out = ctx.saved_tensors
        with torch.enable_grad():
            w_ = w.detach().requires_grad_(True)
            dw, = torch.autograd.grad(F.conv3d(x.detach(), w_.permute(4, 3, 0, 1, 2), padding=1) * m_out, w_, dy)
        dx = F.conv3d(dy * m_out, w.permute(3, 4, 0, 1, 2), padding=1) * m_out
        return dx, dw, None


# A layer that outputs a volume, on a level with neighbours (on isolated rows offset 13 is its own mirror): the wrong data
# gradient reaches the previous layer's weight and BatchNorm gradients.
@pytest.mark.parametrize("name,layer", (("batch3", 4), ("batch3", 8), ("batch3", 12), ("odd40", 16)))
def test_comparator_sees_a_wrong_offset_mirror_in_a_data_gradient(name, layer):
    c, net, code, cots, want, t, _ = _reference(name)

    def mirror(j, x_in, x_out, conv, m_in, m_out):
        return _WrongMirror.apply(x_in, conv.weight, m_out) if j == layer else x_out
    emu = S.emulation(net).eval()
    emu.conv_hook = mirror
    got = S.run(emu, code.double(), c["coord"], c["out_sh"], c["B"], cots)
    assert all(torch.equal(got[k], want[k]) for k in ("net1", "net2", "net3", "net4"))
    assert _flagged(got, want, t, c["counts"]), "a mirrored data gradient in layer %d passes the gate" % layer
